"""The ftrl updater on the device, against the fp64 model and error bound of test_ftrl_cpu.

Every path that steps a table element is covered at world size 1: the fused whole-table Add (its 16-byte and
element-wise bodies, several workers' deltas on one device), the stand-alone updater, the one-sided whole-table push,
the owner-side row Add (the path of every embedding layer's backward), the row mailbox, the layers, and the eviction
and checkpoint of a HashMatrixTable. Values, z and n are held to the model; an element with a zero delta keeps its
bits; memory a kernel must not write keeps a sentinel; with a large lambda1 the elements and rows the model puts
inside the threshold are exactly 0."""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from multiverso_b200.ops import PSEmbedding
from test_ftrl_cpu import OPTS, FtrlModel, _sparse_delta, fopt
from test_table_numerics import _delta, _on_device, _row_case, _start_values

UPD = "ftrl"
SENT = -123.5
SHAPES = [("array", 1), ("array", 5), ("array", 4099), ("array", (1 << 20) + 3),
          ("matrix", (1, 1)), ("matrix", (7, 3)), ("matrix", (1000, 300)), ("matrix", (513, 1025))]


def _table(mv, kind, shape, dtype, **kw):
    if kind == "array":
        t, cols = mv.ArrayTable(shape, dtype, updater=UPD, init_value=0.75), 1
    else:
        (rows, cols) = shape
        t = mv.MatrixTable(rows, cols, dtype, updater=UPD, min_value=-1.0, max_value=1.0, **kw)
    return t, FtrlModel(t.get().cpu().numpy(), cols, dtype)


def _state(t):
    """(z, n) of a device table, per element."""
    return t.state[0][:t.my_len].cpu().numpy(), t.state[1][:t.my_len].cpu().numpy()


def _check(t, model, what):
    model.check_values(t.get().cpu().numpy(), what)
    model.check_state(*_state(t), what)


def _kopt(k, worker_id):
    """The k-th AddOption of test_ftrl_cpu.OPTS for ``worker_id``, and its C struct."""
    from multiverso_b200.tables.device import _opt_struct
    from multiverso_b200.tables.options import AddOption
    lr, alpha, l1, l2 = OPTS[k % len(OPTS)]
    o = AddOption(worker_id=worker_id, momentum=l2, learning_rate=lr, rho=alpha, lambda_=l1)
    return o, _opt_struct(o)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("kind,shape", SHAPES)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_whole_table_add(mv_device, dtype, kind, shape, offset):
    """Five whole-table Adds through the fused Add, the AddOption changing at every step and a fifth of the deltas 0;
    offset 1 puts the delta one element into a larger buffer, so the element-wise body runs."""
    mv = mv_device
    t, model = _table(mv, kind, shape, dtype)
    rng = np.random.default_rng(5)
    full = (shape,) if kind == "array" else shape
    for k in range(5):
        d = _sparse_delta(rng, full, dtype)
        t.add(_on_device(d, offset), fopt(mv, k))
        model.add(d, fopt(mv, k))
    _check(t, model, f"{dtype} {kind}{shape} offset={offset}")


@pytest.mark.gpu
def test_zero_delta_keeps_bits(mv_device):
    """A whole-table Add whose delta is 0 everywhere but one element leaves every other element, z and n bitwise as
    they were, on a randomly initialised table."""
    mv = mv_device
    t = mv.MatrixTable(64, 33, "float32", updater=UPD, min_value=-1.0, max_value=1.0)
    before = t.get().clone()
    d = torch.zeros(64, 33, device="cuda")
    d[5, 7] = 0.01
    t.add(d, fopt(mv, 0))
    after = t.get().view(64, 33)
    mask = torch.ones(64, 33, dtype=torch.bool, device="cuda")
    mask[5, 7] = False
    assert torch.equal(after[mask], before.view(64, 33)[mask])
    z, n = (s[:64 * 33].view(64, 33) for s in t.state)
    assert not bool(z[mask].any()) and not bool(n[mask].any()) and bool(n[5, 7] > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [1, 5, 68])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_fused_add_three_workers(mv_device, dtype, cols):
    """``mvb_add_dense_fused`` with three workers' deltas on one device (scale 0.5): one step per worker in worker
    order, each with its own AddOption, on the shared z and n; the padding after each slab keeps its sentinel."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    rows, W = 37, 3
    n = rows * cols
    stride = (n + 3) // 4 * 4 + 8
    tdt = getattr(torch, dtype)
    rng = np.random.default_rng(31 + cols)
    start = _start_values(rng, n, dtype)
    shard = torch.from_numpy(start).cuda()
    s0 = torch.full((stride + 5,), SENT, dtype=tdt, device="cuda")
    s1 = torch.full((stride + 5,), SENT, dtype=tdt, device="cuda")
    s0[:n] = 0
    s1[:n] = 0
    model = FtrlModel(start, cols, dtype)
    a = N.DenseAdd()
    a.dtype, a.updater = N.dtype_code(tdt), N.UPD_FTRL
    a.shard, a.state0, a.state1 = shard.data_ptr(), s0.data_ptr(), s1.data_ptr()
    a.shard_len, a.shard_off, a.state_stride, a.num_col = n, 0, stride, cols
    a.nworkers, a.worker_mask, a.world = W, (1 << W) - 1, 1
    a.scale, a.clip, a.my_worker = 0.5, 0.0, 0
    for k in range(3):
        deltas = [torch.from_numpy(_sparse_delta(rng, (n,), dtype)).cuda() for _ in range(W)]
        for w in range(W):
            opt, a.opts[w] = _kopt(k * W + w, w)
            a.delta_ptrs[w] = deltas[w].data_ptr()
            model.add(deltas[w].cpu().numpy() * 0.5, opt)
        lib.mvb_add_dense_fused(a, st)
        torch.cuda.synchronize()
    what = f"fused Add {dtype} C={cols} W={W}"
    model.check_values(shard.cpu().numpy(), what)
    model.check_state(s0[:n].cpu().numpy(), s1[:n].cpu().numpy(), what)
    assert model.nupd.max() >= 6
    assert bool((s0[n:] == SENT).all()) and bool((s1[n:] == SENT).all()), f"{what}: padding written"


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_updater_apply(mv_device, dtype):
    """The stand-alone updater (``mvb_updater_apply``, scale 0.5) over more elements than its grid covers at once."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    n = (1 << 21) + 5
    tdt = getattr(torch, dtype)
    rng = np.random.default_rng(17)
    start = _start_values(rng, n, dtype)
    data = torch.from_numpy(start).cuda()
    z = torch.zeros(n + 3, dtype=tdt, device="cuda")
    nn_ = torch.zeros(n + 3, dtype=tdt, device="cuda")
    z[n:] = SENT
    nn_[n:] = SENT
    model = FtrlModel(start, 1, dtype)
    for k in range(4):
        d = _sparse_delta(rng, (n,), dtype)
        opt, copt = _kopt(k, 0)
        lib.mvb_updater_apply(N.dtype_code(tdt), N.UPD_FTRL, data, torch.from_numpy(d).cuda(), z, nn_, n, copt, 0.5,
                              st)
        model.add(d * 0.5, opt)                       # exact: the kernel scales by 0.5 too
    torch.cuda.synchronize()
    model.check_values(data.cpu().numpy(), f"updater_apply {dtype}")
    model.check_state(z[:n].cpu().numpy(), nn_[:n].cpu().numpy(), f"updater_apply {dtype}")
    assert bool((z[n:] == SENT).all()) and bool((nn_[n:] == SENT).all())


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [1, 7, 40])
@pytest.mark.parametrize("worker_id", [0, 2])
@pytest.mark.parametrize("nservers", [1, 3])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_push_dense_stateful(mv_device, dtype, nservers, worker_id, cols):
    """``mvb_push_dense_stateful`` of worker ``worker_id`` into ``nservers`` servers emulated as slices of one buffer,
    laid out last server first with sentinel gaps, each server's z and n slabs at a padded stride. Three pushes of one
    worker: values, z and n against the model (the value is the old value plus the step, within the bound), every
    other word unchanged."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    gap = 16
    srows = [1001] if nservers == 1 else [300, 300, 401]
    rows = sum(srows)
    lens = [r * cols for r in srows]
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
    strides = [(n + 3) // 4 * 4 + 8 for n in lens]
    tdt = getattr(torch, dtype)
    data_at, st_at, pos, spos = {}, {}, gap, gap
    for s in reversed(range(nservers)):
        data_at[s], st_at[s] = pos, spos
        pos += lens[s] + gap
        spos += strides[s] + gap
    rng = np.random.default_rng(nservers * 10 + worker_id + cols)
    start = _start_values(rng, rows * cols, dtype)
    data = torch.full((pos,), SENT, dtype=tdt, device="cuda")
    z = torch.full((spos,), SENT, dtype=tdt, device="cuda")
    n = torch.full((spos,), SENT, dtype=tdt, device="cuda")
    for s in range(nservers):
        data[data_at[s]:data_at[s] + lens[s]] = torch.from_numpy(start[offs[s]:offs[s] + lens[s]]).cuda()
        z[st_at[s]:st_at[s] + lens[s]] = 0
        n[st_at[s]:st_at[s] + lens[s]] = 0
    data0, z0, n0 = data.clone(), z.clone(), n.clone()
    esz = data.element_size()
    sp = (C.c_void_p * nservers)(*[data.data_ptr() + data_at[s] * esz for s in range(nservers)])
    s0 = (C.c_void_p * nservers)(*[z.data_ptr() + st_at[s] * esz for s in range(nservers)])
    s1 = (C.c_void_p * nservers)(*[n.data_ptr() + st_at[s] * esz for s in range(nservers)])
    so, sl = (C.c_int64 * nservers)(*offs), (C.c_int64 * nservers)(*lens)
    ss = (C.c_int64 * nservers)(*strides)
    model = FtrlModel(start, cols, dtype)
    for k in range(3):
        opt, copt = _kopt(k, worker_id)
        d = _sparse_delta(rng, (rows * cols,), dtype)
        lib.mvb_push_dense_stateful(N.dtype_code(tdt), N.UPD_FTRL, torch.from_numpy(d).cuda(), nservers, sp, s0, s1,
                                    so, sl, ss, copt, 1, st)
        model.add(d, opt)
    torch.cuda.synchronize()
    what = f"push_dense_stateful {dtype} S={nservers} worker {worker_id} C={cols}"
    cat = lambda buf, at, ln: torch.cat([buf[at[s]:at[s] + ln[s]] for s in range(nservers)]).cpu().numpy()
    model.check_values(cat(data, data_at, lens), what)
    model.check_state(cat(z, st_at, lens), cat(n, st_at, lens), what)
    for buf, ref, at in ((data, data0, data_at), (z, z0, st_at), (n, n0, st_at)):
        mask = torch.ones_like(buf, dtype=torch.bool)
        for s in range(nservers):
            mask[at[s]:at[s] + lens[s]] = False
        assert torch.equal(buf[mask], ref[mask]), f"{what}: written outside the shards"


@pytest.mark.gpu
@pytest.mark.parametrize("ids_kind", ["unique", "repeated"])
@pytest.mark.parametrize("cols", [1, 3, 4, 5, 300, 1025])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_row_add(mv_device, dtype, cols, ids_kind):
    """Row Adds through the owner kernel: a repeated row (up to 50 times) is one step per occurrence in list order,
    ids -1 and num_row are ignored, rows never named keep their value and zero state."""
    mv = mv_device
    rows = 200
    rng = np.random.default_rng(cols)
    t, model = _table(mv, "matrix", (rows, cols), dtype)
    start = model.data.copy()
    named = set()
    for k in range(3):
        ids = _row_case(rng, rows, ids_kind == "repeated")
        if k == 1:
            ids = rng.permutation(np.concatenate([ids, [-1, rows]])).astype(np.int64)
        v = _sparse_delta(rng, (ids.size, cols), dtype)
        t.add_rows(torch.from_numpy(ids).cuda(), _on_device(v), fopt(mv, k))
        model.add_rows(ids, v, fopt(mv, k))
        named.update(r for r in ids.tolist() if 0 <= r < rows)
    what = f"row Add {dtype} C={cols} {ids_kind}"
    _check(t, model, what)
    if ids_kind == "repeated":
        assert model.nupd.max() >= 40
    untouched = np.setdiff1d(np.arange(rows), sorted(named))
    assert np.array_equal(t.get().cpu().numpy().reshape(rows, cols)[untouched], start[untouched])
    z, n = _state(t)
    assert not z.reshape(rows, cols)[untouched].any() and not n.reshape(rows, cols)[untouched].any()


@pytest.mark.gpu
def test_row_mailbox_apply(mv_device):
    """push_vals then drain(wait=True) on one process: ``rowbox_apply`` steps the named rows, one step per entry of a
    repeated row in list order; unnamed rows stay bitwise unchanged with zero state."""
    from multiverso_b200.runtime import Runtime
    mv = mv_device
    rows, cols = 300, 68
    rng = np.random.default_rng(41)
    t, model = _table(mv, "matrix", (rows, cols), "float32")
    start = model.data.copy()
    mb = t.enable_row_mailbox()
    named = set()
    for k in range(4):
        ids = np.sort(np.concatenate([rng.choice(rows, 90, replace=False), [7, 7, 7]])).astype(np.int32)
        v = _sparse_delta(rng, (ids.size, cols), "float32")
        opt, _ = _kopt(k, 0)
        mb.push_vals(torch.from_numpy(ids).cuda(), torch.from_numpy(v).cuda(), opt)
        torch.cuda.synchronize()
        mb.drain(wait=True)
        mb.drain_stream.synchronize()
        model.add_rows(ids.astype(np.int64), v, opt)
        named.update(ids.tolist())
    Runtime.get().check_watchdog()
    _check(t, model, "row mailbox")
    untouched = np.setdiff1d(np.arange(rows), sorted(named))
    assert np.array_equal(t.get().cpu().numpy().reshape(rows, cols)[untouched], start[untouched])
    assert not _state(t)[1].reshape(rows, cols)[untouched].any()


@pytest.mark.gpu
def test_option_checks(mv_device):
    """An ftrl table refuses an AddOption with lr <= 0, rho <= 0, lambda_ < 0 or momentum < 0 before any kernel runs."""
    mv = mv_device
    t = mv.MatrixTable(8, 4, "float32", updater=UPD, min_value=-1, max_value=1)
    before = t.get().clone()
    for lr, rho, l1, l2 in ((0.0, 0.1, 0.1, 0.0), (0.1, 0.0, 0.1, 0.0), (0.1, 0.1, -0.1, 0.0), (0.1, 0.1, 0.1, -1.0)):
        bad = mv.AddOption(worker_id=0, momentum=l2, learning_rate=lr, rho=rho, lambda_=l1)
        with pytest.raises(ValueError):
            t.add(torch.ones(8, 4, device="cuda"), bad)
        with pytest.raises(ValueError):
            t.add_rows(torch.tensor([1, 2], device="cuda"), torch.ones(2, 4, device="cuda"), bad)
    assert torch.equal(t.get(), before) and not _state(t)[1].any()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fused", "rows"])
def test_sparsity(mv_device, path):
    """With lambda1 = 2: every element whose model |z| is below lambda1 by more than the bound is exactly 0.0 on the
    device, every element the model puts beyond it is not, and the rows the model zeroes as a whole are zero rows.
    Rows get gradients of different sizes, so some rows go to zero and some do not."""
    mv = mv_device
    rows, cols = 256, 24
    rng = np.random.default_rng(77)
    t, model = _table(mv, "matrix", (rows, cols), "float32")
    row_scale = 10.0 ** rng.uniform(-1.5, 1.5, (rows, 1))
    opt = mv.AddOption(worker_id=0, momentum=0.1, learning_rate=0.05, rho=0.1, lambda_=2.0)
    for k in range(6):
        d = (_delta(rng, (rows, cols), "float32") * row_scale).astype(np.float32)
        if path == "fused":
            t.add(_on_device(d), opt)
            model.add(d, opt)
        else:
            ids = np.arange(rows, dtype=np.int64)
            t.add_rows(torch.from_numpy(ids).cuda(), _on_device(d), opt)
            model.add_rows(ids, d, opt)
    _check(t, model, f"sparsity {path}")
    got = t.get().cpu().numpy().reshape(rows, cols)
    l1 = np.float32(2.0)
    inside = np.abs(model.z) < l1 - 4 * model.ez
    outside = np.abs(model.z) > l1 + 4 * model.ez
    assert inside.sum() > rows * cols // 4 and outside.sum() > rows * cols // 4
    assert (got[inside] == 0.0).all(), "an element inside lambda1 is not exactly 0"
    assert (got[outside] != 0.0).all()
    zero_rows = inside.all(axis=1)
    assert zero_rows.sum() >= 10 and (~(model.data == 0).all(axis=1)).sum() >= 10
    assert (got[zero_rows] == 0.0).all()


# ------------------------------------------------------------------------------------------------ layers
def _exact_dout(g, shape):
    """Upstream gradients that are small multiples of 2^-6: every coalesced row gradient is exact in fp32."""
    return torch.randint(-4, 5, shape, device="cuda", generator=g).float() * 2.0 ** -6


def _coalesce(V, ids, bag, dout):
    G = torch.zeros(V, dout.shape[1], dtype=torch.float64, device="cuda")
    G.index_add_(0, ids, dout.double()[bag])
    return G


@pytest.mark.gpu
def test_ps_embedding_steps(mv_device):
    """Three PSEmbedding forward + backward steps: one step per touched row with the coalesced gradient."""
    mv = mv_device
    V, dim, B, L = 500, 36, 64, 12
    t, model = _table(mv, "matrix", (V, dim), "float32")
    g = torch.Generator(device="cuda").manual_seed(7)
    for k in range(3):
        opt, _ = _kopt(k, 0)
        emb = PSEmbedding(t, push_scale=0.5, option=opt)
        ids = torch.randint(0, 60, (B * L,), device="cuda", generator=g)
        offsets = torch.arange(0, B * L, L, device="cuda")
        dout = _exact_dout(g, (B, dim))
        emb(ids, offsets).backward(dout)
        torch.cuda.synchronize()
        G = _coalesce(V, ids, torch.arange(B * L, device="cuda") // L, dout) * 0.5
        uniq = torch.unique(ids)
        model.add_rows(uniq.cpu().numpy(), G[uniq].cpu().numpy(), opt)
    _check(t, model, "PSEmbedding")
    assert model.nupd.max() == 3


@pytest.mark.gpu
def test_ps_embedding_collection_shared_table(mv_device):
    """Two features over one table: a row named by both features gets one step per backward, with the sum of both
    features' gradients."""
    from multiverso_b200.ops.embedding_collection import EmbeddingBagConfig, PSEmbeddingCollection
    mv = mv_device
    V, dim, B, L = 400, 20, 50, 8
    t, model = _table(mv, "matrix", (V, dim), "float32")
    g = torch.Generator(device="cuda").manual_seed(3)
    for k in range(2):
        opt, _ = _kopt(k, 0)
        ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["q", "k"], push_scale=1.0, option=opt)])
        ids = torch.randint(0, 80, (2 * B * L,), device="cuda", generator=g)
        lengths = torch.full((2, B), L, device="cuda")
        dout = _exact_dout(g, (B, 2 * dim))
        ebc(ids, lengths).backward(dout)
        torch.cuda.synchronize()
        bag = torch.arange(B * L, device="cuda") // L
        G = _coalesce(V, ids[:B * L], bag, dout[:, :dim]) + _coalesce(V, ids[B * L:], bag, dout[:, dim:])
        uniq = torch.unique(ids)
        model.add_rows(uniq.cpu().numpy(), G[uniq].cpu().numpy(), opt)
    _check(t, model, "PSEmbeddingCollection")
    assert model.nupd.max() == 2


class _Spy:
    """Records what a layer pushes through one of a table's Add methods, then lets it through."""

    def __init__(self, table, name):
        self.calls, self._f, self._t = [], getattr(table, name), table
        setattr(table, name, self)

    def __call__(self, *args, **kw):
        rec = tuple(a.detach().clone() if torch.is_tensor(a) else a for a in args)
        if kw.get("staged"):                  # a staged Add: the delta is the table's staging buffer
            rec = (self._t._cur_stage.tensor(self._t.dtype, self._t.size).clone(),) + rec[1:] + (kw.get("option"),)
        self.calls.append(rec)
        return self._f(*args, **kw)


@pytest.mark.gpu
def test_ps_sampled_softmax_steps(mv_device):
    """PSSampledSoftmax pushes each backward's coalesced row gradients (labels and candidates, each row once) with
    one row Add; the table steps each of those rows once, as the model does with the pushed rows."""
    mv = mv_device
    n, d, B = 3000, 32, 48
    t, model = _table(mv, "matrix", (n, d), "float32")
    spy = _Spy(t, "add_rows_async")
    g = torch.Generator(device="cuda").manual_seed(5)
    for k in range(3):
        opt, _ = _kopt(k, 0)
        ssm = mv.ops.PSSampledSoftmax(t, num_sampled=256, sampler="log_uniform", push_scale=0.25, option=opt, seed=k)
        x = torch.randn(B, d, device="cuda", generator=g, requires_grad=True)
        y = torch.randint(0, n, (B,), device="cuda", generator=g)
        ssm(x, y).sum().backward()
        torch.cuda.synchronize()
        assert len(spy.calls) == k + 1
        ids, vals, popt = spy.calls[-1][:3]
        assert ids.numel() == torch.unique(ids).numel() and popt is opt
        model.add_rows(ids.cpu().numpy(), vals.double().cpu().numpy(), opt)
    _check(t, model, "PSSampledSoftmax")


@pytest.mark.gpu
def test_ps_full_softmax_steps(mv_device):
    """PSFullSoftmax stages push_scale * dL/dW for every row and issues one whole-table Add per backward; the table
    steps every element with a non-zero gradient once, as the model does with the staged delta."""
    mv = mv_device
    n, d, B = 1000, 64, 40
    t, model = _table(mv, "matrix", (n, d), "float32")
    spy = _Spy(t, "add_async")
    g = torch.Generator(device="cuda").manual_seed(9)
    for k in range(3):
        opt, _ = _kopt(k, 0)
        fsm = mv.ops.PSFullSoftmax(t, push_scale=0.5, option=opt)
        x = torch.randn(B, d, device="cuda", generator=g, requires_grad=True)
        y = torch.randint(0, n, (B,), device="cuda", generator=g)
        fsm(x, y).sum().backward()
        torch.cuda.synchronize()
        assert len(spy.calls) == k + 1
        model.add(spy.calls[-1][0].double().cpu().numpy(), opt)
    _check(t, model, "PSFullSoftmax")
    assert model.nupd.max() == 3


@pytest.mark.gpu
def test_ps_linear_steps(mv_device):
    """PSLinear pushes dW = dy^T x * push_scale as one whole-table Add per backward: every weight with a non-zero
    gradient steps once."""
    mv = mv_device
    out_f, in_f, B = 24, 36, 16
    t, model = _table(mv, "matrix", (out_f, in_f), "float32")
    spy = _Spy(t, "add_async")
    g = torch.Generator(device="cuda").manual_seed(8)
    for k in range(4):
        opt, _ = _kopt(k, 0)
        lin = mv.ops.PSLinear(t, push_scale=0.5, option=opt)
        x = _exact_dout(g, (B, in_f)).requires_grad_()
        dy = _exact_dout(g, (B, out_f))
        lin(x).backward(dy)
        torch.cuda.synchronize()
        dw = (dy.double().t() @ x.detach().double()) * 0.5
        assert len(spy.calls) == k + 1 and torch.equal(spy.calls[-1][0].double().view(out_f, in_f), dw)
        model.add(dw.cpu().numpy(), opt)
    _check(t, model, "PSLinear")
    assert model.nupd.max() == 4


# ------------------------------------------------------------------------------------------------ hash tables
def _hash_state(t, rows):
    z = t.state[0][:t.my_len].view(-1, t.num_col)[rows]
    n = t.state[1][:t.my_len].view(-1, t.num_col)[rows]
    return z, n


@pytest.mark.gpu
def test_hash_table_train_evict_checkpoint(mv_device, tmp_path):
    """A HashMatrixTable trained through PSEmbedding steps each key's row as the model says. An eviction then moves
    every survivor's row, z and n bitwise, leaves zeros in every slot it does not hold, and a returning key starts
    like a new one (initial row, zero state). A checkpoint of the evicted table loads back with z and n in place."""
    from test_gpu_hash_embedding import _init_model, _spread
    mv = mv_device
    dim, B, L = 16, 40, 6
    mk = lambda: mv.HashMatrixTable(1000, dim, updater=UPD, min_value=-1, max_value=1, seed=9, track_access=True)
    t = mk()
    keys = torch.tensor(_spread(120, 33), dtype=torch.int64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(11)
    offsets = torch.arange(0, B * L, L, device="cuda")
    uk = torch.sort(keys)[0]
    t.clock = 0
    t.lookup(uk)                                          # insert every key, then read the starting rows
    model = FtrlModel(t.get(uk).cpu().numpy(), dim, "float32")
    for k in range(3):
        t.clock = k
        opt, _ = _kopt(k, 0)
        sel = keys[torch.randint(0, 60 if k == 2 else 120, (B * L,), device="cuda", generator=g)]
        dout = _exact_dout(g, (B, dim))
        PSEmbedding(t, push_scale=1.0, option=opt)(sel, offsets).backward(dout)
        torch.cuda.synchronize()
        pos = torch.searchsorted(uk, sel)
        G = _coalesce(uk.numel(), pos, torch.arange(B * L, device="cuda") // L, dout)
        touched = torch.unique(pos)
        model.add_rows(touched.cpu().numpy(), G[touched].cpu().numpy(), opt)
    model.check_values(t.get(uk).cpu().numpy(), "HashMatrixTable")
    rows = t.lookup(uk, insert=False)
    model.check_state(*[x.cpu().numpy() for x in _hash_state(t, rows)], "HashMatrixTable")
    # evict the keys idle in the last step
    ls = t.last_seen(uk)
    idle, keep = uk[ls < 2], uk[ls == 2]
    assert idle.numel() and keep.numel()
    before = [x.clone() for x in _hash_state(t, t.lookup(keep, insert=False))]
    vals = t.get(keep)
    assert t.evict(older_than=2) == idle.numel()
    after = _hash_state(t, t.lookup(keep, insert=False))
    for b, a, name in zip(before, after, ("z", "n")):
        assert torch.equal(a, b), f"survivor {name} moved"
        assert bool(b.any()), f"survivor {name} is all zero"
    assert torch.equal(t.get(keep), vals)
    live_keys, live_rows = t._dump(0)
    free = torch.ones(t.slots, dtype=torch.bool, device="cuda")
    free[live_rows] = False
    for x, name in zip(_hash_state(t, torch.arange(t.slots, device="cuda")), ("z", "n")):
        assert not bool(x[free].any()), f"a free slot holds {name}"
    # a checkpoint of the evicted table carries z and n
    assert mv.save_table(t, str(tmp_path / "ck"))
    t2 = mk()
    assert mv.load_table(t2, str(tmp_path / "ck"))
    for i in range(2):
        assert torch.equal(t2.state[i], t.state[i])
    assert torch.equal(t2.get(keep), vals)
    # a returning key starts like a new one
    back = idle[:5]
    for tab in (t, t2):
        r = tab.lookup(back)
        assert np.array_equal(tab.get(back).cpu().numpy(), _init_model(back.tolist(), 9, -1, 1, dim))
        assert all(not bool(x.any()) for x in _hash_state(tab, r))
        opt, _ = _kopt(0, 0)
        tab.add(back, torch.full((5, dim), 0.01, device="cuda"), opt)
    fresh = FtrlModel(_init_model(back.tolist(), 9, -1, 1, dim), dim, "float32")
    fresh.add(np.full((5, dim), 0.01, np.float32), opt)
    fresh.check_values(t.get(back).cpu().numpy(), "returning keys")
    assert torch.equal(t2.get(back), t.get(back))


# ------------------------------------------------------------------------------------- size and round trip
@pytest.mark.gpu
@pytest.mark.parametrize("kind,shape", [("array", 1), ("array", 4099), ("matrix", (7, 3)), ("matrix", (513, 1025))])
def test_state_size(mv_device, kind, shape):
    """Two slabs of round4(R C) elements for a shard of R rows x C."""
    mv = mv_device
    t, _ = _table(mv, kind, shape, "float32")
    R, C_ = (shape, 1) if kind == "array" else shape
    r4 = (R * C_ + 3) // 4 * 4
    assert len(t.state) == 2 and t.state[0].numel() == r4 and t.state[1].numel() == r4


def _run(mv, t, rng, k0, k1, rows, cols):
    for k in range(k0, k1):
        if k % 2:
            ids = _row_case(rng, rows, True)
            t.add_rows(torch.from_numpy(ids).cuda(),
                       torch.from_numpy(_sparse_delta(rng, (ids.size, cols), "float32")).cuda(), fopt(mv, k))
        else:
            t.add(torch.from_numpy(_sparse_delta(rng, (rows, cols), "float32")).cuda(), fopt(mv, k))


@pytest.mark.gpu
def test_store_load_continues_bitwise(mv_device, tmp_path):
    """save_table / load_table carry z and n: a table loaded halfway continues bitwise like one that ran
    uninterrupted, and two identical runs are bitwise equal."""
    mv = mv_device
    rows, cols = 200, 12
    mk = lambda: mv.MatrixTable(rows, cols, "float32", updater=UPD, min_value=-1, max_value=1, seed=3)
    a, b = mk(), mk()
    _run(mv, a, np.random.default_rng(1), 0, 6, rows, cols)
    rng = np.random.default_rng(1)
    _run(mv, b, rng, 0, 3, rows, cols)
    assert mv.save_table(b, str(tmp_path / "ck"))
    c = mv.MatrixTable(rows, cols, "float32", updater=UPD)
    assert mv.load_table(c, str(tmp_path / "ck"))
    for i in range(2):
        assert torch.equal(c.state[i], b.state[i]) and bool(c.state[i].any())
    _run(mv, c, rng, 3, 6, rows, cols)
    assert torch.equal(c.get(), a.get()) and all(torch.equal(c.state[i], a.state[i]) for i in range(2))
    d = mk()
    _run(mv, d, np.random.default_rng(1), 0, 6, rows, cols)
    assert torch.equal(d.get(), a.get()) and all(torch.equal(d.state[i], a.state[i]) for i in range(2))


# ------------------------------------------------------------------------------------------------ multi-GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bsp", "async"])
@pytest.mark.parametrize("nproc", [2, 4])
def test_multi_gpu(nproc, mode):
    """tests/mp_ftrl_check.py under torchrun on ``nproc`` GPUs: BSP fused Adds with per-worker options and row Adds
    (``bsp``); async whole-table pushes of one worker (exact), of every worker (Hogwild), and async row Adds through
    the row mailboxes (``async``)."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = Path(__file__).resolve().parents[1]
    port = 29500 + (os.getpid() % 150) + 1300 + nproc + (0 if mode == "bsp" else 10)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           str(root / "tests" / "mp_ftrl_check.py"), mode]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
