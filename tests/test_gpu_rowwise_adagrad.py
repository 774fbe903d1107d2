"""The rowwise_adagrad updater on the device, against the fp64 model and error bound of test_rowwise_adagrad_cpu.

Every path that steps a table row is covered at world size 1: the fused whole-table Add (its 16-byte and element-wise
bodies, several workers' deltas on one device), the one-sided whole-table push, the owner-side row Add (the path of
every embedding layer's backward), the row mailbox, and the layers themselves. Values and every worker's accumulators
are held to the model; memory a kernel must not write keeps a sentinel."""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from multiverso_b200.ops import PSEmbedding
from test_rowwise_adagrad_cpu import RowwiseModel
from test_table_numerics import _delta, _kopt, _on_device, _opt, _row_case, _start_values

UPD = "rowwise_adagrad"
SENT = -123.5
SHAPES = [("array", 1), ("array", 5), ("array", 4099), ("array", (1 << 20) + 3),
          ("matrix", (1, 1)), ("matrix", (7, 3)), ("matrix", (1000, 300)), ("matrix", (513, 1025))]


def _table(mv, kind, shape, dtype, **kw):
    if kind == "array":
        t, cols = mv.ArrayTable(shape, dtype, updater=UPD, init_value=0.75), 1
    else:
        (rows, cols) = shape
        t = mv.MatrixTable(rows, cols, dtype, updater=UPD, min_value=-1.0, max_value=1.0, **kw)
    return t, RowwiseModel(t.get().cpu().numpy(), cols, dtype)


def _state(t, w=0):
    """Worker w's accumulators of a device table (one per local row)."""
    rows = t.my_len // t.num_col
    return t.state[0][w * t.state_stride:w * t.state_stride + rows].cpu().numpy()


def _check(t, model, dtype, what):
    model.check_values(t.get().cpu().numpy(), dtype, what)
    model.check_state(_state(t), 0, dtype, what)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("kind,shape", SHAPES)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_whole_table_add(mv_device, dtype, kind, shape, offset):
    """Five whole-table Adds through the fused Add, the AddOption changing at every step; offset 1 puts the delta
    one element into a larger buffer, so the element-wise body runs."""
    mv = mv_device
    t, model = _table(mv, kind, shape, dtype)
    rng = np.random.default_rng(5)
    full = (shape,) if kind == "array" else shape
    for k in range(5):
        d = _delta(rng, full, dtype)
        t.add(_on_device(d, offset), _opt(mv, k))
        model.add(d, _opt(mv, k))
    _check(t, model, dtype, f"{dtype} {kind}{shape} offset={offset}")


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [5, 68])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_fused_add_three_workers(mv_device, dtype, cols):
    """``mvb_add_dense_fused`` with three workers' deltas on one device (scale 0.5): worker w steps with its own
    AddOption and its own accumulator slab; the padding after each slab keeps its sentinel."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    rows, W = 37, 3
    n = rows * cols
    stride = (rows + 3) // 4 * 4 + 8
    tdt = getattr(torch, dtype)
    rng = np.random.default_rng(31 + cols)
    start = _start_values(rng, n, dtype)
    shard = torch.from_numpy(start).cuda()
    state = torch.full((stride * W,), SENT, dtype=tdt, device="cuda")
    state.view(W, stride)[:, :rows] = 0
    model = RowwiseModel(start, cols, dtype, workers=W)
    a = N.DenseAdd()
    a.dtype, a.updater = N.dtype_code(tdt), N.UPD_ROWWISE_ADAGRAD
    a.shard, a.state0 = shard.data_ptr(), state.data_ptr()
    a.shard_len, a.shard_off, a.state_stride, a.num_col = n, 0, stride, cols
    a.nworkers, a.worker_mask, a.world = W, (1 << W) - 1, 1
    a.scale, a.clip, a.my_worker = 0.5, 0.0, 0
    for k in range(3):
        deltas = [torch.from_numpy(_delta(rng, (n,), dtype)).cuda() for _ in range(W)]
        for w in range(W):
            opt, a.opts[w] = _kopt(k * W + w, w)
            a.delta_ptrs[w] = deltas[w].data_ptr()
            model.add(deltas[w].cpu().numpy() * 0.5, opt)
        lib.mvb_add_dense_fused(a, st)
        torch.cuda.synchronize()
    what = f"fused Add {dtype} C={cols} W={W}"
    model.check_values(shard.cpu().numpy(), dtype, what)
    slabs = state.view(W, stride)
    for w in range(W):
        model.check_state(slabs[w, :rows].cpu().numpy(), w, dtype, what)
    assert bool((slabs[:, rows:] == SENT).all()), f"{what}: slab padding written"


@pytest.mark.gpu
@pytest.mark.parametrize("worker_id", [0, 2])
@pytest.mark.parametrize("nservers", [1, 3])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_push_dense_rowwise(mv_device, dtype, nservers, worker_id):
    """``mvb_push_dense_rowwise`` of worker ``worker_id`` into ``nservers`` servers emulated as slices of one buffer
    laid out last server first with sentinel gaps, each server's state three worker slabs at a padded stride. Three
    pushes; values and the worker's accumulators against the model, every other word unchanged."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    cols, W, gap = 7, 3, 16
    srows = [1001] if nservers == 1 else [300, 300, 401]
    rows = sum(srows)
    lens = [r * cols for r in srows]
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
    strides = [(r + 3) // 4 * 4 + 8 for r in srows]
    tdt = getattr(torch, dtype)
    data_at, state_at, pos, spos = {}, {}, gap, gap
    for s in reversed(range(nservers)):
        data_at[s], state_at[s] = pos, spos
        pos += lens[s] + gap
        spos += strides[s] * W + gap
    rng = np.random.default_rng(nservers * 10 + worker_id)
    start = _start_values(rng, rows * cols, dtype)
    data = torch.full((pos,), SENT, dtype=tdt, device="cuda")
    state = torch.full((spos,), SENT, dtype=tdt, device="cuda")
    mine = torch.zeros(spos, dtype=torch.bool, device="cuda")
    written = torch.zeros(pos, dtype=torch.bool, device="cuda")
    for s in range(nservers):
        data[data_at[s]:data_at[s] + lens[s]] = torch.from_numpy(start[offs[s]:offs[s] + lens[s]]).cuda()
        o = state_at[s] + worker_id * strides[s]
        state[o:o + srows[s]] = 0
        mine[o:o + srows[s]] = True
        written[data_at[s]:data_at[s] + lens[s]] = True
    data0, state0 = data.clone(), state.clone()
    esz = data.element_size()
    sp = (C.c_void_p * nservers)(*[data.data_ptr() + data_at[s] * esz for s in range(nservers)])
    s0 = (C.c_void_p * nservers)(*[state.data_ptr() + state_at[s] * esz for s in range(nservers)])
    so, sl = (C.c_int64 * nservers)(*offs), (C.c_int64 * nservers)(*lens)
    ss = (C.c_int64 * nservers)(*strides)
    model = RowwiseModel(start, cols, dtype, workers=W)
    for k in range(3):
        opt, copt = _kopt(k, worker_id)
        d = _delta(rng, (rows * cols,), dtype)
        lib.mvb_push_dense_rowwise(N.dtype_code(tdt), N.UPD_ROWWISE_ADAGRAD, torch.from_numpy(d).cuda(), nservers,
                                   sp, s0, so, sl, ss, cols, copt, 1, st)
        model.add(d, opt)
    torch.cuda.synchronize()
    what = f"push_dense_rowwise {dtype} S={nservers} worker {worker_id}"
    got = torch.cat([data[data_at[s]:data_at[s] + lens[s]] for s in range(nservers)]).cpu().numpy()
    model.check_values(got, dtype, what)
    h = torch.cat([state[state_at[s] + worker_id * strides[s]:][:srows[s]] for s in range(nservers)])
    model.check_state(h.cpu().numpy(), worker_id, dtype, what)
    assert torch.equal(data[~written], data0[~written]), f"{what}: data written outside the shards"
    assert torch.equal(state[~mine], state0[~mine]), f"{what}: state written outside the worker's slab"


@pytest.mark.gpu
@pytest.mark.parametrize("ids_kind", ["unique", "repeated"])
@pytest.mark.parametrize("cols", [1, 3, 4, 5, 300, 1025])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_row_add(mv_device, dtype, cols, ids_kind):
    """Row Adds through the owner kernel: a repeated row (up to 50 times) is stepped once per occurrence in list
    order, ids -1 and num_row are ignored, rows never named keep their value and a zero accumulator."""
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
        v = _delta(rng, (ids.size, cols), dtype)
        t.add_rows(torch.from_numpy(ids).cuda(), _on_device(v), _opt(mv, k))
        model.add_rows(ids, v, _opt(mv, k))
        named.update(r for r in ids.tolist() if 0 <= r < rows)
    what = f"row Add {dtype} C={cols} {ids_kind}"
    _check(t, model, dtype, what)
    untouched = np.setdiff1d(np.arange(rows), sorted(named))
    assert np.array_equal(t.get().cpu().numpy().reshape(rows, cols)[untouched], start[untouched])
    assert not _state(t)[untouched].any(), f"{what}: accumulator of a row never named changed"


@pytest.mark.gpu
def test_row_mailbox_apply(mv_device):
    """push_vals then drain(wait=True) on one process: ``rowbox_apply`` steps the named rows; unnamed rows stay
    bitwise unchanged and keep a zero accumulator."""
    from multiverso_b200.runtime import Runtime
    mv = mv_device
    rows, cols = 300, 68
    rng = np.random.default_rng(41)
    t, model = _table(mv, "matrix", (rows, cols), "float32")
    start = model.data.copy()
    mb = t.enable_row_mailbox()
    named = set()
    for k in range(4):
        ids = np.sort(rng.choice(rows, 90, replace=False)).astype(np.int32)
        v = _delta(rng, (ids.size, cols), "float32")
        opt, _ = _kopt(k, 0)
        mb.push_vals(torch.from_numpy(ids).cuda(), torch.from_numpy(v).cuda(), opt)
        torch.cuda.synchronize()
        mb.drain(wait=True)
        mb.drain_stream.synchronize()
        model.add_rows(ids.astype(np.int64), v, opt)
        named.update(ids.tolist())
    Runtime.get().check_watchdog()
    _check(t, model, "float32", "row mailbox")
    untouched = np.setdiff1d(np.arange(rows), sorted(named))
    assert np.array_equal(t.get().cpu().numpy().reshape(rows, cols)[untouched], start[untouched])
    assert not _state(t)[untouched].any()


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
    _check(t, model, "float32", "PSEmbedding")


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
    _check(t, model, "float32", "PSEmbeddingCollection")


@pytest.mark.gpu
def test_hash_table_steps(mv_device):
    """A HashMatrixTable under PSEmbedding: the rows of the keys step as the model says; each key's accumulator is
    the one of its slot's row."""
    mv = mv_device
    dim, B, L = 16, 32, 6
    t = mv.HashMatrixTable(1000, dim, updater=UPD, min_value=-1, max_value=1, seed=9)
    g = torch.Generator(device="cuda").manual_seed(11)
    keys = (torch.randint(0, 50, (B * L,), device="cuda", generator=g) * 1_000_003 + 17).long()
    offsets = torch.arange(0, B * L, L, device="cuda")
    uk = torch.unique(keys)
    rows = t.lookup(uk)                                   # insert every key, then read the starting rows
    model = RowwiseModel(t.get(uk).cpu().numpy(), dim, "float32")
    for k in range(3):
        opt, _ = _kopt(k, 0)
        dout = _exact_dout(g, (B, dim))
        PSEmbedding(t, push_scale=1.0, option=opt)(keys, offsets).backward(dout)
        torch.cuda.synchronize()
        pos = torch.searchsorted(uk, keys)
        G = _coalesce(uk.numel(), pos, torch.arange(B * L, device="cuda") // L, dout)
        model.add(G.cpu().numpy(), opt)
    model.check_values(t.get(uk).cpu().numpy(), "float32", "HashMatrixTable")
    model.check_state(t.state[0][rows.long()].cpu().numpy(), 0, "float32", "HashMatrixTable")


# ------------------------------------------------------------------------------------- size and round trip
@pytest.mark.gpu
@pytest.mark.parametrize("rows,cols", [(1, 1), (7, 3), (1000, 300), (513, 1025)])
def test_state_size(mv_device, rows, cols):
    mv = mv_device
    r = mv.MatrixTable(rows, cols, "float32", updater=UPD)
    a = mv.MatrixTable(rows, cols, "float32", updater="adagrad")
    assert r.state[0].numel() == (rows + 3) // 4 * 4
    assert a.state[0].numel() == (rows * cols + 3) // 4 * 4


def _run(mv, t, rng, k0, k1, rows, cols):
    for k in range(k0, k1):
        if k % 2:
            ids = _row_case(rng, rows, True)
            t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(_delta(rng, (ids.size, cols), "float32")).cuda(),
                       _opt(mv, k))
        else:
            t.add(torch.from_numpy(_delta(rng, (rows, cols), "float32")).cuda(), _opt(mv, k))


@pytest.mark.gpu
def test_store_load_continues_bitwise(mv_device, tmp_path):
    """save_table / load_table carry the accumulators: a table loaded halfway continues bitwise like one that ran
    uninterrupted, and two identical runs are bitwise equal."""
    mv = mv_device
    rows, cols = 200, 12
    a = mv.MatrixTable(rows, cols, "float32", updater=UPD, min_value=-1, max_value=1, seed=3)
    b = mv.MatrixTable(rows, cols, "float32", updater=UPD, min_value=-1, max_value=1, seed=3)
    _run(mv, a, np.random.default_rng(1), 0, 6, rows, cols)
    rng = np.random.default_rng(1)
    _run(mv, b, rng, 0, 3, rows, cols)
    assert mv.save_table(b, str(tmp_path / "ck"))
    c = mv.MatrixTable(rows, cols, "float32", updater=UPD)
    assert mv.load_table(c, str(tmp_path / "ck"))
    assert torch.equal(c.state[0], b.state[0]) and bool(c.state[0].any())
    _run(mv, c, rng, 3, 6, rows, cols)
    assert torch.equal(c.get(), a.get()) and torch.equal(c.state[0], a.state[0])
    d = mv.MatrixTable(rows, cols, "float32", updater=UPD, min_value=-1, max_value=1, seed=3)
    _run(mv, d, np.random.default_rng(1), 0, 6, rows, cols)
    assert torch.equal(d.get(), a.get()) and torch.equal(d.state[0], a.state[0])


# ------------------------------------------------------------------------------------------------ multi-GPU
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bsp", "async"])
@pytest.mark.parametrize("nproc", [2, 4])
def test_multi_gpu(nproc, mode):
    """tests/mp_rowwise_adagrad_check.py under torchrun on ``nproc`` GPUs: BSP fused Adds with per-worker options
    (``bsp``); async whole-table pushes and async row Adds through the row mailboxes (``async``); values and every
    worker's accumulators against the model."""
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = Path(__file__).resolve().parents[1]
    port = 29500 + (os.getpid() % 150) + 800 + nproc + (0 if mode == "bsp" else 10)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           str(root / "tests" / "mp_rowwise_adagrad_check.py"), mode]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
