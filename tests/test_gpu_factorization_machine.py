"""PSFactorizationMachine on the GPU (csrc/cuda/fm.cu): y and the pushed row gradient (fused red.add and compact)
against fp64 within the bounds derived in the op's docstring, at every register class and slab edge of C; S' bitwise
embedding_bag; bitwise equality over runs and over 1 / 2 / 3 / 8 shards; one updater step per touched row for sgd,
adagrad, rowwise_adagrad, adam and ftrl; HashMatrixTable insertion, eval mode and admission; host synchronisations; a
planted FM trained end to end; errors raised without a launch."""
import types
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _sharded(W, S, gap=37):
    """W [n, C] as S shards of a row pitch round4(C) at separate places of one buffer with NaN rows between them
    (reference rows_per_server rule, the last shard takes the remainder), and a function reading the table back."""
    from multiverso_b200 import _native as N
    n, C = W.shape
    pitch = (C + 3) // 4 * 4
    rps = n // S
    buf = torch.full((n + S * gap, pitch), float("nan"), device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, rps
    spans = []
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo, :C] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
        spans.append((at, hi - lo))
    return rm, buf, lambda: torch.cat([buf[a:a + k, :C] for a, k in spans])


def _fake_table(rm, num_row, num_col, updater=None):
    """A MatrixTable handle over an explicit row map: what the op reads of a device table."""
    from multiverso_b200 import _native as N
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=num_row, num_col=num_col,
                                 updater=N.UPD_DEFAULT if updater is None else updater, is_sparse=False,
                                 rt=types.SimpleNamespace(device=torch.device("cuda", 0)))


def _zipf_ids(n, L, gen, s=1.05):
    w = torch.from_numpy(1.0 / np.arange(1, n + 1) ** s).cuda()
    return torch.multinomial(w / w.sum(), L, replacement=True, generator=gen)


def _batch(n, B, gen, long_bag=600):
    """Zipf ids in bags of 0..40 lookups: bag 0 empty, bag 1 one lookup, bag 2 long_bag lookups; signed values."""
    lens = torch.randint(0, 41, (B,), device="cuda", generator=gen)
    lens[0], lens[1], lens[2] = 0, 1, long_bag
    L = int(lens.sum())
    ids = _zipf_ids(n, L, gen)
    x = torch.randn(L, device="cuda", generator=gen)
    return ids, torch.cumsum(lens, 0) - lens, x


def _reference(W, ids, offsets, x, g):
    """fp64 y, its bound, the row gradient G of sum(g * y) and its bound (the op's docstring)."""
    n, C = W.shape
    k = C - 1
    B, L = offsets.numel(), ids.numel()
    lens = torch.diff(offsets, append=torch.tensor([L], device=offsets.device))
    bag = torch.repeat_interleave(torch.arange(B, device=ids.device), lens)
    Wd, xd, gd = W.double(), x.double(), g.double()
    zeros = lambda *s: torch.zeros(*s, dtype=torch.float64, device=W.device)    # noqa: E731
    R = Wd[ids]
    S = zeros(B, C).index_add_(0, bag, xd[:, None] * R)
    A = zeros(B, C).index_add_(0, bag, (xd[:, None] * R).abs())
    q = zeros(B).index_add_(0, bag, xd ** 2 * (R[:, :k] ** 2).sum(1))
    ss = (S[:, :k] ** 2).sum(1)
    y = S[:, k] + 0.5 * (ss - q)
    nb = lens.double()
    P = (A[:, :k] ** 2).sum(1)
    tol_y = U * ((nb + 5) * (A[:, k] + P) + 9 * ss + (nb + 7) * q + 0.5 * (ss - q).abs() + y.abs())
    Sp = S.clone()
    Sp[:, k] = 1
    vp = R.clone()
    vp[:, k] = 0
    gx = gd[bag] * xd
    G = zeros(n, C).index_add_(0, ids, gx[:, None] * (Sp[bag] - xd[:, None] * vp))
    m = torch.bincount(ids, minlength=n).double()
    Ae = A.clone()
    Ae[:, k] = 0                                   # column k of S' is exactly 1
    tol_G = U * zeros(n, C).index_add_(0, ids, gx.abs()[:, None] * (nb[bag][:, None] + 5) * Ae[bag]) \
        + (2 * m + 4)[:, None] * U * (zeros(n, C).index_add_(0, ids, gx.abs()[:, None] * Sp[bag].abs())
                                      + zeros(n, C).index_add_(0, ids, (gd[bag].abs() * xd ** 2)[:, None] * vp.abs()))
    return y, tol_y, G, tol_G, torch.unique(ids)


def _run(W, ids, offsets, x, g, S=1, updater=None, push_scale=1.0):
    """One forward + backward over a fake table of S shards: (y, table after, compact pushes)."""
    from multiverso_b200.ops import PSFactorizationMachine
    rm, keep, back = _sharded(W, S, 0 if S == 1 else 37)
    t = _fake_table(rm, W.shape[0], W.shape[1], updater)
    pushes = []
    t.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    fm = PSFactorizationMachine(t, push_scale=push_scale)
    y = fm(ids, offsets, x)
    (y * g).sum().backward()
    torch.cuda.synchronize()
    return y.detach(), back(), pushes


def _assert_within(got, exp, tol, what):
    err = (got.double() - exp).abs()
    assert (err <= tol).all(), (what, (err / tol.clamp_min(1e-300)).max().item())


@pytest.mark.parametrize("C", [2, 5, 8, 64, 128, 129, 512, 513, 1024])
def test_matches_fp64(cuda, C):
    """B = 2048 bags over 5000 Zipf rows (the hottest row has thousands of lookups, so its run crosses many
    chunks), with an empty, a one-lookup and a 600-lookup bag: y against fp64, the row gradient from a default table
    with push_scale = 1 (fused red.add) and from the compact push of an adagrad table; S' bitwise embedding_bag."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFactorizationMachine, embedding_bag
    gen = torch.Generator(device=cuda).manual_seed(C)
    n, B = 5000, 2048
    W = torch.randn(n, C, device=cuda, generator=gen) / C ** 0.5
    ids, offsets, x = _batch(n, B, gen)
    assert int(torch.bincount(ids).max()) > 256
    g = torch.randn(B, device=cuda, generator=gen)
    y, after, _ = _run(W, ids, offsets, x, g)
    y_r, tol_y, G, tol_G, touched = _reference(W, ids, offsets, x, g)
    assert y[0] == 0
    _assert_within(y, y_r, tol_y, f"y C={C}")
    _assert_within(after.double() - W.double(), G, tol_G + U * (W.double() + G).abs(), f"fused C={C}")
    keep = torch.ones(n, dtype=torch.bool, device=cuda)
    keep[touched] = False
    assert torch.equal(after[keep], W[keep])
    y2, after2, pushes = _run(W, ids, offsets, x, g, updater=N.UPD_ADAGRAD)
    assert torch.equal(y2, y) and torch.equal(after2, W) and len(pushes) == 1
    uid, vals = pushes[0]
    assert torch.equal(uid, touched) and vals.shape == (touched.numel(), C)
    _assert_within(vals, G[uid], tol_G[uid], f"compact C={C}")
    # S' is the embedding bag with per-sample weights x, column k set to 1
    rm, buf, _ = _sharded(W, 1, 0)                 # buf holds the shard while rm points into it
    t = _fake_table(rm, n, C)
    fm = PSFactorizationMachine(t)
    _, sp = fm._launch(*fm_inputs(fm, ids, offsets, x), grad=True)
    eb = embedding_bag(t, ids, offsets, per_sample_weights=x)
    assert torch.equal(sp[:, :C - 1], eb[:, :C - 1]) and bool((sp[:, C - 1] == 1).all())
    assert bool((sp[:, C:] == 0).all())


def fm_inputs(fm, ids, offsets, x):
    from multiverso_b200.ops.embedding import _prepare
    i, o, v = _prepare(fm.table, ids, offsets, x, "sum")
    return i, o, None if v is None else v.contiguous()


def _outputs(W, ids, offsets, x, g, S, updater=None):
    from multiverso_b200.ops import PSFactorizationMachine
    rm, keep, back = _sharded(W, S, 0 if S == 1 else 37)
    t = _fake_table(rm, W.shape[0], W.shape[1], updater)
    pushes = []
    t.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    fm = PSFactorizationMachine(t)
    _, sp = fm._launch(*fm_inputs(fm, ids, offsets, x), grad=True)
    y = fm(ids, offsets, x)
    (y * g).sum().backward()
    torch.cuda.synchronize()
    out = [y.detach(), sp, back()]
    for p in pushes:
        out += list(p)
    return out


@pytest.mark.parametrize("C", [16, 129])
def test_bitwise_over_shards_and_runs(cuda, C):
    from multiverso_b200 import _native as N
    gen = torch.Generator(device=cuda).manual_seed(9)
    n, B = 100003, 4096
    W = torch.randn(n, C, device=cuda, generator=gen) * 0.1
    ids, offsets, x = _batch(n, B, gen)
    g = torch.randn(B, device=cuda, generator=gen)
    for updater in (None, N.UPD_ADAGRAD):
        ref = _outputs(W, ids, offsets, x, g, 1, updater)
        for shards in (1, 2, 3, 8):
            got = _outputs(W, ids, offsets, x, g, shards, updater)
            assert len(got) == len(ref)
            for i, (a, b) in enumerate(zip(ref, got)):
                assert torch.equal(a, b), (updater, shards, i)


@pytest.mark.parametrize("updater", ["sgd", "adagrad", "rowwise_adagrad", "adam", "ftrl"])
def test_updaters_step_once_per_touched_row(mv_device, updater):
    """The real table after one backward equals a twin given the recorded coalesced gradient through add_rows;
    touched rows changed, untouched ones did not, and adam counted exactly one step per touched row."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFactorizationMachine
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    n, C, B, scale = 3000, 64, 1024, 0.1
    kw = dict(min_value=-0.5, max_value=0.5, seed=11)
    t = mv.MatrixTable(n, C, "float32", updater=updater, **kw)
    twin = mv.MatrixTable(n, C, "float32", updater=updater, **kw)
    W0 = t.get().view(n, C).clone()
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    gen = torch.Generator(device="cuda").manual_seed(3)
    ids, offsets, x = _batch(n, B, gen, long_bag=300)
    rm, keep, _ = _sharded(W0, 1, 0)
    rec, pushes = _fake_table(rm, n, C, N.UPD_ADAGRAD), []
    rec.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    PSFactorizationMachine(rec, push_scale=scale, option=opt)(ids, offsets, x).mean().backward()
    PSFactorizationMachine(t, push_scale=scale, option=opt)(ids, offsets, x).mean().backward()
    torch.cuda.synchronize()
    assert len(pushes) == 1
    uniq, grads = pushes[0]
    twin.wait(twin.add_rows_async(uniq, grads, opt))
    torch.cuda.synchronize()
    got = t.get().view(n, C)
    assert torch.equal(got, twin.get().view(n, C))
    touched = torch.zeros(n, dtype=torch.bool, device="cuda")
    touched[uniq] = True
    assert torch.equal(got[~touched], W0[~touched])
    assert ((got - W0).abs().max(1).values[touched] > 0).float().mean() > 0.9
    if updater == "adam":
        rows = t.my_len // t.num_col
        steps = t.state[1][t.state_stride:t.state_stride + rows]
        assert torch.equal(steps, touched.to(steps.dtype))


def _spread(n, seed):
    rng = np.random.default_rng(seed)
    return rng.choice(np.arange(1, 1 << 40, 7919), n, replace=False)


def test_hash_table_insert_eval_and_admission(mv_device):
    from multiverso_b200.ops import PSFactorizationMachine, factorization_machine_reference
    mv = mv_device
    # training mode inserts the missing keys; y is the FM of the rows they got
    t = mv.HashMatrixTable(1000, 16, updater="sgd", min_value=-0.5, max_value=0.5, seed=3)
    keys = torch.tensor(_spread(300, 1), dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(2)
    bags = keys[torch.randint(0, 300, (64, 8), device="cuda", generator=gen)]
    fm = PSFactorizationMachine(t, push_scale=0.1)
    y = fm(bags)
    uk, inv = torch.unique(bags, return_inverse=True)
    assert t.num_keys() == uk.numel()
    ref = factorization_machine_reference(t.get(uk), inv)
    assert torch.allclose(y.double(), ref, rtol=1e-5, atol=1e-5)
    y.sum().backward()
    # eval mode: new keys read the zero row and are not inserted; a backward after it raises
    known = uk[:20]
    before = t.get(known)
    new = torch.tensor(_spread(20, 9), dtype=torch.int64, device="cuda") + 3
    pairs = torch.stack([known, new], 1)                                       # bag b: (known b, new b)
    fm.eval()
    ye = fm(pairs)
    assert t.num_keys() == uk.numel()
    assert torch.allclose(ye.double(), factorization_machine_reference(before, torch.arange(20, device="cuda")[:, None]),
                          rtol=0, atol=1e-6)
    with pytest.raises(RuntimeError, match="eval mode"):
        ye.sum().backward()
    with torch.no_grad():
        assert torch.equal(fm(pairs), ye.detach())
    assert torch.equal(t.get(known), before)
    # admit_after=3: keys seen fewer than 3 times add nothing to y and are not pushed; the zero row stays zero
    h = mv.HashMatrixTable(1000, 16, updater="sgd", admit_after=3, min_value=-0.5, max_value=0.5, seed=4)
    adm = torch.tensor(_spread(32, 5), dtype=torch.int64, device="cuda")
    for _ in range(4):
        h.lookup(adm)
    assert bool((h.lookup(adm, insert=False) != h.zero_row).all())
    fresh = torch.tensor(_spread(32, 6), dtype=torch.int64, device="cuda") + 1
    fa = PSFactorizationMachine(h, push_scale=0.5)
    w_adm = h.get(adm)
    yh = fa(torch.stack([adm, fresh, fresh.flip(0)], 1))
    assert bool((h.lookup(fresh, insert=False) == h.zero_row).all())
    assert torch.allclose(yh.double(), factorization_machine_reference(w_adm, torch.arange(32, device="cuda")[:, None]),
                          rtol=0, atol=1e-6)
    yh.sum().backward()
    torch.cuda.synchronize()
    assert bool((h.shard.view(-1, 16)[h.zero_row] == 0).all())
    # one lookup per bag pushed: the factor gradient is ~0, the linear weight moved by -0.5
    assert torch.allclose(h.get(adm)[:, 15], w_adm[:, 15] - 0.5, atol=1e-6)
    assert torch.allclose(h.get(adm)[:, :15], w_adm[:, :15], atol=1e-6)


def _syncs(fn):
    """Synchronising torch calls made by fn (torch's sync debug mode in 'warn')."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def test_host_syncs_and_empty_batch(mv_device):
    """1 per forward (the id and offset checks), 0 per sgd backward, 1 per compact (adagrad) backward; an empty
    batch after a full call pushes nothing."""
    from multiverso_b200.ops import PSFactorizationMachine
    mv = mv_device
    n, C = 4000, 32
    g = torch.Generator(device="cuda").manual_seed(6)
    ids, offsets, x = _batch(n, 512, g, long_bag=50)
    for updater, want in (("sgd", 0), ("adagrad", 1)):
        t = mv.MatrixTable(n, C, "float32", updater=updater, min_value=-0.5, max_value=0.5)
        fm = PSFactorizationMachine(t, push_scale=0.1)
        fm(ids, offsets, x).mean().backward()                          # warm-up
        out = []
        assert _syncs(lambda: out.append(fm(ids, offsets, x))) == 1
        assert _syncs(lambda: out[0].mean().backward()) == want, updater
        torch.cuda.synchronize()
        before = t.get().clone()
        e = torch.zeros(0, dtype=torch.int64, device="cuda")
        y = fm(e, e)
        assert y.shape == (0,)
        y.sum().backward()
        y = fm(e, torch.zeros(4, dtype=torch.int64, device="cuda"))   # four empty bags
        assert torch.equal(y, torch.zeros(4, device="cuda"))
        y.sum().backward()
        torch.cuda.synchronize()
        assert torch.equal(t.get(), before), updater


def test_no_grad_forward_is_bitwise_the_training_forward(cuda):
    from multiverso_b200.ops import PSFactorizationMachine
    n, C = 5000, 96
    gen = torch.Generator(device=cuda).manual_seed(1)
    rm, keep, back = _sharded(torch.randn(n, C, device=cuda, generator=gen), 1, 0)
    fm = PSFactorizationMachine(_fake_table(rm, n, C), push_scale=None)
    ids, offsets, x = _batch(n, 300, gen)
    with torch.no_grad():
        ev = fm(ids, offsets, x)
    tr = fm(ids, offsets, x)
    assert ev.grad_fn is None and tr.grad_fn is not None and torch.equal(ev, tr.detach())


def test_planted_fm_trains_to_the_planted_log_loss(cuda):
    """Labels drawn from a planted FM (k = 8, 200 Zipf ids, bags of 8, linear weights ~ N(0, 0.5^2), factors ~
    N(0, 0.3^2)): PSFactorizationMachine + sgd (lr 1, mean loss, 1500 steps of 2048 bags, start uniform in +-0.1)
    reaches, on fresh data, a log-loss within 0.03 nats of the planted model's own (~0.42). An fp32 torch simulation
    of the same schedule ends ~0.016 above it: what remains is the noise of SGD at this step size and the fit of 1800
    parameters to noisy labels. A model that learnt nothing stays near log 2, ~0.27 above."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFactorizationMachine, factorization_machine_reference
    n, C, BAG, B = 200, 9, 8, 2048
    gen = torch.Generator(device="cuda").manual_seed(0)
    Wp = torch.cat([torch.randn(n, C - 1, device="cuda", generator=gen) * 0.3,
                    torch.randn(n, 1, device="cuda", generator=gen) * 0.5], 1)
    # C = 9 has a row pitch of 12: a table over an explicit row map, pushed to by the fused sgd red.add
    W0 = (torch.rand(n, C, device="cuda", generator=gen) - 0.5) * 0.2
    rm, buf, _ = _sharded(W0, 1, 0)
    fm = PSFactorizationMachine(_fake_table(rm, n, C, N.UPD_SGD), push_scale=1.0)
    bce = torch.nn.functional.binary_cross_entropy_with_logits

    def batch(b):
        ids = _zipf_ids(n, b * BAG, gen).view(b, BAG)
        ys = factorization_machine_reference(Wp, ids).float()
        return ids, (torch.rand(b, device="cuda", generator=gen) < torch.sigmoid(ys)).float(), ys

    def evaluate():
        ids, lab, ys = batch(65536)
        with torch.no_grad():
            return bce(fm(ids), lab).item(), bce(ys, lab).item()

    start, floor = evaluate()
    for _ in range(1500):
        ids, lab, _ = batch(B)
        bce(fm(ids), lab).backward()
    end, floor2 = evaluate()
    print(f"planted FM: start {start:.4f} end {end:.4f} planted {floor:.4f} / {floor2:.4f}")
    assert start > floor + 0.15, (start, floor)
    assert end < floor2 + 0.03, (end, floor2)


def _fm_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "fm_fwd_kernel" in e.name or "fm_bwd_" in e.name)


def test_errors_raise_without_launching(cuda):
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFactorizationMachine
    n, C = 1000, 32
    W = torch.randn(n, C, device=cuda)
    rm, keep, _ = _sharded(W, 1, 0)
    t = _fake_table(rm, n, C, N.UPD_ADAGRAD)
    t.add_rows_async = lambda ids, vals, option=None: None
    fm = PSFactorizationMachine(t)
    ids = torch.arange(8, device=cuda)
    offs = torch.tensor([0, 3], device=cuda)
    x = torch.rand(8, device=cuda)

    def step():
        fm(ids, offs, x).sum().backward()
    assert _fm_kernels(step) == 7          # the counter sees the op: forward, count + scan, count + scan + main + merge
    cases = [
        (ValueError, r"\[0, 1000\), got min 0 max 1000", (torch.tensor([0, 1, 2, 1000], device=cuda), offs[:1], None)),
        (ValueError, "got min -3", (torch.tensor([0, -3], device=cuda, dtype=torch.int32), offs[:1], None)),
        (TypeError, "int32 or int64", (ids.float(), offs, None)),
        (ValueError, "must start at 0", (ids, offs + 1, None)),
        (ValueError, "non-decreasing", (ids, torch.tensor([0, 5, 3], device=cuda), None)),
        (ValueError, "exceed the number of ids", (ids, torch.tensor([0, 9], device=cuda), None)),
        (ValueError, "shape of ids", (ids, offs, x[:7])),
        (TypeError, "floating point", (ids, offs, torch.ones(8, dtype=torch.int64, device=cuda))),
        (ValueError, "get no gradient", (ids, offs, x.clone().requires_grad_())),
    ]
    for exc, msg, args in cases:
        def call():
            with pytest.raises(exc, match=msg):
                fm(*args)
        assert _fm_kernels(call) == 0, msg
    # the layer's refusals of the table
    with pytest.raises(TypeError, match="MatrixTable"):
        PSFactorizationMachine(W)
    with pytest.raises(TypeError, match="float32"):
        PSFactorizationMachine(types.SimpleNamespace(**{**vars(t), "dtype": torch.float64}))
    for bad in (1, 1025):
        with pytest.raises(ValueError, match=r"\[2, 1024\]"):
            PSFactorizationMachine(_fake_table(rm, n, bad))
    rm6 = N.RowMap()
    rm6.num_row, rm6.num_col, rm6.nservers, rm6.rows_per_server = n, 34, 1, n
    rm6.shard_ptrs[0] = W.data_ptr()
    with pytest.raises(ValueError, match="row pitch"):
        PSFactorizationMachine(_fake_table(rm6, n, 32))
    # every error code of the entry points, each before any launch
    i, o, v = fm_inputs(fm, ids, offs, x)
    y, sp = fm._launch(i, o, v, grad=True)
    nbytes = N.cuda_lib().mvb_embedding_bag_scratch_bytes(8, C)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=cuda)
    grads = torch.empty(8, C, device=cuda)
    uniq = torch.empty(8, dtype=torch.int64, device=cuda)
    dy = torch.ones(2, device=cuda)

    def args(**kw):
        a = fm._args(i, o, v)
        a.y, a.sp, a.lds, a.dy, a.perm = y.data_ptr(), sp.data_ptr(), C, dy.data_ptr(), i.data_ptr()
        a.scratch, a.scratch_bytes, a.epilogue = scratch.data_ptr(), nbytes, N.EMB_COMPACT
        a.grads, a.ldg, a.uniq = grads.data_ptr(), C, uniq.data_ptr()
        for k, val in kw.items():
            if k == "shard0":
                a.wmap.shard_ptrs[0] = val
            elif k.startswith("map_"):
                setattr(a.wmap, k[4:], val)
            else:
                setattr(a, k, val)
        return a
    lib = N.cuda_lib()
    lib.mvb_fm_fwd(args(), N.stream_ptr())
    lib.mvb_fm_bwd(args(), N.stream_ptr())
    common = [(N.BAD_ROW_MAP, dict(map_nservers=0)), (N.BAD_ROW_MAP, dict(map_nservers=9)),
              (N.BAD_ROW_MAP, dict(map_rows_per_server=0)),
              (-90, dict(dim=1)), (-90, dict(dim=1025)), (-90, dict(dim=36)), (-90, dict(map_num_col=30)),
              (-90, dict(shard0=W.data_ptr() + 4)),
              (-91, dict(B=-1)), (-91, dict(L=-1)), (-91, dict(offsets=None)), (-91, dict(ids=None))]
    fwd = common + [(-92, dict(y=None)), (-92, dict(lds=30)), (-92, dict(lds=34)), (-92, dict(sp=sp.data_ptr() + 4))]
    bwd = common + [(-93, dict(dy=None)), (-93, dict(perm=None)), (-93, dict(sp=None)), (-93, dict(lds=28)),
                    (-93, dict(scratch=None)), (-93, dict(scratch_bytes=nbytes - 1)),
                    (-94, dict(epilogue=7)), (-94, dict(uniq=None)), (-94, dict(ldg=30)),
                    (-94, dict(grads=grads.data_ptr() + 4))]
    for entry, cases in ((lib.mvb_fm_fwd, fwd), (lib.mvb_fm_bwd, bwd)):
        for rc, kw in cases:
            def call():
                with pytest.raises(N.NativeError, match=f"rc={rc}:"):
                    entry(args(**kw), N.stream_ptr())
            assert _fm_kernels(call) == 0, (entry.__name__, kw)
    a0, l0 = args(B=0), args(L=0, n_unique=None)
    assert _fm_kernels(lambda: lib.mvb_fm_fwd(a0, N.stream_ptr())) == 0
    assert _fm_kernels(lambda: lib.mvb_fm_bwd(l0, N.stream_ptr())) == 0


def test_factorization_machine_peer_shards_multi_gpu():
    """A table sharded over 2 GPUs (tests/mp_factorization_machine_check.py under torchrun): the forward bitwise
    equal to a single-shard copy, async sgd pushes from every rank landing as W0 - lr * sum."""
    import os
    import subprocess
    import sys
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 1200
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_factorization_machine_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == 2, tail
