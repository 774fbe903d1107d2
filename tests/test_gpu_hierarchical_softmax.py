"""PSHierarchicalSoftmax on the GPU (csrc/cuda/hier_softmax.cu): loss, dL/dhidden and the node gradient (fused and
compact push) against fp64 within the bound derived in the op's docstring, at every width class and tree shape;
bitwise equality over runs and over 1 / 2 / 3 / 8 shards; one updater step per touched node for sgd, adagrad,
rowwise_adagrad, adam and ftrl; host synchronisations; a planted classification task trained end to end; errors
raised without a launch."""
import math
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
    """W as S shards at separate places of one buffer with NaN rows between them (reference rows_per_server rule,
    the last shard takes the remainder), and a function reading the table back."""
    from multiverso_b200 import _native as N
    n, pitch = W.shape
    rps = n // S
    buf = torch.full((n + S * gap, pitch), float("nan"), device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, rps
    spans = []
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
        spans.append((at, hi - lo))
    return rm, buf, lambda: torch.cat([buf[a:a + k] for a, k in spans])


def _fake_table(rm, num_row, num_col, updater=None):
    """A MatrixTable handle over an explicit row map: what the op reads of a device table."""
    from multiverso_b200 import _native as N
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=num_row, num_col=num_col,
                                 updater=N.UPD_DEFAULT if updater is None else updater, is_sparse=False,
                                 rt=types.SimpleNamespace(device=torch.device("cuda", 0)))


def _zipf(n, s=1.05):
    w = 1.0 / np.arange(1, n + 1) ** s
    return w / w.sum()


def _fib(n):
    f = [1, 1]
    while len(f) < n:
        f.append(f[-1] + f[-2])
    return np.array(f[:n], dtype=np.float64)


def _reference(W, x, y, counts, dl):
    """fp64 loss, dL/dhidden of sum(dl * loss) and the node gradient, with the device bounds of the op's docstring."""
    from multiverso_b200.ops.hierarchical_softmax import _steps, huffman_tree
    points, codes, lens = (t.to(x.device) for t in huffman_tree(counts))
    B, d = x.shape
    bag, ids, cds, _ = _steps(points, codes, lens, y)
    x64, dl64 = x.double(), dl.double()
    w = W[ids].double()
    h = x64[bag]
    prod = h * w
    z = prod.sum(1)
    a = prod.abs().sum(1)
    c = cds.double()
    sp = torch.nn.functional.softplus(-(1 - 2 * c) * z)
    Lb = lens[y].double()
    zeros = lambda *s: torch.zeros(*s, dtype=torch.float64, device=x.device)    # noqa: E731
    loss = zeros(B).index_add_(0, bag, sp)
    dz = d * U * a
    tol_loss = zeros(B).index_add_(0, bag, dz + 4 * U * (1 + sp)) + Lb * U * loss
    g = torch.sigmoid(z) - (1 - c)
    dg = dz / 4 + 4 * U
    u = zeros(B, d).index_add_(0, bag, g[:, None] * w)
    dx = dl64[:, None] * u
    tol_dx = dl64.abs()[:, None] * (zeros(B, d).index_add_(0, bag, dg[:, None] * w.abs())
                                    + (Lb + 1)[:, None] * U * zeros(B, d).index_add_(0, bag, (g[:, None] * w).abs())) \
        + U * dx.abs()
    n = W.shape[0]
    dlb = dl64[bag]
    G = zeros(n, d).index_add_(0, ids, (dlb * g)[:, None] * h)
    m = torch.bincount(ids, minlength=n).double()
    tol_G = zeros(n, d).index_add_(0, ids, (dlb.abs() * dg)[:, None] * h.abs()) \
        + (m + 2)[:, None] * U * zeros(n, d).index_add_(0, ids, (dlb * g).abs()[:, None] * h.abs())
    return loss, tol_loss, dx, tol_dx, G, tol_G, torch.unique(ids)


def _check_all(W, x, y, counts, dl, loss, dx, G_dev, what):
    loss_r, tol_loss, dx_r, tol_dx, G, tol_G, touched = _reference(W, x, y, counts, dl)
    err = (loss.double() - loss_r).abs()
    assert (err <= tol_loss).all(), (what, (err / tol_loss).max().item())
    if dx is not None:
        err = (dx.double() - dx_r).abs()
        assert (err <= tol_dx).all(), (what, (err / tol_dx).max().item())
    if G_dev is not None:
        ids, rows, base = G_dev
        tol = tol_G[ids]
        if base is not None:                       # rows = (base + G) - base: the red.add rounds once more
            tol = tol + U * (base.double()[ids] + G[ids]).abs()
        err = (rows.double() - G[ids]).abs()
        assert (err <= tol).all(), (what, (err / tol).max().item())
    return touched


def _run(W, counts, x, y, dl, S=1, updater=None, push_scale=1.0):
    """One forward + backward over a fake table of S shards: (loss, dhidden, table after, compact pushes)."""
    from multiverso_b200.ops import PSHierarchicalSoftmax
    rm, keep, back = _sharded(W, S, 0 if S == 1 else 37)
    t = _fake_table(rm, W.shape[0], W.shape[1], updater)
    pushes = []
    t.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    hsm = PSHierarchicalSoftmax(t, counts, push_scale=push_scale)
    xx = x.clone().requires_grad_()
    loss = hsm(xx, y)
    (loss * dl).sum().backward()
    torch.cuda.synchronize()
    return loss.detach(), xx.grad, back(), pushes


@pytest.mark.parametrize("d", [4, 12, 128, 132, 300, 512, 1024])
def test_matches_fp64(cuda, d):
    """Zipf labels over 1000 classes, B = 8192: loss and dL/dhidden against fp64, the node gradient from a default
    table with push_scale = 1 (fused red.add) and from the compact push of an adagrad table."""
    from multiverso_b200 import _native as N
    gen = torch.Generator(device=cuda).manual_seed(d)
    n, B = 1000, 8192
    p = _zipf(n)
    W = torch.randn(n - 1, d, device=cuda, generator=gen) / d ** 0.5
    x = torch.randn(B, d, device=cuda, generator=gen)
    y = torch.multinomial(torch.from_numpy(p).to(cuda), B, replacement=True, generator=gen)
    dl = torch.rand(B, device=cuda, generator=gen) + 0.5
    loss, dx, after, _ = _run(W, p, x, y, dl)
    rows = torch.arange(n - 1, device=cuda)
    touched = _check_all(W, x, y, p, dl, loss, dx, (rows, after.double() - W.double(), W), f"fused d={d}")
    # the red.add rounds the sum once more: untouched rows are bitwise unchanged
    keep = torch.ones(n - 1, dtype=torch.bool, device=cuda)
    keep[touched] = False
    assert torch.equal(after[keep], W[keep])
    loss2, dx2, after2, pushes = _run(W, p, x, y, dl, updater=N.UPD_ADAGRAD)
    assert len(pushes) == 1 and torch.equal(pushes[0][0], touched) and torch.equal(after2, W)
    assert torch.equal(loss2, loss) and torch.equal(dx2, dx)
    _check_all(W, x, y, p, dl, loss, None, (*pushes[0], None), f"compact d={d}")


_SHAPES = {
    "N2": (lambda: np.array([3.0, 5.0]), "uniform"),
    "N3": (lambda: np.array([1.0, 1.0, 2.0]), "uniform"),
    "N1000003": (lambda: _zipf(1000003), "zipf"),
    "depth61": (lambda: _fib(62), "deepest"),
    "same_label": (lambda: _zipf(1000), "same"),
}


@pytest.mark.parametrize("B", [0, 1, 8192])
@pytest.mark.parametrize("shape", list(_SHAPES))
def test_tree_shapes_and_batches(cuda, shape, B):
    """Paths of length 1 (N = 2), 61 (Fibonacci counts, every label the deepest leaf), a 1M-class Zipf tree, one
    label for the whole batch; B = 0 pushes nothing and returns an empty loss."""
    from multiverso_b200.ops.hierarchical_softmax import huffman_tree
    make, labels = _SHAPES[shape]
    counts = make()
    n, d = counts.size, 128
    gen = torch.Generator(device=cuda).manual_seed(B + n)
    W = torch.randn(n - 1, d, device=cuda, generator=gen) * 0.1
    x = torch.randn(B, d, device=cuda, generator=gen)
    lens = huffman_tree(counts)[2]
    if labels == "zipf":
        y = torch.multinomial(torch.from_numpy(counts).to(cuda), max(B, 1), replacement=True, generator=gen)[:B]
    elif labels == "deepest":
        assert int(lens.max()) == 61
        y = torch.full((B,), int(lens.argmax()), device=cuda)
    elif labels == "same":
        y = torch.full((B,), 7, device=cuda)
    else:
        y = torch.randint(0, n, (B,), device=cuda, generator=gen)
    if shape == "N2":
        assert lens.tolist() == [1, 1]
    dl = torch.rand(B, device=cuda, generator=gen) + 0.5
    loss, dx, after, _ = _run(W, counts, x, y, dl)
    assert loss.shape == (B,) and dx.shape == (B, d)
    if B == 0:
        assert torch.equal(after, W)
        return
    _check_all(W, x, y, counts, dl, loss, dx, (torch.arange(n - 1, device=cuda), after.double() - W.double(), W),
               f"{shape} B={B}")


def _outputs(W, counts, x, y, S):
    """loss, ids, g, u of the kernel and the table after a fused push, over S shards."""
    from multiverso_b200.ops import PSHierarchicalSoftmax
    rm, keep, back = _sharded(W, S, 0 if S == 1 else 37)
    hsm = PSHierarchicalSoftmax(_fake_table(rm, W.shape[0], W.shape[1]), counts, push_scale=1.0)
    y, ln, L = hsm._check(x, y)
    loss, _, ids, offsets, g, u = hsm._launch(x, y, ln, L, grad=True)
    xx = x.clone().requires_grad_()
    hsm(xx, y).sum().backward()
    torch.cuda.synchronize()
    return loss, ids, offsets, g, u, xx.grad, back()


def test_bitwise_over_shards_and_runs(cuda):
    gen = torch.Generator(device=cuda).manual_seed(9)
    n, d, B = 100003, 132, 4096
    p = _zipf(n)
    W = torch.randn(n - 1, d, device=cuda, generator=gen) * 0.1
    x = torch.randn(B, d, device=cuda, generator=gen)
    y = torch.multinomial(torch.from_numpy(p).to(cuda), B, replacement=True, generator=gen)
    ref = _outputs(W, p, x, y, 1)
    for shards in (1, 2, 3, 8):
        got = _outputs(W, p, x, y, shards)
        for i, (a, b) in enumerate(zip(ref, got)):
            assert torch.equal(a, b), (shards, i)


@pytest.mark.parametrize("updater", ["sgd", "adagrad", "rowwise_adagrad", "adam", "ftrl"])
def test_updaters_step_once_per_touched_node(mv_device, updater):
    """The real table after one backward equals a twin given the recorded coalesced gradient through add_rows;
    touched nodes changed, untouched ones did not, and adam counted exactly one step per touched row."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSHierarchicalSoftmax
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    n, d, B, scale = 2000, 64, 1024, 0.1
    p = _zipf(n)
    kw = dict(min_value=-0.5, max_value=0.5, seed=11)
    t = mv.MatrixTable(n - 1, d, "float32", updater=updater, **kw)
    twin = mv.MatrixTable(n - 1, d, "float32", updater=updater, **kw)
    W0 = t.get().view(n - 1, d).clone()
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    gen = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, d, device="cuda", generator=gen)
    y = torch.multinomial(torch.from_numpy(p).cuda(), B, replacement=True, generator=gen)
    rm, keep, _ = _sharded(W0, 1, 0)
    rec, pushes = _fake_table(rm, n - 1, d, N.UPD_ADAGRAD), []
    rec.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    PSHierarchicalSoftmax(rec, p, push_scale=scale, option=opt)(x, y).mean().backward()
    PSHierarchicalSoftmax(t, p, push_scale=scale, option=opt)(x, y).mean().backward()
    torch.cuda.synchronize()
    assert len(pushes) == 1
    uniq, grads = pushes[0]
    twin.wait(twin.add_rows_async(uniq, grads, opt))
    torch.cuda.synchronize()
    got = t.get().view(n - 1, d)
    assert torch.equal(got, twin.get().view(n - 1, d))
    touched = torch.zeros(n - 1, dtype=torch.bool, device="cuda")
    touched[uniq] = True
    assert torch.equal(got[~touched], W0[~touched])
    assert ((got - W0).abs().max(1).values[touched] > 0).float().mean() > 0.9
    if updater == "adam":
        rows = t.my_len // t.num_col
        steps = t.state[1][t.state_stride:t.state_stride + rows]
        assert torch.equal(steps, touched.to(steps.dtype))


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
    """1 per forward (the label checks and the path total), 0 per sgd backward, 1 per compact (adagrad) backward;
    an empty batch after a full call pushes nothing."""
    from multiverso_b200.ops import PSHierarchicalSoftmax
    mv = mv_device
    n, d = 4000, 64
    p = _zipf(n)
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(512, d, device="cuda", generator=g, requires_grad=True)
    y = torch.randint(0, n, (512,), device="cuda", generator=g)
    for updater, want in (("sgd", 0), ("adagrad", 1)):
        t = mv.MatrixTable(n - 1, d, "float32", updater=updater, min_value=-0.5, max_value=0.5)
        hsm = PSHierarchicalSoftmax(t, p, push_scale=0.1)
        hsm(x, y).mean().backward()                                   # warm-up
        out = []
        assert _syncs(lambda: out.append(hsm(x, y))) == 1
        assert _syncs(lambda: out[0].mean().backward()) == want, updater
        torch.cuda.synchronize()
        before = t.get().clone()
        e = torch.zeros(0, d, device="cuda", requires_grad=True)
        loss = hsm(e, torch.zeros(0, dtype=torch.int64, device="cuda"))
        assert loss.shape == (0,)
        loss.sum().backward()
        torch.cuda.synchronize()
        assert torch.equal(t.get(), before) and e.grad.shape == (0, d), updater


def test_no_grad_forward_is_the_evaluation(cuda):
    """Under no_grad the forward writes only the loss: bitwise the training forward's loss, nothing saved."""
    from multiverso_b200.ops import PSHierarchicalSoftmax
    n, d = 5000, 96
    p = _zipf(n)
    gen = torch.Generator(device=cuda).manual_seed(1)
    rm, keep, back = _sharded(torch.randn(n - 1, d, device=cuda, generator=gen), 1, 0)
    hsm = PSHierarchicalSoftmax(_fake_table(rm, n - 1, d), p)
    x = torch.randn(300, d, device=cuda, generator=gen, requires_grad=True)
    y = torch.randint(0, n, (300,), device=cuda, generator=gen)
    with torch.no_grad():
        ev = hsm(x, y)
    assert ev.grad_fn is None and torch.equal(ev, hsm(x, y).detach())


def test_planted_classification_trains_to_the_planted_entropy(mv_device):
    """fastText-style: a bag of one topic word and 7 noise words, PSEmbedding (mean) -> PSHierarchicalSoftmax over
    64 Zipf classes; the label is the topic word's class, replaced by a uniform class with probability 0.1. The
    no-grad loss on fresh data falls from ~log 64 to near the conditional entropy of the label."""
    from multiverso_b200.ops import PSEmbedding, PSHierarchicalSoftmax
    mv = mv_device
    K, TOP, NOISE, D, BAG, EPS = 64, 4, 1000, 32, 8, 0.1
    p = _zipf(K)
    q = 1 - EPS + EPS / K
    H = -(q * math.log(q) + (K - 1) * (EPS / K) * math.log(EPS / K))
    emb_t = mv.MatrixTable(K * TOP + NOISE, D, "float32", updater="sgd", min_value=-0.5 / D, max_value=0.5 / D,
                           seed=2)
    out_t = mv.MatrixTable(K - 1, D, "float32", updater="sgd", init_value=0.0)
    emb = PSEmbedding(emb_t, push_scale=1000.0, mode="mean")
    hsm = PSHierarchicalSoftmax(out_t, p * 1e6, push_scale=20.0)
    gen = torch.Generator(device="cuda").manual_seed(0)
    pd = torch.from_numpy(p).cuda()

    def batch(B):
        y0 = torch.multinomial(pd, B, replacement=True, generator=gen)
        topic = y0 * TOP + torch.randint(0, TOP, (B,), device="cuda", generator=gen)
        noise = K * TOP + torch.randint(0, NOISE, (B, BAG - 1), device="cuda", generator=gen)
        flip = torch.rand(B, device="cuda", generator=gen) < EPS
        return torch.cat([topic[:, None], noise], 1), torch.where(
            flip, torch.randint(0, K, (B,), device="cuda", generator=gen), y0)

    def evaluate():
        ids, y = batch(8192)
        with torch.no_grad():
            return hsm(emb(ids), y).mean().item()

    start = evaluate()
    for _ in range(600):
        ids, y = batch(1024)
        hsm(emb(ids), y).mean().backward()
    end = evaluate()
    assert start > 2.0 and H - 0.05 < end < H + 0.25, (start, end, H)


def _hsm_kernels(fn, control):
    """hsm_fwd_kernel launches of fn, from a profiler session that runs fn and then `control`, a call that launches
    the kernel exactly once. A session without the control's launch recorded no kernel activity and proves nothing,
    so it is run again (at most 5 sessions); the count returned excludes the control's launch."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            control()
            torch.cuda.synchronize()
        n = sum(1 for e in prof.events() if "hsm_fwd_kernel" in e.name)
        if n:
            return n - 1
    raise AssertionError("5 profiler sessions recorded no hsm_fwd_kernel launch")


def test_errors_raise_without_launching(cuda):
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSHierarchicalSoftmax
    n, d = 1000, 32
    p = _zipf(n)
    W = torch.randn(n - 1, d, device=cuda)
    rm, keep, _ = _sharded(W, 1, 0)
    hsm = PSHierarchicalSoftmax(_fake_table(rm, n - 1, d), p)
    x = torch.randn(8, d, device=cuda)
    ok = torch.arange(8, device=cuda)
    def control():                                                     # launches the kernel exactly once
        hsm(x, ok)
    assert _hsm_kernels(control, control) == 1                         # the counter does see the op's kernel
    cases = [
        (ValueError, r"\[0, 1000\), got min 0 max 1000", x, torch.tensor([0, 1, 2, 3, 4, 6, 7, 1000], device=cuda)),
        (ValueError, "got min -3", x, torch.tensor([0, 1, 2, -3, 4, 6, 7, 9], device=cuda, dtype=torch.int32)),
        (TypeError, "int32 or int64", x, ok.float()),
        (ValueError, "hidden has 16 columns", torch.randn(8, 16, device=cuda), ok),
        (ValueError, "one label per row", x, ok[:7]),
        (TypeError, "2-D float32", x.half(), ok),
        (ValueError, "hidden must be too", x.cpu(), ok.cpu()),
    ]
    for exc, msg, h, y in cases:
        def call():
            with pytest.raises(exc, match=msg):
                hsm(h, y)
        assert _hsm_kernels(call, control) == 0, msg
    # the layer's refusals of the table
    wide, _, _ = _sharded(torch.zeros(4, 1028, device=cuda), 1, 0)
    with pytest.raises(ValueError, match="at most 1024"):
        PSHierarchicalSoftmax(_fake_table(wide, 4, 1028), np.ones(5))
    rm6 = N.RowMap()
    rm6.num_row, rm6.num_col, rm6.nservers, rm6.rows_per_server = n - 1, 34, 1, n - 1
    rm6.shard_ptrs[0] = W.data_ptr()
    with pytest.raises(ValueError, match="row pitch"):
        PSHierarchicalSoftmax(_fake_table(rm6, n - 1, 32), p)
    with pytest.raises(ValueError, match="need 999 inner-node rows"):
        PSHierarchicalSoftmax(_fake_table(rm, n - 2, d), p)
    # every error code of the entry point, each before any launch
    y, ln, L = hsm._check(x, ok)
    loss, _, ids, offsets, g, u = hsm._launch(x, y, ln, L, grad=True)

    def args(**kw):
        a = N.Hsm()
        a.wmap, a.dim, a.hidden, a.B, a.ldh = rm, d, x.data_ptr(), 8, d
        a.labels, a.n_classes = y.data_ptr(), n
        a.points, a.codes, a.lens, a.ldp = hsm.points.data_ptr(), hsm.codes.data_ptr(), hsm.lens.data_ptr(), hsm.depth
        a.offsets, a.loss, a.ids, a.g, a.u, a.ldu = offsets.data_ptr(), loss.data_ptr(), ids.data_ptr(), \
            g.data_ptr(), u.data_ptr(), d
        for k, v in kw.items():
            if k.startswith("map_"):
                setattr(a.wmap, k[4:], v)
            else:
                setattr(a, k, v)
        return a
    lib = N.cuda_lib()
    lib.mvb_hsm_fwd(args(), N.stream_ptr())
    cases = [(N.BAD_ROW_MAP, dict(map_nservers=0)), (N.BAD_ROW_MAP, dict(map_nservers=9)),
             (N.BAD_ROW_MAP, dict(map_rows_per_server=0)),
             (-80, dict(dim=0)), (-80, dict(dim=30)), (-80, dict(dim=1028)), (-80, dict(map_num_col=30)),
             (-81, dict(n_classes=1)), (-81, dict(n_classes=n + 1)), (-81, dict(ldp=0)), (-81, dict(ldp=65)),
             (-82, dict(B=-1)), (-82, dict(ldh=16)), (-82, dict(ldh=34)), (-82, dict(ldu=30)),
             (-83, dict(hidden=None)), (-83, dict(labels=None)), (-83, dict(points=None)), (-83, dict(codes=None)),
             (-83, dict(lens=None)), (-83, dict(offsets=None)), (-83, dict(hidden=x.data_ptr() + 4)),
             (-83, dict(u=u.data_ptr() + 8))]
    for rc, kw in cases:
        def call():
            with pytest.raises(N.NativeError, match=f"rc={rc}:"):
                lib.mvb_hsm_fwd(args(**kw), N.stream_ptr())
        assert _hsm_kernels(call, control) == 0, kw
    a = args(B=0)
    assert _hsm_kernels(lambda: lib.mvb_hsm_fwd(a, N.stream_ptr()), control) == 0


def test_hierarchical_softmax_peer_shards_multi_gpu():
    """A table sharded over 2 GPUs (tests/mp_hierarchical_softmax_check.py under torchrun): forward and dL/dhidden
    bitwise equal to a single-shard copy, async sgd pushes from every rank landing as W0 - lr * sum."""
    import os
    import subprocess
    import sys
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 1000
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_hierarchical_softmax_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == 2, tail
