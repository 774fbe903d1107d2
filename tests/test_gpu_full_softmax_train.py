"""PSFullSoftmax on the device (csrc/cuda/full_softmax_bwd.cu) against fp64: dX and dW of the fused backward within
the documented bound at tile, width and class edges, bitwise determinism and sharding independence of dW, the table
after one step of sgd / adagrad / adam, a planted problem, host synchronisations, the kernels each backward launches
and errors raised before any launch."""
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu

T = 2.0 ** -10            # tf32 truncation of one operand


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _data(dev, B, n, d, seed, same_label=False):
    gen = torch.Generator().manual_seed(seed)
    W = (torch.randn(n, d, generator=gen) * (2.0 / d ** 0.5)).to(dev)
    X = torch.randn(B, d, generator=gen).to(dev)
    y = torch.full((B,), n // 2, dtype=torch.int64) if same_label else torch.randint(0, n, (B,), generator=gen)
    g = torch.randn(B, generator=gen)
    g[4::5] = 0.0                         # every fifth query, so that B = 1 still has a gradient
    return W, X, y.to(dev), g.to(dev)


def _sharded(W, S, gap=37):
    """W as S shards at separate places of one buffer, ``gap`` rows of garbage between them."""
    from multiverso_b200 import _native as N
    n, pitch = W.shape
    rps = n // S
    buf = torch.full((n + S * gap, pitch), 1e3, device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, rps
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
    return rm, buf


def _run(rm, X, y, lse, g, scale=1.0, dq=True, dw=True):
    from multiverso_b200.ops.full_softmax import full_softmax_bwd
    from multiverso_b200.ops.topk import padded_queries
    B, d = X.shape
    q = padded_queries(X)
    dX = torch.full((B, d), float("nan"), device=X.device) if dq else None
    dW = torch.full((rm.num_row, rm.num_col), float("nan"), device=X.device) if dw else None
    full_softmax_bwd(rm, q, d, y, lse, g, dX, dW, scale)
    torch.cuda.synchronize()
    return dX, dW


def _bounds(W, X, y, g, lse32, scale, e_z=None):
    """fp64 dX, dW and the documented element bounds (see PSFullSoftmax's docstring). ``e_z``: the logit error, by
    default the tf32 one; 0 for operands that tf32 represents exactly with exact fp32 partial sums."""
    W64, X64, g64 = W.double(), X.double(), g.double()
    Z = X64 @ W64.T
    lse64 = Z.logsumexp(1)
    P = torch.exp(Z - lse64[:, None])
    G = g64[:, None] * P
    G[torch.arange(len(y)), y] -= g64
    dX, dW = G @ W64, scale * (G.T @ X64)
    wmax = W64.norm(dim=1).max()
    if e_z is None:
        e_z = 2 * T * X64.norm(dim=1) * wmax + 1e-6
    e_lse = (lse32.double() - lse64).abs()
    f = (2 * e_z + e_lse + 2 * T)[:, None]                                  # [B, 1]
    n, B = W.shape[0], X.shape[0]
    U = 2.0 ** -24                                                          # fp32 accumulation over N (dX), B (dW)
    Y = torch.zeros_like(P)
    Y[torch.arange(len(y)), y] = 1.0
    bx = g64.abs()[:, None] * ((1.1 * f + n * U) * (P @ W64.abs()) + (2 * T + n * U) * W64[y].abs()) + 1e-6
    bw = abs(scale) * ((g64.abs()[:, None] * ((1.1 * f + B * U) * P + (2 * T + B * U) * Y)).T @ X64.abs()) \
        + 1e-6 * abs(scale)
    return dX, dW, bx, bw


CASES = [(1, 1000, 300), (130, 100, 4), (200, 5003, 128), (257, 129, 128), (77, 20000, 1024), (4100, 3001, 100),
         (64, 1000003, 128)]


@pytest.mark.parametrize("B,n,d", CASES)
@pytest.mark.parametrize("same_label", [False, True])
def test_kernel_vs_fp64(cuda, B, n, d, same_label):
    from multiverso_b200.ops import full_softmax
    W, X, y, g = _data(cuda, B, n, d, seed=B + n + d, same_label=same_label)
    lse = full_softmax(W, X).lse
    rm, _ = _sharded(W, 1, 0)
    dX, dW = _run(rm, X, y, lse, g, scale=0.5)
    dX64, dW64, bx, bw = _bounds(W, X, y, g, lse, 0.5)
    ex = (dX.double() - dX64).abs()
    ew = (dW.double() - dW64).abs()
    assert not torch.isnan(dX).any() and not torch.isnan(dW).any()
    assert (ex <= bx).all(), (ex / bx).max().item()
    assert (ew <= bw).all(), (ew / bw).max().item()


def test_deterministic_and_sharding(cuda):
    from multiverso_b200.ops import full_softmax
    B, n, d = 300, 20011, 200
    W, X, y, g = _data(cuda, B, n, d, seed=5)
    lse = full_softmax(W, X).lse
    rm, keep = _sharded(W, 1, 0)
    dX0, dW0 = _run(rm, X, y, lse, g, scale=-0.25)
    dX1, dW1 = _run(rm, X, y, lse, g, scale=-0.25)
    assert torch.equal(dX0, dX1) and torch.equal(dW0, dW1)
    _, _, bx, _ = _bounds(W, X, y, g, lse, -0.25)
    dX64 = _bounds(W, X, y, g, lse, -0.25)[0]
    for S in (2, 3, 8):
        rm, keep = _sharded(W, S)
        dX, dW = _run(rm, X, y, lse, g, scale=-0.25)
        assert torch.equal(dW, dW0), S
        assert ((dX.double() - dX64).abs() <= bx).all(), S


def test_int32_labels_layer(mv_device):
    mv = mv_device
    n, d, B = 3000, 64, 200
    _, X, y, _ = _data(torch.device("cuda"), B, n, d, seed=3)
    outs = []
    for yy in (y, y.to(torch.int32)):
        t = mv.MatrixTable(n, d, "float32", updater="sgd", min_value=-0.5, max_value=0.5, seed=3)
        fsm = mv.ops.PSFullSoftmax(t, push_scale=0.1)
        x = X.clone().requires_grad_()
        loss = fsm(x, yy)
        loss.sum().backward()
        torch.cuda.synchronize()
        outs.append((loss.detach(), x.grad, t.get().clone()))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


@pytest.mark.parametrize("updater", ["sgd", "adagrad", "adam"])
def test_table_step_equals_staged_delta(mv_device, updater):
    """The table after one step equals a twin given the recorded staged delta through add; sgd also against fp64
    and against the PSLinear + cross_entropy arm."""
    mv = mv_device
    from multiverso_b200.ops import full_softmax
    from multiverso_b200.tables.options import AddOption
    n, d, B, lr = 4000, 128, 300, 0.5
    _, X, y, g = _data(torch.device("cuda"), B, n, d, seed=7)
    opt = AddOption(momentum=0.9, learning_rate=lr, rho=0.1)
    t, twin = (mv.MatrixTable(n, d, "float32", updater=updater, min_value=-0.5, max_value=0.5, seed=11)
               for _ in range(2))
    Wt = t.get().clone().view(n, d)
    assert torch.equal(Wt.view(-1), twin.get())
    fsm = mv.ops.PSFullSoftmax(t, push_scale=lr, option=opt)
    x = X.clone().requires_grad_()
    recorded = []
    orig = t.add_async

    def rec(delta=None, option=None, staged=False):
        recorded.append(t._cur_stage.tensor(torch.float32, t.size).clone())
        return orig(delta, option, staged)
    t.add_async = rec
    (fsm(x, y) * g).sum().backward()
    torch.cuda.synchronize()
    assert len(recorded) == 1
    twin.add(recorded[0], opt)
    torch.cuda.synchronize()
    assert torch.equal(t.get(), twin.get())
    if updater != "sgd":
        return
    lse = full_softmax(Wt, X).lse
    _, dW64, _, bw = _bounds(Wt, X, y, g, lse, lr)
    got = t.get().view(n, d).double()
    slack = 2.0 ** -23 * Wt.double().abs()                  # the fp32 rounding of the step
    err = (got - (Wt.double() - dW64)).abs()
    assert (err <= bw + slack).all(), (err / bw).max().item()
    # the unfused arm: PSLinear + cross_entropy from the same initial table
    t2 = mv.MatrixTable(n, d, "float32", updater="sgd", min_value=-0.5, max_value=0.5, seed=11)
    lin = mv.ops.PSLinear(t2, push_scale=lr)
    loss = torch.nn.functional.cross_entropy(lin(X.clone().requires_grad_()), y, reduction="none")
    (loss * g).sum().backward()
    torch.cuda.synchronize()
    err = (t2.get().view(n, d).double() - got).abs()
    assert (err <= 2 * bw + 2 * slack).all(), (err / bw).max().item()


def test_planted_problem_learns(mv_device):
    mv = mv_device
    n, d, B = 1000, 32, 512
    gen = torch.Generator().manual_seed(1)
    proto = torch.randn(n, d, generator=gen)
    y = torch.randint(0, n, (B,), generator=gen)
    X = (proto[y] + 0.1 * torch.randn(B, d, generator=gen)).cuda()
    y = y.cuda()
    t = mv.MatrixTable(n, d, "float32", updater="sgd")
    fsm = mv.ops.PSFullSoftmax(t, push_scale=0.05)
    losses = []
    for _ in range(6):
        loss = fsm(X, y)
        loss.sum().backward()
        losses.append(fsm.evaluate(X, y).loss.mean().item())
    assert losses[-1] < 0.5 * losses[0], losses


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        try:
            torch.cuda.set_sync_debug_mode("warn")
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def test_host_syncs_and_empty_batch(mv_device):
    mv = mv_device
    t = mv.MatrixTable(4000, 64, "float32", updater="sgd")
    fsm = mv.ops.PSFullSoftmax(t, push_scale=0.1)
    x = torch.randn(300, 64, device="cuda", requires_grad=True)
    y = torch.randint(0, 4000, (300,), device="cuda")
    out = []
    assert _syncs(lambda: out.append(fsm(x, y))) == 1
    assert _syncs(lambda: out[0].mean().backward()) == 0
    # empty batch: an empty loss and one zero Add
    before = t.get().clone()
    calls = []
    orig = t.add_async
    t.add_async = lambda *a, **k: (calls.append(t._cur_stage.tensor(torch.float32, t.size).clone()), orig(*a, **k))[1]
    loss = fsm(torch.zeros(0, 64, device="cuda", requires_grad=True), torch.zeros(0, dtype=torch.int64, device="cuda"))
    assert loss.shape == (0,)
    loss.sum().backward()
    torch.cuda.synchronize()
    assert len(calls) == 1 and not calls[0].any()
    assert torch.equal(t.get(), before)


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in p.events() if e.device_type.name == "CUDA"]


def test_passes_launched(mv_device):
    """No dX pass without requires_grad; no dW pass and no Add with push_scale=None."""
    mv = mv_device
    t = mv.MatrixTable(3000, 64, "float32", updater="sgd")
    y = torch.randint(0, 3000, (200,), device="cuda")
    x0 = torch.randn(200, 64, device="cuda")
    seen = {}
    for push, grad in ((0.1, True), (0.1, False), (None, True)):
        fsm = mv.ops.PSFullSoftmax(t, push_scale=push)
        x = x0.clone().requires_grad_(grad)
        loss = fsm(x, y).sum()
        names = _kernels(loss.backward)
        seen[push, grad] = set(names)
        assert sum("fsm_bwd_kernel<false>" in k for k in names) == (1 if grad else 0), names
        assert sum("fsm_bwd_kernel<true>" in k for k in names) == (1 if push is not None else 0), names
    # push_scale=None launches a subset of the full backward: no dW pass and no Add kernel
    assert seen[None, True] < seen[0.1, True]
    extra = seen[0.1, True] - seen[None, True]
    assert len([k for k in extra if "fsm_" not in k]) >= 1, extra


def test_errors_before_launch(mv_device):
    mv = mv_device
    from multiverso_b200 import _native as N
    t = mv.MatrixTable(300, 64, "float32", updater="sgd")
    fsm = mv.ops.PSFullSoftmax(t, push_scale=0.1)
    x = torch.randn(10, 64, device="cuda")
    x32, xc, xd = x[:, :32].contiguous(), x.cpu(), x.double()
    y0, yc, ybad = (torch.zeros(10, dtype=torch.int64, device="cuda"), torch.zeros(10, dtype=torch.int64),
                    torch.full((10,), 300, dtype=torch.int64, device="cuda"))
    cases = [
        lambda: fsm(x32, y0),
        lambda: fsm(xc, yc),
        lambda: fsm(x, ybad),
        lambda: fsm(xd, y0),
        lambda: mv.ops.PSFullSoftmax(mv.MatrixTable(30, 8, "float64")),
        lambda: mv.ops.PSFullSoftmax(mv.MatrixTable(30, 8, "float32", is_sparse=True)),
        lambda: mv.ops.PSFullSoftmax(mv.MatrixTable(30, 6, "float32")),
        lambda: mv.ops.PSFullSoftmax(mv.HashMatrixTable(64, 8)),
    ]
    for i, c in enumerate(cases):
        names = []
        try:
            names = _kernels(lambda: pytest.raises((TypeError, ValueError), c))
        except Exception as e:          # construction of the refused table itself may launch its init
            raise AssertionError(f"case {i}: {e!r}")
        if i in (0, 1, 3):
            assert not names, (i, names)
        elif i == 2:                    # the label range check is the forward's one device read
            assert not any("fsm_" in k or "topk" in k for k in names), names
    # the C entry point: bad row map and every argument error before any CUDA call
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = 300, 64, 0, 300
    a = N.FullSoftmaxBwd()
    a.M, a.ldq, a.dim, a.wmap = 10, 64, 64, rm
    with pytest.raises(N.NativeError, match="rc=-70"):
        N.cuda_lib().mvb_full_softmax_bwd(a, 0)
    # every other argument error, each from an otherwise valid call, with no kernel launched
    W = torch.randn(300, 64, device="cuda")
    q = torch.randn(10, 64, device="cuda")
    yy = torch.zeros(10, dtype=torch.int64, device="cuda")
    lse, gg = torch.zeros(10, device="cuda"), torch.ones(10, device="cuda")
    dq, dw = torch.empty(10, 64, device="cuda"), torch.empty(300, 64, device="cuda")
    lib = N.cuda_lib()
    scratch = torch.empty(lib.mvb_full_softmax_bwd_scratch_bytes(10, 64, 300, 1, 1), dtype=torch.uint8, device="cuda")

    def call(**kw):
        rm = N.RowMap()
        rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = kw.get("num_row", 300), kw.get("num_col", 64), 1, 300
        rm.shard_ptrs[0] = W.data_ptr()
        a = N.FullSoftmaxBwd()
        a.q, a.M, a.ldq, a.dim, a.wmap = q.data_ptr(), kw.get("M", 10), kw.get("ldq", 64), kw.get("dim", 64), rm
        a.labels, a.lse, a.g = yy.data_ptr(), lse.data_ptr(), kw.get("g", gg.data_ptr())
        a.dq, a.lddq = kw.get("dq", dq.data_ptr()), kw.get("lddq", 64)
        a.dw, a.lddw, a.scale = kw.get("dw", dw.data_ptr()), kw.get("lddw", 64), 1.0
        a.scratch, a.scratch_bytes = scratch.data_ptr(), kw.get("scratch_bytes", scratch.numel())
        lib.mvb_full_softmax_bwd(a, N.stream_ptr())
    bad = [(-42, dict(ldq=62)), (-42, dict(num_col=62)), (-43, dict(dim=0)), (-43, dict(dim=68, ldq=68)),
           (-44, dict(num_row=0)), (-45, dict(M=-1)), (-45, dict(scratch_bytes=16)), (-46, dict(dq=None, dw=None)),
           (-46, dict(g=None)), (-47, dict(lddq=32, dim=64)), (-47, dict(lddw=32))]
    for rc, kw in bad:
        names = _kernels(lambda: pytest.raises(N.NativeError, call, **kw))
        assert not names, (rc, kw, names)
        with pytest.raises(N.NativeError, match=f"rc={rc}:"):
            call(**kw)
    call()                                                  # the same call with valid arguments runs
    torch.cuda.synchronize()
