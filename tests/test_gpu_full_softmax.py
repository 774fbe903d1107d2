"""Fused full softmax and inner-product top-k (csrc/cuda/topk_cos.cu, dot-product form) against fp64: the tf32 bound
of lse / loss, exact top-k outside near-ties, bitwise determinism, sharding and chunk independence of the top-k,
padded pitches, the row limit, empty batches, errors raised before any launch, and PSSampledSoftmax.evaluate after
training on a planted problem."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _fp64(W, X, rows):
    return X.double() @ W[:rows, :X.shape[1]].double().T


def _tol(W, X, rows, lse64):
    """The documented bound: 2^-10 ||x_b|| max_n ||w_n|| + 1e-5 (1 + |lse_fp64|)."""
    wmax = W[:rows, :X.shape[1]].double().norm(dim=1).max()
    return 2.0 ** -10 * X.double().norm(dim=1) * wmax + 1e-5 * (1 + lse64.abs())


def _check(W, X, y, k, rows, r):
    Z = _fp64(W, X, rows)
    lse64 = Z.logsumexp(1)
    tol = _tol(W, X, rows, lse64)
    err = (r.lse.double() - lse64).abs()
    assert (err <= tol).all(), (err / tol).max().item()
    if y is None:
        assert r.loss is None
    else:
        loss64 = lse64 - Z.gather(1, y[:, None].long())[:, 0]
        err = (r.loss.double() - loss64).abs()
        assert (err <= tol + 1e-6 * (1 + loss64.abs())).all(), (err / tol).max().item()
    if k == 0:
        assert r.scores is None and r.ids is None
        return
    s, i = r.scores, r.ids
    kk = min(k, rows)
    assert (i[:, kk:] == -1).all() and torch.isneginf(s[:, kk:]).all()
    got, sg = i[:, :kk], s[:, :kk]
    assert (got >= 0).all() and (got < rows).all()
    assert torch.equal(sg, Z.gather(1, got).float())                # fp64 dot products rounded to fp32
    assert (sg[:, 1:] <= sg[:, :-1]).all()
    tie = sg[:, 1:] == sg[:, :-1]
    assert (got[:, 1:][tie] > got[:, :-1][tie]).all()
    # outside near-ties (rows within the tf32 error of the k-th score) the ids are the fp64 top-k
    eps = (2.0 ** -10 * X.double().norm(dim=1) * W[:rows, :X.shape[1]].double().norm(dim=1).max())[:, None]
    kth = Z.topk(kk, dim=1).values[:, -1:]
    sure = Z > kth + eps
    member = torch.zeros_like(Z, dtype=torch.bool).scatter_(1, got, True)
    assert not (sure & ~member).any()
    assert (Z.gather(1, got) >= kth - eps).all()


def _data(cuda, B, N, d, pitch=None, seed=0, scale=0.35):
    g = torch.Generator(device=cuda).manual_seed(seed)
    pitch = pitch or (d + 3) // 4 * 4
    W = torch.randn(N, pitch, device=cuda, generator=g) * scale
    W[:, d:] = 0
    X = torch.randn(B, d, device=cuda, generator=g)
    y = torch.randint(0, N, (B,), device=cuda, generator=g)
    return W, X, y


@pytest.mark.parametrize("B,N,d,k,labels", [
    (1, 1000, 300, 10, True),             # one query
    (130, 100, 4, 1, True),               # N < 128, B crosses one query tile
    (200, 5003, 128, 0, True),            # loss only, N not a multiple of 128
    (77, 20000, 1024, 64, False),         # widest rows, the largest k
    (257, 129, 128, 64, True),            # one full tile and one row
    (3, 50, 100, 64, True),               # k > N: -1 / -inf slots
    (150, 3001, 300, 0, False),           # log-partition alone
    (4100, 3001, 100, 10, True),          # crosses the host chunk of 4096 queries
])
def test_matches_fp64(cuda, B, N, d, k, labels):
    from multiverso_b200.ops import full_softmax
    W, X, y = _data(cuda, B, N, d, seed=B + N + d)
    if not labels:
        y = None
    r = full_softmax(W, X, y, k=k)
    _check(W, X, y, k, N, r)
    assert not r.lse.requires_grad


def test_int32_labels_and_topk_dot(cuda):
    from multiverso_b200.ops import full_softmax, topk_dot
    W, X, y = _data(cuda, 300, 7777, 64, seed=3)
    r64 = full_softmax(W, X, y, k=12)
    r32 = full_softmax(W, X, y.int(), k=12)
    assert torch.equal(r64.loss, r32.loss) and torch.equal(r64.lse, r32.lse)
    s, i = topk_dot(W, X, 12)
    assert torch.equal(s, r64.scores) and torch.equal(i, r64.ids)
    _check(W, X, None, 12, 7777, types.SimpleNamespace(lse=r64.lse, loss=None, scores=s, ids=i))


def test_bitwise_repeatable(cuda):
    from multiverso_b200.ops import full_softmax
    W, X, y = _data(cuda, 600, 40000, 128, seed=5)
    a = full_softmax(W, X, y, k=10)
    b = full_softmax(W, X, y, k=10)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    c = full_softmax(W, X, y)
    assert torch.equal(a.lse, c.lse) and torch.equal(a.loss, c.loss)   # top-k on or off: same fold


def _sharded(W, S, gap=37):
    """W as S shards at separate places of one buffer, ``gap`` rows of garbage between them (the reference's
    rows_per_server rule, the last shard takes the remainder)."""
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


@pytest.mark.parametrize("n", [100003, 1003])
def test_sharded_topk_bitwise_lse_within_bound(cuda, n):
    from multiverso_b200.ops import full_softmax
    from multiverso_b200.ops.full_softmax import _device
    W, X, y = _data(cuda, 140, n, 300, seed=n)
    ref = full_softmax(W, X, y, k=16)
    Z = _fp64(W, X, n)
    lse64 = Z.logsumexp(1)
    tol = _tol(W, X, n, lse64)
    for S in (1, 2, 3, 8):
        rm, keep = _sharded(W, S, 0 if S == 1 else 37)
        r = _device(rm, W.shape[1], X, y, 16, n, True)
        torch.cuda.synchronize()
        assert torch.equal(r.ids, ref.ids) and torch.equal(r.scores, ref.scores), S
        assert ((r.lse.double() - lse64).abs() <= tol).all(), S
        assert ((r.loss.double() - ref.loss.double()).abs() <= 2 * tol).all(), S


def test_query_chunks(cuda):
    """A batch larger than one kernel call: every chunk gives the top-k a call of its own gives."""
    from multiverso_b200.ops import FullSoftmaxResult, full_softmax
    from multiverso_b200.ops.topk import _Q_CHUNK
    W, X, y = _data(cuda, _Q_CHUNK + 300, 20000, 64, seed=21)
    r = full_softmax(W, X, y, k=10)
    t = full_softmax(W, X[_Q_CHUNK:], y[_Q_CHUNK:], k=10)
    assert torch.equal(r.ids[_Q_CHUNK:], t.ids) and torch.equal(r.scores[_Q_CHUNK:], t.scores)
    _check(W, X[-300:], y[-300:], 10, 20000, FullSoftmaxResult(*(v[-300:] for v in r)))


def test_padded_pitch_and_row_limit(cuda):
    from multiverso_b200.ops import full_softmax, topk_dot
    g = torch.Generator(device=cuda).manual_seed(5)
    big = torch.randn(5000, 320, device=cuda, generator=g) * 0.3
    big[:, 300:] = 1e6 * torch.rand(5000, 20, device=cuda, generator=g)      # padding garbage must not count
    W = big[:, :300]                                                          # a column slice of a wider pitch
    X = torch.randn(33, 300, device=cuda, generator=g)
    for rows in (None, 1037):                                                 # 1037 ends inside a 128-row tile
        n = 5000 if rows is None else rows
        y = torch.randint(0, n, (33,), device=cuda, generator=g)
        r = full_softmax(W, X, y, k=20, rows=rows)
        _check(big, X, y, 20, n, r)
        s, i = topk_dot(W, X[:, :200], 5, rows=rows)                          # fewer columns than the row
        assert (i < n).all()
        _check(big, X[:, :200], None, 5, n, types.SimpleNamespace(lse=_fp64(big, X[:, :200], n).logsumexp(1).float(),
                                                                   loss=None, scores=s, ids=i))


def test_duplicates_and_zero_rows(cuda):
    from multiverso_b200.ops import full_softmax
    W, X, y = _data(cuda, 50, 3000, 32, seed=9)
    W[2345] = W[77]
    W[10:20] = 0
    X[0] = W[77] * 10
    r = full_softmax(W, X, y, k=10)
    assert r.ids[0, :2].tolist() == [77, 2345] and r.scores[0, 0] == r.scores[0, 1]
    _check(W, X, y, 10, 3000, r)


def _kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "topk_" in e.name)


def test_empty_batch_and_errors_without_launching(cuda):
    from multiverso_b200.ops import full_softmax, topk_dot
    W, X, y = _data(cuda, 8, 1000, 32, seed=1)
    assert _kernels(lambda: full_softmax(W, X, y, k=3)) == 2               # the counter sees the op's kernels

    def empty():
        r = full_softmax(W, X[:0], y[:0], k=5)
        assert r.lse.shape == (0,) and r.loss.shape == (0,) and r.scores.shape == (0, 5) and r.ids.shape == (0, 5)
        s, i = topk_dot(W, X[:0], 4)
        assert s.shape == (0, 4) and i.shape == (0, 4)
    assert _kernels(empty) == 0
    cases = [
        (TypeError, "2-D float32", lambda: full_softmax(W, X.double(), y)),
        (ValueError, "33 columns", lambda: full_softmax(W, torch.randn(8, 33, device=cuda), y)),
        (ValueError, r"k must be in \[0, 64\]", lambda: full_softmax(W, X, y, k=65)),
        (ValueError, r"k must be in \[0, 64\]", lambda: full_softmax(W, X, y, k=-1)),
        (ValueError, r"k must be in \[1, 64\]", lambda: topk_dot(W, X, 0)),
        (ValueError, r"\[0, 1000\)", lambda: full_softmax(W, X, torch.arange(993, 1001, device=cuda))),
        (ValueError, r"\[0, 500\)", lambda: full_softmax(W, X, y * 0 + 700, rows=500)),
        (ValueError, r"\[0, 1000\)", lambda: full_softmax(W, X, -1 - y)),
        (TypeError, "int32 or int64", lambda: full_softmax(W, X, y.float())),
        (ValueError, "one label per row", lambda: full_softmax(W, X, y[:7])),
        (ValueError, r"rows=0 outside \[1, 1000\]", lambda: full_softmax(W, X, rows=0)),
        (ValueError, r"rows=1001 outside \[1, 1000\]", lambda: topk_dot(W, X, 3, rows=1001)),
        (ValueError, "multiple of 4", lambda: full_softmax(torch.randn(100, 30, device=cuda), X[:, :30])),
        (ValueError, "must be too", lambda: full_softmax(W, X.cpu(), y)),
    ]
    for exc, msg, f in cases:
        def call():
            with pytest.raises(exc, match=msg):
                f()
        assert _kernels(call) == 0, msg


def _fake_table(rm, num_row, num_col):
    from multiverso_b200 import _native as N
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=num_row, num_col=num_col,
                                 updater=N.UPD_SGD, is_sparse=False,
                                 rt=types.SimpleNamespace(device=torch.device("cuda", 0)))


def test_sampled_softmax_evaluate_after_training(cuda):
    """A planted problem: hidden = 3 * prototype of the label + noise. A few steps of PSSampledSoftmax lower the exact
    full-softmax cross-entropy, which evaluate() gives as fp64 does over the table's rows; evaluate draws nothing."""
    from multiverso_b200.ops import PSSampledSoftmax
    g = torch.Generator(device=cuda).manual_seed(7)
    n, d, B = 3000, 32, 512
    P = torch.randn(n, d, device=cuda, generator=g) / d ** 0.5
    W0 = torch.randn(n, d, device=cuda, generator=g) * 0.01
    rm, buf = _sharded(W0, 3)
    ssm = PSSampledSoftmax(_fake_table(rm, n, d), num_sampled=256, sampler="log_uniform", push_scale=0.5, seed=3)

    def batch():
        y = torch.randint(0, n, (B,), device=cuda, generator=g)
        return 3 * P[y] + 0.1 * torch.randn(B, d, device=cuda, generator=g), y

    xe, ye = batch()
    before = ssm.evaluate(xe, ye)
    for _ in range(30):
        x, y = batch()
        ssm(x, y).sum().backward()
    torch.cuda.synchronize()
    steps = ssm.steps
    after = ssm.evaluate(xe, ye, k=5)
    assert ssm.steps == steps and not after.loss.requires_grad
    rps = n // 3
    W = torch.cat([buf[37 * (s + 1) + s * rps: 37 * (s + 1) + (n if s == 2 else (s + 1) * rps)] for s in range(3)])
    _check(W, xe, ye, 5, n, after)
    print(f"full-softmax cross-entropy {before.loss.mean().item():.3f} -> {after.loss.mean().item():.3f}")
    assert after.loss.mean() < before.loss.mean() - 0.5
    with pytest.raises(ValueError, match="hidden has 16 columns"):
        ssm.evaluate(xe[:, :16], ye)
