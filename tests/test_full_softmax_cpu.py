"""full_softmax / topk_dot without a GPU: full_softmax_reference against a brute-force fp64 logsumexp and top-k
(row limit, k beyond the rows, ties on duplicated rows, zero rows), the host-backend table and
PSSampledSoftmax.evaluate against the reference, and every documented error."""
import pytest
import torch

from multiverso_b200.ops import FullSoftmaxResult, PSSampledSoftmax, full_softmax, full_softmax_reference, topk_dot


def _brute(W, X, y, k, rows):
    """fp64 logits, then logsumexp, loss and the k best by (fp32 score desc, id asc) by a full sort."""
    Z = X.double() @ W[:rows, :X.shape[1]].double().T
    lse = Z.logsumexp(1)
    loss = None if y is None else (lse - Z[torch.arange(X.shape[0]), y]).float()
    s32 = Z.float()
    ids = torch.arange(rows).expand_as(s32)
    o = torch.argsort(ids, dim=1, stable=True)
    o = torch.argsort(-s32.gather(1, o), dim=1, stable=True)
    kk = min(k, rows)
    best_i = torch.full((X.shape[0], k), -1, dtype=torch.int64)
    best_s = torch.full((X.shape[0], k), float("-inf"))
    best_i[:, :kk] = o[:, :kk]
    best_s[:, :kk] = s32.gather(1, o[:, :kk])
    return lse.float(), loss, best_s, best_i


def _data(N=700, width=20, B=9, seed=0):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(N, width, generator=g)
    X = torch.randn(B, width - 3, generator=g)
    y = torch.randint(0, N, (B,), generator=g)
    return W, X, y


@pytest.mark.parametrize("k,rows", [(0, None), (1, None), (10, 333), (64, 40), (5, 1)])
def test_reference_matches_brute_force(k, rows):
    W, X, y = _data()
    n = rows or W.shape[0]
    y = y % n
    r = full_softmax_reference(W, X, y, k=k, rows=rows, row_chunk=128)       # several row chunks
    lse, loss, s, i = _brute(W, X, y, k, n)
    assert torch.allclose(r.lse, lse, rtol=1e-6, atol=1e-6)
    assert torch.allclose(r.loss, loss, rtol=1e-6, atol=1e-6)
    if k == 0:
        assert r.scores is None and r.ids is None
    else:
        assert torch.equal(r.ids, i) and torch.equal(r.scores, s)
        assert (r.ids[:, min(k, n):] == -1).all() and torch.isneginf(r.scores[:, min(k, n):]).all()


def test_reference_ties_and_zero_rows():
    W, X, y = _data(N=300)
    W[200] = W[17]
    W[250] = W[17]
    W[30:40] = 0
    X[0] = W[17, :17] * 3
    r = full_softmax_reference(W, X, y, k=8, row_chunk=64)
    assert r.ids[0, :3].tolist() == [17, 200, 250] and r.scores[0, 0] == r.scores[0, 2]
    lse, loss, s, i = _brute(W, X, y, 8, 300)
    assert torch.equal(r.ids, i) and torch.equal(r.scores, s)
    Z = torch.zeros(5, 8)
    r = full_softmax_reference(Z, torch.randn(2, 8), torch.tensor([0, 4]), k=7)
    assert torch.allclose(r.lse, torch.full((2,), float(torch.log(torch.tensor(5.0)))))
    assert r.ids[:, :5].tolist() == [[0, 1, 2, 3, 4]] * 2 and (r.ids[:, 5:] == -1).all()


def test_cpu_tensor_calls_equal_reference():
    W, X, y = _data(seed=4)
    y = y % 500
    ref = full_softmax_reference(W, X, y, k=6, rows=500)
    r = full_softmax(W, X, y.int(), k=6, rows=500)
    for a, b in zip(r, ref):
        assert torch.equal(a, b)
    s, i = topk_dot(W, X, 6, rows=500)
    assert torch.equal(s, ref.scores) and torch.equal(i, ref.ids)
    r = full_softmax(W, X[:0], y[:0], k=3)
    assert isinstance(r, FullSoftmaxResult) and r.lse.shape == (0,) and r.loss.shape == (0,)
    assert r.scores.shape == (0, 3) and r.ids.shape == (0, 3)
    assert full_softmax(W, X).loss is None


@pytest.fixture
def mv_host():
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.init()
    yield mv
    mv.shutdown(finalize_net=False)
    mv.FLAGS.reset()


def test_host_table_and_evaluate(mv_host):
    W, X, y = _data(N=1000, width=16, seed=7)
    X = torch.randn(9, 16)
    t = mv_host.MatrixTable(1000, 16, "float32")
    t.add(W.numpy())
    Wt = torch.as_tensor(t.get()).view(1000, 16).clone()
    ref = full_softmax_reference(Wt, X, y, k=5)
    r = full_softmax(t, X, y, k=5)
    for a, b in zip(r, ref):
        assert torch.equal(a, b)
    s, i = topk_dot(t, X, 5)
    assert torch.equal(s, ref.scores) and torch.equal(i, ref.ids)
    ssm = PSSampledSoftmax(t, num_sampled=50, sampler="log_uniform", push_scale=None)
    steps = ssm.steps
    e = ssm.evaluate(X.requires_grad_(), y, k=5)
    assert ssm.steps == steps and not e.loss.requires_grad
    for a, b in zip(e, ref):
        assert torch.equal(a, b)
    with pytest.raises(ValueError, match="hidden has 12 columns"):
        ssm.evaluate(X[:, :12], y)


def test_errors():
    W, X, y = _data()
    cases = [
        (TypeError, "2-D float32", lambda: full_softmax(W, X.double(), y)),
        (TypeError, "2-D float32", lambda: full_softmax(W, X[0], y)),
        (TypeError, "2-D float32", lambda: full_softmax(W.double(), X, y)),
        (ValueError, "21 columns", lambda: full_softmax(W, torch.randn(9, 21), y)),
        (ValueError, r"k must be in \[0, 64\], got 65", lambda: full_softmax(W, X, y, k=65)),
        (ValueError, r"k must be in \[0, 64\], got -1", lambda: full_softmax_reference(W, X, y, k=-1)),
        (ValueError, r"k must be in \[1, 64\], got 0", lambda: topk_dot(W, X, 0)),
        (ValueError, r"k must be in \[1, 64\], got 65", lambda: topk_dot(W, X, 65)),
        (ValueError, r"labels must be in \[0, 700\)", lambda: full_softmax(W, X, y + 700)),
        (ValueError, r"labels must be in \[0, 700\)", lambda: full_softmax(W, X, y - 700)),
        (ValueError, r"labels must be in \[0, 10\)", lambda: full_softmax(W, X, y, rows=10)),
        (TypeError, "int32 or int64", lambda: full_softmax(W, X, y.float())),
        (ValueError, "one label per row", lambda: full_softmax(W, X, y[:3])),
        (ValueError, "one label per row", lambda: full_softmax(W, X, y[:, None])),
        (ValueError, r"rows=0 outside \[1, 700\]", lambda: full_softmax(W, X, rows=0)),
        (ValueError, r"rows=701 outside \[1, 700\]", lambda: topk_dot(W, X, 3, rows=701)),
        (ValueError, r"rows=701 outside \[1, 700\]", lambda: full_softmax_reference(W, X, rows=701)),
    ]
    for exc, msg, f in cases:
        with pytest.raises(exc, match=msg):
            f()
