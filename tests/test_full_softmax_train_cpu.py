"""PSFullSoftmax without a GPU: the fp64 host formula against torch autograd of F.cross_entropy, row chunking, one sgd
step against PSLinear + cross_entropy on the host backend, and every refusal."""
import pytest
import torch
import torch.nn.functional as F


def _data(B, n, d, seed):
    gen = torch.Generator().manual_seed(seed)
    W = torch.randn(n, d, generator=gen) * (2.0 / d ** 0.5)
    X = torch.randn(B, d, generator=gen)
    y = torch.randint(0, n, (B,), generator=gen)
    g = torch.randn(B, generator=gen)
    g[::3] = 0.0
    g[1::4] = -g[1::4].abs()
    return W, X, y, g


@pytest.mark.parametrize("B,n,d", [(1, 7, 4), (33, 500, 12), (64, 1000, 8)])
def test_reference_matches_autograd(B, n, d):
    from multiverso_b200.ops import full_softmax_grad_reference
    W, X, y, g = _data(B, n, d, seed=B + n)
    W64, X64 = W.double().requires_grad_(), X.double().requires_grad_()
    loss64 = F.cross_entropy(X64 @ W64.T, y, reduction="none")
    (loss64 * g.double()).sum().backward()
    loss, dX, dW = full_softmax_grad_reference(W, X, y, g, row_chunk=97)
    assert torch.allclose(loss, loss64.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(dX, X64.grad, rtol=1e-10, atol=1e-12)
    assert torch.allclose(dW, W64.grad, rtol=1e-10, atol=1e-12)


def test_row_chunks_agree():
    from multiverso_b200.ops import full_softmax_grad_reference
    W, X, y, g = _data(40, 1000, 16, seed=2)
    one = full_softmax_grad_reference(W, X, y, g, row_chunk=1 << 20)
    for chunk in (1, 7, 128):
        got = full_softmax_grad_reference(W, X, y, g, row_chunk=chunk)
        for a, b in zip(one, got):
            assert torch.allclose(a, b, rtol=1e-12, atol=1e-13), chunk


@pytest.fixture
def host_mv():
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.init()
    yield mv
    mv.shutdown(finalize_net=False)
    mv.FLAGS.reset()


def test_host_layer_matches_autograd_and_pslinear(host_mv):
    mv = host_mv
    n, d, B, lr = 300, 12, 50, 0.25
    W, X, y, g = _data(B, n, d, seed=9)
    t = mv.MatrixTable(n, d, "float32", init_value=W.numpy())
    W0 = torch.as_tensor(t.get()).clone()
    fsm = mv.ops.PSFullSoftmax(t, push_scale=-lr)           # the default updater adds: -lr is a descent step
    x = X.clone().requires_grad_()
    loss = fsm(x, y)
    (loss * g).sum().backward()
    W64, X64 = W0.double().requires_grad_(), X.double().requires_grad_()
    loss64 = F.cross_entropy(X64 @ W64.T, y, reduction="none")
    (loss64 * g.double()).sum().backward()
    assert torch.allclose(loss.double(), loss64.detach(), rtol=1e-6, atol=1e-6)
    assert torch.allclose(x.grad.double(), X64.grad, rtol=1e-6, atol=1e-7)
    W1 = torch.as_tensor(t.get()).double()
    assert torch.allclose(W1, (W0.double() - lr * W64.grad), rtol=0, atol=1e-6)
    # one step of PSLinear + cross_entropy from the same table
    t2 = mv.MatrixTable(n, d, "float32", init_value=W.numpy())
    lin = mv.ops.PSLinear(t2, push_scale=-lr)
    (F.cross_entropy(lin(X.clone().requires_grad_()), y, reduction="none") * g).sum().backward()
    W2 = torch.as_tensor(t2.get()).double()
    assert torch.allclose(W1, W2, rtol=0, atol=4 * 2.0 ** -24 * (1 + W1.abs().max().item()))
    # evaluate is the full softmax, and an empty batch still pushes one (zero) Add
    r = fsm.evaluate(X, y, k=3)
    assert r.ids.shape == (B, 3)
    before = torch.as_tensor(t.get()).clone()
    e = fsm(torch.zeros(0, d, requires_grad=True), torch.zeros(0, dtype=torch.int64))
    assert e.shape == (0,)
    e.sum().backward()
    assert torch.equal(torch.as_tensor(t.get()), before)


def test_push_scale_none_pushes_nothing(host_mv):
    mv = host_mv
    W, X, y, _ = _data(20, 50, 8, seed=4)
    t = mv.MatrixTable(50, 8, "float32", init_value=W.numpy())
    before = torch.as_tensor(t.get()).clone()
    fsm = mv.ops.PSFullSoftmax(t, push_scale=None)
    x = X.clone().requires_grad_()
    fsm(x, y).sum().backward()
    assert x.grad is not None
    assert torch.equal(torch.as_tensor(t.get()), before)


def test_refusals(host_mv):
    mv = host_mv
    t = mv.MatrixTable(30, 8, "float32")
    fsm = mv.ops.PSFullSoftmax(t, push_scale=0.1)
    with pytest.raises(TypeError):
        mv.ops.PSFullSoftmax(torch.zeros(30, 8))
    with pytest.raises(TypeError):
        mv.ops.PSFullSoftmax(mv.MatrixTable(30, 8, "float64"))
    with pytest.raises(ValueError, match="is_sparse"):
        mv.ops.PSFullSoftmax(mv.MatrixTable(30, 8, "float32", is_sparse=True))
    with pytest.raises(ValueError, match="columns"):
        fsm(torch.zeros(4, 6), torch.zeros(4, dtype=torch.int64))
    with pytest.raises(TypeError):
        fsm(torch.zeros(4, 8, dtype=torch.float64), torch.zeros(4, dtype=torch.int64))
    with pytest.raises(ValueError, match="labels"):
        fsm(torch.zeros(4, 8), torch.full((4,), 30, dtype=torch.int64))
    with pytest.raises(TypeError, match="labels"):
        fsm(torch.zeros(4, 8), torch.zeros(4))


def test_device_refusals_without_gpu():
    """The device-only refusals are checked from the table's attributes, before anything touches a GPU."""
    from types import SimpleNamespace
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFullSoftmax
    from multiverso_b200.tables.device import HashMatrixTable
    with pytest.raises(TypeError, match="HashMatrixTable"):
        PSFullSoftmax(HashMatrixTable.__new__(HashMatrixTable))
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = 30, 6, 1, 30
    fake = SimpleNamespace(num_row=30, num_col=6, dtype=torch.float32, is_sparse=False, _rowmap=rm,
                           rt=SimpleNamespace(device=torch.device("cuda", 0)))
    with pytest.raises(ValueError, match="multiple of 4"):
        PSFullSoftmax(fake)
    rm.num_col = 8
    fake.num_col = 8
    fsm = PSFullSoftmax(fake)
    with pytest.raises(ValueError, match="GPU"):
        fsm(torch.zeros(4, 8), torch.zeros(4, dtype=torch.int64))
