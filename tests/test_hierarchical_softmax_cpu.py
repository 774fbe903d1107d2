"""PSHierarchicalSoftmax without a GPU: the normalisation of the fp64 reference over every label, the host layer's loss,
dL/dhidden and pushed node gradient against fp64 autograd of the path formula written out step by step, one sgd step
on the host backend, one coalesced add_rows for a stateful table, and every refusal."""
import types

import numpy as np
import pytest
import torch


def _fib(n):
    f = [1, 1]
    while len(f) < n:
        f.append(f[-1] + f[-2])
    return np.array(f[:n], dtype=np.float64)


def _counts(kind, n):
    if kind == "zipf":
        return 1.0 / np.arange(1, n + 1)
    if kind == "equal":
        return np.full(n, 7.0)
    return _fib(n)


class _HostTable:
    """What the layer reads of a host-backend table, with every add_rows recorded."""

    def __init__(self, W, updater="adagrad"):
        self.W, self.num_row, self.num_col = W, W.shape[0], W.shape[1]
        self.npdt, self.updater, self.adds = np.float32, updater, []

    def get_rows(self, ids):
        return self.W[torch.from_numpy(np.asarray(ids))].numpy()

    def add_rows(self, ids, vals, option=None):
        self.adds.append((np.array(ids), np.array(vals), option))


def _path_formula(W64, x64, y, counts):
    """The loss [B] as the sum over each label's path, one step at a time, from the encoder's tables."""
    from multiverso_b200.models.wordembedding import HuffmanTables
    P, Cd, lens, _ = HuffmanTables.encode(counts)
    out = []
    for b, lab in enumerate(y.tolist()):
        terms = [torch.nn.functional.softplus(-(1.0 - 2.0 * float(Cd[lab, i])) * (x64[b] @ W64[int(P[lab, i])]))
                 for i in range(int(lens[lab]))]
        out.append(torch.stack(terms).sum())
    return torch.stack(out)


@pytest.mark.parametrize("n", [2, 3, 5, 1000])
@pytest.mark.parametrize("kind", ["zipf", "equal", "fib"])
def test_reference_is_normalised(kind, n):
    """exp(-loss) over all N labels sums to 1 for any hidden vector and any table."""
    from multiverso_b200.ops import hierarchical_softmax_reference
    from multiverso_b200.ops.hierarchical_softmax import huffman_tree
    counts = _counts(kind, n if kind != "fib" or n < 1000 else 61)
    N = counts.size
    gen = torch.Generator().manual_seed(n)
    W = torch.randn(N - 1, 8, generator=gen, dtype=torch.float64)
    for _ in range(3):
        x = torch.randn(1, 8, generator=gen, dtype=torch.float64) * 2
        loss = hierarchical_softmax_reference(W, x.expand(N, 8), torch.arange(N), counts)
        assert abs(torch.exp(-loss).sum().item() - 1.0) <= 1e-12
    if kind == "fib" and N == 61:
        assert huffman_tree(counts)[2].max().item() == 60


def test_depth_64_is_accepted_and_65_refused():
    from multiverso_b200.models.wordembedding import HuffmanTables
    from multiverso_b200.ops import PSHierarchicalSoftmax
    from multiverso_b200.utils import FatalError
    t = _HostTable(torch.zeros(70, 4))
    hsm = PSHierarchicalSoftmax(t, _fib(65))
    assert hsm.depth == 64
    with pytest.raises(ValueError, match="longer than 64"):
        PSHierarchicalSoftmax(t, _fib(66))
    with pytest.raises(FatalError, match="Huffman code longer than 64"):
        HuffmanTables(_fib(66), "cpu")


@pytest.mark.parametrize("n,d,B", [(2, 4, 5), (37, 12, 64), (1000, 8, 200)])
def test_host_layer_matches_fp64_path_formula(n, d, B):
    from multiverso_b200.ops import PSHierarchicalSoftmax, hierarchical_softmax_reference
    gen = torch.Generator().manual_seed(n + d)
    counts = np.floor(1e4 / np.arange(1, n + 1) ** 1.1)
    W = torch.randn(n + 3, d, generator=gen) / d ** 0.5                  # rows past N - 2 are never read
    x = torch.randn(B, d, generator=gen).requires_grad_()
    y = torch.randint(0, n, (B,), generator=gen)
    y[: B // 4] = 0                                                       # repeated labels share whole paths
    dl = torch.rand(B, generator=gen) + 0.5
    t = _HostTable(W.clone())
    loss = PSHierarchicalSoftmax(t, counts, push_scale=0.5)(x, y)
    (loss * dl).sum().backward()
    W64, x64 = W.double().requires_grad_(), x.detach().double().requires_grad_()
    ref = _path_formula(W64, x64, y, counts)
    (ref * dl.double()).sum().backward()
    assert torch.allclose(hierarchical_softmax_reference(W, x.detach(), y, counts), ref.detach(), rtol=1e-12,
                          atol=1e-12)
    assert torch.allclose(loss.double(), ref.detach(), rtol=1e-5, atol=1e-5)
    assert torch.allclose(x.grad.double(), x64.grad, rtol=1e-4, atol=1e-5)
    assert len(t.adds) == 1
    ids, vals, _ = t.adds[0]
    touched = torch.nonzero(W64.grad.abs().sum(1)).view(-1).numpy()
    assert np.array_equal(ids, np.unique(ids)) and set(touched) <= set(ids.tolist())
    assert (ids < n - 1).all()
    assert np.allclose(vals, 0.5 * W64.grad[ids].numpy(), rtol=1e-4, atol=1e-5)


def test_stateful_table_gets_one_add_rows_over_the_unique_nodes():
    from multiverso_b200.ops import PSHierarchicalSoftmax
    from multiverso_b200.ops.hierarchical_softmax import huffman_tree
    from multiverso_b200.tables.options import AddOption
    n, d = 500, 16
    counts = 1.0 / np.arange(1, n + 1)
    t = _HostTable(torch.randn(n, d) * 0.1, updater="adam")
    opt = AddOption(learning_rate=0.1)
    hsm = PSHierarchicalSoftmax(t, counts, push_scale=1.0, option=opt)
    y = torch.tensor([0, 0, 3, 499, 250, 3])
    hsm(torch.randn(6, d), y).sum().backward()
    points, _, lens = huffman_tree(counts)
    nodes = sorted({int(points[v, i]) for v in y.tolist() for i in range(int(lens[v]))})
    assert len(t.adds) == 1
    ids, vals, option = t.adds[0]
    assert ids.tolist() == nodes and vals.shape == (len(nodes), d) and option is opt


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


def test_host_sgd_step(host_mv):
    """One SGD step on the host backend (the default updater adds, so push_scale=-lr): table - lr * the node
    gradient coalesced over the batch; other rows unchanged; a no-grad forward after it is the loss of the new
    table."""
    mv = host_mv
    n, d, B, lr = 300, 12, 50, 0.25
    gen = torch.Generator().manual_seed(4)
    counts = np.floor(1e5 / np.arange(1, n + 1))
    W = torch.randn(n - 1, d, generator=gen) * 0.3
    t = mv.MatrixTable(n - 1, d, "float32", init_value=W.numpy())
    W0 = torch.as_tensor(np.asarray(t.get())).view(n - 1, d).clone()
    hsm = mv.ops.PSHierarchicalSoftmax(t, counts, push_scale=-lr)
    x = torch.randn(B, d, generator=gen)
    y = torch.randint(0, n, (B,), generator=gen)
    hsm(x, y).mean().backward()
    W64 = W0.double().requires_grad_()
    _path_formula(W64, x.double(), y, counts).mean().backward()
    got = torch.as_tensor(np.asarray(t.get())).view(n - 1, d)
    exp = W0.double() - lr * W64.grad
    assert torch.allclose(got.double(), exp, rtol=1e-5, atol=1e-6)
    untouched = W64.grad.abs().sum(1) == 0
    assert untouched.any() and torch.equal(got[untouched], W0[untouched])
    with torch.no_grad():
        ev = hsm(x, y)
    assert torch.allclose(ev.double(), _path_formula(got.double(), x.double(), y, counts), rtol=1e-5, atol=1e-5)


def test_empty_batch_pushes_nothing():
    from multiverso_b200.ops import PSHierarchicalSoftmax
    t = _HostTable(torch.randn(10, 4))
    hsm = PSHierarchicalSoftmax(t, np.arange(1.0, 12.0), push_scale=1.0)
    x = torch.zeros(0, 4, requires_grad=True)
    loss = hsm(x, torch.zeros(0, dtype=torch.int64))
    assert loss.shape == (0,)
    loss.sum().backward()
    assert t.adds == [] and x.grad.shape == (0, 4)


def test_refusals():
    from multiverso_b200.ops import PSHierarchicalSoftmax
    from multiverso_b200.tables.device import HashMatrixTable
    counts = np.arange(1.0, 9.0)
    t = _HostTable(torch.zeros(8, 4))
    cases = [
        (TypeError, "MatrixTable", lambda: PSHierarchicalSoftmax(torch.zeros(8, 4), counts)),
        (TypeError, "HashMatrixTable", lambda: PSHierarchicalSoftmax(HashMatrixTable.__new__(HashMatrixTable),
                                                                    counts)),
        (TypeError, "float32", lambda: PSHierarchicalSoftmax(types.SimpleNamespace(num_row=8, num_col=4,
                                                                                   npdt=np.float64), counts)),
        (ValueError, "multiple of 4", lambda: PSHierarchicalSoftmax(_HostTable(torch.zeros(8, 6)), counts)),
        (ValueError, "at least 2 classes", lambda: PSHierarchicalSoftmax(t, [3.0])),
        (ValueError, "at least 2 classes", lambda: PSHierarchicalSoftmax(t, [])),
        (ValueError, "finite and non-negative", lambda: PSHierarchicalSoftmax(t, [1.0, -1.0, 2.0])),
        (ValueError, "finite and non-negative", lambda: PSHierarchicalSoftmax(t, [1.0, float("nan"), 2.0])),
        (ValueError, "finite and non-negative", lambda: PSHierarchicalSoftmax(t, [1.0, float("inf"), 2.0])),
        (ValueError, "1-D", lambda: PSHierarchicalSoftmax(t, np.ones((3, 3)))),
        (ValueError, "need 9 inner-node rows", lambda: PSHierarchicalSoftmax(t, np.arange(1.0, 11.0))),
    ]
    for exc, msg, make in cases:
        with pytest.raises(exc, match=msg):
            make()
    PSHierarchicalSoftmax(t, np.arange(1.0, 10.0))                     # 9 classes: 8 rows are enough
    hsm = PSHierarchicalSoftmax(t, counts)
    x = torch.randn(3, 4)
    calls = [
        (TypeError, "2-D float32", x.double(), torch.arange(3)),
        (TypeError, "2-D float32", x[0], torch.arange(3)),
        (ValueError, "hidden has 8 columns", torch.randn(3, 8), torch.arange(3)),
        (TypeError, "int32 or int64", x, torch.arange(3).float()),
        (ValueError, "one label per row", x, torch.arange(2)),
        (ValueError, r"\[0, 8\), got min 0 max 8", x, torch.tensor([0, 8, 1])),
        (ValueError, r"got min -1", x, torch.tensor([0, -1, 1], dtype=torch.int32)),
    ]
    for exc, msg, h, y in calls:
        with pytest.raises(exc, match=msg):
            hsm(h, y)
    assert t.adds == []
