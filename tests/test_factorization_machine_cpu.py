"""PSFactorizationMachine without a GPU: the fp64 reference against the pair sum written out one pair at a time (with
duplicate ids, empty bags and values None / negative / 0), the host layer and its one coalesced add_rows against
fp64 autograd, 50 sgd steps on the host backend against a torch FM trained by torch.optim.SGD, and every refusal."""
import itertools
import types

import numpy as np
import pytest
import torch


class _HostTable:
    """What the layer reads of a host-backend table, with every add_rows recorded."""

    def __init__(self, W, updater="adagrad"):
        self.W, self.num_row, self.num_col = W, W.shape[0], W.shape[1]
        self.npdt, self.updater, self.adds = np.float32, updater, []

    def get_rows(self, ids):
        return self.W[torch.from_numpy(np.asarray(ids))].numpy()

    def add_rows(self, ids, vals, option=None):
        self.adds.append((np.array(ids), np.array(vals), option))


def _pairs(W64, ids, offsets, x):
    """y [B] as the linear terms plus the pair terms j < l, one at a time."""
    k = W64.shape[1] - 1
    ends = offsets[1:].tolist() + [ids.numel()]
    out = []
    for b, (lo, hi) in enumerate(zip(offsets.tolist(), ends)):
        y = torch.zeros((), dtype=torch.float64)
        for j in range(lo, hi):
            y = y + x[j] * W64[ids[j], k]
        for j, l in itertools.combinations(range(lo, hi), 2):
            y = y + x[j] * x[l] * (W64[ids[j], :k] @ W64[ids[l], :k])
        out.append(y)
    return torch.stack(out) if out else torch.zeros(0, dtype=torch.float64)


def _bags(gen, n, B, max_len):
    lens = torch.randint(0, max_len + 1, (B,), generator=gen)
    lens[0] = 0                                                   # an empty bag
    lens[1] = 1                                                   # a bag of one lookup
    ids = torch.randint(0, n, (int(lens.sum()),), generator=gen)
    ids[2:5] = ids[1]                                             # duplicate ids, in one bag or across bags
    offsets = torch.cumsum(lens, 0) - lens
    return ids, offsets


@pytest.mark.parametrize("C", [2, 5, 9, 64])
@pytest.mark.parametrize("vals", ["none", "signed", "zeros"])
def test_reference_matches_pair_loop(C, vals):
    from multiverso_b200.ops import factorization_machine_reference
    gen = torch.Generator().manual_seed(C)
    n, B = 40, 12
    W = torch.randn(n, C, generator=gen, dtype=torch.float64)
    ids, offsets = _bags(gen, n, B, 7)
    L = ids.numel()
    x = {"none": None, "signed": torch.randn(L, generator=gen, dtype=torch.float64),
         "zeros": torch.randn(L, generator=gen, dtype=torch.float64) * (torch.rand(L, generator=gen) < 0.5)}[vals]
    y = factorization_machine_reference(W, ids, offsets, x)
    exp = _pairs(W, ids, offsets, torch.ones(L, dtype=torch.float64) if x is None else x)
    assert y.dtype == torch.float64 and y.shape == (B,) and y[0] == 0
    assert torch.allclose(y, exp, rtol=1e-12, atol=1e-12)
    # one lookup: the linear term only
    assert torch.allclose(y[1], (1.0 if x is None else x[int(offsets[1])]) * W[ids[int(offsets[1])], C - 1])
    # 2-D bags are the same as 1-D bags with offsets
    ids2 = torch.randint(0, n, (5, 3), generator=gen)
    assert torch.equal(factorization_machine_reference(W, ids2),
                       factorization_machine_reference(W, ids2.reshape(-1), torch.arange(0, 15, 3)))


def test_reference_is_differentiable_in_weights():
    """Its gradient is G_r = sum g x (S' - x v'_r), the gradient the layer pushes."""
    from multiverso_b200.ops import factorization_machine_reference
    gen = torch.Generator().manual_seed(1)
    n, C, B = 30, 6, 9
    W = torch.randn(n, C, generator=gen, dtype=torch.float64, requires_grad=True)
    ids, offsets = _bags(gen, n, B, 6)
    x = torch.randn(ids.numel(), generator=gen, dtype=torch.float64)
    g = torch.randn(B, generator=gen, dtype=torch.float64)
    (factorization_machine_reference(W, ids, offsets, x) * g).sum().backward()
    bag = torch.repeat_interleave(torch.arange(B), torch.diff(offsets, append=torch.tensor([ids.numel()])))
    Wd = W.detach()
    S = torch.zeros(B, C, dtype=torch.float64).index_add_(0, bag, x[:, None] * Wd[ids])
    Sp = S.clone()
    Sp[:, C - 1] = 1
    vp = Wd[ids].clone()
    vp[:, C - 1] = 0
    G = torch.zeros(n, C, dtype=torch.float64).index_add_(0, ids, (g[bag] * x)[:, None] * (Sp[bag] - x[:, None] * vp))
    assert torch.allclose(W.grad, G, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("C", [2, 7, 16])
def test_host_layer_and_coalesced_push(C):
    """The host layer's y against fp64, and its one add_rows over the unique ids: push_scale * fp64 G."""
    from multiverso_b200.ops import PSFactorizationMachine, factorization_machine_reference
    from multiverso_b200.tables.options import AddOption
    gen = torch.Generator().manual_seed(C + 10)
    n, B, scale = 50, 20, 0.3
    W = torch.randn(n, C, generator=gen) * 0.5
    t = _HostTable(W)
    opt = AddOption(learning_rate=0.5)
    fm = PSFactorizationMachine(t, push_scale=scale, option=opt)
    ids, offsets = _bags(gen, n, B, 8)
    x = torch.randn(ids.numel(), generator=gen)
    y = fm(ids, offsets, x)
    W64 = W.double().requires_grad_()
    y64 = factorization_machine_reference(W64, ids, offsets, x.double())
    assert y.dtype == torch.float32 and torch.allclose(y.double(), y64, rtol=1e-5, atol=1e-5)
    g = torch.randn(B, generator=gen)
    (y * g).sum().backward()
    (y64 * g.double()).sum().backward()
    assert len(t.adds) == 1
    uid, vals, option = t.adds[0]
    assert uid.tolist() == torch.unique(ids).tolist() and option is opt
    assert np.allclose(vals, scale * W64.grad[torch.from_numpy(uid)].numpy(), rtol=1e-4, atol=1e-5)
    with torch.no_grad():
        assert torch.equal(fm(ids, offsets, x), y.detach())
    assert len(t.adds) == 1


def test_empty_batch_and_no_push():
    from multiverso_b200.ops import PSFactorizationMachine
    t = _HostTable(torch.randn(10, 4))
    fm = PSFactorizationMachine(t, push_scale=1.0)
    y = fm(torch.zeros(0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64))
    assert y.shape == (0,)
    y.sum().backward()
    y = fm(torch.zeros(0, dtype=torch.int64), torch.zeros(3, dtype=torch.int64))      # three empty bags
    assert torch.equal(y, torch.zeros(3))
    y.sum().backward()
    PSFactorizationMachine(t, push_scale=None)(torch.tensor([[1, 2]])).sum().backward()
    assert t.adds == []


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


def test_sgd_training_matches_torch(host_mv):
    """50 steps on the host backend (the default updater adds, so push_scale=-lr: W -= lr * G) against an
    nn.Parameter FM trained with torch.optim.SGD on the same batches and the same logistic loss."""
    from multiverso_b200.ops import PSFactorizationMachine, factorization_machine_reference
    mv = host_mv
    n, C, B, lr = 200, 9, 32, 0.05
    gen = torch.Generator().manual_seed(7)
    W0 = torch.randn(n, C, generator=gen) * 0.1
    t = mv.MatrixTable(n, C, "float32", init_value=W0.numpy())
    fm = PSFactorizationMachine(t, push_scale=-lr)
    P = torch.nn.Parameter(W0.clone())
    opt = torch.optim.SGD([P], lr=lr)
    for _ in range(50):
        ids = torch.randint(0, n, (B, 6), generator=gen)
        x = torch.rand(B, 6, generator=gen)
        lab = (torch.rand(B, generator=gen) < 0.5).float()
        torch.nn.functional.binary_cross_entropy_with_logits(fm(ids, values=x), lab, reduction="sum").backward()
        opt.zero_grad()
        yt = factorization_machine_reference(P, ids, values=x).float()
        torch.nn.functional.binary_cross_entropy_with_logits(yt, lab, reduction="sum").backward()
        opt.step()
    got = torch.as_tensor(np.asarray(t.get())).view(n, C)
    assert (got - W0).abs().max() > 0.05
    assert torch.allclose(got, P.detach(), rtol=1e-4, atol=1e-5), (got - P.detach()).abs().max()


def test_refusals():
    from multiverso_b200.ops import PSFactorizationMachine
    t = _HostTable(torch.zeros(8, 5))
    cases = [
        (TypeError, "MatrixTable", lambda: PSFactorizationMachine(torch.zeros(8, 4))),
        (TypeError, "float32", lambda: PSFactorizationMachine(types.SimpleNamespace(num_row=8, num_col=4,
                                                                                    npdt=np.float64))),
        (ValueError, r"\[2, 1024\], got 1", lambda: PSFactorizationMachine(_HostTable(torch.zeros(8, 1)))),
        (ValueError, r"\[2, 1024\], got 1025", lambda: PSFactorizationMachine(_HostTable(torch.zeros(2, 1025)))),
    ]
    for exc, msg, make in cases:
        with pytest.raises(exc, match=msg):
            make()
    PSFactorizationMachine(_HostTable(torch.zeros(2, 1024)))
    fm = PSFactorizationMachine(t)
    ids, offs = torch.tensor([0, 1, 2, 3]), torch.tensor([0, 2])
    calls = [
        (TypeError, "values must be floating point", (ids, offs, torch.ones(4, dtype=torch.int64))),
        (ValueError, "shape of ids", (ids, offs, torch.ones(3))),
        (ValueError, "get no gradient", (ids, offs, torch.ones(4, requires_grad=True))),
        (ValueError, r"ids must be in \[0, 8\), got min 0 max 8", (torch.tensor([0, 1, 2, 8]), offs, None)),
        (ValueError, "got min -1", (torch.tensor([0, -1, 2, 3]), offs, None)),
        (ValueError, "must start at 0", (ids, torch.tensor([1, 2]), None)),
        (ValueError, "non-decreasing", (ids, torch.tensor([0, 3, 2]), None)),
        (ValueError, "exceed the number of ids", (ids, torch.tensor([0, 5]), None)),
        (TypeError, "int32 or int64", (ids.float(), offs, None)),
        (ValueError, "1-D ids need offsets", (ids, None, None)),
    ]
    for exc, msg, args in calls:
        with pytest.raises(exc, match=msg):
            fm(*args)
    assert t.adds == []
