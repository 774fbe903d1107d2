"""PSFieldAwareFactorizationMachine without a GPU: the fp64 reference against the pair sum written out one pair at a
time (empty and one-lookup bags, duplicate ids, repeated fields, values None / signed / 0), F = 1 against the FM
reference, the reference's gradient against sum g H, the host layer and its one coalesced add_rows against fp64
autograd, 50 sgd steps on the host backend against a torch FFM trained by torch.optim.SGD, and every refusal."""
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


def _seg(W64, i, f, k):
    return W64[i, f * k:(f + 1) * k]


def _pairs(W64, ids, fields, offsets, x, F, k):
    """y [B] as the linear terms plus the pair terms j < l, one at a time."""
    D = F * k
    ends = offsets[1:].tolist() + [ids.numel()]
    out = []
    for lo, hi in zip(offsets.tolist(), ends):
        y = torch.zeros((), dtype=torch.float64)
        for j in range(lo, hi):
            y = y + x[j] * W64[ids[j], D]
        for j, l in itertools.combinations(range(lo, hi), 2):
            y = y + x[j] * x[l] * (_seg(W64, ids[j], fields[l], k) @ _seg(W64, ids[l], fields[j], k))
        out.append(y)
    return torch.stack(out) if out else torch.zeros(0, dtype=torch.float64)


def _H(W64, ids, fields, offsets, x, F, k):
    """H [L, D + 1]: segment f of row j is x_j sum_{l != j, f_l = f} x_l V_{i_l}[f_j], column D is x_j."""
    D, L = F * k, ids.numel()
    H = torch.zeros(L, D + 1, dtype=torch.float64)
    ends = offsets[1:].tolist() + [L]
    for lo, hi in zip(offsets.tolist(), ends):
        for j in range(lo, hi):
            H[j, D] = x[j]
            for l in range(lo, hi):
                if l != j:
                    f = int(fields[l])
                    H[j, f * k:(f + 1) * k] += x[j] * x[l] * _seg(W64, ids[l], fields[j], k)
    return H


def _bags(gen, n, B, max_len, F):
    lens = torch.randint(0, max_len + 1, (B,), generator=gen)
    lens[0] = 0                                                   # an empty bag
    lens[1] = 1                                                   # a bag of one lookup
    lens[2] = max(int(lens[2]), 4)
    L = int(lens.sum())
    ids = torch.randint(0, n, (L,), generator=gen)
    ids[2:5] = ids[1]                                             # duplicate ids, in one bag or across bags
    fields = torch.randint(0, F, (L,), generator=gen)
    fields[2:4] = fields[4]                                       # a repeated field in one bag
    offsets = torch.cumsum(lens, 0) - lens
    return ids, fields, offsets


@pytest.mark.parametrize("F,k", [(1, 4), (3, 4), (5, 8)])
@pytest.mark.parametrize("vals", ["none", "signed", "zeros"])
def test_reference_matches_pair_loop(F, k, vals):
    from multiverso_b200.ops import field_aware_factorization_machine_reference as ref
    gen = torch.Generator().manual_seed(F * 10 + k)
    n, B, D = 40, 12, F * k
    W = torch.randn(n, D + 3, generator=gen, dtype=torch.float64)
    W[:, D + 1:] = float("nan")                                   # columns past D are never read
    ids, fields, offsets = _bags(gen, n, B, 7, F)
    L = ids.numel()
    x = {"none": None, "signed": torch.randn(L, generator=gen, dtype=torch.float64),
         "zeros": torch.randn(L, generator=gen, dtype=torch.float64) * (torch.rand(L, generator=gen) < 0.5)}[vals]
    y = ref(W, ids, fields, offsets, x, num_fields=F, num_factors=k)
    exp = _pairs(W, ids, fields, offsets, torch.ones(L, dtype=torch.float64) if x is None else x, F, k)
    assert y.dtype == torch.float64 and y.shape == (B,) and y[0] == 0
    assert torch.allclose(y, exp, rtol=1e-12, atol=1e-12)
    j = int(offsets[1])                                           # one lookup: the linear term only
    assert torch.allclose(y[1], (1.0 if x is None else x[j]) * W[ids[j], D])
    # 2-D bags are the same as 1-D bags with offsets
    ids2 = torch.randint(0, n, (5, 3), generator=gen)
    f2 = torch.randint(0, F, (5, 3), generator=gen)
    assert torch.equal(ref(W, ids2, f2, num_fields=F, num_factors=k),
                       ref(W, ids2.reshape(-1), f2.reshape(-1), torch.arange(0, 15, 3), num_fields=F, num_factors=k))


def test_one_field_is_the_factorization_machine():
    from multiverso_b200.ops import factorization_machine_reference, field_aware_factorization_machine_reference
    gen = torch.Generator().manual_seed(3)
    n, B, k = 30, 10, 8
    W = torch.randn(n, k + 1, generator=gen, dtype=torch.float64)
    ids, _, offsets = _bags(gen, n, B, 9, 1)
    x = torch.randn(ids.numel(), generator=gen, dtype=torch.float64)
    y = field_aware_factorization_machine_reference(W, ids, torch.zeros_like(ids), offsets, x, num_fields=1,
                                                    num_factors=k)
    assert torch.allclose(y, factorization_machine_reference(W, ids, offsets, x), rtol=1e-12, atol=1e-12)


def test_reference_gradient_is_sum_g_H():
    from multiverso_b200.ops import field_aware_factorization_machine_reference as ref
    gen = torch.Generator().manual_seed(1)
    n, F, k, B = 30, 3, 4, 9
    D = F * k
    W = torch.randn(n, D + 1, generator=gen, dtype=torch.float64, requires_grad=True)
    ids, fields, offsets = _bags(gen, n, B, 6, F)
    L = ids.numel()
    x = torch.randn(L, generator=gen, dtype=torch.float64)
    g = torch.randn(B, generator=gen, dtype=torch.float64)
    (ref(W, ids, fields, offsets, x, num_fields=F, num_factors=k) * g).sum().backward()
    bag = torch.repeat_interleave(torch.arange(B), torch.diff(offsets, append=torch.tensor([L])))
    H = _H(W.detach(), ids, fields, offsets, x, F, k)
    G = torch.zeros(n, D + 1, dtype=torch.float64).index_add_(0, ids, g[bag][:, None] * H)
    assert torch.allclose(W.grad, G, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("F,k,width", [(1, 4, 5), (4, 4, 20), (3, 8, 28)])
def test_host_layer_and_coalesced_push(F, k, width):
    """The host layer's y against fp64, and its one add_rows over the unique ids: push_scale * fp64 G."""
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine, field_aware_factorization_machine_reference
    from multiverso_b200.tables.options import AddOption
    gen = torch.Generator().manual_seed(F + k)
    n, B, scale = 50, 20, 0.3
    W = torch.randn(n, width, generator=gen) * 0.5
    t = _HostTable(W)
    opt = AddOption(learning_rate=0.5)
    ffm = PSFieldAwareFactorizationMachine(t, F, k, push_scale=scale, option=opt)
    ids, fields, offsets = _bags(gen, n, B, 8, F)
    x = torch.randn(ids.numel(), generator=gen)
    y = ffm(ids, fields, offsets, x)
    W64 = W.double().requires_grad_()
    y64 = field_aware_factorization_machine_reference(W64, ids, fields, offsets, x.double(), num_fields=F,
                                                      num_factors=k)
    assert y.dtype == torch.float32 and torch.allclose(y.double(), y64, rtol=1e-5, atol=1e-5)
    g = torch.randn(B, generator=gen)
    (y * g).sum().backward()
    (y64 * g.double()).sum().backward()
    assert len(t.adds) == 1
    uid, vals, option = t.adds[0]
    assert uid.tolist() == torch.unique(ids).tolist() and option is opt and vals.shape == (uid.size, width)
    assert np.allclose(vals, scale * W64.grad[torch.from_numpy(uid)].numpy(), rtol=1e-4, atol=1e-5)
    assert not vals[:, F * k + 1:].any()
    with torch.no_grad():
        assert torch.equal(ffm(ids, fields, offsets, x), y.detach())
    assert len(t.adds) == 1


def test_empty_batch_and_no_push():
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine
    t = _HostTable(torch.randn(10, 9))
    ffm = PSFieldAwareFactorizationMachine(t, 2, 4, push_scale=1.0)
    e = torch.zeros(0, dtype=torch.int64)
    y = ffm(e, e, e)
    assert y.shape == (0,)
    y.sum().backward()
    y = ffm(e, e, torch.zeros(3, dtype=torch.int64))                # three empty bags
    assert torch.equal(y, torch.zeros(3))
    y.sum().backward()
    PSFieldAwareFactorizationMachine(t, 2, 4, push_scale=None)(torch.tensor([[1, 2]]), torch.tensor([[0, 1]])) \
        .sum().backward()
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
    nn.Parameter FFM trained with torch.optim.SGD on the same batches and the same logistic loss."""
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine, field_aware_factorization_machine_reference
    mv = host_mv
    n, F, k, B, lr = 200, 3, 4, 32, 0.05
    C = F * k + 1
    gen = torch.Generator().manual_seed(7)
    W0 = torch.randn(n, C, generator=gen) * 0.1
    t = mv.MatrixTable(n, C, "float32", init_value=W0.numpy())
    ffm = PSFieldAwareFactorizationMachine(t, F, k, push_scale=-lr)
    P = torch.nn.Parameter(W0.clone())
    opt = torch.optim.SGD([P], lr=lr)
    for _ in range(50):
        ids = torch.randint(0, n, (B, 6), generator=gen)
        fields = torch.randint(0, F, (B, 6), generator=gen)
        x = torch.rand(B, 6, generator=gen)
        lab = (torch.rand(B, generator=gen) < 0.5).float()
        torch.nn.functional.binary_cross_entropy_with_logits(ffm(ids, fields, values=x), lab,
                                                             reduction="sum").backward()
        opt.zero_grad()
        yt = field_aware_factorization_machine_reference(P, ids, fields, values=x, num_fields=F,
                                                         num_factors=k).float()
        torch.nn.functional.binary_cross_entropy_with_logits(yt, lab, reduction="sum").backward()
        opt.step()
    got = torch.as_tensor(np.asarray(t.get())).view(n, C)
    assert (got - W0).abs().max() > 0.05
    assert torch.allclose(got, P.detach(), rtol=1e-4, atol=1e-5), (got - P.detach()).abs().max()


def test_refusals():
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine as FFM
    from multiverso_b200.ops import field_aware_factorization_machine_reference as ref
    t = _HostTable(torch.zeros(8, 9))
    cases = [
        (TypeError, "MatrixTable", lambda: FFM(torch.zeros(8, 9), 2, 4)),
        (TypeError, "float32", lambda: FFM(types.SimpleNamespace(num_row=8, num_col=9, npdt=np.float64), 2, 4)),
        (ValueError, "num_fields must be a positive integer, got 0", lambda: FFM(t, 0, 4)),
        (ValueError, "num_fields must be a positive integer, got 1.5", lambda: FFM(t, 1.5, 4)),
        (ValueError, "multiple of 4, got 0", lambda: FFM(t, 1, 0)),
        (ValueError, "multiple of 4, got 6", lambda: FFM(t, 1, 6)),
        (ValueError, "multiple of 4, got -4", lambda: FFM(t, 1, -4)),
        (ValueError, "at most 1024, got 1025", lambda: FFM(_HostTable(torch.zeros(2, 1028)), 256, 4)),
        (ValueError, r"width \(8\) must be at least .* = 9", lambda: FFM(_HostTable(torch.zeros(8, 8)), 2, 4)),
    ]
    for exc, msg, make in cases:
        with pytest.raises(exc, match=msg):
            make()
    FFM(_HostTable(torch.zeros(2, 1021)), 255, 4)
    ffm = FFM(t, 2, 4)
    ids, offs, f = torch.tensor([0, 1, 2, 3]), torch.tensor([0, 2]), torch.tensor([0, 1, 1, 0])
    calls = [
        (TypeError, "values must be floating point", (ids, f, offs, torch.ones(4, dtype=torch.int64))),
        (ValueError, "values must have the shape of ids", (ids, f, offs, torch.ones(3))),
        (ValueError, "get no gradient", (ids, f, offs, torch.ones(4, requires_grad=True))),
        (TypeError, "fields must be integers", (ids, f.float(), offs, None)),
        (TypeError, "fields must be integers", (ids, f.bool(), offs, None)),
        (ValueError, "fields must have the shape of ids", (ids, f[:3], offs, None)),
        (ValueError, r"fields must be in \[0, 2\), got min 0 max 2", (ids, torch.tensor([0, 1, 2, 0]), offs, None)),
        (ValueError, r"fields must be in \[0, 2\), got min -1", (ids, torch.tensor([0, -1, 1, 0]), offs, None)),
        (ValueError, r"ids must be in \[0, 8\), got min 0 max 8", (torch.tensor([0, 1, 2, 8]), f, offs, None)),
        (ValueError, "got min -1", (torch.tensor([0, -1, 2, 3]), f, offs, None)),
        (ValueError, "must start at 0", (ids, f, torch.tensor([1, 2]), None)),
        (ValueError, "non-decreasing", (ids, f, torch.tensor([0, 3, 2]), None)),
        (ValueError, "exceed the number of ids", (ids, f, torch.tensor([0, 5]), None)),
        (TypeError, "int32 or int64", (ids.float(), f, offs, None)),
        (ValueError, "1-D ids need offsets", (ids, f, None, None)),
    ]
    for exc, msg, args in calls:
        with pytest.raises(exc, match=msg):
            ffm(*args)
    assert t.adds == []
    with pytest.raises(ValueError, match=r"fields must be in \[0, 2\)"):
        ref(t.W, ids, torch.tensor([0, 1, 2, 0]), offs, num_fields=2, num_factors=4)
    with pytest.raises(ValueError, match=r"weights must be \[num_row, >= 9\]"):
        ref(torch.zeros(8, 8), ids, f, offs, num_fields=2, num_factors=4)
