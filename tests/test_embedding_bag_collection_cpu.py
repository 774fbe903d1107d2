"""PSEmbeddingCollection without a GPU: the host backend against torch (forward, one step of per-table EmbeddingBag +
SGD), one updater step per row of a table that two features share, the per-sample-weight gradient, split() and the
input checks."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from multiverso_b200.ops import EmbeddingBagConfig, PSEmbedding, PSEmbeddingCollection
from multiverso_b200.tables.options import AddOption


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


def _host_table(mv, W):
    t = mv.MatrixTable(W.shape[0], W.shape[1], "float32")
    t.add(W.numpy())
    return t


class StatefulTable:
    """A host table stand-in whose add_rows applies momentum_sgd or adagrad in fp64, with the device updaters'
    rules (csrc/cuda/mvb_common.cuh), and counts the steps each row takes."""

    def __init__(self, W, updater):
        self.w = W.double().numpy().copy()
        self.s = np.zeros_like(self.w)
        self.steps = np.zeros(W.shape[0], dtype=np.int64)
        self.num_row, self.num_col = W.shape
        self.npdt, self.updater = np.float32, updater

    def get_rows(self, ids):
        return self.w[np.asarray(ids)].astype(np.float32)

    def add_rows(self, ids, vals, option=None):
        ids, g = np.asarray(ids), np.asarray(vals, dtype=np.float64)
        assert len(np.unique(ids)) == len(ids)               # one coalesced row per id and call
        self.steps[ids] += 1
        step(self.w, self.s, ids, g, self.updater, option)


def step(w, s, ids, g, updater, option):
    if updater == "momentum_sgd":
        s[ids] = option.momentum * s[ids] + (1.0 - option.momentum) * g
        w[ids] -= s[ids]
    else:
        gn = g / option.learning_rate
        s[ids] += gn * gn
        w[ids] -= option.rho / np.sqrt(s[ids] + 1e-6) * gn


def _batch(seed, nrows, F_, B, max_len=4):
    """ids and lengths in the jagged layout, with empty bags and heavy duplicates."""
    g = torch.Generator().manual_seed(seed)
    lengths = torch.randint(0, max_len + 1, (F_, B), generator=g)
    lengths[:, ::5] = 0
    parts = [torch.randint(0, n, (int(lengths[f].sum()),), generator=g) for f, n in enumerate(nrows)]
    for p in parts:
        p[::3] = 1
    return torch.cat(parts), lengths


def _feature(ids, lengths, f):
    """(ids, offsets) of feature f."""
    starts = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(lengths.sum(1), 0)])
    lo, hi = int(starts[f]), int(starts[f + 1])
    return ids[lo:hi], torch.cumsum(lengths[f], 0) - lengths[f]


@pytest.mark.parametrize("mode", ["sum", "mean"])
def test_host_step_equals_embeddingbag_sgd(mv_host, mode):
    """Two tables, one of them shared by two features: forward = F.embedding_bag per feature, and one step = per-table
    nn.EmbeddingBag(sparse=True) + SGD on the features' bags."""
    g = torch.Generator().manual_seed(0)
    Wa, Wb = torch.randn(40, 8, generator=g), torch.randn(30, 12, generator=g)
    ta, tb = _host_table(mv_host, Wa), _host_table(mv_host, Wb)
    lr = 0.1
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(ta, ["a"], push_scale=-lr, mode=mode),
                                 EmbeddingBagConfig(tb, ["b1", "b2"], push_scale=-lr, mode=mode)])
    ids, lengths = _batch(1, [40, 30, 30], 3, 16)
    out = ebc(ids.to(torch.int32), lengths)
    assert out.shape == (16, 8 + 12 + 12)
    target = torch.randn(16, 32, generator=g)
    ((out - target) ** 2).sum().backward()
    refs = [torch.nn.EmbeddingBag(*W.shape, mode=mode, sparse=True) for W in (Wa, Wb)]
    for r, W in zip(refs, (Wa, Wb)):
        with torch.no_grad():
            r.weight.copy_(W)
    parts = [refs[0](*_feature(ids, lengths, 0)), refs[1](*_feature(ids, lengths, 1)),
             refs[1](*_feature(ids, lengths, 2))]
    y = torch.cat(parts, 1)
    assert torch.allclose(out, y.detach(), atol=1e-6)
    ((y - target) ** 2).sum().backward()
    opt = torch.optim.SGD([r.weight for r in refs], lr=lr)
    opt.step()
    assert torch.allclose(torch.from_numpy(ta.get()), refs[0].weight.detach(), atol=1e-5)
    assert torch.allclose(torch.from_numpy(tb.get()), refs[1].weight.detach(), atol=1e-5)


@pytest.mark.parametrize("updater", ["momentum_sgd", "adagrad"])
def test_shared_table_one_step_per_row(updater):
    """A row that two features touch in one step gets one updater step with the summed gradient; two separate
    PSEmbedding calls give it two steps, which is a different result."""
    g = torch.Generator().manual_seed(2)
    W = torch.randn(20, 8, generator=g)
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    ids, lengths = _batch(3, [20, 20], 2, 10)
    dout = torch.randn(10, 16, generator=g)
    t = StatefulTable(W, updater)
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["query", "title"], push_scale=1.0, option=opt)])
    ebc(ids, lengths).backward(dout)
    (i0, o0), (i1, o1) = _feature(ids, lengths, 0), _feature(ids, lengths, 1)
    # fp64 expectation: the gradient summed over both features, then one step per touched row
    G = np.zeros((20, 8))
    for (i, o), d in (((i0, o0), dout[:, :8]), ((i1, o1), dout[:, 8:])):
        bag = torch.repeat_interleave(torch.arange(10), torch.diff(o, append=torch.tensor([i.numel()])))
        np.add.at(G, i.numpy(), d.double()[bag].numpy())
    touched = np.unique(torch.cat([i0, i1]).numpy())
    w, s = W.double().numpy().copy(), np.zeros((20, 8))
    step(w, s, touched, G[touched], updater, opt)
    assert (t.steps[touched] == 1).all() and t.steps.sum() == len(touched)
    assert np.abs(t.w - w).max() < 1e-5
    both = np.intersect1d(i0.numpy(), i1.numpy())
    assert len(both) > 0
    # per-feature layers: the rows both features touch take two steps and end up elsewhere
    t2 = StatefulTable(W, updater)
    PSEmbedding(t2, push_scale=1.0, option=opt)(i0, o0).backward(dout[:, :8])
    PSEmbedding(t2, push_scale=1.0, option=opt)(i1, o1).backward(dout[:, 8:])
    assert (t2.steps[both] == 2).all()
    assert np.abs(t2.w[both] - w[both]).max() > 1e-3


def test_psw_grad_and_split(mv_host):
    g = torch.Generator().manual_seed(4)
    Wa, Wb = torch.randn(25, 4, generator=g), torch.randn(35, 6, generator=g)
    ta, tb = _host_table(mv_host, Wa), _host_table(mv_host, Wb)
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(ta, ["x", "y"], push_scale=None),
                                 EmbeddingBagConfig(tb, ["z"], push_scale=None)])
    ids, lengths = _batch(5, [25, 25, 35], 3, 9)
    p = torch.rand(ids.numel(), generator=g).requires_grad_()
    dout = torch.randn(9, 14, generator=g)
    out = ebc(ids, lengths, p)
    (out * dout).sum().backward()
    p2 = p.detach().clone().requires_grad_()
    starts = [0] + torch.cumsum(lengths.sum(1), 0).tolist()
    ys = []
    for f, W in enumerate((Wa, Wa, Wb)):
        i, o = _feature(ids, lengths, f)
        ys.append(F.embedding_bag(i, W, o, mode="sum", per_sample_weights=p2[starts[f]:starts[f + 1]]))
    (torch.cat(ys, 1) * dout).sum().backward()
    assert torch.allclose(out, torch.cat(ys, 1).detach(), atol=1e-6)
    assert torch.allclose(p.grad, p2.grad, atol=1e-5)
    assert torch.equal(torch.from_numpy(ta.get()), Wa)        # push_scale=None: nothing pushed
    parts = ebc.split(out)
    assert list(parts) == ["x", "y", "z"]
    assert [v.shape for v in parts.values()] == [(9, 4), (9, 4), (9, 6)]
    assert parts["z"].data_ptr() == out[:, 8:].data_ptr() and torch.equal(parts["y"], out[:, 4:8])
    with pytest.raises(ValueError, match=r"split: expected \[B, 14\]"):
        ebc.split(out[:, :10])


def test_empty_batch_and_empty_feature(mv_host):
    W = torch.randn(10, 4)
    t = _host_table(mv_host, W)
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["u", "v"], push_scale=-0.1)])
    out = ebc(torch.zeros(0, dtype=torch.int64), torch.zeros(2, 0, dtype=torch.int64))
    assert out.shape == (0, 8)
    ids, lengths = torch.tensor([3, 4, 3]), torch.tensor([[0, 0], [2, 1]])      # feature u has no lookups
    out = ebc(ids, lengths)
    assert (out[:, :4] == 0).all() and torch.allclose(out[0, 4:], W[3] + W[4])
    out.sum().backward()
    exp = W.clone()
    exp[3] -= 0.2
    exp[4] -= 0.1
    assert torch.allclose(torch.from_numpy(t.get()), exp, atol=1e-6)


def test_validation_errors(mv_host):
    g = torch.Generator().manual_seed(6)
    ta, tb = _host_table(mv_host, torch.randn(10, 4, generator=g)), _host_table(mv_host, torch.randn(50, 8, generator=g))
    with pytest.raises(ValueError, match="use the same table; list both features in one config"):
        PSEmbeddingCollection([EmbeddingBagConfig(ta, ["a"]), EmbeddingBagConfig(ta, ["b"])])
    with pytest.raises(ValueError, match="duplicate feature name 'a'"):
        PSEmbeddingCollection([EmbeddingBagConfig(ta, ["a"]), EmbeddingBagConfig(tb, ["a"])])
    t64 = mv_host.MatrixTable(10, 4, "float64")
    with pytest.raises(TypeError, match="the table must be float32"):
        PSEmbeddingCollection([EmbeddingBagConfig(t64, ["a"])])
    with pytest.raises(TypeError, match="a tensor table has no updater"):
        PSEmbeddingCollection([EmbeddingBagConfig(torch.randn(5, 4), ["a"])])
    with pytest.raises(ValueError, match="mode must be one of"):
        PSEmbeddingCollection([EmbeddingBagConfig(ta, ["a"], mode="max")])
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(ta, ["a"]), EmbeddingBagConfig(tb, ["b"], mode="mean")])
    ids, lengths = torch.tensor([1, 2, 40]), torch.tensor([[1, 1], [0, 1]])
    bad = [
        (dict(lengths=torch.tensor([1, 1, 0, 1])), ValueError, r"lengths must be \[F, B\] with F = 2"),
        (dict(lengths=torch.tensor([[2, 1], [0, 1]])), ValueError, "lengths sum to 4 but ids has 3 entries"),
        (dict(lengths=torch.tensor([[3, -1], [0, 1]])), ValueError, "lengths must be non-negative"),
        # 40 is a valid row of table b but not of feature a's table
        (dict(lengths=torch.tensor([[1, 0], [1, 1]]), ids=torch.tensor([40, 1, 2])), ValueError,
         r"ids of feature 'a' must be in \[0, 10\)"),
        (dict(ids=torch.tensor([1, 2, 50])), ValueError, r"ids of feature 'b' must be in \[0, 50\)"),
        (dict(ids=torch.tensor([-1, 2, 40])), ValueError, r"ids of feature 'a' must be in \[0, 10\)"),
        (dict(per_sample_weights=torch.ones(3)), ValueError, "per_sample_weights need every table to pool with"),
        (dict(ids=ids.float()), TypeError, "ids must be int32 or int64"),
        (dict(lengths=lengths.float()), TypeError, "lengths must be int32 or int64"),
        (dict(ids=ids.view(3, 1)), ValueError, "ids must be 1-D"),
    ]
    for kw, exc, msg in bad:
        args = dict(ids=ids, lengths=lengths)
        args.update(kw)
        with pytest.raises(exc, match=msg):
            ebc(**args)
    assert ebc(ids, torch.tensor([[1, 1, 0], [0, 0, 1]])).shape == (3, 12)      # B follows lengths
    ebc_sum = PSEmbeddingCollection([EmbeddingBagConfig(ta, ["a"]), EmbeddingBagConfig(tb, ["b"])])
    with pytest.raises(ValueError, match="per_sample_weights must have the shape of ids"):
        ebc_sum(ids, lengths, torch.ones(2))
