"""PSSampledSoftmax without a GPU: the host backend against an explicit fp64 formula over ssm.draw(step), one sgd step
against a local nn.Parameter + torch.optim.SGD, one momentum / AdaGrad step per touched row, accidental-hit masking,
the draws (a pure function of (seed, step), frequencies matching q) and every named error."""
import math
import types

import numpy as np
import pytest
import torch
from scipy import stats

from multiverso_b200.ops import PSSampledSoftmax
from multiverso_b200.ops.sampled_softmax import draw_reference
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
    """A host table stand-in whose add_rows applies momentum_sgd or adagrad in fp64 with the device updaters' rules
    (csrc/cuda/mvb_common.cuh) and counts the steps of every row."""

    def __init__(self, W, updater):
        self.w = W.double().numpy().copy()
        self.s = np.zeros_like(self.w)
        self.steps = np.zeros(W.shape[0], dtype=np.int64)
        self.num_row, self.num_col = W.shape
        self.npdt, self.updater = np.float32, updater
        self.calls = 0

    def get_rows(self, ids):
        return self.w[np.asarray(ids)].astype(np.float32)

    def add_rows(self, ids, vals, option=None):
        ids, g = np.asarray(ids), np.asarray(vals, dtype=np.float64)
        assert len(np.unique(ids)) == len(ids)               # one coalesced row per id and call
        self.steps[ids] += 1
        self.calls += 1
        step(self.w, self.s, ids, g, self.updater, option)


def step(w, s, ids, g, updater, option):
    if updater == "momentum_sgd":
        s[ids] = option.momentum * s[ids] + (1.0 - option.momentum) * g
        w[ids] -= s[ids]
    else:
        gn = g / option.learning_rate
        s[ids] += gn * gn
        w[ids] -= option.rho / np.sqrt(s[ids] + 1e-6) * gn


def _q(n, counts=None, power=0.75):
    """q in fp64: log-uniform, or counts^power normalised."""
    if counts is None:
        k = np.arange(n, dtype=np.float64)
        return np.log((k + 2) / (k + 1)) / math.log(n + 1)
    w = np.power(np.asarray(counts, dtype=np.float64), power)
    return w / w.sum()


def _loss64(x, W, y, cand, q):
    """The defining formula in fp64: loss_b = logsumexp(t_b, s_b.) - t_b with log(S q) corrections, hits masked."""
    S = cand.numel()
    logq = torch.from_numpy(np.log(S * q))
    t = (x * W[y]).sum(1) - logq[y]
    s = x @ W[cand].t() - logq[cand][None, :]
    s = s.masked_fill(cand[None, :] == y[:, None], float("-inf"))
    return torch.logsumexp(torch.cat([t[:, None], s], 1), 1) - t


@pytest.mark.parametrize("sampler", ["log_uniform", "counts"])
def test_loss_and_grad_match_fp64_formula(mv_host, sampler):
    g = torch.Generator().manual_seed(0)
    n, d, B, S = 300, 12, 40, 64
    W = torch.randn(n, d, generator=g) * 0.5
    counts = torch.randint(1, 1000, (n,), generator=g) if sampler == "counts" else None
    ssm = PSSampledSoftmax(_host_table(mv_host, W), num_sampled=S, push_scale=None, seed=7,
                           **({"counts": counts} if counts is not None else {"sampler": "log_uniform"}))
    x = torch.randn(B, d, generator=g, requires_grad=True)
    y = torch.randint(0, n, (B,), generator=g)
    for step in range(2):
        x.grad = None
        loss = ssm(x, y.to(torch.int32))
        loss.sum().backward()
        cand = ssm.draw(step)
        x64 = x.detach().double().requires_grad_()
        ref = _loss64(x64, W.double(), y, cand, _q(n, counts))
        ref.sum().backward()
        assert torch.allclose(loss.detach().double(), ref.detach(), rtol=1e-5, atol=1e-5)
        assert torch.allclose(x.grad.double(), x64.grad, rtol=1e-4, atol=1e-5)
    assert ssm.steps == 2


def test_sgd_step_equals_local_parameter(mv_host):
    """push_scale = -lr on the default (adding) updater: the touched rows take one SGD step of the summed gradient,
    exactly as a local nn.Parameter with the same loss and torch.optim.SGD; the other rows stay unchanged."""
    g = torch.Generator().manual_seed(1)
    n, d, B, S, lr = 200, 8, 32, 48, 0.3
    W = torch.randn(n, d, generator=g)
    t = _host_table(mv_host, W)
    ssm = PSSampledSoftmax(t, num_sampled=S, sampler="log_uniform", push_scale=-lr, seed=3)
    x = torch.randn(B, d, generator=g)
    y = torch.randint(0, n, (B,), generator=g)
    ssm(x, y).mean().backward()
    P = torch.nn.Parameter(W.double().clone())
    opt = torch.optim.SGD([P], lr=lr)
    _loss64(x.double(), P, y, ssm.draw(0), _q(n)).mean().backward()
    opt.step()
    got = torch.from_numpy(t.get()).double()
    touched = torch.unique(torch.cat([y, ssm.draw(0)]))
    untouched = torch.ones(n, dtype=torch.bool)
    untouched[touched] = False
    assert torch.allclose(got[touched], P.detach()[touched], atol=2e-6)
    assert torch.equal(got[untouched].float(), W[untouched])
    assert not torch.allclose(got[touched], W.double()[touched])


@pytest.mark.parametrize("updater", ["momentum_sgd", "adagrad"])
def test_one_stateful_step_per_row(updater):
    """A row that is a label and a (duplicated) candidate in one call takes one momentum / AdaGrad step with its
    summed gradient; pushing the label part and the candidate part separately would not give that result."""
    g = torch.Generator().manual_seed(2)
    n, d, B, S, scale = 16, 4, 12, 40, 0.5                    # S >> n: candidates repeat
    W = torch.randn(n, d, generator=g)
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    tab = StatefulTable(W, updater)
    ssm = PSSampledSoftmax(tab, num_sampled=S, sampler="log_uniform", push_scale=scale, option=opt, seed=5)
    cand = ssm.draw(0)
    ids, cnt = torch.unique(cand, return_counts=True)
    dup = int(ids[cnt > 1][0])
    y = torch.randint(0, n, (B,), generator=g)
    y[:3] = dup                                              # the duplicated candidate is also a label
    x = torch.randn(B, d, generator=g)
    ssm(x, y).sum().backward()
    touched = torch.unique(torch.cat([y, cand])).numpy()
    assert tab.calls == 1 and (tab.steps[touched] == 1).all() and tab.steps.sum() == touched.size
    P = W.double().clone().requires_grad_()
    _loss64(x.double(), P, y, cand, _q(n)).sum().backward()
    G = P.grad.numpy() * scale
    w, s = W.double().numpy().copy(), np.zeros((n, d))
    step(w, s, touched, G[touched], updater, opt)
    assert np.abs(tab.w - w).max() < 1e-6
    # two pushes (label rows, then candidate rows) take two steps for `dup`: a different result
    Pl = W.double().clone().requires_grad_()
    x64 = x.double()
    logq = torch.from_numpy(np.log(S * _q(n)))
    t = (x64 * Pl[y]).sum(1) - logq[y]
    s_ = (x64 @ W.double()[cand].t() - logq[cand][None, :]).masked_fill(cand[None, :] == y[:, None], float("-inf"))
    (torch.logsumexp(torch.cat([t[:, None], s_], 1), 1) - t).sum().backward()
    Gl = Pl.grad.numpy() * scale
    w2, s2 = W.double().numpy().copy(), np.zeros((n, d))
    lab = np.unique(y.numpy())
    step(w2, s2, lab, Gl[lab], updater, opt)
    cu = np.unique(cand.numpy())
    step(w2, s2, cu, G[cu] - Gl[cu], updater, opt)
    assert np.abs(w2[dup] - w[dup]).max() > 1e-4


def test_accidental_hits_are_masked(mv_host):
    g = torch.Generator().manual_seed(4)
    n, d, S = 100, 8, 32
    W = torch.randn(n, d, generator=g)
    ssm = PSSampledSoftmax(_host_table(mv_host, W), num_sampled=S, sampler="log_uniform", push_scale=None, seed=9)
    y = ssm.draw(ssm.steps)[:16].clone()                   # every label is one of this call's candidates
    x = torch.randn(16, d, generator=g)
    loss = ssm(x, y)
    cand = ssm.draw(0)
    ref = _loss64(x.double(), W.double(), y, cand, _q(n))
    assert torch.allclose(loss.double(), ref, rtol=1e-5, atol=1e-5)
    logq = torch.from_numpy(np.log(S * _q(n)))
    t = (x.double() * W.double()[y]).sum(1) - logq[y]
    unmasked = torch.logsumexp(torch.cat([t[:, None], x.double() @ W.double()[cand].t() - logq[cand]], 1), 1) - t
    assert (unmasked > ref).all() and (unmasked - ref).max() > 1e-2     # the hit columns really were removed


def test_draw_is_a_pure_function_of_seed_and_step(mv_host):
    W = torch.zeros(500, 4)
    t = _host_table(mv_host, W)
    a = PSSampledSoftmax(t, num_sampled=256, sampler="log_uniform", push_scale=None, seed=11)
    b = PSSampledSoftmax(t, num_sampled=256, sampler="log_uniform", push_scale=None, seed=11)
    c = PSSampledSoftmax(t, num_sampled=256, sampler="log_uniform", push_scale=None, seed=12)
    d3 = a.draw(3)
    a(torch.zeros(2, 4), torch.tensor([0, 1]))
    assert torch.equal(a.draw(3), d3) and torch.equal(b.draw(3), d3)
    assert not torch.equal(a.draw(4), d3) and not torch.equal(c.draw(3), d3)
    assert d3.dtype == torch.int64 and d3.min() >= 0 and d3.max() < 500
    assert np.array_equal(draw_reference(a._prob, a._alias, 11, 3, 256), d3.numpy())


@pytest.mark.parametrize("sampler", ["log_uniform", "counts"])
def test_draw_frequencies_match_q(sampler):
    """Seeded chi-square test of 10^6 draws against q (bins with an expectation below 20 merged)."""
    n, draws = 1000, 10**6
    rng = np.random.default_rng(0)
    counts = rng.zipf(1.3, n).astype(np.float64) if sampler == "counts" else None
    if counts is not None:
        counts[::97] = 0                                     # rows that must never be drawn
    tab = types.SimpleNamespace(num_row=n, num_col=4, npdt=np.float32)
    ssm = PSSampledSoftmax(tab, num_sampled=draws, push_scale=None, seed=1,
                           **({"counts": counts} if counts is not None else {"sampler": "log_uniform"}))
    got = np.bincount(ssm.draw(0).numpy(), minlength=n).astype(np.float64)
    q = _q(n, counts)
    if counts is not None:
        assert got[counts == 0].sum() == 0
    exp = q * draws
    big = exp >= 20
    obs_b, exp_b = np.append(got[big], got[~big].sum()), np.append(exp[big], exp[~big].sum())
    keep = exp_b > 0
    p = stats.chisquare(obs_b[keep], exp_b[keep]).pvalue
    assert p > 1e-4, p


def test_named_errors(mv_host):
    W = torch.randn(50, 8)
    t = _host_table(mv_host, W)
    ok = dict(num_sampled=8, sampler="log_uniform")
    with pytest.raises(ValueError, match="exactly one of"):
        PSSampledSoftmax(t, num_sampled=8)
    with pytest.raises(ValueError, match="exactly one of"):
        PSSampledSoftmax(t, num_sampled=8, sampler="log_uniform", counts=torch.ones(50))
    with pytest.raises(ValueError, match="sampler must be one of"):
        PSSampledSoftmax(t, num_sampled=8, sampler="uniform")
    with pytest.raises(ValueError, match="one entry per table row"):
        PSSampledSoftmax(t, num_sampled=8, counts=torch.ones(49))
    with pytest.raises(ValueError, match="non-negative"):
        PSSampledSoftmax(t, num_sampled=8, counts=torch.cat([torch.ones(49), -torch.ones(1)]))
    with pytest.raises(ValueError, match="all zero"):
        PSSampledSoftmax(t, num_sampled=8, counts=torch.zeros(50))
    with pytest.raises(ValueError, match="num_sampled must be >= 1"):
        PSSampledSoftmax(t, num_sampled=0, sampler="log_uniform")
    with pytest.raises(TypeError, match="must be float32"):
        PSSampledSoftmax(types.SimpleNamespace(num_row=50, num_col=8, npdt=np.float64), **ok)
    with pytest.raises(ValueError, match="multiple of 4"):
        PSSampledSoftmax(_host_table(mv_host, torch.randn(50, 6)), **ok)
    with pytest.raises(ValueError, match=r"< 2\^31 rows"):
        PSSampledSoftmax(types.SimpleNamespace(num_row=1 << 31, num_col=8, npdt=np.float32), **ok)
    with pytest.raises(TypeError, match="must be a MatrixTable"):
        PSSampledSoftmax(W, **ok)
    ssm = PSSampledSoftmax(t, **ok)
    x = torch.randn(4, 8)
    cases = [
        (TypeError, "2-D float32", x.double(), torch.arange(4)),
        (TypeError, "2-D float32", x[0], torch.arange(4)),
        (ValueError, "hidden has 6 columns", torch.randn(4, 6), torch.arange(4)),
        (ValueError, "one label per row", x, torch.arange(5)),
        (TypeError, "int32 or int64", x, torch.arange(4).float()),
        (ValueError, r"\[0, 50\).*max 50", x, torch.tensor([0, 1, 2, 50])),
        (ValueError, r"\[0, 50\).*min -1", x, torch.tensor([0, -1, 2, 3])),
    ]
    for exc, msg, h, y in cases:
        with pytest.raises(exc, match=msg):
            ssm(h, y)
    for power in (0.0, -0.75, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="power must be finite and > 0"):
            PSSampledSoftmax(t, num_sampled=8, counts=torch.ones(50), power=power)
    with pytest.raises(ValueError, match="overflows"):
        PSSampledSoftmax(t, num_sampled=8, counts=torch.full((50,), 1e6), power=100.0)
    counts = torch.ones(50)
    counts[7] = 0
    zc = PSSampledSoftmax(t, num_sampled=8, counts=counts)
    with pytest.raises(ValueError, match="count zero"):
        zc(x, torch.tensor([0, 7, 1, 2]))
    assert ssm.steps == 0 and zc.steps == 0                 # failed calls draw nothing


@pytest.mark.parametrize("updater", ["default", "momentum_sgd"])
def test_empty_batch_pushes_nothing(mv_host, updater):
    """B = 0: an empty loss whose backward runs and pushes nothing (a momentum table takes no step either)."""
    W = torch.randn(30, 8, generator=torch.Generator().manual_seed(5))
    t = _host_table(mv_host, W) if updater == "default" else StatefulTable(W, updater)
    ssm = PSSampledSoftmax(t, num_sampled=16, sampler="log_uniform", push_scale=0.5,
                           option=AddOption(momentum=0.9, learning_rate=0.5, rho=0.2))
    before = t.get_rows(np.arange(30)).copy()
    for requires_grad in (True, False):
        x = torch.zeros(0, 8, requires_grad=requires_grad)
        loss = ssm(x, torch.zeros(0, dtype=torch.int64))
        assert loss.shape == (0,)
        loss.sum().backward()
    assert np.array_equal(t.get_rows(np.arange(30)), before) and ssm.steps == 2
    if updater != "default":
        assert t.calls == 0


def test_second_backward_raises(mv_host):
    """A call's gradient is pushed once: backpropagating a retained graph a second time raises."""
    W = torch.randn(40, 8, generator=torch.Generator().manual_seed(6))
    t = _host_table(mv_host, W)
    ssm = PSSampledSoftmax(t, num_sampled=16, sampler="log_uniform", push_scale=-0.1)
    loss = ssm(torch.randn(5, 8, requires_grad=True), torch.arange(5))
    loss.sum().backward(retain_graph=True)
    after = t.get().copy()
    with pytest.raises(RuntimeError, match="backward ran twice"):
        loss.sum().backward()
    assert np.array_equal(t.get(), after)
