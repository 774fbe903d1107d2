"""The vectorised fp64 model of the deterministic skip-gram schedule (tests/sgns_det_model.py), which the GPU tests
of `mvb_sgns_train_det` hold the kernel to, against a plain loop over positions: one centre, one context, one output
row at a time, with Python-integer hashes.  Small random cases span breaks, K = 1..7, W = 1..15, alias and pool
negatives, a pool size smaller than the pool, a one-word pool equal to every centre, compact row maps with padded
rows, step scales, waves of a few centres and blocks split over several calls."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sgns_det_model as sdm  # noqa: E402

M64 = sdm.M64


def _hash64(x):
    x &= M64
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


def _loop(case, wave):
    """The schedule one position at a time (the loop of test_gpu_sgns_det_tiles._check_schedule, with waves,
    calls, maps, the pool size, the loss and the rows read)."""
    c = case["c"]
    V, D, W, K, lr = c["V"], c["D"], c["W"], c["K"], case["lr"]
    mi, mo = sdm.word_maps(case)
    si = np.ones(V) if case["s_in"] is None else case["s_in"].double().numpy()
    so = np.ones(V) if case["s_out"] is None else case["s_out"].double().numpy()
    IN, OUT = case["w_in"][:, :D].double().numpy().copy(), case["w_out"][:, :D].double().numpy().copy()
    read_in, read_out = np.zeros(IN.shape[0], dtype=bool), np.zeros(OUT.shape[0], dtype=bool)
    tokens = case["tokens"].tolist()
    pairs, loss = 0, 0.0
    cuts = c.get("calls", (0, len(tokens)))
    for s, e in zip(cuts[:-1], cuts[1:]):
        tl, seed, n = tokens[s:e], case["seed"] + s, e - s
        for p0 in range(0, n, wave):
            i0, o0 = IN.copy(), OUT.copy()                   # the tables as the previous wave left them
            for p in range(p0, min(p0 + wave, n)):
                x = tl[p]
                if x < 0 or mo[x] < 0:
                    continue
                prng = _hash64(seed ^ (((p + 1) * sdm.GOLD) & M64))
                hw = W - ((prng >> 16) % W)
                ctxs = []
                for sgn in (-1, 1):
                    for d in range(1, hw + 1):
                        q = p + sgn * d
                        if q < 0 or q >= n or tl[q] < 0 or mi[tl[q]] < 0:
                            break
                        ctxs.append(tl[q])
                outs = [(x, 1.0)]
                for k in range(1, K + 1):
                    r = _hash64(prng ^ ((k * sdm.NEG) & M64))
                    if case["pool"] is not None:
                        pool_n = case.get("pool_n", len(case["pool"]))
                        t = int(case["pool"][(r >> 8) % pool_n]) if pool_n > 0 else -1
                    else:
                        idx = (r >> 32) % V
                        u = np.float32(r & 0xFFFFFF) * np.float32(1.0 / 16777216.0)
                        t = idx if u < case["prob"][idx] else int(case["alias"][idx])
                    if t >= 0 and t != x and mo[t] >= 0:
                        outs.append((t, 0.0))
                for y in ctxs:
                    h = i0[mi[y]]
                    read_in[mi[y]] = True
                    for (o, label) in outs:
                        f = float(h @ o0[mo[o]])
                        g = (label - 1.0 / (1.0 + np.exp(-f))) * lr
                        IN[mi[y]] += g * si[y] * o0[mo[o]]
                        OUT[mo[o]] += g * so[o] * h
                        read_out[mo[o]] = True
                        if p % 8 == 0:
                            loss += 8.0 * float(np.logaddexp(0.0, -f if label else f))
                    pairs += 1
    return IN, OUT, read_in, read_out, pairs, loss


def _case(seed, *, V=48, D=5, W=5, K=5, n=120, breaks=(), neg="pool", pool=None, pool_n=None, maps=False,
          scales=True, calls=None, word=None):
    g = torch.Generator().manual_seed(seed)
    rows = V + 7 if maps else V
    LD = D + 3 if maps else D
    w_in, w_out = torch.full((rows, LD), 9.0), torch.full((rows, LD), -9.0)
    w_in[:, :D] = (torch.rand(rows, D, generator=g) - 0.5) * 1.2        # scores of order 1: varied gradients
    w_out[:, :D] = (torch.rand(rows, D, generator=g) - 0.5) * 1.2
    toks = torch.full((n,), word, dtype=torch.int32) if word is not None else \
        torch.randint(0, V, (n,), generator=g, dtype=torch.int32)
    for b in breaks:
        toks[b] = -1
    c = dict(V=V, D=D, LD=LD, W=W, K=K, n_tok=n)
    if calls is not None:
        c["calls"] = calls
    case = dict(c=c, tokens=toks, w_in=w_in, w_out=w_out, map=None, prob=None, alias=None, pool=None,
                s_in=0.5 + torch.rand(V, generator=g) if scales else None,
                s_out=0.5 + torch.rand(V, generator=g) if scales else None, lr=0.02, seed=0x5EED + seed)
    if maps:
        case["map_in"] = torch.randperm(rows, generator=g)[:V].to(torch.int32)
        case["map_out"] = torch.randperm(rows, generator=g)[:V].to(torch.int32)
    if neg == "pool":
        case["pool"] = torch.randint(0, V, (11,), generator=g, dtype=torch.int32) if pool is None else \
            torch.tensor(pool, dtype=torch.int32)
        if pool_n is not None:
            case["pool_n"] = pool_n
    else:
        case["prob"] = torch.rand(V, generator=g).numpy().astype(np.float32)
        case["alias"] = torch.randint(0, V, (V,), generator=g).numpy()
    return case


CASES = {
    "w1_k1": dict(W=1, K=1, breaks=(0, 7, 8, 50)),
    "w2_k2_alias": dict(W=2, K=2, neg="alias"),
    "w3_k3_maps": dict(W=3, K=3, maps=True, breaks=(119,)),
    "w4_k4_pool_n": dict(W=4, K=4, pool_n=3),
    "w6_k5_noscale": dict(W=6, K=5, scales=False, breaks=range(0, 120, 13)),
    "w7_k6_alias_maps": dict(W=7, K=6, neg="alias", maps=True),
    "w9_k7": dict(W=9, K=7, D=9),
    "w11_k7_breaks": dict(W=11, K=7, breaks=range(1, 120, 4)),
    "w13_k2_3calls": dict(W=13, K=2, calls=(0, 37, 38, 120)),
    "w15_k5_3calls_alias": dict(W=15, K=5, neg="alias", calls=(0, 50, 90, 120), maps=True),
    "w15_k7_long": dict(W=15, K=7, n=300),
    "w8_k3_one_word_pool": dict(W=8, K=3, word=4, pool=[4]),   # every negative is the centre: skipped
    "w5_k7_one_word": dict(W=5, K=7, word=4, calls=(0, 60, 120)),
    "w10_k1_all_breaks_but_one": dict(W=10, K=1, breaks=[i for i in range(120) if i != 60]),
    "w12_k6_pool_n0": dict(W=12, K=6, pool_n=0),               # no negatives at all
}


@pytest.mark.parametrize("wave", [7, 16, 1000])
@pytest.mark.parametrize("name", sorted(CASES))
def test_sgns_det_model_matches_loop(name, wave):
    case = _case(sorted(CASES).index(name) + 1, **CASES[name])
    got = sdm.model(case, wave)
    IN, OUT, read_in, read_out, pairs, loss = _loop(case, wave)
    D = case["c"]["D"]
    assert got["pairs"] == pairs
    assert np.array_equal(got["read_in"], read_in) and np.array_equal(got["read_out"], read_out)
    for ref, mine, init in ((IN, got["w_in"], case["w_in"]), (OUT, got["w_out"], case["w_out"])):
        d_ref = ref - init[:, :D].double().numpy()
        d_mine = mine.numpy() - init[:, :D].double().numpy()
        scale = max(np.linalg.norm(d_ref), 1e-300)
        assert np.linalg.norm(d_mine - d_ref) <= 1e-12 * scale, (np.linalg.norm(d_mine - d_ref), scale)
    assert abs(got["loss"] - loss) <= 1e-12 * abs(loss)
    if name == "w10_k1_all_breaks_but_one":
        assert pairs == 0 and loss == 0.0
    else:
        assert pairs > 0 and loss > 0


def test_sgns_det_model_waves_see_previous_wave():
    """A one-centre wave reads what the wave before it wrote: the model differs from one wave over the block."""
    case = _case(99, W=3, K=2, n=40)
    a, b = sdm.model(case, 1), sdm.model(case, 1000)
    assert a["pairs"] == b["pairs"]
    assert not torch.allclose(a["w_in"], b["w_in"], rtol=0, atol=1e-9)
    assert a["loss"] != b["loss"]
