"""The generic word2vec kernel (`w2v_generic_kernel`: CBOW, hierarchical softmax, AdaGrad and row widths the
register kernels do not take) against a plain fp64 re-implementation of its sample schedule, through
`mvb_sgns_train`.

The model reproduces the kernel's integer RNG exactly: per centre p, rng = hash64(seed ^ (p+1) * golden),
rng = lcg(rng), half-window W - (rng >> 16) % W stopped at sentence breaks and block ends; contexts in position
order; negatives drawn from the block pool (pool[(lcg(rng) >> 8) % n]) or the alias table, K per skip-gram
sample and one set per CBOW centre, skipped when equal to the centre.  The maths is the reference's
FeedForward / BPOutputLayer / TrainSample: CBOW averages its context rows when there are several and gives each
of them the full input step; the HS error is 1 - code - sigma(f), the NS error label - sigma(f); the HS loss
is softplus(-f) for code 0 and softplus(f) for code 1.

The model evaluates every sample on the initial rows.  The kernel runs the centres of these small blocks
concurrently, so a warp may read a row that other samples of the launch have already stepped.  A row stepped
k times (the HS root is on every path: ~1000 samples here) moves by up to lr * k * |err| * |row| (the same
context words repeat), and every step rounds to fp32 (relative to the step, about 2^-24 / (sqrt(12) lr |err|)).
With rows of norm ~1, lr = 2e-5 and |err| ~ 0.5, lr * k * |row|^2 is ~2e-2 at the root, and both effects stay
below ~7e-3 relative Frobenius error of the table deltas on an H100.  The tolerance is 1.5e-2.  Each mutation
of the kernel maths this suite was checked against fails at least one case by 10x that or more: CBOW average
dropped (0.9 to 11), HS error or branch code flipped (~2), the centre drawn as a negative (up to 0.22), a
half-window off by one (the pair count, and 0.13 to 1.0).  Loss sums are compared to 1e-3 relative (measured
<= 2e-4; a flipped loss sign moves them by up to 1.5e-2) and pair counts exactly.

AdaGrad runs with lr = init_learning_rate (0.025), as the callers pass it, in two regimes:
  * contention-free: sentences of two distinct words, window 1, no negatives: every row is stepped by exactly
    one sample, so the model matches to fp32 rounding (the first step is lr * sign(e), through the
    s > 1e-10 guard);
  * contended: repeated words and G^2 tables starting at G0 = 1024, far above a launch's sum of e^2 (~2 on
    the HS root), so sqrt(G) is the same to 1e-3 in any order, a row's delta is the order-free
    lr * sum(e) / sqrt(G0) and its G^2 delta the plain sum of e^2.  With steps of lr / 32 and 2 negatives
    the stale reads cost up to 2.6e-2 (measured on an H100); the tolerance is 5e-2.  A kernel whose plain
    read-modify-writes lose updates misses by 0.56 to 0.95."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15
TOL = 1.5e-2
LOSS_TOL = 1e-3
CONTENDED_TOL = 5e-2


def _hash64(x):
    x &= M64
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


def _lcg(x):
    return (x * 25214903917 + 11) & M64


def _softplus(x):
    return max(x, 0.0) + np.log1p(np.exp(-abs(x)))


def _model(tl, W, K, cbow, hs, lr, i0, o0, seed, pool=None, alias=None, huff=None,
           adagrad=False, g2i0=None, g2o0=None):
    """fp64 deltas (in, out, g2_in, g2_out), loss sum and pair count of one launch; every read sees the
    initial rows i0 / o0.  AdaGrad G^2 sums accumulate in schedule order."""
    n = len(tl)
    d_in, d_out = np.zeros_like(i0), np.zeros_like(o0)
    G_in = None if g2i0 is None else g2i0.copy()
    G_out = None if g2o0 is None else g2o0.copy()
    loss, pairs = 0.0, 0

    def negative(rng):
        rng = _lcg(rng)
        if pool is not None:
            return pool[(rng >> 8) % len(pool)], rng
        prob, idx = alias
        j = (rng >> 16) % len(prob)
        rng = _lcg(rng)
        u = ((rng >> 24) & 0xFFFFFF) / 16777216.0            # exact in fp32 and fp64
        return (j if u < prob[j] else int(idx[j])), rng

    def step(G, r, e):
        G[r] += e * e
        return np.where(G[r] > 1e-10, e * lr / np.sqrt(np.maximum(G[r], 1e-30)), 0.0)

    for p, c in enumerate(tl):
        if c < 0:
            continue
        rng = _lcg(_hash64(seed ^ (((p + 1) * GOLD) & M64)))
        hw = W - (rng >> 16) % W
        ctx = []
        for sgn in (-1, 1):
            for s in range(1, hw + 1):
                q = p + sgn * s
                if q < 0 or q >= n or tl[q] < 0:
                    break
                ctx.append(q)
        ctx.sort()
        if not ctx:
            continue
        for ins in ([[tl[q] for q in ctx]] if cbow else [[tl[q]] for q in ctx]):
            hid = sum(i0[x] for x in ins)
            if len(ins) > 1:
                hid = hid / len(ins)
            if hs:
                pts, cds, ln = huff
                outs = [(int(pts[c, d]), int(cds[c, d])) for d in range(ln[c])]
            else:
                outs = [(c, 1)]
                for _ in range(K):
                    t, rng = negative(rng)
                    if t != c:
                        outs.append((t, 0))
            herr = np.zeros_like(hid)
            for o, label in outs:
                f = float(hid @ o0[o])
                sg = 1.0 / (1.0 + np.exp(-f))
                err = (1.0 - label - sg) if hs else (label - sg)
                loss += _softplus(-f) if (label == 0 if hs else label == 1) else _softplus(f)
                herr += err * o0[o]
                d_out[o] += step(G_out, o, err * hid) if adagrad else lr * err * hid
            for x in ins:
                d_in[x] += step(G_in, x, herr) if adagrad else lr * herr
            pairs += 1
    dg_in = None if G_in is None else G_in - g2i0
    dg_out = None if G_out is None else G_out - g2o0
    return d_in, d_out, dg_in, dg_out, loss, pairs


def _rel(d, r):
    return float(np.linalg.norm(d - r) / np.linalg.norm(r))


def _zipf_counts(V):
    return np.maximum(np.round(1e6 / np.arange(1, V + 1)), 1.0)


def _tokens(n_tok, V, rng, pairs_only=False):
    """Zipf tokens with sentence breaks on the first and last position, two adjacent breaks, an isolated word
    (a centre with no context) and, at 80..82, a CBOW centre whose window holds the same word twice."""
    if pairs_only:                                            # a b -1 c d -1 ...: every word once
        ids = rng.permutation(V)[: 2 * (n_tok // 3)]
        tl = []
        for i in range(0, len(ids), 2):
            tl += [int(ids[i]), int(ids[i + 1]), -1]
        return tl
    w = 1.0 / np.arange(1, V + 1)
    tl = rng.choice(V, size=n_tok, p=w / w.sum()).tolist()
    for b in [0, n_tok - 1, 30, 31] + list(range(45, n_tok, 41)):
        tl[b] = -1
    tl[60], tl[61], tl[62] = -1, 999, -1
    tl[79:84] = [5, 7, 8, 7, 6]
    return tl


def _run(mode, out, dim, *, n_tok=200, W=5, K=5, V=1000, ld=None, maps=False, hogwild=0,
         adagrad=None, seed=0x5EED, lr=2e-5, scale=1.0, G0=1024.0):
    """One launch of `mvb_sgns_train` on the generic kernel and the fp64 model of it.  `out` is "hs", "pool"
    or "alias"; adagrad is None, "exact", "exact_zero_out" or "contended"."""
    from multiverso_b200 import _native as N
    from multiverso_b200.models.wordembedding import HuffmanTables
    cbow, hs = mode == "cbow", out == "hs"
    rng = np.random.default_rng(dim * 131 + W + K + len(out) + (7 if cbow else 0))
    D, LD = dim, ld or dim
    a_ = scale * np.sqrt(3.0 / D)                            # rows uniform in +-a_: norm ~ scale
    i0 = rng.uniform(-a_, a_, (V, D))
    o0 = rng.uniform(-a_, a_, (V, D))
    if adagrad == "exact_zero_out":
        o0[:] = 0.0
    tl = _tokens(n_tok, V, rng, pairs_only=adagrad is not None and adagrad.startswith("exact"))
    g2i0 = g2o0 = None
    if adagrad is not None:
        G0 = G0 if adagrad == "contended" else 0.0
        g2i0, g2o0 = np.full((V, D), G0), np.full((V, D), G0)
        lr = 0.025
    counts = _zipf_counts(V)
    pool_l = alias_np = huff_np = None
    dev = {}
    if hs:
        h = HuffmanTables(counts, "cuda")
        huff_np = (h.points.cpu().numpy(), h.codes.cpu().numpy(), h.lens.cpu().numpy())
        dev["huff"] = h
    elif out == "pool":
        # hot words, which are often the centre too; the contended AdaGrad runs draw from 20 colder words so
        # that no pool row collects more steps than the HS root
        pool_l = list(range(100, 120)) if adagrad == "contended" else [0, 1, 2, 3, 1, 40, 500]
        dev["pool"] = torch.tensor(pool_l, dtype=torch.int32, device="cuda")
    else:
        prob = np.empty(V, dtype=np.float32)
        idx = np.empty(V, dtype=np.int32)
        w = np.power(counts, 0.75)
        N.cuda_lib().mvb_build_alias_table(w.ctypes.data, V, prob.ctypes.data, idx.ctypes.data)
        alias_np = (prob.astype(np.float64), idx)
        dev["prob"], dev["idx"] = torch.from_numpy(prob).cuda(), torch.from_numpy(idx).cuda()
    kK = 0 if hs else K

    # device tables: rows by id, or by slot through id -> slot maps, in rows of pitch LD (the pad must stay 0)
    perm_in = rng.permutation(V) if maps else np.arange(V)
    perm_out = rng.permutation(V) if maps else np.arange(V)

    def table(x, perm):
        t = np.zeros((V, LD), dtype=np.float32)
        t[perm, :D] = x
        return torch.from_numpy(t).cuda()

    w_in, w_out = table(i0, perm_in), table(o0, perm_out)
    i0, o0 = w_in.double().cpu().numpy()[perm_in, :D], w_out.double().cpu().numpy()[perm_out, :D]   # fp32 values
    before = (w_in.clone(), w_out.clone())
    g2 = [table(g2i0, perm_in), table(g2o0, perm_out)] if adagrad is not None else [None, None]
    toks = torch.tensor(tl, dtype=torch.int32, device="cuda")
    loss = torch.zeros(1, device="cuda")
    pairs = torch.zeros(1, dtype=torch.int64, device="cuda")
    m_in = torch.from_numpy(perm_in.astype(np.int32)).cuda() if maps else None
    m_out = torch.from_numpy(perm_out.astype(np.int32)).cuda() if maps else None

    a = N.Sgns()
    a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
    a.w_in, a.w_out, a.dim, a.ld = w_in.data_ptr(), w_out.data_ptr(), D, LD
    a.g2_in, a.g2_out = N.ptr(g2[0]), N.ptr(g2[1])
    a.window, a.negative, a.lr = W, kK, lr
    a.cbow, a.hs, a.use_adagrad, a.hogwild = int(cbow), int(hs), int(adagrad is not None), hogwild
    a.vocab = V
    if hs:
        h = dev["huff"]
        a.hs_points, a.hs_codes = h.points.data_ptr(), h.codes.data_ptr()
        a.hs_len, a.hs_max_code = h.lens.data_ptr(), h.max_code
    elif out == "pool":
        a.neg_pool, a.neg_pool_size = dev["pool"].data_ptr(), len(pool_l)
    else:
        a.alias_prob, a.alias_idx = dev["prob"].data_ptr(), dev["idx"].data_ptr()
    a.map_in, a.map_out = N.ptr(m_in), N.ptr(m_out)
    a.seed, a.loss_sum, a.pair_count = seed, loss.data_ptr(), pairs.data_ptr()
    N.cuda_lib().mvb_sgns_train(a, N.stream_ptr())
    torch.cuda.synchronize()
    assert N.cuda_lib().mvb_sgns_last_launches() == 1          # one generic-kernel launch

    huff_m = None if huff_np is None else (huff_np[0], huff_np[1], huff_np[2])
    r_in, r_out, rg_in, rg_out, r_loss, r_pairs = _model(
        tl, W, kK, cbow, hs, lr, i0, o0, seed, pool=pool_l, alias=alias_np, huff=huff_m,
        adagrad=adagrad is not None, g2i0=g2i0, g2o0=g2o0)
    res = dict(tl=tl, r_in=r_in, r_out=r_out, r_loss=r_loss, r_pairs=r_pairs, rg_in=rg_in, rg_out=rg_out,
               pairs=int(pairs.item()), loss=float(loss.item()))
    new_in, new_out = w_in.double().cpu().numpy(), w_out.double().cpu().numpy()
    res["d_in"] = new_in[perm_in, :D] - i0
    res["d_out"] = new_out[perm_out, :D] - o0
    if adagrad is not None:
        res["dg_in"] = g2[0].double().cpu().numpy()[perm_in, :D] - g2i0
        res["dg_out"] = g2[1].double().cpu().numpy()[perm_out, :D] - g2o0
        res["g2_pad"] = [g[:, D:] for g in g2]
    # rows the model never steps, and the pad columns, keep their bits
    for side, (new, old, r, perm) in enumerate([(w_in, before[0], r_in, perm_in), (w_out, before[1], r_out, perm_out)]):
        still = torch.from_numpy(perm[~np.any(r != 0, axis=1)]).cuda()
        assert torch.equal(new[still], old[still]), f"untouched {'output' if side else 'input'} rows changed"
        assert torch.equal(new[:, D:], old[:, D:]), "pad columns changed"
    return res


def _check(res, tol=TOL, loss_tol=LOSS_TOL):
    assert res["pairs"] == res["r_pairs"], (res["pairs"], res["r_pairs"])
    e_in, e_out = _rel(res["d_in"], res["r_in"]), _rel(res["d_out"], res["r_out"])
    e_loss = abs(res["loss"] - res["r_loss"]) / res["r_loss"]
    assert e_in < tol and e_out < tol and e_loss < loss_tol, (e_in, e_out, e_loss)
    return e_in, e_out, e_loss


CASES = [
    # mode, negatives, dim, extra
    ("sg", "hs", 64, {}), ("sg", "hs", 100, {}), ("sg", "hs", 300, {}),
    ("cbow", "hs", 64, {}), ("cbow", "hs", 100, {}), ("cbow", "hs", 300, {}),
    ("cbow", "pool", 64, {}), ("cbow", "pool", 100, {}), ("cbow", "pool", 300, {}),
    ("cbow", "alias", 64, {}), ("cbow", "alias", 100, {}), ("cbow", "alias", 300, {}),
    ("sg", "hs", 37, {}), ("cbow", "pool", 37, {}), ("cbow", "alias", 37, {}),
    ("sg", "pool", 37, {"hogwild": 1}),                      # skip-gram + NS off the register kernels' widths
    ("sg", "alias", 37, {"K": 8}),                           # 8 negatives: the deterministic kernel declines
    ("sg", "pool", 50, {"K": 8}),
    ("cbow", "hs", 100, {"ld": 112, "maps": True}),           # block-cache layout: slots and padded rows
    ("sg", "hs", 37, {"ld": 40, "maps": True}),
    ("cbow", "pool", 100, {"ld": 104, "maps": True}),
    ("sg", "hs", 100, {"W": 1}), ("cbow", "alias", 100, {"W": 1}),
    ("sg", "hs", 64, {"W": 15, "n_tok": 120}), ("cbow", "pool", 100, {"W": 15}),
]


@pytest.mark.parametrize("mode,out,dim,extra", CASES,
                         ids=[f"{m}-{o}-d{d}" + "".join(f"-{k}{v}" for k, v in e.items()) for m, o, d, e in CASES])
def test_generic_kernel_matches_fp64_schedule(mv_device, mode, out, dim, extra):
    res = _run(mode, out, dim, **extra)
    assert res["tl"][60] == res["tl"][62] == -1 and res["r_pairs"] > 0     # position 61 is a centre with no context
    _check(res)


@pytest.mark.parametrize("mode", ["sg", "cbow"])
def test_generic_kernel_adagrad_contention_free_is_exact(mv_device, mode):
    """Each row is stepped by exactly one sample, from G^2 = 0: the step is lr * sign(e) and G^2 = e^2."""
    res = _run(mode, "pool", 100, W=1, K=0, n_tok=300, adagrad="exact")
    assert res["pairs"] == res["r_pairs"] == 200
    for got, want in [(res["d_in"], res["r_in"]), (res["d_out"], res["r_out"]),
                      (res["dg_in"], res["rg_in"]), (res["dg_out"], res["rg_out"])]:
        assert _rel(got, want) < 1e-5, _rel(got, want)
    stepped = res["r_out"] != 0
    assert np.allclose(np.abs(res["d_out"][stepped]), 0.025, rtol=1e-5)
    assert abs(res["loss"] - res["r_loss"]) / res["r_loss"] < 1e-5


@pytest.mark.parametrize("mode", ["sg", "cbow"])
def test_generic_kernel_adagrad_zero_output_rows(mv_device, mode):
    """The reference's initial output rows are zero: the input error is zero, so the input rows and their
    G^2 sums stay exactly as they were while every output row takes a step of lr * sign(g)."""
    res = _run(mode, "pool", 64, W=1, K=0, n_tok=300, adagrad="exact_zero_out")
    assert np.abs(res["d_in"]).max() == 0 and np.abs(res["dg_in"]).max() == 0 and np.abs(res["r_in"]).max() == 0
    assert _rel(res["d_out"], res["r_out"]) < 1e-5 and _rel(res["dg_out"], res["rg_out"]) < 1e-5
    assert np.allclose(np.abs(res["d_out"][res["r_out"] != 0]), 0.025, rtol=1e-5)


@pytest.mark.parametrize("mode,out", [("sg", "pool"), ("sg", "hs"), ("cbow", "pool"), ("cbow", "hs")])
def test_generic_kernel_adagrad_contended_loses_no_update(mv_device, mode, out):
    """Repeated words: many warps step the same rows and G^2 sums at once.  With G0 = 1024 every step is
    lr * e / 32 to 1e-3 in any order, so the row deltas and the G^2 deltas (plain sums of e^2) must match."""
    res = _run(mode, out, 100, K=2, adagrad="contended")
    e = [_rel(res["d_in"], res["r_in"]), _rel(res["d_out"], res["r_out"]),
         _rel(res["dg_in"], res["rg_in"]), _rel(res["dg_out"], res["rg_out"])]
    assert res["pairs"] == res["r_pairs"]
    assert max(e) < CONTENDED_TOL, e
