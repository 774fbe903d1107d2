"""The Hogwild skip-gram kernels (the window kernel `sgns_win_kernel`, locally and in direct mode, and the register
kernel `sgns_fast_kernel`), the alias draws and loss estimator of the deterministic kernel, and the dispatch of
`mvb_sgns_train`, against fp64 models of their sample schedules.

Two models, each reproducing its kernel's integer RNG exactly:

  * per position (window and deterministic kernels): prng = hash64(seed ^ (p+1) phi); half window
    W - (prng >> 16) % W stopped at breaks and block ends; K negatives drawn once per position,
    r_k = hash64(prng ^ k 0xD6E8FEB86659FD93), then pool[(r_k >> 8) % n] or the hash alias rule
    j = (r_k >> 32) % V, u = (r_k & 0xFFFFFF) / 2^24, j if u < prob[j] else alias[j]; a draw equal to the centre
    is skipped.  Every score is taken on the pre-update rows; context c gets s_in(c) sum_k g_ck out_k, output row k
    gets s_out(k) sum_c g_ck in_c, g = (label - sigma(f)) lr.  Loss: 8 sum softplus(-+f) over the centres with
    p % 8 == 0.
  * per pair (register kernel): rng = lcg(hash64(seed ^ (p+1) phi)), half window W - (rng >> 16) % W; contexts in
    position order; each (context, centre) pair draws K fresh negatives from the continuing LCG stream
    (pool[(lcg >> 8) % n], or the alias rule j = (lcg >> 16) % V, u = ((lcg' >> 24) & 0xFFFFFF) / 2^24 over two
    steps).  The centre row is stepped in registers after every context; negatives go in batches of KB = 5, 5, 1,
    2 rows (row widths of 1-4 float4 per lane), a batch's reads taken before its updates.  No scales; the loss is
    the full sum.

Exact regime.  Sentences of two distinct words (a b -1 c d -1 ...), every input row one-hot on a column of its own
with a value in {1/2, 1, 2}, output rows uniform in +-1/2, negatives drawn from words that are never tokens, and
a seed for which no negative row is drawn twice in the whole call.  Then every row is read and written by one
sample only, the kernels are order-free, and each score f = v o[col] is exact in fp32 (|f| <= 1).  What remains
is the sigmoid: sigm_fast = __fdividef(1, 1 + __expf(-f)) is within (3 + 2 + 1/2) ulp of sigma for |f| <= 1
(__expf: 2 + |1.17 f| ulp, __fdividef: 2 ulp), so |g - g_model| <= 2^-20.5 lr; and fp32 rounding: each product
g s x and each of the <= 16 accumulation steps rounds to 2^-24 relative, and the store to half an ulp.  Per
element the bound is

    |got - model| <= 2^-19 lr sum_k s_k |x_k| + 2^-20 sum_k |g_k s_k x_k| + 2^-24 |model|,

where x_k runs over the terms of the element's delta.  The measured worst case on an H100 is below 0.3 of it.
Pair counts are exact, rows outside the touched set and padding columns keep their bits, and the window kernel
gives the same bits on identity tables, on id -> slot caches with padded rows, and in direct mode over 2, 3 and 8
shards.  Loss sums match to 1e-5 relative (fp32 sums of <= 8 __expf / log1pf terms per lane).

Contended regime.  Zipf tokens over a small vocabulary, windows up to 15, breaks at block ends, at CTA chunk
boundaries (computed from the SM count) and at the edges of the register kernel's lane window; negatives are
tokens too, so the centre skip matters.  Thousands of warps read rows that others have already stepped, which
the model (initial rows) cannot follow: a row stepped k times in flight costs an O(lr k) relative error.  With
lr = 2e-5, rows of norm ~1 and a pool of 40 words, the relative Frobenius error of the table deltas measured on an
H100 (80GB HBM3, 700 W) is at most 3.3e-2 for the window kernel (six-word device pool) and 2.1e-2 for the register
kernel (window 15, pool), most cases below 1e-2; the tolerance is 5e-2.  Loss sums measured at most 2.1e-3 off;
the tolerance is 1e-2.  Dropping the centre skip misses by more than that in every case that draws hot words.
Pair counts are exact and the rows outside the model's touched set keep their bits.

The deterministic kernel (one wave: every read sees the initial rows) is held to 1e-4 with a non-uniform
Vose table (measured 7e-7), and its loss estimator to 1e-5 (measured 4e-8).

The dispatch table runs each input of the comment above `mvb_sgns_train` and tells the kernel by its launch count
(deterministic: plan + 2 per wave; the others 1) and by which model matches on the elements no other sample
touches: the per-position model (window, deterministic), the per-pair model with batched negative reads
(register), or with sequential reads, each draw seeing the row after the previous draw's update (generic)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

M64 = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15
KMUL = 0xD6E8FEB86659FD93
KB = {1: 5, 2: 5, 3: 1, 4: 2}          # register kernel: negative rows in flight per batch, by float4 per lane
VX = (1 << 16) + 7                     # exact regime: words (not divisible by 2, 3 or 8)
WIN_TOL, REG_TOL = 5e-2, 5e-2          # contended regime, relative Frobenius error of the table deltas
LOSS_TOL = 1e-2                        # contended regime, loss sums
PAD = -3.25                            # padding columns and gaps between shards hold this / GARBAGE
GARBAGE = 1e3


def _hash64(x):
    x &= M64
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


def _lcg(x):
    return (x * 25214903917 + 11) & M64


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def _softplus(x):
    return np.logaddexp(0.0, x)


class _Sampler:
    """Negative draws of both RNG rules from a pool (n of its entries) or an alias table."""

    def __init__(self, pool=None, n=None, prob=None, idx=None):
        self.pool, self.prob, self.idx = pool, prob, idx
        self.n = len(pool) if pool is not None and n is None else n

    def hashed(self, r):                      # window / deterministic kernels; -1: no draw
        if self.pool is not None:
            return self.pool[(r >> 8) % self.n] if self.n > 0 else -1
        j = (r >> 32) % len(self.prob)
        return j if (r & 0xFFFFFF) / 16777216.0 < self.prob[j] else int(self.idx[j])

    def lcg(self, rng):                       # register / generic kernels
        rng = _lcg(rng)
        if self.pool is not None:
            return self.pool[(rng >> 8) % self.n], rng
        j = (rng >> 16) % len(self.prob)
        rng = _lcg(rng)
        return (j if ((rng >> 24) & 0xFFFFFF) / 16777216.0 < self.prob[j] else int(self.idx[j])), rng


def _window(tl, p, hw):
    ctx = []
    for sgn in (-1, 1):
        for d in range(1, hw + 1):
            q = p + sgn * d
            if q < 0 or q >= len(tl) or tl[q] < 0:
                break
            ctx.append(q)
    return sorted(ctx)


def _sched_pos(tl, W, K, seed, smp):
    """[(p, centre, context positions, negatives)] of the window / deterministic kernels."""
    out = []
    for p, c in enumerate(tl):
        if c < 0:
            continue
        prng = _hash64(seed ^ (((p + 1) * GOLD) & M64))
        ctx = _window(tl, p, W - (prng >> 16) % W)
        negs = []
        for k in range(1, K + 1):
            t = smp.hashed(_hash64(prng ^ ((k * KMUL) & M64)))
            if t >= 0 and t != c:
                negs.append(t)
        if ctx:
            out.append((p, c, ctx, negs))
    return out


def _sched_pair(tl, W, K, seed, smp, kb):
    """[(p, centre, [(context position, [negatives of each batch of kb draws])])] of the register kernel."""
    out = []
    for p, c in enumerate(tl):
        if c < 0:
            continue
        rng = _lcg(_hash64(seed ^ (((p + 1) * GOLD) & M64)))
        samples = []
        for q in _window(tl, p, W - (rng >> 16) % W):
            batches = []
            for d0 in range(0, K, kb):
                b = []
                for d in range(kb):
                    if d0 + d < K:
                        t, rng = smp.lcg(rng)
                        if t != c:
                            b.append(t)
                batches.append(b)
            samples.append((q, batches))
        if samples:
            out.append((p, c, samples))
    return out


class _Model:
    """fp64 deltas of the rows a schedule touches (compact: row i of `din` is word `ids_in[i]`), the element bound
    terms of the exact regime, loss and pair count."""

    def __init__(self, ids_in, ids_out, I0, O0):
        self.ids_in, self.ids_out = ids_in, ids_out
        self.ix_in = {w: i for i, w in enumerate(ids_in)}
        self.ix_out = {w: i for i, w in enumerate(ids_out)}
        self.I0, self.O0 = I0, O0
        z = np.zeros_like
        self.din, self.dout, self.xin, self.xout, self.tin, self.tout = z(I0), z(O0), z(I0), z(O0), z(I0), z(O0)
        self.loss, self.pairs = 0.0, 0


def _ids(sched_rows):
    ins, outs = set(), set()
    for x, o in sched_rows:
        ins.update(x)
        outs.update(o)
    return sorted(ins), sorted(outs)


def _model_pos(sched, tl, lr, rows, s_in=None, s_out=None):
    ids_in, ids_out = _ids([([tl[q] for q in ctx], [c] + negs) for _, c, ctx, negs in sched])
    m = _Model(ids_in, ids_out, rows("in", ids_in), rows("out", ids_out))
    for p, c, ctx, negs in sched:
        xs = [m.ix_in[tl[q]] for q in ctx]
        words = [c] + negs
        os_ = [m.ix_out[o] for o in words]
        H, O = m.I0[xs], m.O0[os_]
        lab = np.array([1.0] + [0.0] * len(negs))
        F = H @ O.T
        G = (lab[None, :] - _sig(F)) * lr
        si = np.ones(len(xs)) if s_in is None else s_in[[tl[q] for q in ctx]].astype(np.float64)
        so = np.ones(len(os_)) if s_out is None else s_out[words].astype(np.float64)
        np.add.at(m.din, xs, si[:, None] * (G @ O))
        np.add.at(m.dout, os_, so[:, None] * (G.T @ H))
        np.add.at(m.tin, xs, si[:, None] * (np.abs(G) @ np.abs(O)))
        np.add.at(m.tout, os_, so[:, None] * (np.abs(G).T @ np.abs(H)))
        np.add.at(m.xin, xs, lr * si[:, None] * np.abs(O).sum(0)[None, :])
        np.add.at(m.xout, os_, lr * so[:, None] * np.abs(H).sum(0)[None, :])
        m.pairs += len(ctx)
        if p % 8 == 0:
            m.loss += 8.0 * float(_softplus(np.where(lab[None, :] > 0, -F, F)).sum())
    return m


def _model_pair(sched, tl, lr, rows):
    ids_in, ids_out = _ids([([tl[q] for q, _ in smp], [c] + [t for _, bs in smp for b in bs for t in b])
                            for _, c, smp in sched])
    m = _Model(ids_in, ids_out, rows("in", ids_in), rows("out", ids_out))
    for p, c, samples in sched:
        ci = m.ix_out[c]
        crow = m.O0[ci].copy()
        for q, batches in samples:
            xi = m.ix_in[tl[q]]
            h = m.I0[xi]
            f = h @ crow
            g = (1.0 - _sig(f)) * lr
            herr, tin, xin = g * crow, np.abs(g * crow), lr * np.abs(crow)
            crow = crow + g * h
            m.dout[ci] += g * h
            m.tout[ci] += np.abs(g * h)
            m.xout[ci] += lr * np.abs(h)
            m.loss += float(_softplus(-f))
            own = {}                                  # this pair's updates of its negative rows so far
            for b in batches:
                read = [m.O0[m.ix_out[t]] + own.get(t, 0.0) for t in b]
                for t, n in zip(b, read):
                    f = h @ n
                    g = -_sig(f) * lr
                    herr, tin, xin = herr + g * n, tin + np.abs(g * n), xin + lr * np.abs(n)
                    ti = m.ix_out[t]
                    m.dout[ti] += g * h
                    m.tout[ti] += np.abs(g * h)
                    m.xout[ti] += lr * np.abs(h)
                    own[t] = own.get(t, 0.0) + g * h
                    m.loss += float(_softplus(f))
            m.din[xi] += herr
            m.tin[xi] += tin
            m.xin[xi] += xin
            m.pairs += 1
    return m


def _bound(x, t, model):
    return 2.0 ** -19 * x + 2.0 ** -20 * t + 2.0 ** -24 * np.abs(model) + 1e-30


def _rel(d, r):
    return float(np.linalg.norm(d - r) / np.linalg.norm(r))


# ---------------------------------------------------------------------------------------------- device tables
class _Table:
    """One table in a layout: "id" (rows by word id, pitch dim), "map" (rows by slot through an id -> slot map,
    padded pitch) or "direct" (S shards at separate places of one buffer, garbage rows between them, padded pitch;
    the reference rows_per_server rule, the last shard takes the remainder)."""

    def __init__(self, base, kind, D, S=1, perm=None, pad=4, gap=37):
        V = base.shape[0]
        self.kind, self.D, self.S = kind, D, S
        self.LD = D if kind == "id" else D + pad
        dev = base.device
        if kind == "id":
            self.t = base.clone()
            self.rows = torch.arange(V, device=dev)
        elif kind == "map":
            self.t = torch.full((V, self.LD), PAD, device=dev)
            self.rows = perm
            self.t[perm, :D] = base
        else:
            self.rps = V // S
            self.t = torch.full((V + S * gap, self.LD), GARBAGE, device=dev)
            self.rows = torch.empty(V, dtype=torch.int64, device=dev)
            self.shards = []
            for s in range(S):
                lo, hi = s * self.rps, (V if s == S - 1 else (s + 1) * self.rps)
                at = lo + (s + 1) * gap
                self.t[at:at + hi - lo, :D] = base[lo:hi]
                self.t[at:at + hi - lo, D:] = PAD
                self.rows[lo:hi] = torch.arange(at, at + hi - lo, device=dev)
                self.shards.append(self.t[at].data_ptr())
        self.before = self.t.clone()

    def get(self, ids=None):
        r = self.rows if ids is None else self.rows[torch.as_tensor(ids, dtype=torch.int64, device=self.t.device)]
        return self.t[r, :self.D]

    def check_untouched(self, touched):
        """Rows outside `touched`, padding columns and garbage rows keep their bits."""
        keep = torch.ones(self.t.shape[0], dtype=torch.bool, device=self.t.device)
        if len(touched):
            keep[self.rows[torch.as_tensor(touched, dtype=torch.int64, device=self.t.device)]] = False
        assert torch.equal(self.t[keep], self.before[keep]), f"{self.kind}: a row outside the touched set changed"
        assert torch.equal(self.t[:, self.D:], self.before[:, self.D:]), f"{self.kind}: padding columns changed"


def _train(fn, tab_in, tab_out, toks, D, W, K, lr, seed, smp_dev, *, hogwild=0, scales=None, pool_ptr=None):
    """One call of `fn`; (loss, pairs, launches)."""
    from multiverso_b200 import _native as N
    a = N.Sgns()
    a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
    a.w_in, a.w_out, a.dim, a.ld = tab_in.t.data_ptr(), tab_out.t.data_ptr(), D, tab_in.LD
    a.window, a.negative, a.lr, a.seed, a.hogwild = W, K, lr, seed, hogwild
    a.vocab = tab_in.rows.numel()
    if "pool" in smp_dev:
        a.neg_pool, a.neg_pool_size = smp_dev["pool"].data_ptr(), smp_dev["pool"].numel()
    else:
        a.alias_prob, a.alias_idx = smp_dev["prob"].data_ptr(), smp_dev["idx"].data_ptr()
    a.neg_pool_size_ptr = N.ptr(pool_ptr)
    maps = []
    if tab_in.kind == "map":
        maps = [tab_in.rows.to(torch.int32), tab_out.rows.to(torch.int32)]
        a.map_in, a.map_out = maps[0].data_ptr(), maps[1].data_ptr()
    if tab_in.kind == "direct":
        a.nservers, a.rows_per_server = tab_in.S, tab_in.rps
        for s in range(tab_in.S):
            a.w_in_peers[s], a.w_out_peers[s] = tab_in.shards[s], tab_out.shards[s]
    if scales is not None:
        a.scale_in, a.scale_out = scales[0].data_ptr(), scales[1].data_ptr()
    loss = torch.zeros(1, device="cuda")
    pairs = torch.zeros(1, dtype=torch.int64, device="cuda")
    a.loss_sum, a.pair_count = loss.data_ptr(), pairs.data_ptr()
    getattr(N.cuda_lib(), fn)(a, N.stream_ptr())
    launches = N.cuda_lib().mvb_sgns_last_launches()
    torch.cuda.synchronize()
    return float(loss.item()), int(pairs.item()), launches


def _alias(w):
    from multiverso_b200 import _native as N
    prob = np.empty(len(w), dtype=np.float32)
    idx = np.empty(len(w), dtype=np.int32)
    assert N.cuda_lib().mvb_build_alias_table(np.ascontiguousarray(w, dtype=np.float64).ctypes.data, len(w),
                                               prob.ctypes.data, idx.ctypes.data) == 0
    return prob, idx


def _samplers(kind, V, non_tokens, rng, weights=None, pool_n=None):
    """(host sampler, device tensors) over the words `non_tokens` (pool) or a Vose table of `weights`."""
    if kind == "pool":
        pool = [int(x) for x in non_tokens]
        dev = {"pool": torch.tensor(pool, dtype=torch.int32, device="cuda")}
        return _Sampler(pool=pool, n=pool_n), dev
    prob, idx = _alias(weights)
    assert (prob < 1).sum() > len(prob) // 4                    # the alias branch is taken
    return _Sampler(prob=prob.astype(np.float64), idx=idx), {"prob": torch.from_numpy(prob).cuda(),
                                                              "idx": torch.from_numpy(idx).cuda()}


# ---------------------------------------------------------------------------------------------- exact regime
def _exact_inputs(dim, K, W, kind, tag, small_pool=False):
    """Pair sentences over one-hot input rows; non-token negatives.  Returns the pieces of a run."""
    rng = np.random.default_rng(dim * 1009 + K * 31 + W * 7 + len(kind) + tag)
    n_sent = max(1, min(dim // 2, 24))
    words = rng.choice(VX - 2, 2 * n_sent - 2, replace=False).tolist() + [VX - 1, VX - 2]   # the last shard's rest
    rng.shuffle(words)
    tl = []
    for i in range(0, len(words), 2):
        tl += [words[i], words[i + 1], -1]
    tl = tl[:-1]                                                 # the block ends on a word
    cols = rng.permutation(dim)[:len(words)]
    vals = 2.0 ** rng.integers(-1, 2, len(words))
    i0 = torch.zeros(VX, dim)
    i0[torch.tensor(words), torch.from_numpy(cols)] = torch.from_numpy(vals).float()
    g = torch.Generator(device="cuda").manual_seed(int(rng.integers(1 << 30)))
    o0 = torch.rand(VX, dim, device="cuda", generator=g) - 0.5
    is_tok = np.zeros(VX, dtype=bool)
    is_tok[words] = True
    non_tokens = np.flatnonzero(~is_tok)
    if small_pool:
        non_tokens = non_tokens[rng.choice(len(non_tokens), 2, replace=False)]
    else:
        non_tokens = rng.permutation(non_tokens)
    weights = np.where(is_tok, 0.0, 1.0 + (np.arange(VX) * 2654435761 % 7))
    smp, dev = _samplers(kind, VX, non_tokens, rng, weights)
    return tl, i0.cuda(), o0, smp, dev


def _distinct(draws):
    return len(set(draws)) == len(draws)


def _exact_seed(tl, W, K, smp, per_pair, kb, want_dup=False):
    """First seed whose schedule draws no negative row twice in the call (want_dup: one that draws a row twice
    within one batch of a pair)."""
    for seed in range(0x1000, 0x1000 + 5000):
        if per_pair:
            s = _sched_pair(tl, W, K, seed, smp, kb)
            per = [sum(bs, []) for _, _, smp_ in s for _, bs in smp_]
            if want_dup:
                if any(not _distinct(b) for _, _, smp_ in s for _, bs in smp_ for b in bs):
                    return seed, s
                continue
            if _distinct(sum(per, [])):
                return seed, s
        else:
            s = _sched_pos(tl, W, K, seed, smp)
            if _distinct([t for _, _, _, negs in s for t in negs]):
                return seed, s
    raise AssertionError("no seed with distinct draws")


def _rows_of(tab_in, tab_out):
    def rows(side, ids):
        t = tab_in if side == "in" else tab_out
        return t.get(ids).double().cpu().numpy() if len(ids) else np.zeros((0, t.D))
    return rows


def _check_exact(m, tab_in, tab_out, loss, pairs, loss_rel=1e-5):
    assert pairs == m.pairs, (pairs, m.pairs)
    worst = 0.0
    for tab, ids, R0, d, x, t in [(tab_in, m.ids_in, m.I0, m.din, m.xin, m.tin),
                                  (tab_out, m.ids_out, m.O0, m.dout, m.xout, m.tout)]:
        got = tab.get(ids).double().cpu().numpy()
        want = R0 + d
        ratio = np.abs(got - want) / _bound(x, t, want)
        worst = max(worst, float(ratio.max()))
        assert ratio.max() <= 1.0, (tab.kind, float(ratio.max()), np.unravel_index(ratio.argmax(), ratio.shape))
        assert np.abs(d).max() > 0
        tab.check_untouched(ids)
    assert abs(loss - m.loss) <= loss_rel * m.loss, (loss, m.loss)
    return worst


EXACT_WIN = [
    # dim, K, W, sampler: all 8 Row<NF4, TAIL> cases (dims 4..512), KO = 6 (K <= 5) and KO = 8 (K 6, 7)
    (4, 1, 1, "pool"), (64, 5, 15, "alias"), (100, 6, 1, "pool"), (128, 7, 15, "alias"), (132, 5, 5, "pool"),
    (256, 1, 15, "alias"), (300, 5, 5, "alias"), (324, 6, 15, "pool"), (448, 7, 1, "alias"), (452, 5, 15, "pool"),
    (512, 7, 15, "alias"),
]


@pytest.mark.parametrize("dim,K,W,kind", EXACT_WIN, ids=[f"d{d}-K{k}-W{w}-{s}" for d, k, w, s in EXACT_WIN])
def test_window_kernel_exact_regime_in_every_layout(mv_device, dim, K, W, kind):
    """The window kernel on identity tables matches the model element by element; id -> slot caches with padded
    rows and direct mode over 2, 3 and 8 shards give the same bits."""
    tl, i0, o0, smp, dev = _exact_inputs(dim, K, W, kind, 1)
    seed, sched = _exact_seed(tl, W, K, smp, False, 0)
    toks = torch.tensor(tl, dtype=torch.int32, device="cuda")
    lr = 0.25
    ref = None
    g = torch.Generator().manual_seed(dim)
    layouts = [("id", 1), ("map", 1), ("direct", 2), ("direct", 3), ("direct", 8)]
    for kind_l, S in layouts:
        perm = [torch.randperm(VX, generator=g).cuda() if kind_l == "map" else None for _ in range(2)]
        ti, to = _Table(i0, kind_l, dim, S, perm[0]), _Table(o0, kind_l, dim, S, perm[1])
        loss, pairs, launches = _train("mvb_sgns_train", ti, to, toks, dim, W, K, lr, seed, dev, hogwild=1)
        assert launches == 1
        if ref is None:
            m = _model_pos(sched, tl, lr, _rows_of(_Table(i0, "id", dim), _Table(o0, "id", dim)))
            worst = _check_exact(m, ti, to, loss, pairs)
            print(f"exact win d{dim} K{K} W{W} {kind}: worst/bound {worst:.3g}")
            ref = (ti.get(), to.get(), loss, pairs)
        else:
            ti.check_untouched(m.ids_in)
            to.check_untouched(m.ids_out)
            assert torch.equal(ti.get(), ref[0]) and torch.equal(to.get(), ref[1]), (kind_l, S)
            assert pairs == ref[3] and abs(loss - ref[2]) <= 1e-6 * ref[2], (kind_l, S)     # fp32 atomics


def test_window_kernel_exact_regime_with_step_scales(mv_device):
    """scale_in / scale_out (powers of two, so the model's products are exact) on the window kernel."""
    dim, K, W = 300, 5, 5
    tl, i0, o0, smp, dev = _exact_inputs(dim, K, W, "pool", 2)
    seed, sched = _exact_seed(tl, W, K, smp, False, 0)
    rng = np.random.default_rng(5)
    s_in = (2.0 ** -rng.integers(0, 3, VX)).astype(np.float32)
    s_out = (2.0 ** -rng.integers(0, 3, VX)).astype(np.float32)
    ti, to = _Table(i0, "id", dim), _Table(o0, "id", dim)
    m = _model_pos(sched, tl, 0.25, _rows_of(ti, to), s_in, s_out)
    sc = (torch.from_numpy(s_in).cuda(), torch.from_numpy(s_out).cuda())
    loss, pairs, _ = _train("mvb_sgns_train_win", ti, to, torch.tensor(tl, dtype=torch.int32, device="cuda"),
                            dim, W, K, 0.25, seed, dev, scales=sc)
    _check_exact(m, ti, to, loss, pairs)


EXACT_REG = [
    # dim (float4 per lane 1..4), K (every tail of the KB batches), sampler, layout, hogwild
    (64, 8, "pool", "id", 0), (128, 9, "alias", "map", 1), (132, 10, "pool", "id", 1), (256, 15, "alias", "id", 0),
    (300, 8, "alias", "map", 0), (300, 15, "pool", "id", 1), (512, 9, "pool", "map", 0), (512, 10, "alias", "id", 1),
    (4, 8, "alias", "id", 0),
]


@pytest.mark.parametrize("dim,K,kind,layout,hogwild", EXACT_REG,
                         ids=[f"d{d}-K{k}-{s}-{l}-hw{h}" for d, k, s, l, h in EXACT_REG])
def test_register_kernel_exact_regime(mv_device, dim, K, kind, layout, hogwild):
    """The register kernel (K >= 8, with hogwild 0 and 1) matches the per-pair model element by element."""
    W = 3
    vpl = (dim // 4 + 31) // 32
    tl, i0, o0, smp, dev = _exact_inputs(dim, K, W, kind, 3)
    seed, sched = _exact_seed(tl, W, K, smp, True, KB[vpl])
    g = torch.Generator().manual_seed(dim + K)
    perm = [torch.randperm(VX, generator=g).cuda() if layout == "map" else None for _ in range(2)]
    ti, to = _Table(i0, layout, dim, 1, perm[0]), _Table(o0, layout, dim, 1, perm[1])
    m = _model_pair(sched, tl, 0.25, _rows_of(_Table(i0, "id", dim), _Table(o0, "id", dim)))
    loss, pairs, launches = _train("mvb_sgns_train", ti, to, torch.tensor(tl, dtype=torch.int32, device="cuda"),
                                   dim, W, K, 0.25, seed, dev, hogwild=hogwild)
    assert launches == 1
    worst = _check_exact(m, ti, to, loss, pairs)
    print(f"exact reg d{dim} K{K} {kind} {layout}: worst/bound {worst:.3g}")


# ---------------------------------------------------------------------------------------------- contended regime
def _zipf_tokens(n, V, rng, breaks):
    w = 1.0 / np.arange(1, V + 1)
    tl = rng.choice(V, size=n, p=w / w.sum()).tolist()
    for b in breaks:
        if 0 <= b < n:
            tl[b] = -1
    return tl


def _contended(dim, n, V, W, K, kind, rng, breaks, lr):
    tl = _zipf_tokens(n, V, rng, breaks)
    a_ = np.sqrt(3.0 / dim)
    g = torch.Generator(device="cuda").manual_seed(int(rng.integers(1 << 30)))
    i0 = (torch.rand(V, dim, device="cuda", generator=g) * 2 - 1) * a_
    o0 = (torch.rand(V, dim, device="cuda", generator=g) * 2 - 1) * a_
    counts = np.maximum(np.round(1e6 / np.arange(1, V + 1)), 1.0)
    # the pool repeats hot words, which are often the centre too, among 30 colder ones
    smp, dev = _samplers(kind, V, [0, 1, 2, 3, 1, 40, 500, 7, 0, 11] + list(range(1000, 1030)), rng,
                         np.power(counts, 0.75))
    return tl, i0, o0, smp, dev


def _check_contended(m, ti, to, loss, pairs, tol, loss_tol):
    assert pairs == m.pairs, (pairs, m.pairs)
    errs = []
    for tab, ids, R0, d in [(ti, m.ids_in, m.I0, m.din), (to, m.ids_out, m.O0, m.dout)]:
        got = tab.get(ids).double().cpu().numpy() - R0
        errs.append(_rel(got, d))
        tab.check_untouched(ids)
    e_loss = abs(loss - m.loss) / m.loss
    print(f"contended: e_in {errs[0]:.3g} e_out {errs[1]:.3g} e_loss {e_loss:.3g}")
    assert max(errs) < tol and e_loss < loss_tol, (errs, e_loss)


def _chunk_breaks(n):
    """Breaks on both sides of the window kernel's CTA chunk boundaries (one chunk per CTA, <= one per SM)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    blocks = min(sms, (n + 63) // 64)
    chunk = (n + blocks - 1) // blocks
    return [b for c in range(chunk, n, chunk) for b in (c - 1, c)][::3] + [0, n - 1]


CONT_WIN = [
    # dim, K, W, sampler, layout, extra
    (300, 5, 5, "pool", "id", {}),
    (512, 7, 15, "alias", "id", {}),                                   # wide rows, W 15, KO 8: < 10 consumer warps
    (128, 6, 5, "pool", "map", {"pool_n": 6}),                         # device pool size below neg_pool_size
    (64, 5, 5, "pool", "id", {"pool_n": 0}),                           # ... and 0: positives only
    (100, 1, 1, "alias", "id", {"scales": True}),
    (324, 5, 5, "alias", "direct", {"S": 3}),
    (132, 7, 15, "pool", "direct", {"S": 8}),
    (256, 5, 5, "alias", "direct", {"S": 2}),
]


@pytest.mark.parametrize("dim,K,W,kind,layout,extra", CONT_WIN,
                         ids=[f"d{d}-K{k}-W{w}-{s}-{l}" + "".join(f"-{a}{b}" for a, b in e.items())
                              for d, k, w, s, l, e in CONT_WIN])
def test_window_kernel_contended_regime(mv_device, dim, K, W, kind, layout, extra):
    n, V, lr = 4000, 3001, 2e-5
    rng = np.random.default_rng(dim * 17 + K + W)
    breaks = _chunk_breaks(n) + list(range(97, n, 211))
    tl, i0, o0, smp, dev = _contended(dim, n, V, W, K, kind, rng, breaks, lr)
    pool_ptr = None
    if "pool_n" in extra:
        smp.n = extra["pool_n"]
        pool_ptr = torch.tensor([extra["pool_n"]], dtype=torch.int32, device="cuda")
    s_in = s_out = sc = None
    if extra.get("scales"):
        s_in = (0.25 + 0.75 * rng.random(V)).astype(np.float32)
        s_out = (0.25 + 0.75 * rng.random(V)).astype(np.float32)
        sc = (torch.from_numpy(s_in).cuda(), torch.from_numpy(s_out).cuda())
    g = torch.Generator().manual_seed(dim)
    perm = [torch.randperm(V, generator=g).cuda() if layout == "map" else None for _ in range(2)]
    S = extra.get("S", 1)
    ti, to = _Table(i0, layout, dim, S, perm[0]), _Table(o0, layout, dim, S, perm[1])
    sched = _sched_pos(tl, W, K, 0xBEEF, smp)
    m = _model_pos(sched, tl, lr, _rows_of(ti, to), s_in, s_out)
    loss, pairs, _ = _train("mvb_sgns_train", ti, to, torch.tensor(tl, dtype=torch.int32, device="cuda"), dim, W, K,
                            lr, 0xBEEF, dev, hogwild=1, scales=sc, pool_ptr=pool_ptr)
    if extra.get("pool_n") == 0:
        assert all(not negs for *_, negs in sched)
    _check_contended(m, ti, to, loss, pairs, WIN_TOL, LOSS_TOL)


CONT_REG = [
    # dim, K, W, sampler, layout, hogwild
    (64, 8, 15, "pool", "id", 0), (128, 9, 7, "alias", "map", 1), (300, 10, 1, "pool", "id", 1),
    (512, 15, 5, "alias", "id", 0),
]


@pytest.mark.parametrize("dim,K,W,kind,layout,hogwild", CONT_REG,
                         ids=[f"d{d}-K{k}-W{w}-{s}-{l}-hw{h}" for d, k, w, s, l, h in CONT_REG])
def test_register_kernel_contended_regime(mv_device, dim, K, W, kind, layout, hogwild):
    n, V, lr = 1500, 3001, 2e-5
    rng = np.random.default_rng(dim * 13 + K + W)
    # breaks at the block ends and at lane 0 / lane 2W of the centres 2W + 1 apart
    breaks = [0, n - 1] + list(range(50, n, 4 * W + 3)) + list(range(50 + 2 * W, n, 4 * W + 3))
    tl, i0, o0, smp, dev = _contended(dim, n, V, W, K, kind, rng, breaks, lr)
    g = torch.Generator().manual_seed(dim)
    perm = [torch.randperm(V, generator=g).cuda() if layout == "map" else None for _ in range(2)]
    ti, to = _Table(i0, layout, dim, 1, perm[0]), _Table(o0, layout, dim, 1, perm[1])
    vpl = (dim // 4 + 31) // 32
    sched = _sched_pair(tl, W, K, 0xFACE, smp, KB[vpl])
    m = _model_pair(sched, tl, lr, _rows_of(ti, to))
    loss, pairs, launches = _train("mvb_sgns_train", ti, to, torch.tensor(tl, dtype=torch.int32, device="cuda"), dim,
                                   W, K, lr, 0xFACE, dev, hogwild=hogwild)
    assert launches == 1
    _check_contended(m, ti, to, loss, pairs, REG_TOL, LOSS_TOL)


@pytest.mark.parametrize("dim,pool_n", [(300, None), (100, None), (64, 6)])
def test_deterministic_kernel_alias_draws_and_loss_estimator(mv_device, dim, pool_n):
    """One wave of the deterministic kernel: every read sees the initial rows, so the hash alias draws over a
    non-uniform Vose table (or a device pool size) and the loss estimator match the model tightly."""
    n, V, W, K, lr = 2000, 3001, 5, 5, 1e-2
    rng = np.random.default_rng(dim)
    kind = "alias" if pool_n is None else "pool"
    tl, i0, o0, smp, dev = _contended(dim, n, V, W, K, kind, rng, [0, n - 1] + list(range(40, n, 67)), lr)
    pool_ptr = None
    if pool_n is not None:
        smp.n = pool_n
        pool_ptr = torch.tensor([pool_n], dtype=torch.int32, device="cuda")
    ti, to = _Table(i0, "id", dim), _Table(o0, "id", dim)
    sched = _sched_pos(tl, W, K, 0xD0D0, smp)
    m = _model_pos(sched, tl, lr, _rows_of(ti, to))
    loss, pairs, launches = _train("mvb_sgns_train", ti, to, torch.tensor(tl, dtype=torch.int32, device="cuda"), dim,
                                   W, K, lr, 0xD0D0, dev, pool_ptr=pool_ptr)
    assert launches == 8                                          # the plan's 6 and one wave
    _check_contended(m, ti, to, loss, pairs, 1e-4, 1e-5)


# ---------------------------------------------------------------------------------------------- dispatch
DISPATCH = [
    # hogwild, K, dim, w_in 16-byte aligned, nservers -> kernel
    (0, 5, 64, True, 1, "det"), (0, 5, 37, True, 1, "det"), (0, 5, 64, False, 1, "det"),
    (0, 8, 64, True, 1, "reg"), (0, 8, 37, True, 1, "generic"), (0, 9, 64, False, 1, "generic"),
    (1, 5, 64, True, 1, "win"), (1, 5, 64, False, 1, "generic"), (1, 5, 37, True, 1, "generic"),
    (1, 8, 64, True, 1, "reg"), (0, 5, 64, True, 2, "win"), (1, 7, 64, True, 3, "win"),
]


@pytest.mark.parametrize("hogwild,K,dim,aligned,S,kernel", DISPATCH,
                         ids=[f"hw{h}-K{k}-d{d}-{'al' if a else 'mis'}-S{s}-{x}" for h, k, d, a, s, x in DISPATCH])
def test_dispatch_runs_the_promised_kernel(mv_device, hogwild, K, dim, aligned, S, kernel):
    """Exact-regime input with a two-word pool, so that a pair draws the same row twice within one batch: the
    register kernel reads both before either update, the generic kernel reads the second after the first.  Only
    elements no other sample reads or writes are compared (each input row's own column, each centre's output row,
    the pool rows' token columns)."""
    W = 2
    tl, i0, o0, smp, dev = _exact_inputs(dim, K, W, "pool", 4, small_pool=True)
    words = [t for t in tl if t >= 0]
    kb = KB[(dim // 4 + 31) // 32] if dim % 4 == 0 else 5
    seed, _ = _exact_seed(tl, W, K, smp, True, kb, want_dup=True)
    base_in = _Table(i0, "id", dim)
    base_out = _Table(o0, "id", dim)
    ti, to = _Table(i0, "direct" if S > 1 else "id", dim, S), _Table(o0, "direct" if S > 1 else "id", dim, S)
    if not aligned:                                               # rows start 4 bytes past a 16-byte boundary
        buf = torch.empty(ti.t.numel() + 1, device="cuda")
        buf[1:] = ti.t.reshape(-1)
        ti.t = buf[1:].view(ti.t.shape)
        ti.before = ti.t.clone()
    loss, pairs, launches = _train("mvb_sgns_train", ti, to, torch.tensor(tl, dtype=torch.int32, device="cuda"), dim,
                                   W, K, 0.25, seed, dev, hogwild=hogwild)
    assert (launches > 1) == (kernel == "det"), launches
    rows = _rows_of(base_in, base_out)
    models = {"pos": _model_pos(_sched_pos(tl, W, K, seed, smp), tl, 0.25, rows),
              "batched": _model_pair(_sched_pair(tl, W, K, seed, smp, kb), tl, 0.25, rows),
              "sequential": _model_pair(_sched_pair(tl, W, K, seed, smp, 1), tl, 0.25, rows)}
    col = {int(w): int(i0[w].abs().argmax()) for w in words}
    errs = {}
    for name, m in models.items():
        worst = 0.0
        for tab, ids, R0, d, x, t, side in [(ti, m.ids_in, m.I0, m.din, m.xin, m.tin, "in"),
                                            (to, m.ids_out, m.O0, m.dout, m.xout, m.tout, "out")]:
            got = tab.get(ids).double().cpu().numpy()
            want = R0 + d
            ratio = np.abs(got - want) / (_bound(x, t, want) + 2.0 ** -38)   # fixed point of the deterministic kernel
            for r, w in enumerate(ids):
                if side == "in":
                    sel = [col[w]] if w in col else []
                elif w in col:
                    sel = list(range(dim))                         # a centre's output row
                else:
                    sel = list(col.values())                       # a pool row at the token columns
                if sel:
                    worst = max(worst, float(ratio[r, sel].max()))
        errs[name] = worst if m.pairs == pairs else np.inf
    want = {"det": "pos", "win": "pos", "reg": "batched", "generic": "sequential"}[kernel]
    assert errs[want] <= 1.0, errs
    assert all(v > 1.0 for k, v in errs.items() if k != want), errs


def test_k8_model_has_no_step_scales(mv_device):
    """K >= 8 runs on the register kernel, which applies no hot-row step scales: none are built or reported."""
    from multiverso_b200 import _native as N
    from multiverso_b200.models.wordembedding import WordEmbedding, WordEmbeddingOption
    assert N.cuda_lib().mvb_sgns_win_inflight(300, 10, 5) == 0
    assert N.cuda_lib().mvb_sgns_win_inflight(300, 7, 5) > 0
    we = WordEmbedding(WordEmbeddingOption(embeding_size=300, window_size=5, negative_num=10), 5000)
    assert we.scale_in is None and we.scale_out is None and not hasattr(we, "hot_rows_capped")
    we5 = WordEmbedding(WordEmbeddingOption(embeding_size=300, window_size=5, negative_num=5), 5000)
    assert we5.scale_in is not None and we5.scale_out is not None
