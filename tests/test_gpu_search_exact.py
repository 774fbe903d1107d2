"""Top-k search, the full softmax and its backward (csrc/cuda/topk_cos.cu, csrc/cuda/full_softmax_bwd.cu) on operands
that tf32 represents exactly: small integers, or small integers times one power of two, whose partial sums stay exact
in fp32 (|v| <= 2048, sums < 2^24). Every logit of the tf32 wgmma is then exact, so

* top-k ids and scores must be bitwise those of an exact sort of the fp64 logits by (float32(z) desc, id asc), ties
  included, with -1 / -inf in missing slots;
* lse and loss differ from fp64 only by the exp approximation and the fp32 summation order (``lse_bound``);
* the backward differs from fp64 only by the tf32 truncation of G in the second product (``_bounds`` of
  test_gpu_full_softmax_train with ``e_z = 0``).

The shapes sit on the edges of the kernels: the two 64-query consumer warp groups, the 128-query and 128-row tiles,
the 4096-query host chunk, k around the candidate buffer, shards shorter than a tile, a row limit inside a tile and a
shard, 1 / 16 / 17 / SM-count W-tile ranges (one merge round, a second round whose last group is one list, the
largest grid), and the ``num_kb`` / ``DC`` column chunks of the backward. Ties are planted on both sides of every range
and shard boundary.

The data generators and references come first; tests/test_search_exact_cpu.py imports them and shows on the CPU that
each bound accepts rounding-sized errors and rejects the bugs it is meant to catch.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

BM = BN = 128             # query tile and W tile of both kernels
DC = 128                  # output columns per item of the backward
KSLACK = 8                # candidates kept beyond k by the tf32 pass
U = 2.0 ** -24            # fp32 unit roundoff
EX2 = 2.0 ** -22          # ex2.approx.ftz.f32: within 2 ulp of 2^a, 2^-22 relative
LOG2E_F32 = float(np.float32(math.log2(math.e)))
DELTA = abs(LOG2E_F32 * math.log(2.0) - 1.0)     # the fp32 log2(e) of the kernels: 1.33e-8 relative
SENTINEL = 0x7FD1CE5D     # a quiet NaN with a payload, in output columns no kernel may write


# ------------------------------------------------------------------------------------------------ layout
def shard_rows(num_row, S, n_rows=None):
    """[lo, hi) searched by each of S shards under the row-map rule (rows_per_server = num_row // S, the last shard
    takes the remainder), clipped to a row limit."""
    n_rows = num_row if n_rows is None else n_rows
    rps = num_row // S
    return [(min(s * rps, n_rows), min(num_row if s == S - 1 else (s + 1) * rps, n_rows)) for s in range(S)]


def tiles_of(num_row, S, n_rows=None, bn=BN):
    """(first global row, valid rows) of every W tile, in the kernels' order: tiles never straddle shards."""
    return [(t, min(bn, hi - t)) for lo, hi in shard_rows(num_row, S, n_rows) for t in range(lo, hi, bn)]


def fwd_ranges(M, n_rows, sms):
    """W-tile ranges per query tile of one search call over M queries (ranges_for in topk_cos.cu)."""
    m_tiles = -(-M // BM)
    r = min(-(-sms // m_tiles), max(1, -(-n_rows // BN) // 16))
    return max(1, r)


def bwd_ranges(M, num_row, d, sms):
    """W-tile ranges of the backward's dX pass (ranges_for in full_softmax_bwd.cu)."""
    per = -(-M // BM) * -(-d // DC)
    return max(1, min(-(-sms // per), max(1, -(-num_row // BM) // 16)))


def range_bounds(n_tiles, R):
    """[t0, t1) tile index range of each of R ranges."""
    return [(r * n_tiles // R, (r + 1) * n_tiles // R) for r in range(R)]


def chunks(M, q_chunk):
    return [(lo, min(M, lo + q_chunk)) for lo in range(0, M, q_chunk)]


def tiles_per_range(M, num_row, S, n_rows, sms, q_chunk):
    """[M] the most W tiles any range of query m's search call covers."""
    tiles = tiles_of(num_row, S, n_rows)
    out = torch.empty(M, dtype=torch.float64)
    for lo, hi in chunks(M, q_chunk):
        R = fwd_ranges(hi - lo, n_rows, sms)
        out[lo:hi] = max(t1 - t0 for t0, t1 in range_bounds(len(tiles), R))
    return out


def boundary_rows(num_row, S, n_rows, R):
    """Rows on both sides of every range boundary (last valid row of range r's last tile, first row of range r + 1)
    and of every shard boundary."""
    tiles = tiles_of(num_row, S, n_rows)
    rows = set()
    for t0, _ in range_bounds(len(tiles), R)[1:]:
        if 0 < t0 < len(tiles):
            rows.add(tiles[t0][0])
            rows.add(tiles[t0 - 1][0] + tiles[t0 - 1][1] - 1)
    for lo, hi in shard_rows(num_row, S, n_rows):
        if hi > lo:
            rows.update((lo, hi - 1))
    return sorted(rows)


def edge_labels(num_row, S):
    """Classes on the first and last row of a tile and of a shard, and row num_row - 1."""
    rows = {0, num_row - 1}
    for t, v in tiles_of(num_row, S):
        rows.update((t, t + v - 1))
    return sorted(rows)


# ------------------------------------------------------------------------------------------------ data
def exp_scale(d):
    """2^-e with 2^e near sqrt(d): a dot product of d entries in [-2, 2] then has a spread of about 2."""
    return 2.0 ** -round(math.log2(math.sqrt(d)))


def ints(gen, shape, lo, hi):
    return torch.randint(lo, hi + 1, shape, generator=gen).to(torch.float32)


def tie_data(M, n, d, pitch, seed, plant=()):
    """Top-k data with many equal logits: X in [0, 3], W in [-3, 3] (integers), the rows ``plant`` all 3, which ties
    them for the best logit of every query. Columns [d, pitch) of W hold garbage no kernel may read."""
    gen = torch.Generator().manual_seed(seed)
    W = torch.full((n, pitch), 1e6)
    W[:, :d] = ints(gen, (n, d), -3, 3)
    if len(plant):
        W[list(plant), :d] = 3.0
    X = ints(gen, (M, d), 0, 3)
    return W, X


def lse_data(M, n, d, pitch, seed):
    """Log-partition data: X in [-2, 2] 2^-e, W in [-2, 2] (integers), so the logits spread about 2 around 0 (|z| <= 8
    or so) and every W tile carries a share of the exp-mass far above the bound."""
    gen = torch.Generator().manual_seed(seed)
    W = torch.full((n, pitch), 1e6)
    W[:, :d] = ints(gen, (n, d), -2, 2)
    X = ints(gen, (M, d), -2, 2) * exp_scale(d)
    return W, X


def positive_data(M, n, d, pitch, seed):
    """The cancellation-free arm of the backward: X in [0, 2] 2^-e and W in [0, 2], so every P part of dX and dW is a
    sum of same-sign terms."""
    gen = torch.Generator().manual_seed(seed)
    W = torch.full((n, pitch), 1e6)
    W[:, :d] = ints(gen, (n, d), 0, 2)
    X = ints(gen, (M, d), 0, 2) * exp_scale(d)
    return W, X


def logits(W, X):
    """Exact fp64 logits (the operands are small integers times powers of two)."""
    return X.double() @ W[:, :X.shape[1]].double().T


# ------------------------------------------------------------------------------------------------ references
def exact_topk(Z, k):
    """(scores [M, k] fp32, ids [M, k] int64): the rows sorted by (float32(z) desc, id asc), -inf / -1 beyond n."""
    M, n = Z.shape
    z = Z.float() + 0.0                       # -0.0 -> +0.0, as the kernels' fp64 sums give
    o = torch.argsort(-z, dim=1, stable=True)[:, :k]
    s = torch.full((M, k), float("-inf"), dtype=torch.float32, device=Z.device)
    i = torch.full((M, k), -1, dtype=torch.int64, device=Z.device)
    s[:, :o.shape[1]] = z.gather(1, o)
    i[:, :o.shape[1]] = o
    return s, i


def same_topk(s, i, rs, ri):
    """Bitwise equality of (scores, ids)."""
    return torch.equal(i.cpu(), ri.cpu()) and torch.equal(s.cpu().view(torch.int32), rs.cpu().view(torch.int32))


def cosine_ref(W, q):
    """float32(d / sqrt(wn qn)) of the finish kernel, in fp64 from the fp32 operands it reads: ``q`` [M, dim] the
    normalised queries, 0 for a zero row or query."""
    W64, q64 = W[:, :q.shape[1]].double(), q.double()
    d = q64 @ W64.T
    wn, qn = (W64 * W64).sum(1), (q64 * q64).sum(1)
    den = torch.sqrt(wn[None, :] * qn[:, None])
    return torch.where(den > 0, d / torch.where(den > 0, den, torch.ones_like(den)), torch.zeros_like(d)).float()


def lse_bound(Z, tiles_per_range):
    """Bound on |lse - lse_fp64| for exact logits Z [M, n] (fp64), from the kernel's order of operations.

    In base 2 with c = float32(log2 e): a range's partial sum is s = sum_n 2^(a_n), a_n = fl(c z_n - m) by one fma,
    m the running maximum (the same float is folded into the result, so its rounding cancels). With
    A = c (max z - min z) >= |a_n| for every term and rescale argument, one ex2 with its argument's rounding is
    within e_ex = 2^-22 + ln2 u A relative (u = 2^-24). Per thread and range (Tr tiles): a term takes one ex2, up to
    31 adds inside its tile, one add into the running sum per tile and up to Tr rescales (an ex2 and a product), so
    it is within (1 + Tr) e_ex + (31 + 2 Tr) u; the quad butterfly adds two combines (an ex2, a product and an add
    each), 2 (e_ex + 2 u). The range fold and lse = ln2 (m + log2 s) run in fp64 (1e-12 covers them). Positive
    terms keep the relative error of the sum, and |ln(1 + E)| <= E (1.01 covers the second-order terms), so

        |lse - lse_fp64| <= 1.01 ((3 + Tr) e_ex + (35 + 2 Tr) u) + |c ln 2 - 1| max|z| + u |lse_fp64| + 1e-12

    where the last two terms are the fp32 log2(e) (1.33e-8 relative on each exponent) and the final fp32 rounding.
    The same holds for loss = fl32(lse - z_y) with u |loss_fp64| in place of u |lse_fp64|: the fp64 lse is used.
    Returns (lse_fp64, bound without the final rounding)."""
    Z = Z.double()
    lse64 = Z.logsumexp(1)
    A = LOG2E_F32 * (Z.amax(1) - Z.amin(1))
    e_ex = EX2 + math.log(2.0) * U * A
    Tr = tiles_per_range.to(Z.device)
    E = 1.01 * ((3 + Tr) * e_ex + (35 + 2 * Tr) * U)
    return lse64, E + DELTA * Z.abs().amax(1) + 1e-12


# ------------------------------------------------------------------------------------------------ device plumbing
@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sharded(W, S, gap=37):
    """W as S shards at separate places of one buffer, ``gap`` rows of NaN garbage between them."""
    from multiverso_b200 import _native as N
    n, pitch = W.shape
    buf = torch.full((n + S * gap, pitch), float("nan"), device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, n // S
    for s, (lo, hi) in enumerate(shard_rows(n, S)):
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
    return rm, buf


def _sentinel(shape, dev):
    return torch.full(shape, SENTINEL, dtype=torch.int32, device=dev).view(torch.float32)


def _kept_sentinel(t):
    return bool((t.contiguous().view(torch.int32) == SENTINEL).all())


# ------------------------------------------------------------------------------------------------ a, c: forward
# (M, n, rows, k, S, d, ranges): ranges is the count the case is meant to hit ("max": the SM count), or None
TINY = [(1, 1, None, 1, 1, 4, None), (1, 1, None, 8, 1, 32, None), (63, 127, None, 9, 1, 36, None),
        (64, 128, None, 63, 2, 28, None), (65, 129, None, 64, 8, 4, None), (3, 50, None, 64, 2, 100, None)]
FWD = TINY + [
    (127, 1003, 1000, 8, 3, 36, None),     # the row limit ends inside the last shard and inside a tile
    (128, 700, 400, 1, 3, 128, None),      # ... inside the middle shard
    (129, 300, None, 64, 3, 132, None),
    (256, 4200, None, 9, 8, 260, None),    # two query tiles x 2 ranges
    (4097, 300, None, 9, 2, 32, None),     # the host chunk and a one-query last chunk
    (1, 33, None, 8, 1, 8, 1),
    (1, 16 * 16 * BN, None, 8, 1, 8, 16),  # one merge round of 16 full lists
    (1, 17 * 16 * BN, None, 9, 3, 8, 17),  # a second round whose last group is one list
    (65, 17 * 16 * BN - 5, 16 * 16 * BN + 50, 64, 8, 4, 16),   # the row limit sets the range count
    (1, "sms", None, 64, 8, 4, "max"),     # one range per SM: 9 groups in round one, 1 in round two
]


def _fwd_id(c):
    M, n, rows, k, S, d, R = c
    tag = "tiny-" if c in TINY else ""
    return f"{tag}M{M}-n{n}-rows{rows}-k{k}-S{S}-d{d}-R{R}"


def _resolve(case, sms):
    M, n, rows, k, S, d, R = case
    if n == "sms":
        n = sms * 16 * BN + 77
    return M, n, rows, k, S, d, (sms if R == "max" else R)


def _search(rm, width, X, y, k, n, want_lse):
    from multiverso_b200.ops.full_softmax import _device
    r = _device(rm, width, X, y, k, n, want_lse)
    torch.cuda.synchronize()
    return r


def _check_forward(W, X, y, k, S, rows, sms, what):
    from multiverso_b200.ops.topk import _Q_CHUNK
    dev = X.device
    n_all = W.shape[0]
    n = n_all if rows is None else rows
    rm, _keep = _sharded(W.to(dev), S, 0 if S == 1 else 37)
    Z = logits(W[:n].to(dev), X)
    rs, ri = exact_topk(Z, k)
    r = _search(rm, X.shape[1], X, y, k, n, True)
    assert same_topk(r.scores, r.ids, rs, ri), what
    s, i = _search(rm, X.shape[1], X, None, k, n, False)[2:]         # topk_dot's kernel: no log-partition
    assert same_topk(s, i, rs, ri), what
    r0 = _search(rm, X.shape[1], X, y, 0, n, True)                    # the loss-only kernel
    assert torch.equal(r0.lse, r.lse) and torch.equal(r0.loss, r.loss), what
    Tr = tiles_per_range(X.shape[0], n_all, S, n, sms, _Q_CHUNK)
    lse64, b = lse_bound(Z, Tr)
    err = (r.lse.double() - lse64).abs()
    ratio = (err / (b + U * lse64.abs())).max().item()
    assert (err <= b + U * lse64.abs()).all(), (what, ratio)
    loss64 = lse64 - Z.gather(1, y[:, None])[:, 0]
    lerr = (r.loss.double() - loss64).abs()
    lratio = (lerr / (b + U * loss64.abs())).max().item()
    assert (lerr <= b + U * loss64.abs()).all(), (what, lratio)
    return max(ratio, lratio)


@pytest.mark.parametrize("case", FWD, ids=_fwd_id)
def test_forward_exact(cuda, case):
    from multiverso_b200 import _native as N
    from multiverso_b200.ops.topk import _Q_CHUNK
    sms = _sms()
    M, n, rows, k, S, d, R = _resolve(case, sms)
    nr = n if rows is None else rows
    pitch = (d + 3) // 4 * 4 + 4
    lib = N.cuda_lib()
    for lo, hi in chunks(M, _Q_CHUNK):
        # the library sizes its scratch by its own range count: it must be the one this test computes
        Rc = fwd_ranges(hi - lo, nr, sms)
        assert lib.mvb_topk_cos_scratch_bytes(hi - lo, k, nr) == 2 * (hi - lo) * Rc * (k + KSLACK) * 8
    if R is not None:
        assert fwd_ranges(M, nr, sms) == R, (M, nr, sms)
    R0 = fwd_ranges(min(M, _Q_CHUNK), nr, sms)
    plant = boundary_rows(n, S, nr, R0)
    worst = 0.0
    for arm, (W, X) in (("ties", tie_data(M, n, d, pitch, seed=M + n + d, plant=plant)),
                        ("lse", lse_data(M, n, d, pitch, seed=M + n + d + 1))):
        gen = torch.Generator().manual_seed(M + k)
        y = torch.randint(0, nr, (M,), generator=gen)
        X, y = X.to(cuda), y.to(cuda)
        ratio = _check_forward(W, X, y, k, S, rows, sms, (arm, M, n, rows, k, S, d))
        if arm == "lse":
            worst = ratio
    print(f"lse / loss max err/bound {worst:.3g}")


def test_all_rows_equal_overflow(cuda):
    """Every row the same: every tile overflows the 48-entry candidate buffer (k = 64, 72 list entries) and the answer
    is ids 0..63 with one score, across 3 shards and several ranges."""
    sms = _sms()
    M, n, d, k = 65, 40 * 16 * BN + 3, 12, 64
    W = torch.zeros(n, 12)
    W[:] = torch.arange(1, 13, dtype=torch.float32) - 6
    X = torch.randint(-3, 4, (M, d), generator=torch.Generator().manual_seed(3)).float()
    assert fwd_ranges(M, n, sms) >= 2
    rm, _keep = _sharded(W.to(cuda), 3)
    z = logits(W[:1], X).float()
    for want_lse in (False, True):
        r = _search(rm, d, X.to(cuda), None, k, n, want_lse)
        assert torch.equal(r.ids.cpu(), torch.arange(k).expand(M, k))
        assert torch.equal(r.scores.cpu(), z.expand(M, k))


# ------------------------------------------------------------------------------------------------ b: cosine
def _cos_search(W, Q, k, S, rows=None):
    from multiverso_b200.ops.topk import _topk_device
    rm, _keep = _sharded(W, S, 0 if S == 1 else 37)
    out = _topk_device(rm, W.shape[1], Q, k, rows)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("S", [1, 3, 8])
def test_cosine_duplicates_across_ranges_and_shards(cuda, S):
    """Copies of one row on both sides of every range and shard boundary score bitwise alike and come out by id."""
    sms = _sms()
    n, d, M, k = 8 * 16 * BN + 11, 60, 3, 40
    gen = torch.Generator().manual_seed(S)
    W = torch.randn(n, 60, generator=gen)
    dup = boundary_rows(n, S, n, fwd_ranges(M, n, sms))
    assert len(dup) >= 8 and len(dup) <= k
    W[dup] = W[5].clone()
    Q = W[5].expand(M, d) + 0.05 * torch.randn(M, d, generator=gen)
    s, i = _cos_search(W.to(cuda), Q.to(cuda), k, S)
    s, i = s.cpu(), i.cpu()
    ids = sorted(set(dup) | {5})
    assert torch.equal(i[:, :len(ids)], torch.tensor(ids).expand(M, len(ids))), i[:, :len(ids)]
    assert (s[:, :len(ids)] == s[:, :1]).all()


def test_cosine_zero_query_and_zero_rows(cuda):
    n, d, k = 3 * BN + 5, 32, 20
    gen = torch.Generator().manual_seed(4)
    W = -torch.rand(n, d, generator=gen) - 0.1          # every nonzero row has a negative cosine with Q[1]
    zero_rows = [3, 127, 128, 200, n - 1]
    W[zero_rows] = 0
    Q = torch.zeros(2, d)
    Q[1] = 1.0
    s, i = _cos_search(W.to(cuda), Q.to(cuda), k, 3)
    s, i = s.cpu(), i.cpu()
    assert torch.equal(i[0], torch.arange(k)) and (s[0] == 0).all() and not torch.signbit(s[0]).any()
    assert i[1, :5].tolist() == zero_rows and (s[1, :5] == 0).all()
    assert (s[1, 5:] < 0).all()


@pytest.mark.parametrize("k,S", [(1, 1), (9, 2), (56, 8)])
def test_cosine_order_below_tf32_resolution(cuda, k, S):
    """k + 8 rows stand clear of the rest by far more than the tf32 error; inside that set the cosines differ by
    about 1e-6 (below tf32 resolution, above an fp32 ulp). The output follows the exact fp64 order."""
    n, d, M = 9000, 64, 4
    gen = torch.Generator().manual_seed(k)
    W = torch.randn(n, d, generator=gen) * 0.1
    top = torch.randperm(n, generator=gen)[:k + KSLACK].tolist()
    # one query direction (queries of different lengths); top row j is qd + sqrt(2e-6 (j + 1)) v with v orthogonal
    # to qd, so its cosine is about 1 - 1e-6 (j + 1)
    qd = torch.randn(d, generator=gen)
    qd = qd / qd.norm()
    v = torch.randn(d, generator=gen)
    v = v - (v @ qd) * qd
    v = v / v.norm()
    for j, row in enumerate(top):
        W[row] = qd + math.sqrt(2e-6 * (j + 1)) * v
    Q = qd[None, :] * torch.tensor([1.0, 2.0, 0.5, 3.0])[:, None]
    s, i = _cos_search(W.to(cuda), Q.to(cuda), k, S)
    from multiverso_b200.ops.topk import _unit_rows
    C = cosine_ref(W, _unit_rows(Q))
    rest = torch.ones(n, dtype=torch.bool)
    rest[top] = False
    assert (C[:, top].min(1).values > 0.99).all() and (C[:, rest].max(1).values < 0.9).all()
    gaps = C[:, top].double().sort(1).values.diff(1)
    assert (gaps < 2.0 ** -11).all() and (gaps > 2.0 ** -23).all()
    rs, ri = exact_topk(C.double(), k)
    assert same_topk(s, i, rs, ri), (i, ri)


# ------------------------------------------------------------------------------------------------ d: backward
# (B, n, d, S)
BWD_TINY = [(1, 1, 4, 1), (1, 129, 28, 1), (63, 127, 32, 2), (64, 128, 36, 3), (65, 129, 4, 8)]
BWD = BWD_TINY + [
    (127, 129, 124, 8),       # shards of 16 rows
    (128, 1003, 128, 3),
    (129, 5003, 256, 2),      # two query tiles, two d-chunks, 2 ranges
    (65, 4500, 132, 1),       # 2 ranges
    (200, 3001, 260, 8),
    (65, 2000, 1024, 3),      # eight d-chunks
    (1, 40000, 36, 3),        # 19 ranges
    (4097, 300, 4, 2),        # the forward's host chunk
]


def _bwd_id(c):
    return ("tiny-" if c in BWD_TINY else "") + "B{}-n{}-d{}-S{}".format(*c)


def _bwd(rm, X, y, lse, g, scale, pad):
    """dX and dW written through full_softmax_bwd into buffers whose ld is larger than d, the extra columns holding
    SENTINEL."""
    from multiverso_b200.ops.full_softmax import full_softmax_bwd
    from multiverso_b200.ops.topk import padded_queries
    B, d = X.shape
    dXb = _sentinel((B, d + pad), X.device)
    dWb = _sentinel((rm.num_row, d + pad + 4), X.device)
    full_softmax_bwd(rm, padded_queries(X), d, y, lse, g, dXb[:, :d], dWb[:, :d], scale)
    torch.cuda.synchronize()
    assert _kept_sentinel(dXb[:, d:]) and _kept_sentinel(dWb[:, d:])
    return dXb[:, :d], dWb[:, :d]


def _labels(B, n, S, gen, spread):
    """Edge labels (tile and shard ends, row n - 1) in turn, and with ``spread`` a random label every third query."""
    edges = torch.tensor(edge_labels(n, S))
    y = edges[torch.arange(B) % len(edges)]
    if spread:
        y[::3] = torch.randint(0, n, (len(y[::3]),), generator=gen)
    return y


@pytest.mark.parametrize("case", BWD, ids=_bwd_id)
def test_backward_exact(cuda, case):
    from test_gpu_full_softmax_train import _bounds
    from multiverso_b200 import _native as N
    B, n, d, S = case
    sms = _sms()
    pitch = (d + 3) // 4 * 4 + 4
    R = bwd_ranges(B, n, d, sms)
    lib = N.cuda_lib()
    mp = -(-B // BM) * BM
    part = -(-(-(-mp * 8 // 256) * 256 + mp * 4) // 256) * 256
    assert lib.mvb_full_softmax_bwd_scratch_bytes(B, d, n, 1, 0) == -(-(part + R * B * d * 4) // 256) * 256
    gen = torch.Generator().manual_seed(B + n + d)
    worst = {}
    for arm in ("signed", "positive"):
        W, X = (lse_data if arm == "signed" else positive_data)(B, n, d, pitch, seed=B + n + d)
        y = _labels(B, n, S, gen, arm == "signed")
        g = torch.randn(B, generator=gen) if arm == "signed" else torch.rand(B, generator=gen) + 0.5
        if arm == "signed" and B > 1:
            g[1::7] = 0.0
        Wd, X, y, g = W.to(cuda), X.to(cuda), y.to(cuda), g.to(cuda)
        rm, _keep = _sharded(Wd, S, 0 if S == 1 else 37)
        lse = _search(rm, d, X, None, 0, n, True).lse
        dX, dW = _bwd(rm, X, y, lse, g, -0.75, pad=3 if arm == "signed" else 8)
        dX64, dW64, bx, bw = _bounds(Wd[:, :d], X, y, g, lse, -0.75, e_z=0.0)
        ex, ew = (dX.double() - dX64).abs(), (dW.double() - dW64).abs()
        worst[arm] = max((ex / bx).max().item(), (ew / bw).max().item())
        assert (ex <= bx).all(), (arm, (ex / bx).max().item())
        assert (ew <= bw).all(), (arm, (ew / bw).max().item())
        # an identically zero upstream gradient gives exactly zero gradients
        dX0, dW0 = _bwd(rm, X, y, lse, torch.zeros_like(g), -0.75, pad=4)
        assert (dX0 == 0).all() and (dW0 == 0).all()
    print("max err/bound", {a: f"{v:.3g}" for a, v in worst.items()}, f"ranges {R}")


def test_backward_empty_batch_keeps_padding(cuda):
    """M = 0: dW is zeroed over its dim columns by one 2-D memset; the columns beyond dim keep their bits."""
    W = torch.ones(300, 40, device=cuda)
    rm, _keep = _sharded(W, 3)
    X = torch.zeros(0, 37, device=cuda)
    e = torch.zeros(0, device=cuda)
    dX, dW = _bwd(rm, X, torch.zeros(0, dtype=torch.int64, device=cuda), e, e, 1.0, pad=5)
    assert dX.shape == (0, 37) and (dW == 0).all()
