"""The references and bounds of tests/test_gpu_search_exact.py, checked without a GPU: the exact top-k sort against
brute force, each bound accepting an fp32 emulation of the kernel's order of operations and rejecting the bugs it is
there to catch, and the host implementations of full_softmax / topk_dot bitwise equal to the exact sort."""
import math

import numpy as np
import pytest
import torch

from test_gpu_full_softmax_train import _bounds
from test_gpu_search_exact import (LOG2E_F32, _labels, bwd_ranges, exact_topk, fwd_ranges, logits, lse_bound,
                                   lse_data, positive_data, range_bounds, same_topk, tie_data, tiles_of, tiles_per_range)

SMS = 132                 # the H100 SXM's SM count: sets the range split of these layouts


def test_exact_topk_matches_brute_force():
    W, X = tie_data(7, 300, 5, 8, seed=1, plant=(0, 127, 128, 299))
    Z = logits(W, X)
    assert (Z == Z.round()).all() and len(torch.unique(Z)) < 60        # many equal logits
    for k in (1, 4, 64):
        s, i = exact_topk(Z, k)
        for m in range(Z.shape[0]):
            ref = sorted(range(Z.shape[1]), key=lambda n: (-float(np.float32(Z[m, n])), n))[:k]
            assert i[m, :len(ref)].tolist() == ref
            assert s[m, :len(ref)].tolist() == [float(np.float32(Z[m, n])) for n in ref]
    s, i = exact_topk(Z[:, :3], 5)                                       # k > n: -1 / -inf
    assert (i[:, 3:] == -1).all() and torch.isneginf(s[:, 3:]).all()


def test_swapped_tied_ids_rejected():
    W, X = tie_data(4, 500, 6, 8, seed=2, plant=(10, 128, 300))
    s, i = exact_topk(logits(W, X), 8)
    assert same_topk(s, i, s.clone(), i.clone())
    assert s[0, 0] == s[0, 1] == s[0, 2] and i[0, :3].tolist() == [10, 128, 300]
    j = i.clone()
    j[0, [0, 1]] = j[0, [1, 0]]
    assert not same_topk(s, j, s, i)


@pytest.mark.parametrize("M,n,rows,k", [(5, 1003, None, 9), (130, 300, 257, 64), (2, 129, None, 1)])
def test_host_full_softmax_and_topk_dot_are_exact(M, n, rows, k):
    """The CPU path promises the kernels' (fp32 score desc, id asc) rule: on exact logits it is the exact sort."""
    from multiverso_b200.ops import full_softmax, full_softmax_reference, topk_dot
    for W, X in (tie_data(M, n, 12, 16, seed=n, plant=(0, 128, n - 1)), lse_data(M, n, 12, 16, seed=n)):
        nr = n if rows is None else rows
        rs, ri = exact_topk(logits(W[:nr], X), k)
        r = full_softmax(W, X, k=k, rows=rows)
        assert same_topk(r.scores, r.ids, rs, ri)
        assert same_topk(*topk_dot(W, X, k, rows=rows), rs, ri)
        r = full_softmax_reference(W, X, k=k, rows=rows, row_chunk=100)   # merges across host chunks
        assert same_topk(r.scores, r.ids, rs, ri)


# ------------------------------------------------------------------------------------------------ lse
def _f32(x):
    return np.float32(x)


def emulate_lse(Z, tiles, R):
    """The kernel's log-partition in fp32 (exact exp2 instead of ex2.approx): per range and lane of a quad, a tile's
    max, one rescale, a 32-term sum per tile; the quad butterfly; the fp64 range fold; lse rounded to fp32."""
    c = _f32(LOG2E_F32)
    z = Z.numpy().astype(np.float32)
    M = z.shape[0]
    lo_f = _f32(-np.finfo(np.float32).max)

    def combine(m, s, m2, s2):
        mn = np.maximum(m, m2)
        return mn, (s * np.exp2(m - mn)).astype(np.float32) + (s2 * np.exp2(m2 - mn)).astype(np.float32)

    parts = []
    for t0, t1 in range_bounds(len(tiles), R):
        lm = np.full((4, M), lo_f, dtype=np.float32)
        ls = np.zeros((4, M), dtype=np.float32)
        for start, valid in tiles[t0:t1]:
            for lane in range(4):
                cols = [8 * j + 2 * lane + cc for j in range(16) for cc in range(2) if 8 * j + 2 * lane + cc < valid]
                if not cols:
                    continue
                tmax = (z[:, [start + x for x in cols]].max(1) * c).astype(np.float32)
                up = tmax > lm[lane]
                ls[lane] = np.where(up, (ls[lane] * np.exp2(lm[lane] - tmax)).astype(np.float32), ls[lane])
                lm[lane] = np.where(up, tmax, lm[lane])
                s = np.zeros(M, dtype=np.float32)
                for x in cols:      # fma(z, c, -m): one rounding of the exact z c - m
                    a = (z[:, start + x].astype(np.float64) * float(c) - lm[lane].astype(np.float64)).astype(np.float32)
                    s = (s + np.exp2(a).astype(np.float32)).astype(np.float32)
                ls[lane] = (ls[lane] + s).astype(np.float32)
        for o in (1, 2):
            m2, s2 = lm[[lane ^ o for lane in range(4)]], ls[[lane ^ o for lane in range(4)]]
            lm, ls = combine(lm, ls, m2, s2)
        parts.append((lm[0].astype(np.float64), ls[0].astype(np.float64)))
    mx, s = np.full(M, -np.finfo(np.float64).max), np.zeros(M)
    for pm, ps in parts:
        mn = np.maximum(mx, pm)
        s = s * np.exp2(mx - mn) + ps * np.exp2(pm - mn)
        mx = mn
    return torch.from_numpy((math.log(2.0) * (mx + np.log2(s))).astype(np.float32))


@pytest.mark.parametrize("M,n,d,S", [(40, 129, 32, 1), (40, 1003, 36, 3), (3, 5003, 128, 2), (1, 40000, 4, 8)])
def test_lse_bound_accepts_emulation_and_rejects_padding(M, n, d, S):
    from multiverso_b200.ops.topk import _Q_CHUNK
    W, X = lse_data(M, n, d, d + 4, seed=n)
    Z = logits(W, X)
    tiles = tiles_of(n, S)
    Tr = tiles_per_range(M, n, S, n, SMS, _Q_CHUNK)
    lse64, b = lse_bound(Z, Tr)
    b = b + 2.0 ** -24 * lse64.abs()
    got = emulate_lse(Z, tiles, fwd_ranges(M, n, SMS))
    err = (got.double() - lse64).abs()
    assert (err <= b).all(), (err / b).max().item()
    print(f"emulated fp32 order: max err/bound {(err / b).max().item():.3g}")
    # one padding row counted as a zero logit, one padding tile (127 zero logits) counted
    for extra in (1, 127):
        bad = torch.logaddexp(lse64, torch.tensor(math.log(extra), dtype=torch.float64))
        ratio = (bad - lse64).abs() / b
        if extra == 127 or n in (129, 1003):
            assert not (ratio <= 1).all() and (ratio > 1).float().mean() > 0.9, (extra, ratio.min().item())


def test_lse_bound_rejects_a_dropped_tile():
    W, X = lse_data(50, 1003, 36, 40, seed=7)
    Z = logits(W, X)
    lse64, b = lse_bound(Z, torch.full((50,), 8.0))
    bad = Z[:, 128:].logsumexp(1)
    assert ((bad - lse64).abs() > b).all()


# ------------------------------------------------------------------------------------------------ backward
def _tf32(x):
    """Truncation to tf32: the low 13 mantissa bits of fp32 cleared."""
    return (x.view(torch.int32) & ~0x1FFF).view(torch.float32)


def _positive_case(B, n, d, S, seed):
    gen = torch.Generator().manual_seed(seed)
    W, X = positive_data(B, n, d, d + 4, seed=seed)
    W = W[:, :d].contiguous()
    y = _labels(B, n, S, gen, False)
    g = torch.rand(B, generator=gen) + 0.5
    Z = logits(W, X)
    lse64 = Z.logsumexp(1)
    return W, X, y, g, Z, lse64


@pytest.mark.parametrize("B,n,d,S", [(300, 5003, 36, 2), (1, 40000, 36, 3), (129, 1003, 132, 8)])
def test_backward_bound_accepts_tf32_g_and_rejects_bugs(B, n, d, S):
    scale = -0.75
    W, X, y, g, Z, lse64 = _positive_case(B, n, d, S, seed=B + n)
    lse32 = lse64.float()
    dX64, dW64, bx, bw = _bounds(W, X, y, g, lse32, scale, e_z=0.0)
    # the kernel's arithmetic in fp32 with G truncated to tf32: accepted
    P32 = torch.exp((Z - lse32.double()[:, None]).float())
    Y = torch.zeros(B, n)
    Y[torch.arange(B), y] = 1.0
    G = _tf32(g[:, None] * (P32 - Y))
    for got, ref, bnd in ((G @ W, dX64, bx), (scale * (G.T @ X), dW64, bw)):
        assert ((got.double() - ref).abs() <= bnd).all(), ((got.double() - ref).abs() / bnd).max().item()
    P = torch.exp(Z - lse64[:, None])
    g64, X64, W64, Y64 = g.double(), X.double(), W.double(), Y.double()

    def rejected(got, ref, bnd):
        return not ((got - ref).abs() <= bnd).all()
    # P scaled by 1.01 (with one query over 40000 classes every dW element is below the bound's 1e-6 floor)
    Gs = g64[:, None] * (1.01 * P - Y64)
    assert rejected(Gs @ W64, dX64, bx) and (B == 1 or rejected(scale * (Gs.T @ X64), dW64, bw))
    # one X tile's P part missing from dW
    if B > 128:
        Gt = g64[:, None] * (P - Y64)
        Gt[:128] = -g64[:128, None] * Y64[:128]
        assert rejected(scale * (Gt.T @ X64), dW64, bw)
    # one W range's P part missing from dX
    R = bwd_ranges(B, n, d, SMS)
    tiles = tiles_of(n, S)
    if R > 1:
        t0, t1 = range_bounds(len(tiles), R)[R // 2]
        keep = torch.ones(n, dtype=torch.bool)
        for start, valid in tiles[t0:t1]:
            keep[start:start + valid] = False
        Gr = g64[:, None] * (P * keep - Y64)
        assert rejected(Gr @ W64, dX64, bx)
