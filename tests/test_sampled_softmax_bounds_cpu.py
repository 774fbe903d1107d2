"""The fp64 bounds of tests/test_gpu_sampled_softmax_fp64.py on the CPU: a numpy fp32 emulation of the sampled-softmax
kernels' order of operations (the logits of the TF32 GEMM, the per-lane fp32 true dot and its butterfly sum, each
lane's online logsumexp over 4-strided columns of 1024-candidate tiles and the warp merge, E and e_true, and E
truncated to TF32 in the two backward GEMMs) lies within every bound, and each seeded bug lies outside one."""
import math

import numpy as np
import pytest
import torch

from test_gpu_sampled_softmax_fp64 import FWD_TILE, bounds, reference

f32 = np.float32


def _tf32(a, truncate=False):
    """fp32 -> TF32 (10 explicit mantissa bits), rounded to nearest or truncated."""
    b = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)
    if not truncate:
        b = b + np.uint32(0x1000)
    return (b & np.uint32(0xFFFFE000)).view(np.float32)


def _warp_sum(v):
    """The xor-butterfly warp_sum of [B, 32] fp32 lane values (every lane ends with the same sum)."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[:, lanes ^ o]).astype(f32)
    return v[:, 0]


def emulate(x, W, y, cand, logq, log_s, g, exact, bug=None):
    """The kernels' loss, dL/dx and dL/dW in fp32 (numpy arrays in, numpy arrays out)."""
    B, d = x.shape
    S = cand.size
    Sp = (S + 3) // 4 * 4
    ws = np.zeros((Sp, d), f32)
    ws[:S] = W[cand]
    if exact:
        logits = (x.astype(np.float64) @ ws.T.astype(np.float64)).astype(f32)
    else:
        logits = (_tf32(x).astype(np.float64) @ _tf32(ws).T.astype(np.float64)).astype(f32)
    lq = (f32(log_s) + logq[cand]).astype(f32)
    # the true logit: lane l takes columns 4l + 128k .. +3 with fmas in order, then the butterfly sum
    dot = np.zeros((B, 32), f32)
    for lane in range(32):
        for c in range(4 * lane, d, 128):
            for q in range(4):
                dot[:, lane] = (x[:, c + q].astype(np.float64) * W[y, c + q] + dot[:, lane]).astype(f32)
    corr = (f32(log_s) + logq[y]).astype(f32)
    t = (_warp_sum(dot) + corr if bug == "logq_sign" else _warp_sum(dot) - corr).astype(f32)
    # each lane's (m, s) over 4-strided columns of every 1024-candidate tile
    m = np.full((B, 32), -np.inf, f32)
    s = np.zeros((B, 32), f32)
    lane4 = 4 * np.arange(32)
    with np.errstate(over="ignore", invalid="ignore"):
        for j0 in range(0, S, FWD_TILE):
            if bug == "one_tile" and j0 > 0:
                break
            if bug == "reset_per_tile":
                m = np.full((B, 32), -np.inf, f32)
                s = np.zeros((B, 32), f32)
            n = min(FWD_TILE, S - j0)
            n_seen = min(FWD_TILE, Sp - j0) if bug == "pad_column" else n
            for k in range(0, n_seen, 128):
                for q in range(4):
                    i = lane4 + k + q
                    ok = i < n_seen
                    j = np.minimum(j0 + i, Sp - 1)
                    c = np.where(j < S, cand[np.minimum(j, S - 1)], -1)
                    lqj = np.where(j < S, lq[np.minimum(j, S - 1)], f32(0))
                    live = ok[None, :] & (c[None, :] != y[:, None])
                    l = (logits[:, j] - lqj[None, :]).astype(f32)
                    up = l > m
                    s_up = (s * np.exp((m - l).astype(f32)) + f32(1)).astype(f32)
                    s_add = (s + np.exp((l - m).astype(f32))).astype(f32)
                    s = np.where(live, np.where(up, s_up, s_add), s).astype(f32)
                    m = np.where(live & up, l, m).astype(f32)
        mx = m.max(1)
        part = np.where(m == -np.inf, f32(0), (s * np.exp((m - mx[:, None]).astype(f32))).astype(f32))
        tot_s = _warp_sum(part.astype(f32))
        top = np.maximum(mx, t)
        tot = (np.where(mx == -np.inf, f32(0), (tot_s * np.exp((mx - top).astype(f32))).astype(f32))
               + np.exp((t - top).astype(f32))).astype(f32)
        lse = (top + np.log(tot).astype(f32)).astype(f32)
    loss = (lse - t).astype(f32)
    # the backward epilogue: E over the sampled columns (0 on masked ones), e_true
    hit = cand[None, :] == y[:, None]
    E = (g[:, None] * np.exp((logits[:, :S] - lq[None, :] - lse[:, None]).astype(f32))).astype(f32)
    if bug != "no_mask_bwd":
        E = np.where(hit, f32(0), E)
    e_true = np.exp((t - lse).astype(f32)).astype(f32)
    e_true = (g * (e_true if bug == "no_minus_one" else e_true - f32(1))).astype(f32)
    # dX = E W_S + e_true w_y and dW_S = E^T X on the GEMM: E truncated to TF32, fp32 results
    Et = _tf32(E, truncate=True).astype(np.float64)
    wop = ws[:S] if exact else _tf32(ws[:S])
    xop = x if exact else _tf32(x)
    dx = ((Et @ wop.astype(np.float64)).astype(f32) + (e_true[:, None] * W[y]).astype(f32)).astype(f32)
    dws = (Et.T @ xop.astype(np.float64)).astype(f32)
    dW = np.zeros(W.shape, f32)
    np.add.at(dW, y, (e_true[:, None] * x).astype(f32))
    np.add.at(dW, cand, dws)
    return loss, dx, dW


def _case(S, exact, seed, n=500, B=9, d=132):
    """Operands, a Zipf-like draw of S candidates with duplicates, labels with accidental hits and a repeat, and
    g with zeros and negatives."""
    rng = np.random.default_rng(seed)
    if exact:
        W = (rng.integers(-3, 4, (n, d)) * 0.125).astype(f32)
        x = (rng.integers(-3, 4, (B, d)) * 0.25).astype(f32)
    else:
        W = (rng.standard_normal((n, d)) / math.sqrt(d)).astype(f32)
        x = (rng.standard_normal((B, d)) * 2).astype(f32)
    k = np.arange(n, dtype=np.float64)
    q = np.log((k + 2) / (k + 1)) / math.log(n + 1)
    logq = np.log(q).astype(f32)
    cand = np.minimum((rng.random(S) ** 3 * n).astype(np.int64), n - 1)
    y = rng.integers(0, n, B)
    y[:3] = cand[rng.integers(0, S, 3)]
    y[3] = y[0]
    g = rng.standard_normal(B).astype(f32)
    g[1::3] = 0
    log_s = f32(math.log(S))
    if exact:
        logsq = (log_s + logq).astype(np.float64)
    else:
        logsq = math.log(S) + np.log(q)
    return x, W, y, cand, logq, log_s, g, logsq


def _ratios(S, exact, seed, bug=None):
    x, W, y, cand, logq, log_s, g, logsq = _case(S, exact, seed)
    loss, dx, dW = emulate(x, W, y, cand, logq, log_s, g, exact, bug)
    T = torch.from_numpy
    args = (T(x), T(W), T(y), T(cand), T(logsq), T(g))
    r = reference(*args)
    tol = bounds(r, *args, exact=exact)

    def ratio(err, b):
        err = err.double()
        return torch.where(err == 0, torch.zeros_like(err), err / b).max().item()
    return dict(loss=ratio((T(loss).double() - r["loss"]).abs(), tol["loss"]),
                dx=ratio((T(dx).double() - r["dx"]).abs().amax(1), tol["dx"]),
                rows=ratio((T(dW).double() - r["dW"]).abs().amax(1), tol["rows"]))


@pytest.mark.parametrize("exact", [False, True], ids=["tf32", "exact"])
@pytest.mark.parametrize("S", [3, 1023, 1025, 2049])
def test_bounds_accept_the_emulation(S, exact):
    got = _ratios(S, exact, S)
    assert all(v <= 1 for v in got.values()), got


# (bug, S, quantities whose bound rejects it on the TF32 arm, on the exact arm). A pad column counted as a candidate
# adds its e^-lse to the partition sum: far below the TF32 logit bound, but not the exact arm's.
@pytest.mark.parametrize("bug,S,tf32,exact", [
    ("one_tile", 2049, ("loss", "dx", "rows"), ("loss", "dx", "rows")),
    ("reset_per_tile", 2049, ("loss", "dx", "rows"), ("loss", "dx", "rows")),
    ("no_mask_bwd", 1025, ("rows",), ("dx", "rows")),
    ("pad_column", 1025, (), ("loss", "rows")),
    ("no_minus_one", 1025, ("dx", "rows"), ("dx", "rows")),
    ("logq_sign", 1025, ("loss",), ("loss", "dx", "rows")),
])
def test_bounds_reject_seeded_bugs(bug, S, tf32, exact):
    for arm, which in ((False, tf32), (True, exact)):
        got = _ratios(S, arm, S, bug)
        assert all(got[k] > 1 for k in which), (arm, got)
