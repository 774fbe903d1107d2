"""fp64 model of the deterministic skip-gram kernel (`mvb_sgns_train_det`) and its wave schedule.

A case is a dict in the layout of tests/golden/record_sgns_det_owner.py:

  c          V (words), D (dim), W (window), K (negatives), optionally calls = (0, cut, ..., n_tok)
  tokens     int32 words, -1 a sentence break
  w_in/w_out float32 tables [rows, LD >= D]; only the first D columns are modelled
  map        word -> table row for both tables, or map_in / map_out for each; None: the word is the row
  pool       int32 negative pool, drawn with its first pool_n entries (pool_n: the size the kernel reads from
             device memory; default the whole pool) -- or prob / alias, an alias table over the V words
  s_in/s_out per-word step scales, or None
  lr, seed

The block is trained in calls [cuts[i], cuts[i+1]): every call starts at position 0, uses seed + start and
sees no word outside itself.  A call is trained in waves of `wave` consecutive centres; every read of a wave sees
the tables as the previous wave left them.  A centre with a context reads its output row (label 1) and those of
its K negatives (label 0; a negative equal to the centre is skipped); its contexts are the positions within its
half window hw = W - prng % W up to the first break or call end on either side.  The loss sums 8 softplus(-f)
(label 1) / 8 softplus(f) (label 0) over the pairs of centres at call positions p with p % 8 == 0.
"""
from __future__ import annotations

import numpy as np
import torch

M64 = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15
NEG = 0xD6E8FEB86659FD93


def hash64(x):
    """The kernel's 64-bit finaliser on a uint64 array."""
    x = np.array(x, dtype=np.uint64)
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33); x *= np.uint64(0xff51afd7ed558ccd)
        x ^= x >> np.uint64(33); x *= np.uint64(0xc4ceb9fe1a85ec53)
        x ^= x >> np.uint64(33)
    return x


def _np(t, dtype):
    return None if t is None else np.asarray(t.numpy() if isinstance(t, torch.Tensor) else t).astype(dtype)


def word_maps(case):
    """(map_in, map_out) as int64 arrays over the V words."""
    V = case["c"]["V"]
    m = case.get("map")
    mi, mo = case.get("map_in", m), case.get("map_out", m)
    ident = np.arange(V, dtype=np.int64)
    return (ident if mi is None else _np(mi, np.int64)), (ident if mo is None else _np(mo, np.int64))


def _schedule(case, tl, seed):
    """One call's plan: per position its input row and scale, per centre its 1+K output rows, scales and labels,
    and the (centre, context) pairs."""
    c = case["c"]
    V, W, K = c["V"], c["W"], c["K"]
    mi, mo = word_maps(case)
    ones = np.ones(V)
    si = ones if case.get("s_in") is None else _np(case["s_in"], np.float64)
    so = ones if case.get("s_out") is None else _np(case["s_out"], np.float64)
    n = len(tl)
    valid = tl >= 0
    t0 = np.maximum(tl, 0)
    in_rid = np.where(valid, mi[t0], -1)
    in_sc = np.where(valid, si[t0], 1.0)
    with np.errstate(over="ignore"):
        pos = np.arange(n, dtype=np.uint64)
        prng = hash64(np.uint64(seed) ^ ((pos + np.uint64(1)) * np.uint64(GOLD)))
        hw = (W - (prng >> np.uint64(16)) % np.uint64(W)).astype(np.int64)
        out_rid = np.full((n, K + 1), -1, dtype=np.int64)
        out_sc = np.ones((n, K + 1))
        out_rid[:, 0] = np.where(valid, mo[t0], -1)
        out_sc[:, 0] = np.where(valid, so[t0], 1.0)
        for k in range(1, K + 1):
            r = hash64(prng ^ np.uint64((k * NEG) & M64))
            if case.get("pool") is not None:
                pool = _np(case["pool"], np.int64)
                pool_n = case.get("pool_n", len(pool))
                t = (pool[((r >> np.uint64(8)) % np.uint64(pool_n)).astype(np.int64)] if pool_n > 0
                     else np.full(n, -1, dtype=np.int64))
            else:
                idx = ((r >> np.uint64(32)) % np.uint64(V)).astype(np.int64)
                u = (r & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(1.0 / 16777216.0)
                prob, alias = _np(case["prob"], np.float32), _np(case["alias"], np.int64)
                t = np.where(u < prob[idx], idx, alias[idx])
            t = np.where(valid & (t != tl), t, -1)
            out_rid[:, k] = np.where(t >= 0, mo[np.maximum(t, 0)], -1)
            out_sc[:, k] = np.where(t >= 0, so[np.maximum(t, 0)], 1.0)
    p = np.arange(n, dtype=np.int64)
    trains = out_rid[:, 0] >= 0
    ps, qs = [], []
    for sgn in (-1, 1):
        ok = trains.copy()
        for d in range(1, W + 1):
            q = p + sgn * d
            ok &= (d <= hw) & (q >= 0) & (q < n)
            ok &= in_rid[np.clip(q, 0, n - 1)] >= 0
            ps.append(p[ok]); qs.append(q[ok])
    return in_rid, in_sc, out_rid, out_sc, np.concatenate(ps), np.concatenate(qs)


def model(case, wave):
    """Trains the case in fp64: dict(w_in, w_out [rows, D] float64 tensors, read_in, read_out [rows] bool arrays
    of the table rows any wave read, pairs, loss)."""
    c = case["c"]
    D, K, lr = c["D"], c["K"], case["lr"]
    tokens = _np(case["tokens"], np.int64)
    IN, OUT = case["w_in"][:, :D].double().clone(), case["w_out"][:, :D].double().clone()
    read_in, read_out = np.zeros(IN.shape[0], dtype=bool), np.zeros(OUT.shape[0], dtype=bool)
    pairs, loss = 0, 0.0
    cuts = c.get("calls", (0, len(tokens)))
    for s, e in zip(cuts[:-1], cuts[1:]):
        in_rid, in_sc, out_rid, out_sc, ps, qs = _schedule(case, tokens[s:e], case["seed"] + s)
        pairs += len(ps)
        for w in range(0, -(-(e - s) // wave)):
            sel = ps // wave == w
            P, Q = ps[sel], qs[sel]
            rq = torch.from_numpy(in_rid[Q])
            read_in[in_rid[Q]] = True
            H = IN[rq]
            d_in, d_out = torch.zeros_like(IN), torch.zeros_like(OUT)
            for k in range(K + 1):
                m = out_rid[P, k] >= 0
                ro = torch.from_numpy(out_rid[P, k][m])
                read_out[out_rid[P, k][m]] = True
                mt = torch.from_numpy(m)
                h, o = H[mt], OUT[ro]
                f = (h * o).sum(1)
                g = ((1.0 if k == 0 else 0.0) - torch.sigmoid(f)) * lr
                d_in.index_add_(0, rq[mt], (g * torch.from_numpy(in_sc[Q][m]))[:, None] * o)
                d_out.index_add_(0, ro, (g * torch.from_numpy(out_sc[P, k][m]))[:, None] * h)
                sampled = torch.from_numpy(P[m] % 8 == 0)
                loss += 8.0 * float(torch.nn.functional.softplus(-f if k == 0 else f)[sampled].sum())
            IN += d_in
            OUT += d_out
    return dict(w_in=IN, w_out=OUT, read_in=read_in, read_out=read_out, pairs=pairs, loss=loss)
