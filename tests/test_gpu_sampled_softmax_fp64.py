"""PSSampledSoftmax (csrc/cuda/sampled_softmax.cu) against fp64 at the edges of its kernels: S on both sides of the
forward's 1024-candidate shared-memory tile (the online logsumexp (m, s) carried from tile to tile), S = 1..5 where
S_pad > S and the pad rows of W_S are zero, B around the 8-example forward CTA and the 32 x 32 backward tile, d
around the 128-float lane stride of the true dot, rows whose every candidate is an accidental hit, logits near +-80,
a non-uniform g, duplicate candidates, 1 / 3 / 8 shards with NaN gaps, the compact push, the two epilogues called
directly on crafted logits, the refusals of the three entry points, and S past the 65535-block grid.y limit.

Bounds. u = 2^-24. For example b let L_b be the largest finite |z_bj| over its true and sampled logits.

* One logit. On random operands the wgmma rounds x and w to TF32 (4 * 2^-11 per product, test_gpu_sampled_softmax)
  and sums d terms in fp32; the correction log(S q) is an fp32 value: ``(TF32 + d u) |x_b| max|w| + 4 u (1 +
  max|log S q| + L_b)``. On the exact arm (x and W small integers times a power of two) every product and sum is
  exact and the reference takes the kernel's fp32 ``log_s + logq[c]`` as given, so only the subtraction of the
  correction rounds: ``u L_b``.
* The logsumexp. Each lane folds at most 32 logits per 1024-candidate tile into (m, s), each through one fp32
  subtraction (|argument| <= 2 L_b), one expf (2 ulp) and one add or rescale, so every push moves s by at most
  (2 L_b + 8) u relative; the warp merge, the true logit and the log add 8 more such steps and 2 u |lse_b|:
  ``sum_b = (32 ceil(S / 1024) + 8) (2 L_b + 8) u + 2 u |lse_b|``. lse is 1-Lipschitz in the logits, so its error is
  ``logit_b + sum_b`` and the loss ``lse - t`` adds one more logit error and one rounding.
* E = g softmax and e_true = g (p_true - 1). The exponent of p_bj is off by the logit and lse errors plus the fp32
  subtractions (3 u (L_b + |lse_b|)) and expf (4 u), so p_bj is within ``rel_b = expm1(that) + u`` relative: E_bj
  within ``|g_b| p_bj rel_b`` (exactly 0 on masked columns, where p = 0), e_true within ``|g_b| (p_true rel_b + 2 u)``.
* dX = E W_S + e_true w_y on the GEMM: the E error, the TF32 rounding of the operands (TF32 per product; 2^-10 for
  the truncated E alone on the exact arm) and an fp32 sum over S terms (2 (S + 8) u, allowing truncating adds), per
  coordinate against the rows' max-norms, plus the fp32 addcmul.
* dW_S = E^T X likewise over B terms; the push coalesces at most B + S uses of a row in fp32 (2 (B + S) u of their
  magnitudes); one sgd step ``W - lr dW`` adds one product and one add rounding.

tests/test_sampled_softmax_bounds_cpu.py emulates the kernels' order of operations in numpy fp32 and shows that these
bounds accept it and reject a dropped second tile, (m, s) reset per tile, the mask missing in the backward, a pad
column counted as a candidate, e_true without its -1 and a flipped log-Q sign on the true logit.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TF32 = 4 * 2.0 ** -11      # a product of two TF32-rounded operands
TF32_ONE = 2.0 ** -10      # one TF32-truncated operand times an exact one
FWD_TILE = 1024            # candidates per shared-memory tile of the forward epilogue
NAN_BITS = 0x7FD1CE5D      # a quiet NaN with a payload, in rows no kernel may write
BIG_S = 65535 * 32 + 33    # S_pad / 32 row tiles of W_S^T past the 65535 grid.y limit


# ------------------------------------------------------------------------------------------------ fp64 model
def reference(x, W, y, cand, logsq, g):
    """fp64 loss, lse, logits z = [t, s], p = softmax(z), E, e_true, dL/dx and dL/dW of (loss * g).sum(); every
    argument is a torch tensor (logsq: log(S q) per table row)."""
    x64 = x.double().requires_grad_()
    W64 = W.double().requires_grad_()
    t = (x64 * W64[y]).sum(1) - logsq[y]
    s = (x64 @ W64[cand].t() - logsq[cand][None, :]).masked_fill(cand[None, :] == y[:, None], float("-inf"))
    z = torch.cat([t[:, None], s], 1)
    lse = torch.logsumexp(z, 1)
    loss = lse - t
    (loss * g.double()).sum().backward()
    with torch.no_grad():
        p = torch.softmax(z, 1)
        g64 = g.double()
        return dict(loss=loss.detach(), lse=lse.detach(), z=z.detach(), p=p, E=g64[:, None] * p[:, 1:],
                    e_true=g64 * (p[:, 0] - 1), dx=x64.grad, dW=W64.grad)


def softmax_bounds(z, lse, loss, g, logit_err):
    """tol_loss [B], tol_E [B, S] and tol_etrue [B] of the epilogues over the fp64 logits z = [t, s] (-inf on masked
    columns), given the error of one logit per example."""
    S = z.shape[1] - 1
    L = torch.where(torch.isfinite(z), z.abs(), torch.zeros_like(z)).amax(1)
    summ = (32 * -(-S // FWD_TILE) + 8) * (2 * L + 8) * U + 2 * U * lse.abs()
    lse_err = logit_err + summ
    tol_loss = logit_err + lse_err + U * (lse.abs() + loss.abs())
    rel = torch.expm1(logit_err + lse_err + 3 * U * (L + lse.abs()) + 4 * U) + U
    p = torch.softmax(z, 1)
    ga = g.double().abs()
    return tol_loss, ga[:, None] * p[:, 1:] * rel[:, None], ga * (p[:, 0] * rel + 2 * U)


def bounds(r, x, W, y, cand, logsq, g, exact=False):
    """The bounds of the module docstring: tol_loss [B], tol_E [B, S], tol_etrue [B], tol_dx [B] (max over
    coordinates) and tol_rows [n] (dL/dW per row, max over coordinates)."""
    B, d = x.shape
    S = cand.numel()
    x64, W64 = x.double(), W.double()
    z = r["z"]
    L = torch.where(torch.isfinite(z), z.abs(), torch.zeros_like(z)).amax(1)
    if exact:
        logit = U * L
    else:
        used = torch.cat([y, cand])
        wmax = W64[used].norm(dim=1).max()
        logit = (TF32 + d * U) * x64.norm(dim=1) * wmax + 4 * U * (1 + logsq[used].abs().max() + L)
    tol_loss, tol_E, tol_et = softmax_bounds(z, r["lse"], r["loss"], g, logit)
    prod = TF32_ONE if exact else TF32
    aE = r["E"].abs() + tol_E
    aet = r["e_true"].abs()
    wI, xI = W64.abs().amax(1), x64.abs().amax(1)
    tol_dx = ((tol_E + (prod + 2 * (S + 8) * U) * aE) @ wI[cand] + (tol_et + 2 * U * aet) * wI[y]
              + 2 * U * r["dx"].abs().amax(1))
    rows = torch.zeros(W.shape[0], dtype=torch.float64, device=x.device)
    rows.index_add_(0, cand, ((tol_E + (prod + 2 * (B + 8) * U) * aE) * xI[:, None]).sum(0))
    rows.index_add_(0, y, (tol_et + 2 * U * aet) * xI)
    mag = torch.zeros_like(rows)
    mag.index_add_(0, cand, (aE * xI[:, None]).sum(0))
    mag.index_add_(0, y, aet * xI)
    rows += 2 * (B + S) * U * mag
    return dict(loss=tol_loss, E=tol_E, e_true=tol_et, dx=tol_dx, rows=rows)


def logsq64(ssm, counts=None):
    """log(S q) per row in fp64 from the sampler's definition (-inf on zero-count rows)."""
    n = ssm.num_classes
    if counts is None:
        k = np.arange(n, dtype=np.float64)
        q = np.log((k + 2) / (k + 1)) / np.log(n + 1)
    else:
        w = np.power(counts.double().numpy(), ssm.power)
        q = w / w.sum()
    with np.errstate(divide="ignore"):
        return torch.from_numpy(np.log(ssm.num_sampled * q))


def logsq32(ssm):
    """The kernels' own fp32 corrections log_s + logq[c] per row, as fp64."""
    return torch.from_numpy((np.float32(ssm._log_s) + ssm._logq.cpu().numpy()).astype(np.float64))


def ratio(err, tol):
    """max err / tol, with 0 / 0 = 0 and anything / 0 = inf."""
    err, tol = err.double(), tol.double()
    q = torch.where(err == 0, torch.zeros_like(err), err / tol)
    return q.max().item() if q.numel() else 0.0


# ------------------------------------------------------------------------------------------------ device set-up
@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _nan_sharded(W, S, gap=3):
    """W as S shards of one buffer (rows_per_server = n // S, the last shard takes the remainder) with `gap` rows of
    payload NaN before every shard and after the last. Returns the row map, the buffer, a reader of the table and a
    mask of the buffer rows that belong to no shard."""
    from multiverso_b200 import _native as N
    n, d = W.shape
    rps = n // S
    buf = torch.empty(n + (S + 1) * gap, d, device=W.device)
    _bits(buf).fill_(NAN_BITS)
    gaps = torch.ones(buf.shape[0], dtype=torch.bool, device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, d, S, rps
    spans = []
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = W[lo:hi]
        gaps[at:at + hi - lo] = False
        rm.shard_ptrs[s] = buf[at].data_ptr()
        spans.append((at, hi - lo))
    return rm, buf, (lambda: torch.cat([buf[a:a + k] for a, k in spans])), gaps


def _fake_table(rm, num_row, num_col, updater=None):
    from test_gpu_sampled_softmax import _fake_table as fake
    return fake(rm, num_row, num_col, updater)


def _labels(gen, ssm, B, allowed):
    """B labels from `allowed` rows, a quarter of them planted on drawn candidates (accidental hits, duplicates
    included) and a quarter repeating one label."""
    dev = allowed.device
    y = allowed[torch.randint(0, allowed.numel(), (B,), device=dev, generator=gen)]
    cand = ssm.draw(0)
    hits = (B + 3) // 4
    y[:hits] = cand[torch.randint(0, cand.numel(), (hits,), device=dev, generator=gen)]
    rep = B // 4
    y[hits:hits + rep] = y[0]
    return y


def _g(gen, B, dev):
    """A non-uniform loss gradient: normal (so half negative) with every third entry zero."""
    g = torch.randn(B, device=dev, generator=gen)
    g[1::3] = 0
    return g


def _step(W, x, y, g, ssm_kw, shards, lr):
    """One forward and backward of (loss * g).sum() over a NaN-gapped sharded copy of W: loss, dL/dx, the table
    after the sgd push, the buffer before and after, the gap mask and the candidates."""
    from multiverso_b200.ops import PSSampledSoftmax
    n, d = W.shape
    rm, buf, back, gaps = _nan_sharded(W, shards)
    before = buf.clone()
    ssm = PSSampledSoftmax(_fake_table(rm, n, d), push_scale=lr, **ssm_kw)
    xx = x.clone().requires_grad_()
    loss = ssm(xx, y)
    (loss * g).sum().backward()
    torch.cuda.synchronize()
    return loss.detach(), xx.grad, back(), before, buf, gaps, ssm


def _check_op(W, x, y, g, ssm_kw, shards=1, lr=0.5, counts=None, exact=False):
    """The op against fp64 (loss, dL/dx, the table after one sgd step), and nothing else of the buffer touched.
    Returns the err / bound ratios."""
    loss, dx, got, before, buf, gaps, ssm = _step(W, x, y, g, ssm_kw, shards, lr)
    cand = ssm.draw(0)
    dev = x.device
    ls = (logsq32(ssm) if exact else logsq64(ssm, counts)).to(dev)
    r = reference(x, W, y, cand, ls, g)
    tol = bounds(r, x, W, y, cand, ls, g, exact)
    exp = W.double() - lr * r["dW"]
    err_w = (got.double() - exp).abs().amax(1)
    tol_w = lr * tol["rows"] + 2 * U * lr * r["dW"].abs().amax(1) + 2 * U * exp.abs().amax(1)
    out = dict(loss=ratio((loss.double() - r["loss"]).abs(), tol["loss"]),
               dx=ratio((dx.double() - r["dx"]).abs().amax(1), tol["dx"]),
               table=ratio(err_w, tol_w))
    assert torch.isfinite(loss).all() and torch.isfinite(dx).all() and torch.isfinite(got).all()
    for k, v in out.items():
        assert v <= 1, (k, out)
    touched = torch.zeros(W.shape[0], dtype=torch.bool, device=dev)
    touched[torch.cat([y, cand])] = True
    assert torch.equal(_bits(got[~touched]), _bits(W[~touched]))          # untouched rows: bitwise unchanged
    assert torch.equal(_bits(buf[gaps]), _bits(before[gaps]))             # the gaps: bitwise unchanged
    return out


# ------------------------------------------------------------------------------------------------ a. the op
# (S, B, d, sampler, n, shards): S on both sides of 1024-candidate tiles and of S_pad, B around the 8-example
# forward CTA and the 32-example backward tile, d around the 128-float lane stride; n = 4011 has an odd
# rows_per_server over 1, 3 and 8 shards, n = 61 makes nearly every candidate a duplicate
CASES = [
    ("S1_B1_d4", 1, 1, 4, "log_uniform", 4011, 1),
    ("S1_B301_d132_all_hits", 1, 301, 132, "log_uniform", 61, 1),
    ("S3_B2_d8_counts", 3, 2, 8, "counts", 4011, 3),
    ("S3_B32_d1024", 3, 32, 1024, "log_uniform", 4011, 1),
    ("S4_B3_d124", 4, 3, 124, "log_uniform", 4011, 8),
    ("S4_B1025_d4", 4, 1025, 4, "log_uniform", 4011, 3),
    ("S5_B7_d128", 5, 7, 128, "log_uniform", 4011, 1),
    ("S5_B8_d132_counts", 5, 8, 132, "counts", 4011, 1),
    ("S1023_B9_d4", 1023, 9, 4, "log_uniform", 4011, 1),
    ("S1023_B2_d516_counts", 1023, 2, 516, "counts", 4011, 8),
    ("S1024_B31_d128", 1024, 31, 128, "log_uniform", 4011, 1),
    ("S1024_B1_d1024", 1024, 1, 1024, "log_uniform", 4011, 3),
    ("S1025_B32_d132", 1025, 32, 132, "log_uniform", 4011, 1),
    ("S1025_B33_d8_counts", 1025, 33, 8, "counts", 4011, 1),
    ("S1025_B9_d124_dups", 1025, 9, 124, "log_uniform", 61, 1),
    ("S2047_B301_d516", 2047, 301, 516, "log_uniform", 4011, 1),
    ("S2047_B7_d8", 2047, 7, 8, "log_uniform", 4011, 8),
    ("S2049_B8_d1024", 2049, 8, 1024, "log_uniform", 4011, 1),
    ("S2049_B1025_d124_counts", 2049, 1025, 124, "counts", 4011, 3),
    ("S2049_B31_d128", 2049, 31, 128, "log_uniform", 4011, 1),
    ("S8192_B1025_d128", 8192, 1025, 128, "log_uniform", 4011, 1),
    ("S8192_B33_d4_counts", 8192, 33, 4, "counts", 4011, 8),
    ("S8192_B3_d132", 8192, 3, 132, "log_uniform", 4011, 1),
    ("S8193_B3_d516", 8193, 3, 516, "log_uniform", 4011, 3),
    ("S8193_B301_d1024", 8193, 301, 1024, "log_uniform", 4011, 1),
    ("S8193_B32_d8_counts", 8193, 32, 8, "counts", 4011, 1),
    ("S8193_B2_d4_dups", 8193, 2, 4, "log_uniform", 61, 1),
    ("S1025_B1_d4_counts", 1025, 1, 4, "counts", 4011, 8),
]


def _counts(gen_cpu, n):
    """Counts with about half the rows zero."""
    c = torch.randint(1, 100, (n,), generator=gen_cpu) * (torch.rand(n, generator=gen_cpu) < 0.5)
    c[0] = 1
    return c


@pytest.mark.parametrize("S,B,d,sampler,n,shards", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_op_matches_fp64(cuda, S, B, d, sampler, n, shards):
    seed = S * 7919 + B * 31 + d
    gen = torch.Generator(device=cuda).manual_seed(seed)
    gcpu = torch.Generator().manual_seed(seed)
    W = torch.randn(n, d, device=cuda, generator=gen) / d ** 0.5
    x = torch.randn(B, d, device=cuda, generator=gen) * 2
    counts = _counts(gcpu, n) if sampler == "counts" else None
    kw = dict(num_sampled=S, seed=seed, **({"counts": counts} if counts is not None else {"sampler": sampler}))
    from multiverso_b200.ops import PSSampledSoftmax
    probe = PSSampledSoftmax(_fake_table(_nan_sharded(W, 1)[0], n, d), push_scale=None, **kw)
    allowed = torch.arange(n, device=cuda) if counts is None else torch.nonzero(counts > 0)[:, 0].to(cuda)
    y = _labels(gen, probe, B, allowed)
    _check_op(W, x, y, _g(gen, B, cuda), kw, shards, counts=counts)


# ------------------------------------------------------------------------------------------------ b. degenerate
def test_every_column_masked_is_exact(cuda):
    """A one-row table, and labels all equal to the only class of a one-hot sampler: every sampled column is an
    accidental hit, so the loss is exactly 0, dX exactly 0 and the pushed rows exactly W."""
    gen = torch.Generator(device=cuda).manual_seed(5)
    for n, counts, S, B, d in ((1, None, 1025, 9, 8), (50, torch.eye(50)[17], 2049, 33, 132)):
        W = torch.randn(n, d, device=cuda, generator=gen)
        x = torch.randn(B, d, device=cuda, generator=gen)
        y = torch.full((B,), n - 1 if counts is None else 17, dtype=torch.int64, device=cuda)
        kw = dict(num_sampled=S, seed=3, **({"counts": counts} if counts is not None else {"sampler": "log_uniform"}))
        loss, dx, got, before, buf, gaps, ssm = _step(W, x, y, _g(gen, B, cuda), kw, 1, 0.5)
        assert (ssm.draw(0) == y[0]).all()
        assert torch.equal(loss, torch.zeros_like(loss))
        assert torch.equal(dx, torch.zeros_like(dx))
        assert torch.equal(_bits(got), _bits(W))
        assert torch.equal(_bits(buf), _bits(before))


@pytest.mark.parametrize("kind", ["pm80", "true_dominates"])
def test_large_logits(cuda, kind):
    """Logits near +-80 (any missing max-shift overflows expf over 8193 columns), and a true logit ~100 above every
    sampled one (a loss near 1e-30): finite, and within the bounds."""
    gen = torch.Generator(device=cuda).manual_seed(11)
    n, S, B = 4011, 8193, 32
    d = 4 if kind == "pm80" else 128
    W = torch.randn(n, d, device=cuda, generator=gen)
    W /= W.norm(dim=1, keepdim=True)
    y = torch.randint(0, n, (B,), device=cuda, generator=gen)
    if kind == "pm80":
        x = torch.randn(B, d, device=cuda, generator=gen)
        x *= 84 / x.norm(dim=1, keepdim=True)
    else:
        x = 100 * W[y]
    out = _check_op(W, x, y, _g(gen, B, cuda), dict(num_sampled=S, seed=2, sampler="log_uniform"), lr=1e-3)
    assert all(v <= 1 for v in out.values())


# ------------------------------------------------------------------------------------------------ c. exact operands
@pytest.mark.parametrize("S", [1025, 4097, 8193])
def test_exact_operands(cuda, S):
    """x and W small integers times a power of two: every wgmma logit and the fp32 true dot are exact, the
    corrections are the kernel's fp32 values, and the tight bound of the exact arm holds."""
    gen = torch.Generator(device=cuda).manual_seed(S)
    n, B, d = 4011, 33, 132
    W = torch.randint(-3, 4, (n, d), device=cuda, generator=gen).float() * 0.125
    x = torch.randint(-3, 4, (B, d), device=cuda, generator=gen).float() * 0.25
    kw = dict(num_sampled=S, seed=S, sampler="log_uniform")
    from multiverso_b200.ops import PSSampledSoftmax
    probe = PSSampledSoftmax(_fake_table(_nan_sharded(W, 1)[0], n, d), push_scale=None, **kw)
    y = _labels(gen, probe, B, torch.arange(n, device=cuda))
    _check_op(W, x, y, _g(gen, B, cuda), kw, 3, lr=0.5, exact=True)


# ------------------------------------------------------------------------------------------------ e. compact push
def test_compact_push_past_one_tile(cuda):
    """An adagrad table gets the compact push: one row per touched id, within the fp64 bound, at S = 8193."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSSampledSoftmax
    gen = torch.Generator(device=cuda).manual_seed(21)
    n, d, B, S, scale = 3001, 36, 65, 8193, 0.1
    W = torch.randn(n, d, device=cuda, generator=gen) * 0.3
    rm, buf, back, gaps = _nan_sharded(W, 3)
    pushes = []
    rec = _fake_table(rm, n, d, N.UPDATER_NAMES["adagrad"])
    rec.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    ssm = PSSampledSoftmax(rec, num_sampled=S, sampler="log_uniform", push_scale=scale, seed=4)
    y = _labels(gen, ssm, B, torch.arange(n, device=cuda))
    x = torch.randn(B, d, device=cuda, generator=gen)
    g = _g(gen, B, cuda)
    (ssm(x, y) * g).sum().backward()
    torch.cuda.synchronize()
    cand = ssm.draw(0)
    ls = logsq64(ssm).to(cuda)
    r = reference(x, W, y, cand, ls, g)
    tol = bounds(r, x, W, y, cand, ls, g)
    assert len(pushes) == 1
    uniq, grads = pushes[0]
    assert torch.equal(uniq, torch.unique(torch.cat([y, cand])))
    err = (grads.double() - scale * r["dW"][uniq]).abs().amax(1)
    bound = scale * tol["rows"][uniq] + 2 * U * scale * r["dW"][uniq].abs().amax(1)
    assert (err <= bound).all(), ratio(err, bound)
    assert torch.equal(back(), W)                                         # a compact push writes no row itself


# ------------------------------------------------------------------------------------------------ f. epilogues
def _round4(n):
    return (n + 3) // 4 * 4


def _epilogue_args(cuda, S, B, seed):
    """Crafted epilogue inputs: logits [B, S_pad] with NaN in the pad columns, duplicate candidates, labels with
    accidental hits (one row fully masked when S == 1), exact true dots, arbitrary fp32 corrections, and g with
    zeros and negatives. Returns the argument struct and its tensors."""
    from multiverso_b200 import _native as N
    gen = torch.Generator(device=cuda).manual_seed(seed)
    n, d = 97, 8
    Sp, Bp = _round4(S), _round4(B)
    T = dict(
        cand=torch.randint(0, n, (S,), device=cuda, generator=gen),
        logq_c=(torch.randn(S, device=cuda, generator=gen) * 2).float(),
        logq=(torch.randn(n, device=cuda, generator=gen) - 4).float(),
        x=torch.randint(-3, 4, (B, d), device=cuda, generator=gen).float() * 0.25,
        w_y=torch.randint(-3, 4, (B, d), device=cuda, generator=gen).float() * 0.125,
        logits=torch.full((B, Sp), float("nan"), device=cuda),
        loss=torch.full((B,), float("nan"), device=cuda), lse=torch.full((B,), float("nan"), device=cuda),
        t_true=torch.full((B,), float("nan"), device=cuda), g=_g(gen, B, cuda),
        e_t=torch.empty(Sp, Bp, device=cuda), e_true=torch.full((B,), float("nan"), device=cuda))
    _bits(T["e_t"]).fill_(NAN_BITS)
    T["logits"][:, :S] = torch.randn(B, S, device=cuda, generator=gen) * 3
    y = torch.randint(0, n, (B,), device=cuda, generator=gen)
    hits = (B + 2) // 3
    y[:hits] = T["cand"][torch.randint(0, S, (hits,), device=cuda, generator=gen)]
    T["labels"] = y
    a = N.SampledSoftmax()
    a.n, a.S, a.S_pad, a.log_s = n, S, Sp, float(np.float32(math.log(S)))
    a.B, a.B_pad, a.d = B, Bp, d
    for k in ("cand", "logq_c", "logq", "x", "w_y", "labels", "logits", "loss", "lse", "t_true", "g", "e_t",
              "e_true"):
        setattr(a, k, T[k].data_ptr())
    return a, T


@pytest.mark.parametrize("S,B", [(1, 8), (5, 33), (1023, 9), (1024, 32), (1024, 7), (1025, 31), (1025, 8),
                                 (2049, 33)])
def test_epilogues_on_crafted_logits(cuda, S, B):
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    a, T = _epilogue_args(cuda, S, B, S * 100 + B)
    lib.mvb_ss_fwd_epilogue(a, st)
    torch.cuda.synchronize()
    y, cand = T["labels"], T["cand"]
    corr = (np.float32(a.log_s) + T["logq"].cpu().numpy()).astype(np.float64)        # the kernel's fp32 correction
    t = (T["x"].double() * T["w_y"].double()).sum(1) - torch.from_numpy(corr).to(cuda)[y]
    s = (T["logits"][:, :S].double() - T["logq_c"].double()[None, :]).masked_fill(
        cand[None, :] == y[:, None], float("-inf"))
    z = torch.cat([t[:, None], s], 1)
    lse = torch.logsumexp(z, 1)
    loss = lse - t
    L = torch.where(torch.isfinite(z), z.abs(), torch.zeros_like(z)).amax(1)
    tol_loss, tol_E, tol_et = softmax_bounds(z, lse, loss, T["g"], U * L)
    assert ratio((T["t_true"].double() - t).abs(), U * L) <= 1
    assert ratio((T["loss"].double() - loss).abs(), tol_loss) <= 1
    assert ratio((T["lse"].double() - lse).abs(), tol_loss) <= 1
    logits_in = T["logits"].clone()
    lib.mvb_ss_bwd_epilogue(a, st)
    torch.cuda.synchronize()
    E = T["logits"]
    p = torch.softmax(z, 1)
    g64 = T["g"].double()
    assert ratio((E[:, :S].double() - g64[:, None] * p[:, 1:]).abs(), tol_E) <= 1
    assert ratio((T["e_true"].double() - g64 * (p[:, 0] - 1)).abs(), tol_et) <= 1
    masked = (cand[None, :] == y[:, None])
    assert (_bits(E[:, :S])[masked] == 0).all()                           # masked columns: exactly +0
    assert (_bits(E[:, S:]) == 0).all()                                   # the NaN pad columns: exactly +0
    assert torch.equal(_bits(T["e_t"][:, :B]), _bits(E.t()))              # E^T, bitwise
    assert (_bits(T["e_t"][:, B:]) == 0).all()                            # the pad columns of E^T: exactly +0
    assert torch.isnan(logits_in[:, S:]).all()


# ------------------------------------------------------------------------------------------------ g. refusals
def _captured(fn):
    """The work fn enqueues, counted exactly: fn(stream) runs while the driver captures that stream into a graph, so
    every launch, copy or memset it makes becomes a graph node instead of running. Returns the node count."""
    import ctypes
    cu = ctypes.CDLL("libcuda.so.1")
    cu.cuStreamBeginCapture_v2.argtypes = [ctypes.c_void_p, ctypes.c_int]
    cu.cuStreamEndCapture.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_void_p)]
    cu.cuGraphGetNodes.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_size_t)]
    cu.cuGraphDestroy.argtypes = [ctypes.c_void_p]
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    assert cu.cuStreamBeginCapture_v2(stream.cuda_stream, 2) == 0            # CU_STREAM_CAPTURE_MODE_RELAXED
    graph = ctypes.c_void_p()
    try:
        with torch.cuda.stream(stream):
            fn(stream.cuda_stream)
    finally:
        rc = cu.cuStreamEndCapture(stream.cuda_stream, ctypes.byref(graph))
    assert rc == 0, rc
    nodes = ctypes.c_size_t()
    assert cu.cuGraphGetNodes(graph, None, ctypes.byref(nodes)) == 0
    cu.cuGraphDestroy(graph)
    return nodes.value


def test_entry_points_refuse_without_launching(cuda):
    """Every return code of mvb_ss_sample / mvb_ss_fwd_epilogue / mvb_ss_bwd_epilogue raises with nothing enqueued,
    and an empty batch returns with nothing enqueued. The capture ends with one valid draw, which must be its one
    node: that also shows the capture records the entry points' launches."""
    from multiverso_b200 import _native as N
    lib = N.cuda_lib()
    a, T = _epilogue_args(cuda, 9, 5, 1)
    prob = torch.ones(a.n, device=cuda)
    alias = torch.zeros(a.n, dtype=torch.int32, device=cuda)
    a.alias_prob, a.alias_idx = prob.data_ptr(), alias.data_ptr()
    shape = [("n", 0), ("n", 1 << 31), ("S", 0), ("S_pad", 8), ("S_pad", 14)]
    cases = [(f, -60, [(k, v)]) for f in ("mvb_ss_sample", "mvb_ss_fwd_epilogue", "mvb_ss_bwd_epilogue")
             for k, v in shape]
    cases += [("mvb_ss_sample", -61, [(k, None)]) for k in ("alias_prob", "alias_idx", "logq", "cand", "logq_c")]
    cases += [("mvb_ss_fwd_epilogue", -62, [(k, v)]) for k, v in (("d", 0), ("d", 6))]
    cases += [("mvb_ss_fwd_epilogue", -62, [(k, getattr(a, k) + 4)]) for k in ("x", "w_y", "logits")]
    cases += [("mvb_ss_fwd_epilogue", -63, [("B", 8 << 31), ("B_pad", 8 << 31)])]
    cases += [("mvb_ss_bwd_epilogue", -64, [(k, v)]) for k, v in (("B_pad", 4), ("B_pad", 10), ("e_t", None),
                                                                  ("e_true", None), ("g", None))]
    cases += [("mvb_ss_bwd_epilogue", -63, [("B", 65536 * 32), ("B_pad", 65536 * 32)])]
    for fname, rc, edits in cases:
        saved = [(k, getattr(a, k)) for k, _ in edits]
        for k, v in edits:
            setattr(a, k, v)

        def refused(st):
            with pytest.raises(N.NativeError, match=f"rc={rc}:"):
                getattr(lib, fname)(a, st)
        assert _captured(refused) == 0, (fname, edits)
        for k, v in saved:
            setattr(a, k, v)
    a.B = 0
    for name in ("mvb_ss_fwd_epilogue", "mvb_ss_bwd_epilogue"):
        assert _captured(lambda st: getattr(lib, name)(a, st)) == 0, name
    assert _captured(lambda st: lib.mvb_ss_sample(a, st)) == 1                # the capture sees a launch


def test_batch_past_the_backward_grid_is_refused(cuda):
    """B above MAX_BATCH is refused with a named error before any draw, launch or copy, and steps does not
    advance. The capture ends with one valid draw, which must be its one node."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSSampledSoftmax
    from multiverso_b200.ops.sampled_softmax import MAX_BATCH
    assert MAX_BATCH == 65535 * 32
    n, d = 1000, 4
    rm, buf, back, gaps = _nan_sharded(torch.randn(n, d, device=cuda), 1)
    ssm = PSSampledSoftmax(_fake_table(rm, n, d), num_sampled=16, sampler="log_uniform")
    x = torch.zeros(MAX_BATCH + 1, d, device=cuda)
    y = torch.zeros(MAX_BATCH + 1, dtype=torch.int64, device=cuda)
    cand = torch.empty(16, dtype=torch.int64, device=cuda)
    logq_c = torch.empty(16, device=cuda)
    a = ssm._args(0)
    a.cand, a.logq_c = cand.data_ptr(), logq_c.data_ptr()

    def refused(st):
        with pytest.raises(ValueError, match="at most 2097120 examples"):
            ssm(x, y)
    assert _captured(refused) == 0
    assert ssm.steps == 0
    assert _captured(lambda st: N.cuda_lib().mvb_ss_sample(a, st)) == 1


# ------------------------------------------------------------------------------------------------ 3. shape limit
def test_num_sampled_past_grid_y_limit(cuda):
    """S = 2,097,153: W_S^T has more 32-row tiles than grid.y holds; the backward's transposes grid-stride over
    them. About 250 MB of device buffers."""
    gen = torch.Generator(device=cuda).manual_seed(17)
    n, B, d = 4011, 5, 4
    W = torch.randn(n, d, device=cuda, generator=gen) / 2
    x = torch.randn(B, d, device=cuda, generator=gen) * 2
    y = torch.randint(0, n, (B,), device=cuda, generator=gen)
    y[0] = 0                                                              # the most drawn row: accidental hits
    _check_op(W, x, y, _g(gen, B, cuda), dict(num_sampled=BIG_S, seed=8, sampler="log_uniform"), 1)
