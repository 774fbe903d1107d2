"""The deterministic skip-gram kernel (`mvb_sgns_train_det`) at the edges of its CTA tiles.

A CTA owns a slice of consecutive centres of a wave, stages the input rows of the slice and a halo of W
positions on each side, and sums every position's input deltas on chip before sending them out.  These
tests check it against a plain fp64 re-implementation of the sample schedule where the tiling could go
wrong (sentence breaks on and next to slice boundaries, a short last slice, rows that are not a multiple
of 32 floats, the widest window, 7 negatives), and check its exact bits on three multi-wave cases
against digests recorded from the per-centre kernel it replaced (tests/golden/record_sgns_det.py)."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
M64 = (1 << 64) - 1


def _hash64(x):
    x &= M64
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


def _check_schedule(n_tok, dim, W, K, breaks, tol=1e-4):
    """One block of at most one wave: every read sees the initial rows, as the fp64 schedule assumes."""
    from multiverso_b200 import _native as N
    V, D, lr, seed = 4096, dim, 1e-4, 0xC0FFEE
    g = torch.Generator().manual_seed(1)
    w_in = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()
    w_out = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()
    tl = torch.randperm(V - 16, generator=g)[:n_tok].tolist()
    for b in breaks:
        if b < n_tok:
            tl[b] = -1
    pool_l = list(range(V - 16, V - 9))                       # 7 pool words, never tokens
    toks = torch.tensor(tl, dtype=torch.int32, device="cuda")
    pool = torch.tensor(pool_l, dtype=torch.int32, device="cuda")
    s_in, s_out = 0.5 + torch.rand(V, generator=g), 0.5 + torch.rand(V, generator=g)   # hot-row step scales
    i0, o0 = w_in.double().cpu().numpy(), w_out.double().cpu().numpy()
    si, so = s_in.double().numpy(), s_out.double().numpy()
    ref_in, ref_out = i0.copy(), o0.copy()
    n_pairs = 0
    for p, c in enumerate(tl):
        if c < 0:
            continue
        prng = _hash64(seed ^ (((p + 1) * 0x9E3779B97F4A7C15) & M64))
        hw = W - ((prng >> 16) % W)
        ctxs = []
        for sgn in (-1, 1):
            for d in range(1, hw + 1):
                q = p + sgn * d
                if q < 0 or q >= n_tok or tl[q] < 0:
                    break
                ctxs.append(tl[q])
        outs = [(c, 1.0)]
        for k in range(1, K + 1):
            r = _hash64(prng ^ ((k * 0xD6E8FEB86659FD93) & M64))
            t = pool_l[(r >> 8) % len(pool_l)]
            if t != c:
                outs.append((t, 0.0))
        for x in ctxs:
            h = i0[x]
            for (o, label) in outs:
                gk = (label - 1.0 / (1.0 + np.exp(-(h @ o0[o])))) * lr
                ref_in[x] += gk * si[x] * o0[o]
                ref_out[o] += gk * so[o] * h
            n_pairs += 1
    a = N.Sgns()
    loss = torch.zeros(1, device="cuda")
    pairs = torch.zeros(1, dtype=torch.int64, device="cuda")
    a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
    a.w_in, a.w_out, a.dim, a.ld = w_in.data_ptr(), w_out.data_ptr(), D, D
    a.window, a.negative, a.lr = W, K, lr
    a.vocab, a.neg_pool, a.neg_pool_size = V, pool.data_ptr(), len(pool_l)
    a.seed, a.loss_sum, a.pair_count = seed, loss.data_ptr(), pairs.data_ptr()
    sic, soc = s_in.cuda(), s_out.cuda()
    a.scale_in, a.scale_out = sic.data_ptr(), soc.data_ptr()
    assert N.cuda_lib().mvb_sgns_train_det(a, N.stream_ptr()) == 0
    torch.cuda.synchronize()
    assert int(pairs.item()) == n_pairs
    d_in, d_out = w_in.double().cpu().numpy() - i0, w_out.double().cpu().numpy() - o0
    r_in, r_out = ref_in - i0, ref_out - o0
    e_in = np.linalg.norm(d_in - r_in) / np.linalg.norm(r_in)
    e_out = np.linalg.norm(d_out - r_out) / np.linalg.norm(r_out)
    assert e_in < tol and e_out < tol, (e_in, e_out)
    # rows that are neither tokens nor pool words are untouched
    untouched = np.ones(V, dtype=bool)
    untouched[[t for t in tl if t >= 0] + pool_l] = False
    assert np.abs(d_in[untouched]).max() == 0 and np.abs(d_out[untouched]).max() == 0
    assert float(loss.item()) > 0


# Slices hold up to 20 centres (dim 300, window 5, 5 negatives): breaks on, just before and just after
# slice boundaries, and on the first and last position.
SLICE_BREAKS = [0, 19, 20, 21, 59, 61, 139, 140, 141, 259, 260, 499, 999]


@pytest.mark.parametrize("n_tok,dim,window,negative,breaks", [
    (1000, 300, 5, 5, SLICE_BREAKS),                 # breaks around slice boundaries
    (1013, 300, 5, 5, None),                         # a last slice of 13 centres
    (13, 300, 5, 5, None),                           # one slice, shorter than S
    (900, 64, 5, 5, None),
    (700, 100, 5, 5, SLICE_BREAKS),
    (500, 37, 5, 5, None),                           # rows of an odd number of floats
    (700, 512, 5, 5, None),
    (1500, 300, 15, 5, None),                        # the widest window
    (1500, 300, 5, 7, None),                         # 7 negatives (8 output rows per centre)
    (600, 512, 15, 7, [0, 5, 6, 7, 11, 12, 13, 599]),  # all three at once; its slices hold 6 centres
])
def test_sgns_det_tiles_match_schedule(mv_device, n_tok, dim, window, negative, breaks):
    _check_schedule(n_tok, dim, window, negative, range(37, n_tok, 53) if breaks is None else breaks)


def _recorder():
    spec = importlib.util.spec_from_file_location("record_sgns_det", os.path.join(GOLDEN, "record_sgns_det.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize("case", ["zipf_v5000", "maps_ld320", "dim512_w15"])
def test_sgns_det_bits_match_recorded(mv_device, case):
    """Multi-wave runs give the same table bits, loss bits and pair count as the per-centre kernel did
    (digests recorded on an H100 SXM: the wave size follows from the SM count)."""
    with open(os.path.join(GOLDEN, "sgns_det_parent.json")) as f:
        want = json.load(f)["cases"][case]
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("digests were recorded with the wave size of a 132-SM H100")
    assert _recorder().run_case(case) == want
