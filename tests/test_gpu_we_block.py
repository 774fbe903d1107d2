"""Device-side WordEmbedding block protocol (csrc/cuda/we_block.cu) against plain PyTorch references:
PrepareData (bitmap-unique + prefix sum + negative pool), bulk-engine row pull and delta push."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _prep(tokens, V, K, prob, alias, cap_in, cap_out, seed=99):
    from multiverso_b200 import _native as N
    words = (V + 31) // 32
    i32 = dict(dtype=torch.int32, device="cuda")
    b = dict(bm_in=torch.empty(words, **i32), bm_out=torch.empty(words, **i32),
             chunk_sums=torch.empty((words + 1023) // 1024 + 1, **i32),
             map_in=torch.full((V,), -7, **i32), map_out=torch.full((V,), -7, **i32),
             ids_in=torch.full((cap_in,), -7, **i32), ids_out=torch.full((cap_out,), -7, **i32),
             neg_pool=torch.full((max(cap_in * K, 1),), -7, **i32), counts=torch.zeros(4, **i32))
    p = N.WePrep()
    p.tokens, p.n_tokens, p.vocab, p.negative = tokens.data_ptr(), tokens.numel(), V, K
    p.alias_prob, p.alias_idx, p.seed = N.ptr(prob), N.ptr(alias), seed
    p.bm_in, p.bm_out, p.chunk_sums = b["bm_in"].data_ptr(), b["bm_out"].data_ptr(), b["chunk_sums"].data_ptr()
    p.map_in, p.map_out = b["map_in"].data_ptr(), b["map_out"].data_ptr()
    p.ids_in, p.ids_out = b["ids_in"].data_ptr(), b["ids_out"].data_ptr()
    p.neg_pool, p.pool_cap, p.counts = b["neg_pool"].data_ptr(), b["neg_pool"].numel(), b["counts"].data_ptr()
    p.cap_in, p.cap_out = cap_in, cap_out
    N.cuda_lib().mvb_we_prepare(p, N.stream_ptr())
    torch.cuda.synchronize()
    return b


@pytest.mark.parametrize("V,n_tok,K", [(100003, 50000, 5), (1000, 20000, 5), (70001, 3000, 0), (2_000_000, 300000, 3)])
def test_we_prepare_matches_torch(mv_device, V, n_tok, K):
    g = torch.Generator().manual_seed(V)
    toks = (torch.rand(n_tok, generator=g).pow(3) * V).to(torch.int32).clamp_(0, V - 1)
    toks[100::101] = -1
    toks = toks.cuda()
    prob = torch.rand(V, generator=g).cuda()
    alias = torch.randint(0, V, (V,), generator=g, dtype=torch.int32).cuda()
    cap_in = min(V, n_tok)
    cap_out = min(V, cap_in * (1 + K))
    b = _prep(toks, V, K, prob if K else None, alias if K else None, cap_in, cap_out)
    n_in, n_out, n_pool = b["counts"][:3].tolist()
    exp_in = torch.unique(toks[toks >= 0].long())
    assert n_in == exp_in.numel()
    assert torch.equal(b["ids_in"][:n_in].long(), exp_in)                 # ascending ids, slot = rank
    exp_map = torch.full((V,), -1, dtype=torch.int32, device="cuda")
    exp_map[exp_in] = torch.arange(n_in, dtype=torch.int32, device="cuda")
    assert torch.equal(b["map_in"], exp_map)
    assert n_pool == K * n_in
    pool = b["neg_pool"][:n_pool].long()
    if K:
        assert int(pool.min()) >= 0 and int(pool.max()) < V
    exp_out = torch.unique(torch.cat([exp_in, pool]))
    assert n_out == exp_out.numel()
    assert torch.equal(b["ids_out"][:n_out].long(), exp_out)
    exp_mo = torch.full((V,), -1, dtype=torch.int32, device="cuda")
    exp_mo[exp_out] = torch.arange(n_out, dtype=torch.int32, device="cuda")
    assert torch.equal(b["map_out"], exp_mo)


def test_we_prepare_pool_distribution(mv_device):
    """Pool draws are the alias method: word i with probability prob-mass of a known table."""
    import numpy as np
    from multiverso_b200 import _native as N
    V, K = 64, 5
    wts = np.arange(1, V + 1, dtype=np.float64)
    prob = np.empty(V, dtype=np.float32); alias = np.empty(V, dtype=np.int32)
    assert N.cuda_lib().mvb_build_alias_table(wts.ctypes.data, V, prob.ctypes.data, alias.ctypes.data) == 0
    toks = torch.arange(200000, dtype=torch.int32, device="cuda") % V     # n_in = 64 -> 320 draws only
    b = _prep(toks, V, K, torch.from_numpy(prob).cuda(), torch.from_numpy(alias).cuda(), V, V)
    assert b["counts"][2].item() == K * V
    # many seeds -> empirical distribution
    hist = torch.zeros(V, dtype=torch.float64)
    for seed in range(200):
        bb = _prep(toks, V, K, torch.from_numpy(prob).cuda(), torch.from_numpy(alias).cuda(), V, V, seed=seed)
        hist += torch.bincount(bb["neg_pool"][:K * V].long().cpu(), minlength=V).double()
    emp = hist / hist.sum()
    exp = torch.from_numpy(wts / wts.sum())
    assert (emp - exp).abs().max().item() < 0.004


@pytest.mark.parametrize("lsu", [False, True])
@pytest.mark.parametrize("rows,cols,k", [(20000, 300, 7001), (5000, 64, 5000), (3000, 512, 33), (1000, 300, 1)])
def test_rows_pull_push_bulk(mv_device, rows, cols, k, lsu):
    """lsu=False: bulk-copy-engine kernels (max_ctas > 0); lsu=True: register-path kernels (max_ctas < 0)."""
    import multiverso_b200 as mv
    from multiverso_b200 import _native as N
    t = mv.MatrixTable(rows, cols, "float32", min_value=-1.0, max_value=1.0, seed=5)
    full0 = t.get().view(rows, cols).clone()
    g = torch.Generator().manual_seed(rows)
    ids = torch.randperm(rows, generator=g)[:k].sort().values.to(torch.int32).cuda()
    cap = k + 100
    ids_buf = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
    ids_buf[:k] = ids
    n_dev = torch.tensor([k], dtype=torch.int32, device="cuda")
    cache = torch.full((cap, cols), 7.0, device="cuda")
    old = torch.full((cap, cols), 7.0, device="cuda")
    lib, st = N.cuda_lib(), N.stream_ptr()
    lib.mvb_rows_pull_bulk(t._rowmap, 4, ids_buf, n_dev, cap, cache, old, cols, -1 if lsu else 5, st)
    torch.cuda.synchronize()
    assert torch.equal(cache[:k], full0[ids.long()]) and torch.equal(old[:k], full0[ids.long()])
    assert bool((cache[k:] == 7.0).all()) and bool((old[k:] == 7.0).all())       # the device count bounds the copy
    # "train": change most rows, leave every 5th untouched
    delta = torch.randn(k, cols, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    delta[::5] = 0
    cache[:k] += delta
    lib.mvb_rows_push_delta_bulk(t._rowmap, ids_buf, n_dev, cap, cache, old, cols, 0.5, -2 if lsu else 3, st)
    torch.cuda.synchronize()
    exp = full0.clone()
    exp[ids.long()] += (cache[:k] - old[:k]) * 0.5
    got = t.get().view(rows, cols)
    assert torch.allclose(got, exp, rtol=0, atol=1e-6)
    untouched = torch.ones(rows, dtype=torch.bool, device="cuda")
    untouched[ids.long()] = False
    assert torch.equal(got[untouched], full0[untouched])
    # host-count variant (n_ptr = NULL)
    cache2 = torch.zeros(k, cols, device="cuda")
    lib.mvb_rows_pull_bulk(t._rowmap, 4, ids, None, k, cache2, None, cols, 0, st)
    torch.cuda.synchronize()
    assert torch.equal(cache2, got[ids.long()])
