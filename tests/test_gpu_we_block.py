"""Device-side WordEmbedding block protocol (csrc/cuda/we_block.cu) against plain PyTorch references:
PrepareData (bitmap-unique + prefix sum + negative pool), row pull and delta push."""
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


def _pull_push(rowmap, full0, read_full, ids, cols, ctas):
    """Pull ids through a device count, push (trained - pulled) / 2 back, pull again with a host count."""
    from multiverso_b200 import _native as N
    k = ids.numel()
    cap = k + 100
    ids_buf = torch.full((cap,), -1, dtype=torch.int32, device="cuda")
    ids_buf[:k] = ids
    n_dev = torch.tensor([k], dtype=torch.int32, device="cuda")
    cache = torch.full((cap, cols), 7.0, device="cuda")
    old = torch.full((cap, cols), 7.0, device="cuda")
    lib, st = N.cuda_lib(), N.stream_ptr()
    lib.mvb_rows_pull(rowmap, 4, ids_buf, n_dev, cap, cache, old, cols, ctas, st)
    torch.cuda.synchronize()
    assert torch.equal(cache[:k], full0[ids.long()]) and torch.equal(old[:k], full0[ids.long()])
    assert bool((cache[k:] == 7.0).all()) and bool((old[k:] == 7.0).all())       # the device count bounds the copy
    # "train": change most rows, leave every 5th untouched
    delta = torch.randn(k, cols, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    delta[::5] = 0
    cache[:k] += delta
    lib.mvb_rows_push_delta(rowmap, ids_buf, n_dev, cap, cache, old, cols, 0.5, ctas, st)
    torch.cuda.synchronize()
    exp = full0.clone()
    exp[ids.long()] += (cache[:k] - old[:k]) * 0.5
    got = read_full()
    assert torch.allclose(got, exp, rtol=0, atol=1e-6)
    untouched = torch.ones(full0.shape[0], dtype=torch.bool, device="cuda")
    untouched[ids.long()] = False
    assert torch.equal(got[untouched], full0[untouched])
    # host-count variant (n_ptr = NULL)
    cache2 = torch.zeros(k, cols, device="cuda")
    lib.mvb_rows_pull(rowmap, 4, ids, None, k, cache2, None, cols, ctas, st)
    torch.cuda.synchronize()
    assert torch.equal(cache2, got[ids.long()])


@pytest.mark.parametrize("ctas", [1, 2])
@pytest.mark.parametrize("rows,cols,k", [(20000, 300, 7001), (5000, 64, 5000), (3000, 512, 33), (1000, 300, 1)])
def test_rows_pull_push(mv_device, rows, cols, k, ctas):
    """Row pull and delta push at 1 and 2 CTAs per SM (the pipelined and the blocking grid)."""
    import multiverso_b200 as mv
    from multiverso_b200 import _native as N
    t = mv.MatrixTable(rows, cols, "float32", min_value=-1.0, max_value=1.0, seed=5)
    full0 = t.get().view(rows, cols).clone()
    g = torch.Generator().manual_seed(rows)
    ids = torch.randperm(rows, generator=g)[:k].sort().values.to(torch.int32).cuda()
    _pull_push(t._rowmap, full0, lambda: t.get().view(rows, cols), ids, cols, ctas)
    with pytest.raises(N.NativeError):           # the grid is a whole number of CTAs per SM
        N.cuda_lib().mvb_rows_pull(t._rowmap, 4, ids, None, k, full0, None, cols, 0, N.stream_ptr())


def _get_add_rows(op, rm, full0, read_full, ids, cols):
    """One of the int64-id row kernels (Get, stateless Add, fused AddDeltaParameter) on the rows ids."""
    from multiverso_b200 import _native as N
    lib, st, k = N.cuda_lib(), N.stream_ptr(), ids.numel()
    ids = ids.long()
    g = torch.Generator(device="cuda").manual_seed(11)
    exp = full0.clone()
    if op == "get_rows":
        out = torch.full((k, cols), 7.0, device="cuda")
        lib.mvb_get_rows(N.F32, rm, ids, k, out, cols, st)
        torch.cuda.synchronize()
        assert torch.equal(out, full0[ids])
    elif op == "add_rows_red":
        vals = torch.randn(k, cols, device="cuda", generator=g)
        lib.mvb_add_rows_red(N.F32, rm, ids, k, vals, cols, -1.0, st)
        exp[ids] -= vals
    else:
        old = torch.randn(k, cols, device="cuda", generator=g)
        cur = old + torch.randn(k, cols, device="cuda", generator=g)
        cur[::5] = old[::5]                                                # unchanged rows push nothing
        lib.mvb_add_rows_delta(rm, ids, k, cur, old, cols, 0.5, st)
        exp[ids] += (cur - old) * 0.5
    torch.cuda.synchronize()
    assert torch.allclose(read_full(), exp, rtol=0, atol=1e-6)


def test_rows_pull_push_three_servers(mv_device):
    """Owner arithmetic of every row kernel: three servers of 6000, 6000 and 8000 rows (the last takes the
    remainder), laid out out of order in one local buffer with sentinel gaps between them, so a row read from or
    added to the wrong server, or past its end, changes a value. Each kernel runs on a fresh copy of the layout:
    row pull / delta push (int32 ids, device count), then mvb_get_rows, mvb_add_rows_red and mvb_add_rows_delta
    (int64 ids)."""
    from multiverso_b200 import _native as N
    rows, cols, rps, gap = 20000, 300, 6000, 16
    lens = [rps, rps, rows - 2 * rps]
    starts = [lens[2] + gap, lens[2] + lens[0] + 2 * gap, 0]          # server 2 first, then 0, then 1
    pick = torch.randperm(rows, generator=torch.Generator().manual_seed(7))[:5000]
    edges = torch.tensor([0, rps - 1, rps, 2 * rps - 1, 2 * rps, rows - 1])
    ids = torch.unique(torch.cat([pick, edges])).to(torch.int32).cuda()      # every owner, both ends of each
    for op in ("pull_push", "get_rows", "add_rows_red", "add_rows_delta"):
        buf = torch.full((rows + 3 * gap, cols), 7.0, device="cuda")
        shards = [buf[s0:s0 + n] for s0, n in zip(starts, lens)]
        g = torch.Generator(device="cuda").manual_seed(3)
        for sh in shards:
            sh.copy_(torch.rand(sh.shape, device="cuda", generator=g) * 2 - 1)
        gaps = torch.ones(buf.shape[0], dtype=torch.bool, device="cuda")
        for s0, n in zip(starts, lens):
            gaps[s0:s0 + n] = False
        rm = N.RowMap()
        rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = rows, cols, 3, rps
        for s, sh in enumerate(shards):
            rm.shard_ptrs[s] = sh.data_ptr()
        full0 = torch.cat(shards)
        if op == "pull_push":
            _pull_push(rm, full0, lambda: torch.cat(shards), ids, cols, 2)
        else:
            _get_add_rows(op, rm, full0, lambda: torch.cat(shards), ids, cols)
        assert bool((buf[gaps] == 7.0).all()), op
