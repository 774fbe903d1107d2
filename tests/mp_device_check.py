"""Multi-GPU end-to-end checks, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_device_check.py

Mirrors the reference's multi-process scenarios (Test/test_array_table.cpp, test_matrix_table.cpp,
test_kv_table.cpp, test_allreduce.cpp) with their exact integer expectations, on the device
backend: fused BSP Add/Get (K1/K2), one-sided async push, row ops (K3/K4), KV (K5),
allreduce (K6), uneven iteration counts + FinishTrain, and a distributed WordEmbedding block.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv

results = {}


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def scenario_sync():
    mv.init(sync=True)
    W, r = mv.num_workers(), mv.rank()
    n = 1 << 20
    t = mv.ArrayTable(n, "float32")
    delta = torch.arange(n, dtype=torch.float32, device="cuda") % 1000 + 1
    ok = True
    for it in range(1, 6):
        t.add(delta)
        got = t.get()
        ok &= bool(torch.equal(got, delta * it * W))
    check("bsp_array_exact", ok)
    # momentum updater: every owner applies the W deltas sequentially in worker order
    tm = mv.ArrayTable(10007, "float32", updater="momentum_sgd")
    d = torch.full((10007,), 1.0, device="cuda") * (r + 1)
    opt = mv.AddOption(momentum=0.5)
    tm.add(d, opt)
    s, x = 0.0, 0.0
    for w in range(W):
        s = 0.5 * s + 0.5 * (w + 1)
        x -= s
    check("bsp_momentum_sequential", torch.allclose(tm.get(), torch.full((10007,), x, device="cuda")))
    # the AddOption travels with each worker's request: per-worker learning rates under AdaGrad (per-worker
    # history): worker w adds delta = lr_w twice -> owner moves by rho/sqrt(1) + rho/sqrt(2) for EVERY worker
    # only if it divides by the pushing worker's own learning rate
    to = mv.ArrayTable(70001, "float32", updater="adagrad")
    lr_w = 0.01 * (r + 1)
    for it in range(2):
        to.add(torch.full((70001,), lr_w, device="cuda"), mv.AddOption(learning_rate=lr_w, rho=0.1))
    exp_o = -W * (0.1 / 1.0 + 0.1 / (2 ** 0.5))
    check("bsp_per_worker_addoption", torch.allclose(to.get(), torch.full((70001,), exp_o, device="cuda"), rtol=1e-4),
          f"{to.get()[:2].tolist()} vs {exp_o}")
    # matrix scenario (test_matrix_table.cpp): whole + rows 0,1,3,7
    rows, cols = 1000, 64
    m = mv.MatrixTable(rows, cols, "float32")
    base = (torch.arange(rows * cols, dtype=torch.float32, device="cuda") % 97 + 1).view(rows, cols)
    ids = torch.tensor([0, 1, 3, 7, 999], device="cuda")
    ok = True
    for count in range(1, 4):
        m.add(base)
        mv.barrier()
        m.add_rows(ids, base[ids])
        mv.barrier()
        exp = base * count * W
        exp[ids] *= 2
        ok &= bool(torch.equal(m.get().view(rows, cols), exp))
        ok &= bool(torch.equal(m.get_rows(ids), exp[ids]))
        mv.barrier()
    check("bsp_matrix_rows_exact", ok)
    # uneven iteration counts (test_array_table.cpp:30) -> FinishTrain on shutdown
    tu = mv.ArrayTable(4096, "float32")
    one = torch.ones(4096, device="cuda")
    iters = 3 + r
    for it in range(iters):
        tu.add(one)
        tu.get()
    mv.shutdown(finalize_net=False)
    check("bsp_uneven_finish_train", True)


def scenario_async():
    mv.init(sync=False)
    W, r = mv.num_workers(), mv.rank()
    n = 300007
    t = mv.ArrayTable(n, "float32")            # default updater -> one-sided red.add push
    delta = torch.arange(n, dtype=torch.float32, device="cuda") % 13 + 1
    for it in range(4):
        t.add(delta)
    mv.barrier()
    check("async_push_red_exact", torch.equal(t.get(), delta * 4 * W))
    ts = mv.ArrayTable(n, "float32", updater="sgd")
    ts.add(delta)
    mv.barrier()
    check("async_sgd_sign", torch.equal(ts.get(), -delta * W))
    # stateful updater in ASYNC mode: one-sided, no lockstep -- ranks add a different number of
    # times; per-worker AdaGrad history makes the result exact: each add of delta=lr moves by
    # rho / sqrt(k) at the k-th add of that worker
    ta = mv.ArrayTable(100003, "float32", updater="adagrad")
    my_adds = 1 + r
    for k in range(my_adds):
        ta.add(torch.full((100003,), 0.01, device="cuda"), mv.AddOption(learning_rate=0.01, rho=0.1))
    mv.barrier()
    exp_a = -sum(0.1 / (k ** 0.5) for w in range(W) for k in range(1, 2 + w))
    check("async_stateful_one_sided", torch.allclose(ta.get(), torch.full((100003,), exp_a, device="cuda"), rtol=1e-4),
          f"{ta.get()[:3].tolist()} vs {exp_a}")
    # rows
    m = mv.MatrixTable(5000, 300, "float32")
    ids = torch.arange(r, 5000, 7, device="cuda")
    vals = torch.ones(ids.numel(), 300, device="cuda") * (r + 1)
    m.add_rows(ids, vals)
    mv.barrier()
    full = m.get().view(5000, 300)
    exp = torch.zeros(5000, 300, device="cuda")
    for w in range(W):
        exp[torch.arange(w, 5000, 7, device="cuda")] += (w + 1)
    check("async_rows_scatter_add", torch.equal(full, exp))
    check("rows_gather", torch.equal(m.get_rows(ids), exp[ids]))
    # stateful rows: owner-applied, exactly once per (worker,row)
    ma = mv.MatrixTable(512, 32, "float32", updater="adagrad")
    rid = torch.arange(0, 512, 3, device="cuda")
    ma.add_rows(rid, torch.ones(rid.numel(), 32, device="cuda") * 0.01, mv.AddOption(learning_rate=0.01, rho=0.1))
    mv.barrier()                       # row mailboxes: pushes are applied by their owners, at the latest here
    got = ma.get().view(512, 32)
    # each worker has its own G^2 history: g=1, G2=1 -> step = rho/sqrt(1+1e-6)
    check("stateful_rows_adagrad", torch.allclose(got[rid], torch.full((rid.numel(), 32), -0.1 * W, device="cuda"), atol=1e-4))
    # device-side mailboxes: workers are NOT in lockstep -- rank r issues r+1 row Adds (unsorted ids, rows of
    # every owner), per-worker learning rates travel with the push; per-worker AdaGrad history makes the
    # result exact: the k-th add of a worker moves its rows by rho / sqrt(k)
    mu = mv.MatrixTable(3001, 64, "float32", updater="adagrad")
    check("row_mailbox_enabled", (mu._mailbox is not None) == (W > 1))
    urid = torch.randperm(3001, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7))[:1500]
    for k in range(r + 1):
        lr_w = 0.01 * (r + 1)
        mu.add_rows(urid, torch.full((1500, 64), lr_w, device="cuda"), mv.AddOption(learning_rate=lr_w, rho=0.1))
    mv.barrier()
    exp_u = -sum(0.1 / (k ** 0.5) for w in range(W) for k in range(1, 2 + w))
    gu = mu.get().view(3001, 64)
    untouched = torch.ones(3001, dtype=torch.bool, device="cuda"); untouched[urid] = False
    check("stateful_rows_uneven_mailbox", torch.allclose(gu[urid], torch.full((1500, 64), exp_u, device="cuda"), rtol=1e-4)
          and bool((gu[untouched] == 0).all()), f"{gu[urid][0, :2].tolist()} vs {exp_u}")
    # momentum (shared state): one push per worker, applied sequentially by the owner -> order-independent only
    # for equal deltas: s = m s + (1-m) g applied W times to rows that start at 0
    mm = mv.MatrixTable(1000, 32, "float32", updater="momentum_sgd")
    mm.add_rows(torch.arange(0, 1000, 2, device="cuda"), torch.ones(500, 32, device="cuda"), mv.AddOption(momentum=0.5))
    mv.barrier()
    sm, dm = 0.0, 0.0
    for w in range(W):
        sm = 0.5 * sm + 0.5 * 1.0
        dm -= sm
    check("stateful_rows_momentum_mailbox", torch.allclose(mm.get().view(1000, 32)[::2], torch.full((500, 32), dm, device="cuda"), rtol=1e-5))
    # staleness instrumentation: everybody pulls, then the workers add one after the other -- worker r's Add is
    # applied after r Adds of other workers since its last Get, a second round sees W - 1 foreign Adds each
    mv.set_flag("staleness", True)
    ts_ = mv.ArrayTable(4096, "float32", updater="momentum_sgd")
    mv.set_flag("staleness", False)
    ts_.get()
    for turn in range(2 * W):
        mv.barrier()
        if turn % W == r:
            ts_.add(torch.ones(4096, device="cuda"), mv.AddOption(momentum=0.5))
            torch.cuda.synchronize()
    mv.barrier()
    hist = mv.Dashboard.staleness()[ts_.table_id]["hist"]
    exp_h = [0] * 64
    # (one histogram entry per (Add, shard): an Add updates all W shards)
    exp_h[r] += W                       # first round: r foreign adds since the Get
    exp_h[W - 1 + r] += W               # second round: no new Get -> foreign adds keep accumulating: (W-1) + r
    check("staleness_histogram", hist == exp_h, f"{hist[:2 * W + 1]} vs {exp_h[:2 * W + 1]}")
    # application-defined tables on the device extension point (LogReg's SparseTable / FTRLTable): keys of every
    # owner, server subtracts, whole-table Get returns the union of the keys anybody wrote
    from multiverso_b200.tables.custom import SparseDeviceTable
    spt = SparseDeviceTable(100003)
    skeys = torch.arange(r, 100003, 11, device="cuda")
    spt.add(skeys, torch.full((skeys.numel(),), float(r + 1), device="cuda"))
    torch.cuda.synchronize(); mv.barrier()
    exp_keys = torch.unique(torch.cat([torch.arange(w, 100003, 11) for w in range(W)]))
    dense = torch.zeros(100003)
    for w in range(W):
        dense[torch.arange(w, 100003, 11)] -= (w + 1)
    ka, va = spt.get()
    check("app_sparse_table", torch.equal(ka.cpu(), exp_keys) and torch.equal(va.cpu(), dense[exp_keys])
          and torch.equal(spt.get(skeys).cpu(), dense[skeys.cpu()]))
    mv.barrier()
    # KV
    kv = mv.KVTable("int64", "float32")
    keys = torch.arange(0, 1000, device="cuda")
    kv.add(keys, torch.ones(1000, device="cuda"))
    mv.barrier()
    check("kv_add_get", torch.equal(kv.get(keys), torch.full((1000,), float(W), device="cuda")))
    # allreduce (test_allreduce.cpp): sum of ones == size; plus large two-shot
    x = torch.ones(1, dtype=torch.int32, device="cuda")
    mv.aggregate(x)
    check("aggregate_int", int(x.item()) == mv.size())
    for n_el in (1000, 3_000_001):
        y = torch.full((n_el,), float(r + 1), device="cuda")
        mv.aggregate(y)
        check(f"aggregate_f32_{n_el}", torch.equal(y, torch.full((n_el,), W * (W + 1) / 2.0, device="cuda")))
    # latency path (one fused launch, double-buffered staging): back-to-back calls, changing sizes / dtypes,
    # interleaved with the staged large-message path
    ok_f = True
    for it in range(24):
        n_el = (1, 7, 1000, 4099, 262144)[it % 5]
        dt = (torch.float32, torch.int32, torch.float64)[it % 3]
        v = torch.full((n_el,), r + 1 + it, device="cuda").to(dt)
        mv.aggregate(v)
        ok_f = ok_f and bool((v == W * (W + 1) // 2 + W * it).all())
        if it % 8 == 7:
            big = torch.ones(600_000, device="cuda")
            mv.aggregate(big)
            ok_f = ok_f and bool((big == W).all())
    un = torch.arange(1001, device="cuda", dtype=torch.float32)[1:]      # 4-byte aligned only
    mv.aggregate(un)
    ok_f = ok_f and bool(torch.equal(un, W * torch.arange(1, 1001, device="cuda", dtype=torch.float32)))
    check("aggregate_fused_small", ok_f)
    # zero-copy aggregate on a tensor in symmetric memory, mixed with the staged path
    zs = mv.symm_tensor(2_000_003, "float32")
    ok_z = True
    for it in range(3):
        zs.fill_(float(r + 1 + it))
        mv.aggregate(zs)
        ok_z = ok_z and bool((zs == W * (W + 1) / 2.0 + W * it).all())
        big = torch.ones(700_001, device="cuda")
        mv.aggregate(big)
        ok_z = ok_z and bool((big == W).all())
    check("aggregate_symm_in_place", ok_z)
    z = torch.full((5_000_000,), float(r + 1), device="cuda")
    from multiverso_b200.parallel import aggregate as _agg
    _agg(z, algo="nvls")
    check("aggregate_nvls_or_fallback", torch.equal(z, torch.full((5_000_000,), W * (W + 1) / 2.0, device="cuda")))
    # fused Get+GEMM with the W tiles streamed from peer shards by TMA (wgmma)
    from multiverso_b200.ops import get_gemm
    wt = mv.MatrixTable(1000, 256, "float32", min_value=-1.0, max_value=1.0, seed=3)
    mv.barrier()
    Wfull = wt.get().view(1000, 256).clone()
    xg = torch.randn(300, 256, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    yg = get_gemm(wt, xg)
    torch.cuda.synchronize()
    ref = xg.double() @ Wfull.double().T
    check("get_gemm_peer_tma", (yg.double() - ref).abs().max().item() < 4e-3 * 16 * 4, str((yg.double() - ref).abs().max().item()))
    mv.barrier()
    # several x-groups over remote shards: the first pass stages each W tile in the local scratch
    # (TMA store), the later passes load from it -- ragged M, shard sizes that are not tile multiples
    wt2 = mv.MatrixTable(3001, 320, "float32", min_value=-1.0, max_value=1.0, seed=4)
    mv.barrier()
    W2 = wt2.get().view(3001, 320).clone()
    for Mrows in (700, 1500):
        x2 = torch.randn(Mrows, 320, device="cuda", generator=torch.Generator(device="cuda").manual_seed(6))
        y2 = get_gemm(wt2, x2)
        torch.cuda.synchronize()
        ref2 = x2.double() @ W2.double().T
        err2 = (y2.double() - ref2).abs().max().item()
        check(f"get_gemm_peer_scratch_M{Mrows}", err2 < 4e-3 * 18 * 4, str(err2))
    mv.barrier()
    # device-side block protocol across ranks: row pull from peer shards, one-sided delta push
    from multiverso_b200 import _native as N
    bt = mv.MatrixTable(40000, 300, "float32", min_value=-1.0, max_value=1.0, seed=11)
    mv.barrier()
    bfull = bt.get().view(40000, 300).clone()
    bids = torch.arange(r, 40000, 3, device="cuda", dtype=torch.int32)          # rows of every owner
    kk = bids.numel()
    ndev = torch.tensor([kk], dtype=torch.int32, device="cuda")
    cache = torch.zeros(kk + 7, 300, device="cuda"); old = torch.zeros(kk + 7, 300, device="cuda")
    lib, stp = N.cuda_lib(), N.stream_ptr()
    lib.mvb_rows_pull(bt._rowmap, 4, bids, ndev, kk + 7, cache, old, 300, 1, stp)
    torch.cuda.synchronize()
    check("rows_pull_peer", torch.equal(cache[:kk], bfull[bids.long()]) and torch.equal(old[:kk], bfull[bids.long()]))
    mv.barrier()
    cache[:kk] += float(r + 1)
    lib.mvb_rows_push_delta(bt._rowmap, bids, ndev, kk + 7, cache, old, 300, 0.5, 2, stp)
    torch.cuda.synchronize()
    mv.barrier()
    bexp = bfull.clone()
    for w in range(W):
        bexp[torch.arange(w, 40000, 3, device="cuda")] += 0.5 * (w + 1)
    check("rows_push_delta_peer", torch.allclose(bt.get().view(40000, 300), bexp, rtol=0, atol=1e-5))
    mv.barrier()
    # distributed WordEmbedding block (block mode)
    from multiverso_b200.models.wordembedding import WordEmbedding, WordEmbeddingOption, synthetic_zipf_corpus
    we = WordEmbedding(WordEmbeddingOption(embeding_size=300, init_learning_rate=0.01), 200000)
    toks = torch.from_numpy(synthetic_zipf_corpus(400000, 200000, 1000, seed=r)).cuda()
    losses = []
    for it in range(4):
        we.loss.zero_(); we.pairs.zero_()
        we.train_block(toks)
        torch.cuda.synchronize()
        losses.append(float(we.loss.item()) / max(int(we.pairs.item()), 1))
    mv.barrier()
    check("wordembedding_block_mode", losses[-1] < losses[0] and all(l == l for l in losses), str(losses))
    # pipelined block mode (-is_pipeline): block i+1 is prepared / pulled on a side stream while block i
    # trains; block i's deltas are pushed while block i+1 trains
    blocks = [torch.from_numpy(synthetic_zipf_corpus(200000, 200000, 1000, seed=10 * r + b)).cuda() for b in range(3)]
    pl = []
    for it in range(6):
        we.loss.zero_(); we.pairs.zero_()
        we.train_block(blocks[it % 3], next_tokens=blocks[(it + 1) % 3] if it < 5 else None)
        torch.cuda.synchronize()
        pl.append(float(we.loss.item()) / max(int(we.pairs.item()), 1))
    we.flush()
    torch.cuda.synchronize()
    mv.barrier()
    emb = we.embeddings()
    check("wordembedding_pipelined", pl[-1] < pl[0] and all(l == l for l in pl) and bool(torch.isfinite(emb).all()), str(pl))
    # direct mode: K7 trains in the row-sharded tables themselves over NVLink (bulk loads from / bulk reductions
    # into peer shards), no block cache
    os.environ["MVB_WE_MODE"] = "direct"
    wd = WordEmbedding(WordEmbeddingOption(embeding_size=300, init_learning_rate=0.01), 200000)
    os.environ.pop("MVB_WE_MODE")
    dl = []
    for it in range(5):
        wd.loss.zero_(); wd.pairs.zero_()
        wd.train_block(blocks[it % 3])
        torch.cuda.synchronize()
        dl.append(float(wd.loss.item()) / max(int(wd.pairs.item()), 1))
    mv.barrier()
    check("wordembedding_direct_mode", wd.mode == "direct" and dl[-1] < dl[0] and all(l == l for l in dl)
          and bool(torch.isfinite(wd.embeddings()).all()), str(dl))
    mv.shutdown()


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    t0 = time.time()
    try:
        if which in ("all", "sync"):
            scenario_sync()
        if which in ("all", "async"):
            scenario_async()
    except Exception as e:
        import traceback
        traceback.print_exc()
        results["exception"] = False
    rank = int(os.environ.get("RANK", "0"))
    ok = all(results.values()) and len(results) > 0
    print(f"[rank {rank}] {'PASS' if ok else 'FAIL'} {json.dumps(results)} ({time.time() - t0:.1f}s)", flush=True)
    os.makedirs("gpurun_out", exist_ok=True)
    with open(f"gpurun_out/mp_check_rank{rank}.json", "w") as f:
        json.dump(results, f)
    sys.exit(0 if ok else 1)
