"""The ftrl updater on tables sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_ftrl_check.py MODE

``bsp``: two BSP whole-table Adds in which every worker adds its own delta with its own AddOption (the owners apply
the workers in worker order, one step each), then two collective row Adds that repeat rows across workers (applied
worker by worker, in list order). Each rank checks its shard, z and n against the fp64 model of
tests/test_ftrl_cpu.py. A fifth of every delta is 0, and those elements must keep their bits.

``async``: rank 0 alone pushes two whole-table deltas one-sided (``mvb_push_dense_stateful``), which is exact; then
every rank pushes two (data, z and n are Hogwild across concurrent pushers, so they are only checked to be finite and
n to have grown); then row Adds through the row mailboxes in which worker w names only rows
r % N == w, so no row's steps depend on the order in which sources arrive.
"""
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np
import torch

import multiverso_b200 as mv
from test_ftrl_cpu import FtrlModel, _sparse_delta, fopt

results = {}
ROWS, COLS = 1001, 36


def check(name, fn):
    try:
        fn()
        results[name] = True
    except AssertionError as e:
        results[name] = False
        print(f"[rank {mv.rank()}] FAIL {name} {str(e)[:500]}", flush=True)


def _local(t):
    lo, hi = t.row_lo[t.sid], t.row_hi[t.sid]
    rows = hi - lo
    z = t.state[0][:rows * COLS].cpu().numpy()
    n = t.state[1][:rows * COLS].cpu().numpy()
    return lo, hi, t.shard.view(rows, COLS).cpu().numpy(), z, n


def check_shard(t, model, what):
    lo, hi, got, z, n = _local(t)
    rows = np.arange(lo, hi)
    check(f"{what}_values", lambda: model.check_values(np.pad(got, ((lo, ROWS - hi), (0, 0))), what, rows))
    full = lambda x: np.pad(x.reshape(hi - lo, -1), ((lo, ROWS - hi), (0, 0)))
    check(f"{what}_state", lambda: model.check_state(full(z), full(n), what, rows))


def main(mode):
    mv.init(["-sync=true"] if mode == "bsp" else ["-sync=false"])
    S, me = mv.size(), mv.rank()
    t = mv.MatrixTable(ROWS, COLS, "float32", updater="ftrl", min_value=-1.0, max_value=1.0, seed=5)
    mv.barrier()
    model = FtrlModel(t.get().view(ROWS, COLS).cpu().numpy(), COLS, "float32")
    mv.barrier()
    if mode == "bsp":
        for k in range(2):
            deltas = [_sparse_delta(np.random.default_rng(1000 * k + w), (ROWS, COLS), "float32") for w in range(S)]
            opts = [fopt(mv, k * S + w, w) for w in range(S)]
            t.add(torch.from_numpy(deltas[me]).cuda(), opts[me])
            for w in range(S):
                model.add(deltas[w], opts[w])
        for k in range(2):
            batches = []
            for w in range(S):
                rng = np.random.default_rng(3000 + 100 * k + w)
                ids = np.concatenate([[0, 0, 500], rng.choice(ROWS, 200, replace=False)]).astype(np.int64)
                batches.append((ids, _sparse_delta(rng, (ids.size, COLS), "float32"), fopt(mv, 2 + k * S + w, w)))
            ids, vals, opt = batches[me]
            t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(vals).cuda(), opt)
            for ids_w, vals_w, opt_w in batches:
                model.add_rows(ids_w, vals_w, opt_w)
        torch.cuda.synchronize()
        mv.barrier()
        check_shard(t, model, "bsp")
    else:
        for k in range(2):
            d = _sparse_delta(np.random.default_rng(1000 * k), (ROWS, COLS), "float32")
            if me == 0:
                t.add(torch.from_numpy(d).cuda(), fopt(mv, k, 0))
            model.add(d, fopt(mv, k, 0))
        torch.cuda.synchronize()
        mv.barrier()
        check_shard(t, model, "async_one_pusher")
        mv.barrier()
        for k in range(2):
            d = _sparse_delta(np.random.default_rng(2000 * k + me), (ROWS, COLS), "float32")
            t.add(torch.from_numpy(d).cuda(), fopt(mv, k, me))
        torch.cuda.synchronize()
        mv.barrier()
        lo, hi, got, z, n = _local(t)
        n_one = model.n[lo:hi].reshape(-1)

        def pushed():
            assert np.isfinite(got).all() and np.isfinite(z).all() and np.isfinite(n).all()
            assert (n > n_one).mean() > 0.5
        check("async_all_pushers", pushed)
        mv.barrier()
        base = FtrlModel(got, COLS, "float32")
        base.z[:], base.n[:] = z.reshape(-1, COLS), n.reshape(-1, COLS)
        for k in range(2):
            for w in range(S):
                rng = np.random.default_rng(5000 + 100 * k + w)
                own = np.arange(w, ROWS, S)
                ids = np.sort(rng.choice(own, min(150, own.size), replace=False)).astype(np.int64)
                vals = _sparse_delta(rng, (ids.size, COLS), "float32")
                if w == me:
                    t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(vals).cuda(), fopt(mv, 3 + k, w))
                local = ids[(ids >= lo) & (ids < hi)]
                base.add_rows(local - lo, vals[(ids >= lo) & (ids < hi)], fopt(mv, 3 + k, w))
        torch.cuda.synchronize()
        mv.barrier()
        _, _, got, z, n = _local(t)
        check("async_row_adds_values", lambda: base.check_values(got, "async row adds"))
        check("async_row_adds_state", lambda: base.check_state(z, n, "async row adds"))
    mv.barrier()
    mv.shutdown()


if __name__ == "__main__":
    t0 = time.time()
    try:
        main(sys.argv[1] if len(sys.argv) > 1 else "bsp")
    except Exception:
        import traceback
        traceback.print_exc()
        results["exception"] = False
    rank = int(os.environ.get("RANK", "0"))
    ok = all(results.values()) and len(results) > 0
    print(f"[rank {rank}] {'PASS' if ok else 'FAIL'} {json.dumps(results)} ({time.time() - t0:.1f}s)", flush=True)
    sys.exit(0 if ok else 1)
