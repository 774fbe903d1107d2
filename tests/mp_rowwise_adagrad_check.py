"""The rowwise_adagrad updater on tables sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_rowwise_adagrad_check.py MODE

``bsp``: two BSP whole-table Adds in which every worker adds its own delta with its own AddOption; the owners apply
the workers in worker order. ``async``: every rank pushes two whole-table deltas one-sided (``mvb_push_dense_rowwise``)
and then two row Adds through the row mailboxes. A step depends only on its own worker's delta and accumulator, never
on the row's value, so the async result is the model's whatever the interleaving, up to the order of the roundings,
which the bound of tests/test_rowwise_adagrad_cpu.py covers. Each rank checks its shard and every worker's accumulators
of its rows against the fp64 model.
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
from test_rowwise_adagrad_cpu import RowwiseModel
from test_table_numerics import _delta, _kopt

results = {}
ROWS, COLS = 1001, 36


def check(name, fn):
    try:
        fn()
        results[name] = True
    except AssertionError as e:
        results[name] = False
        print(f"[rank {mv.rank()}] FAIL {name} {str(e)[:500]}", flush=True)


def check_shard(t, model, what):
    lo, hi = t.row_lo[t.sid], t.row_hi[t.sid]
    rows = hi - lo
    got = t.shard.view(rows, COLS).cpu().numpy()
    sub = RowwiseModel(model.data[lo:hi], COLS, "float32", workers=t.W)
    sub.data, sub.mag, sub.nupd = model.data[lo:hi], model.mag[lo:hi], model.nupd[lo:hi]
    sub.h, sub.hn = model.h[:, lo:hi], model.hn[:, lo:hi]

    def values():
        sub.check_values(got, "float32", what)

    def states():
        for w in range(t.W):
            sub.check_state(t.state[0][w * t.state_stride:w * t.state_stride + rows].cpu().numpy(), w, "float32", what)
    check(f"{what}_values", values)
    check(f"{what}_state", states)


def main(mode):
    mv.init(["-sync=true"] if mode == "bsp" else ["-sync=false"])
    S, me = mv.size(), mv.rank()
    t = mv.MatrixTable(ROWS, COLS, "float32", updater="rowwise_adagrad", min_value=-1.0, max_value=1.0, seed=5)
    mv.barrier()
    model = RowwiseModel(t.get().view(ROWS, COLS).cpu().numpy(), COLS, "float32", workers=S)
    mv.barrier()
    for k in range(2):
        deltas = [_delta(np.random.default_rng(1000 * k + w), (ROWS, COLS), "float32") for w in range(S)]
        opts = [_kopt(k * S + w, w)[0] for w in range(S)]
        t.add(torch.from_numpy(deltas[me]).cuda(), opts[me])
        for w in range(S):
            model.add(deltas[w], opts[w])
    torch.cuda.synchronize()
    mv.barrier()
    check_shard(t, model, f"{mode}_whole_table")
    if mode == "async":
        mv.barrier()
        for k in range(2):
            batches = []
            for w in range(S):
                rng = np.random.default_rng(5000 + 100 * k + w)
                ids = np.sort(rng.choice(ROWS, 300, replace=False)).astype(np.int64)
                batches.append((ids, _delta(rng, (ids.size, COLS), "float32"), _kopt(3 + k * S + w, w)[0]))
            ids, vals, opt = batches[me]
            t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(vals).cuda(), opt)
            for ids_w, vals_w, opt_w in batches:
                model.add_rows(ids_w, vals_w, opt_w)
        torch.cuda.synchronize()
        mv.barrier()
        check_shard(t, model, "async_row_adds")
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
