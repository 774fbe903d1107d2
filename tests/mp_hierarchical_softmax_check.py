"""Hierarchical softmax over a MatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_hierarchical_softmax_check.py

Every rank's forward reads the path rows from the owners' shards through peer pointers and must equal, bitwise, the
same op over a local single-shard copy of the table (loss and dL/dhidden). Then every rank pushes its own node
gradient (one-sided red.add into the owners, no collective); after a barrier the table must equal
W0 - lr * (sum of every rank's node gradient).
"""
import json
import os
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import multiverso_b200 as mv
from multiverso_b200 import _native as N
from multiverso_b200.ops import PSHierarchicalSoftmax, hierarchical_softmax_reference

results = {}
V, D, B, LR = 20011, 128, 512, 0.05
COUNTS = 1.0 / np.arange(1, V + 1) ** 1.05


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def rank_batch(r):
    g = torch.Generator(device="cuda").manual_seed(100 + r)
    x = torch.randn(B, D, device="cuda", generator=g)
    y = torch.randint(0, V, (B,), device="cuda", generator=g)
    y[::4] = 3                                              # a hot path shared by every rank
    return x, y


def local_table(W):
    """A one-shard table over a local copy, with the sgd updater and no pushes."""
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = V - 1, D, 1, V - 1
    rm.shard_ptrs[0] = W.data_ptr()
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=V - 1, num_col=D, updater=N.UPD_SGD,
                                 is_sparse=False, rt=types.SimpleNamespace(device=W.device))


def main():
    mv.init()
    size, me = mv.size(), mv.rank()
    t = mv.MatrixTable(V - 1, D, "float32", updater="sgd", min_value=-0.1, max_value=0.1, seed=7)
    mv.barrier()
    W0 = t.get().view(V - 1, D).clone()
    hsm = PSHierarchicalSoftmax(t, COUNTS, push_scale=LR)
    local = PSHierarchicalSoftmax(local_table(W0), COUNTS, push_scale=None)
    x, y = rank_batch(me)
    xr, xl = x.clone().requires_grad_(), x.clone().requires_grad_()
    loss = hsm(xr, y)
    ref = local(xl, y)
    ref.mean().backward()
    torch.cuda.synchronize()
    check("forward_equals_local", torch.equal(loss.detach(), ref.detach()))
    mv.barrier()
    loss.mean().backward()
    torch.cuda.synchronize()
    check("dhidden_equals_local", torch.equal(xr.grad, xl.grad))
    mv.barrier()
    G = torch.zeros(V - 1, D, dtype=torch.float64)
    for r in range(size):
        xr_, yr = rank_batch(r)
        P = W0.double().cpu().requires_grad_()
        hierarchical_softmax_reference(P, xr_, yr, COUNTS).mean().backward()
        G += P.grad
    got = t.get().view(V - 1, D).double().cpu()
    err = (got - (W0.double().cpu() - LR * G)).abs().max().item()
    check("async_sgd_pushes", err < 1e-4, str(err))
    mv.barrier()
    mv.shutdown()


if __name__ == "__main__":
    t0 = time.time()
    try:
        main()
    except Exception:
        import traceback
        traceback.print_exc()
        results["exception"] = False
    rank = int(os.environ.get("RANK", "0"))
    ok = all(results.values()) and len(results) > 0
    print(f"[rank {rank}] {'PASS' if ok else 'FAIL'} {json.dumps(results)} ({time.time() - t0:.1f}s)", flush=True)
    sys.exit(0 if ok else 1)
