"""Embedding bags over a MatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_embedding_check.py

Every rank looks up rows of the whole table: the forward reads them from the owners' shards through peer
pointers and must equal, bitwise, the same call over a local single-shard copy. Then every rank pushes its own
gradient into the sgd table with PSEmbedding (one-sided red.add into the owners, no collective); after a
barrier the table must equal W0 - lr * (sum of every rank's coalesced gradient).
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import PSEmbedding, embedding_bag

results = {}


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def rank_batch(r, V, B, n, dim):
    g = torch.Generator(device="cuda").manual_seed(100 + r)
    ids = torch.randint(0, V, (B * n,), device="cuda", generator=g)
    ids[::3] = 11                                          # a hot row shared by every rank
    offsets = torch.arange(0, B * n, n, device="cuda")
    dout = torch.randn(B, dim, device="cuda", generator=g)
    return ids, offsets, dout


def main():
    mv.init()
    S, me = mv.size(), mv.rank()
    V, dim, B, n, lr = 5003, 128, 512, 20, 0.05
    t = mv.MatrixTable(V, dim, "float32", updater="sgd", min_value=-1.0, max_value=1.0, seed=7)
    mv.barrier()
    W0 = t.get().view(V, dim).clone()
    ids, offsets, dout = rank_batch(me, V, B, n, dim)
    out = embedding_bag(t, ids, offsets)
    ref = embedding_bag(W0, ids, offsets)
    torch.cuda.synchronize()
    check("forward_equals_local", torch.equal(out, ref), str((out - ref).abs().max().item()))
    mv.barrier()
    PSEmbedding(t, push_scale=lr)(ids, offsets).backward(dout)
    torch.cuda.synchronize()
    mv.barrier()
    G = torch.zeros(V, dim, dtype=torch.float64, device="cuda")
    for r in range(S):
        i, o, d = rank_batch(r, V, B, n, dim)
        G.index_add_(0, i, d.double()[torch.arange(B * n, device="cuda") // n])
    exp = W0.double() - lr * G
    got = t.get().view(V, dim).double()
    err = (got - exp).abs().max().item()
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
