"""A HashMatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_hash_embedding_check.py

Every rank inserts an overlapping key set at the same time (PSEmbedding in training mode: the keys go to their owners'
indexes through system-scope CAS on peer memory). Afterwards every key has exactly one row, ``num_keys`` is the size of
the union, every rank's ``get`` of all keys is bitwise equal, and the async sgd pushes of all ranks have landed as
init - lr * (sum of every rank's coalesced gradient).
"""
import hashlib
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import PSEmbedding
from multiverso_b200.runtime import Runtime

results = {}


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def key_pool(n):
    """n int64 keys spread over the whole range."""
    x = torch.arange(1, n + 1, dtype=torch.int64) * 0x9E3779B97F4A7C15 % (1 << 62)
    return (x * ((torch.arange(n) % 2) * 2 - 1)).cuda()


def rank_batch(r, pool, B, n, dim):
    g = torch.Generator(device="cuda").manual_seed(100 + r)
    ids = pool[torch.randint(0, pool.numel() // 2 + 400 * r, (B * n,), device="cuda", generator=g)]
    ids[::3] = pool[11]                                      # a hot key every rank inserts at once
    offsets = torch.arange(0, B * n, n, device="cuda")
    dout = torch.randn(B, dim, device="cuda", generator=g)
    return ids, offsets, dout


def main():
    mv.init()
    S, me = mv.size(), mv.rank()
    dim, B, n, lr = 64, 512, 16, 0.05
    pool = key_pool(6000)
    t = mv.HashMatrixTable(8000, dim, updater="sgd", min_value=-1.0, max_value=1.0, seed=7)
    mv.barrier()
    ids, offsets, dout = rank_batch(me, pool, B, n, dim)
    PSEmbedding(t, push_scale=lr)(ids, offsets).backward(dout)
    torch.cuda.synchronize()
    mv.barrier()
    batches = [rank_batch(r, pool, B, n, dim) for r in range(S)]
    union = torch.unique(torch.cat([b[0] for b in batches]))
    check("num_keys_is_union", t.num_keys() == union.numel(), f"{t.num_keys()} vs {union.numel()}")
    rows = t.lookup(union, insert=False)
    owner = torch.remainder(union, S)
    check("one_row_per_key", torch.unique(rows).numel() == union.numel() and
          bool(((rows >= owner * t.slots) & (rows < (owner + 1) * t.slots)).all()))
    got = t.get(union)
    digests = Runtime.get().all_gather_object(hashlib.sha256(got.cpu().numpy().tobytes()).hexdigest())
    check("get_equal_on_every_rank", len(set(digests)) == 1, str(digests))
    # expected: the initial row of every key (a fresh table, same seed, one rank inserting) minus lr * sum of grads
    G = torch.zeros(union.numel(), dim, dtype=torch.float64, device="cuda")
    for i, o, d in batches:
        G.index_add_(0, torch.searchsorted(union, i), d.double()[torch.arange(B * n, device="cuda") // n])
    fresh = mv.HashMatrixTable(8000, dim, updater="sgd", min_value=-1.0, max_value=1.0, seed=7)
    mv.barrier()
    if me == 0:
        fresh.lookup(union)
    torch.cuda.synchronize()
    mv.barrier()
    exp = fresh.get(union).double() - lr * G
    err = (got.double() - exp).abs().max().item()
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
