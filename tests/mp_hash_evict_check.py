"""Eviction of a HashMatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_hash_evict_check.py

Every rank trains on an overlapping key set with its own clock (rank r at clock 10 + r), so the shared keys carry
stamps from several ranks and keep the largest. Each rank then lists keys to erase that peers own, and all ranks
evict together with one age limit. Afterwards the listed keys and the keys idle on every rank are gone on every
server, the stamps of the survivors are the largest clock of the ranks that touched them, ``num_keys`` is the
number of survivors, and every rank's ``get`` of the whole key pool is bitwise equal.
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


def rank_keys(r, pool, n):
    g = torch.Generator(device="cuda").manual_seed(200 + r)
    return pool[torch.randint(0, pool.numel(), (n,), device="cuda", generator=g)]


def main():
    mv.init()
    S, me = mv.size(), mv.rank()
    rt = Runtime.get()
    dim, n = 32, 4096
    pool = key_pool(6000)
    t = mv.HashMatrixTable(8000, dim, updater="adagrad", min_value=-1.0, max_value=1.0, seed=7, track_access=True)
    # an old generation, seen by rank 0 only at clock 0, then every rank's own keys at its own clock
    old = pool[5000:]
    if me == 0:
        t.clock = 0
        t.lookup(old)
    torch.cuda.synchronize()
    mv.barrier()
    t.clock = 10 + me
    ids = rank_keys(me, pool[:5000], n)
    PSEmbedding(t, push_scale=0.05)(ids, torch.arange(0, n, 4, device="cuda")).backward(
        torch.randn(n // 4, dim, device="cuda"))
    torch.cuda.synchronize()
    mv.barrier()
    per_rank = [torch.unique(rank_keys(r, pool[:5000], n)) for r in range(S)]
    union = torch.unique(torch.cat(per_rank))
    want_ls = torch.full((union.numel(),), -1, dtype=torch.int64, device="cuda")
    for r, k in enumerate(per_rank):
        pos = torch.searchsorted(union, k)
        want_ls[pos] = torch.maximum(want_ls[pos], torch.full_like(pos, 10 + r))
    check("stamps_are_max_over_ranks", torch.equal(t.last_seen(union), want_ls))
    # rank r erases keys owned by rank (r + 1) % S
    owned_by_next = union[torch.remainder(union, S) == (me + 1) % S]
    erase = owned_by_next[:50]
    all_erased = torch.unique(torch.cat([union[torch.remainder(union, S) == (r + 1) % S][:50] for r in range(S)]))
    removed = t.evict(older_than=5, keys=erase)
    survivors = union[~torch.isin(union, all_erased)]
    check("removed_count", removed == old.numel() + all_erased.numel(),
          f"{removed} vs {old.numel() + all_erased.numel()}")
    check("num_keys", t.num_keys() == survivors.numel(), f"{t.num_keys()} vs {survivors.numel()}")
    check("erased_and_idle_gone", bool((t.last_seen(torch.cat([all_erased, old])) == -1).all()))
    check("survivor_stamps_kept", torch.equal(t.last_seen(survivors), want_ls[torch.searchsorted(union, survivors)]))
    got = t.get(pool)
    check("erased_read_zero", bool((t.get(all_erased) == 0).all()))
    digests = rt.all_gather_object(hashlib.sha256(got.cpu().numpy().tobytes()).hexdigest())
    check("get_equal_on_every_rank", len(set(digests)) == 1, str(digests))
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
