"""Count-based admission of a HashMatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_hash_admission_check.py

Every rank looks up (inserting) its own keys and a shared set, each key once per rank in one call, all ranks at
once, so the shared keys are counted by several ranks into sketches that peers own. With admit_after = N every
shared key reaches N only from the counts of all ranks together: after a barrier it holds a slot on its owner, while
the keys seen by one rank only do not. A later call of every rank trains the shared keys, and afterwards every
rank's ``get`` of the whole pool is bitwise equal and the zero row is zero.
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
    x = torch.arange(1, n + 1, dtype=torch.int64) * 0x9E3779B97F4A7C15 % (1 << 62)
    return (x * ((torch.arange(n) % 2) * 2 - 1)).cuda()


def main():
    mv.init()
    S, me = mv.size(), mv.rank()
    rt = Runtime.get()
    dim = 16
    pool = key_pool(1000 + 200 * S)
    shared, own = pool[:1000], pool[1000 + 200 * me:1000 + 200 * (me + 1)]
    t = mv.HashMatrixTable(1 << 16, dim, updater="sgd", min_value=-1.0, max_value=1.0, admit_after=S)
    t.lookup(torch.cat([shared, own]))             # one count per rank: below S for every key, before the others
    torch.cuda.synchronize()
    mv.barrier()
    # a shared key is admitted by the call that brings its count to S; own keys (count 1) only for S = 1
    t.lookup(shared)                                # held keys are not counted; the rest may still be admitted
    torch.cuda.synchronize()
    mv.barrier()
    held = t.lookup(pool, insert=False) != t.zero_row
    check("shared_admitted", bool(held[:1000].all()))
    if S > 1:
        check("own_not_admitted", not bool(held[1000:].any()), str(int(held[1000:].sum())))
    check("num_keys", t.num_keys() == int(held.sum()), f"{t.num_keys()} vs {int(held.sum())}")
    ids = shared[torch.randint(0, 1000, (2048,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(me))]
    PSEmbedding(t, push_scale=0.05)(ids, torch.arange(0, 2048, 8, device="cuda")).backward(
        torch.randn(256, dim, device="cuda"))
    torch.cuda.synchronize()
    mv.barrier()
    got = t.get(pool)
    check("zero_row_zero", bool((t.get_rows(torch.tensor([t.zero_row], device="cuda")) == 0).all()))
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
