"""Fused cosine top-k over a MatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_topk_check.py

Every rank searches the whole table: the main kernel streams W tiles from the owners' shards with TMA (peer
HBM), the finish kernel re-reads the candidate rows through the row map with plain peer loads. Each rank's
result must equal, bitwise, the same search over a local single-shard copy of the table, and agree with an
fp64 top-k. Cases: shards that are not tile multiples, a row pitch larger than the compared width with
garbage in the padding, and row limits that end inside the first and inside the last shard.
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import topk_cosine

results = {}


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def fp64_agrees(W, Q, k, rows, s, i, tol=1e-5):
    dim = Q.shape[1]
    Wd = W[:rows, :dim].double()
    wn = Wd.norm(dim=1)
    C = (Q.double() / Q.double().norm(dim=1, keepdim=True)) @ (Wd / torch.where(wn > 0, wn, torch.ones_like(wn))[:, None]).T
    if (s.double() - C.gather(1, i)).abs().max().item() >= tol:
        return False
    kth = C.topk(k, dim=1).values[:, -1:]
    must = C > kth + tol                                  # every row clearly above the k-th must be returned
    got = torch.zeros_like(must).scatter_(1, i, True)
    return bool((got | ~must).all()) and bool((C.gather(1, i) >= kth - tol).all())


def main():
    mv.init()
    S = mv.size()
    g = torch.Generator(device="cuda").manual_seed(11)
    for name, V, pitch, dim, k, rows in (("tiles", 5003, 300, 300, 16, None),
                                         ("padded_pitch", 3001, 320, 300, 40, None),
                                         ("rows_in_first_shard", 5003, 300, 300, 10, 5003 // S - 33),
                                         ("rows_in_last_shard", 5003, 300, 300, 10, 5003 - 5003 // (2 * S))):
        t = mv.MatrixTable(V, pitch, "float32", min_value=-1.0, max_value=1.0, seed=7)
        if pitch > dim and t.my_len:
            t.shard.view(-1, pitch)[:, dim:] = 1e6         # padding columns never count
        mv.barrier()
        W = t.get().view(V, pitch).clone()
        Q = torch.randn(150, dim, device="cuda", generator=g)
        s, i = topk_cosine(t, Q, k, rows=rows)
        s1, i1 = topk_cosine(W, Q, k, rows=rows)           # one local shard
        torch.cuda.synchronize()
        check(f"topk_peer_{name}_equals_local", torch.equal(s, s1) and torch.equal(i, i1),
              str((s - s1).abs().max().item()))
        check(f"topk_peer_{name}_fp64", fp64_agrees(W, Q, k, V if rows is None else rows, s, i))
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
