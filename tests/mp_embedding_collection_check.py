"""An embedding-bag collection over MatrixTables sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_embedding_collection_check.py

Two sgd tables, one of them shared by two features. Every rank's forward reads rows from the owners' shards through
peer pointers and must equal, bitwise, the same collection over local single-shard copies of the tables. Then every
rank pushes its own gradient (one-sided red.add into the owners, no collective); after a barrier each table must
equal W0 - lr * (sum of every rank's gradient, coalesced over the table's features).
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection

results = {}
SHAPES = [(5003, 128), (777, 64)]
FEATS = [["item", "history"], ["user"]]


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def rank_batch(r, B, n):
    g = torch.Generator(device="cuda").manual_seed(100 + r)
    nrows = [SHAPES[0][0], SHAPES[0][0], SHAPES[1][0]]
    ids = torch.cat([torch.randint(0, v, (B * n,), device="cuda", generator=g) for v in nrows])
    ids[::3] = 11                                          # a hot row shared by every rank and feature
    lengths = torch.full((3, B), n, device="cuda")
    dout = torch.randn(B, 128 + 128 + 64, device="cuda", generator=g)
    return ids, lengths, dout


def main():
    mv.init()
    S, me = mv.size(), mv.rank()
    B, n, lr = 512, 20, 0.05
    tables = [mv.MatrixTable(V, d, "float32", updater="sgd", min_value=-1.0, max_value=1.0, seed=7 + i)
              for i, (V, d) in enumerate(SHAPES)]
    mv.barrier()
    W0 = [t.get().view(V, d).clone() for t, (V, d) in zip(tables, SHAPES)]
    ids, lengths, dout = rank_batch(me, B, n)
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, f, push_scale=lr) for t, f in zip(tables, FEATS)])
    local = PSEmbeddingCollection([EmbeddingBagConfig(w, f, push_scale=None) for w, f in zip(W0, FEATS)])
    with torch.no_grad():
        out, ref = ebc(ids, lengths), local(ids, lengths)
    torch.cuda.synchronize()
    check("forward_equals_local", torch.equal(out, ref), str((out - ref).abs().max().item()))
    mv.barrier()
    ebc(ids, lengths).backward(dout)
    torch.cuda.synchronize()
    mv.barrier()
    G = [torch.zeros(V, d, dtype=torch.float64, device="cuda") for V, d in SHAPES]
    bag = torch.arange(B * n, device="cuda") // n
    for r in range(S):
        i, _, d = rank_batch(r, B, n)
        G[0].index_add_(0, i[:B * n], d.double()[bag, :128])
        G[0].index_add_(0, i[B * n:2 * B * n], d.double()[bag, 128:256])
        G[1].index_add_(0, i[2 * B * n:], d.double()[bag, 256:])
    for k, (t, (V, d)) in enumerate(zip(tables, SHAPES)):
        got = t.get().view(V, d).double()
        err = (got - (W0[k].double() - lr * G[k])).abs().max().item()
        check(f"async_sgd_pushes_table{k}", err < 1e-4, str(err))
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
