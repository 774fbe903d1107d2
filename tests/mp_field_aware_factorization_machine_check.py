"""A field-aware factorization machine over a MatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_field_aware_factorization_machine_check.py

Every rank's forward reads its rows from the owners' shards through peer pointers and must equal, bitwise, the same
op over a local single-shard copy of the table. Then every rank pushes its own row gradient (one-sided red.add into
the owners, no collective); after a barrier the table must equal W0 - lr * (sum of every rank's row gradient) within
the red.add rounding.
"""
import json
import os
import sys
import time
import types

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200 import _native as N
from multiverso_b200.ops import PSFieldAwareFactorizationMachine, field_aware_factorization_machine_reference

results = {}
V, F, K, B, BAG, LR = 20011, 12, 4, 512, 12, 0.05
C = F * K + 4


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def rank_batch(r):
    g = torch.Generator(device="cuda").manual_seed(100 + r)
    ids = torch.randint(0, V, (B, BAG), device="cuda", generator=g)
    ids[::4, 0] = 3                                         # a hot row shared by every rank
    x = torch.rand(B, BAG, device="cuda", generator=g)
    fields = torch.arange(BAG, device="cuda").expand(B, BAG) % F
    return ids, fields, x


def local_table(W):
    """A one-shard table over a local copy, with the sgd updater and no pushes."""
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = V, C, 1, V
    rm.shard_ptrs[0] = W.data_ptr()
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=V, num_col=C, updater=N.UPD_SGD,
                                 is_sparse=False, rt=types.SimpleNamespace(device=W.device))


def main():
    mv.init()
    size, me = mv.size(), mv.rank()
    t = mv.MatrixTable(V, C, "float32", updater="sgd", min_value=-0.1, max_value=0.1, seed=7)
    mv.barrier()
    W0 = t.get().view(V, C).clone()
    fm = PSFieldAwareFactorizationMachine(t, F, K, push_scale=LR)
    local = PSFieldAwareFactorizationMachine(local_table(W0), F, K, push_scale=None)
    ids, fields, x = rank_batch(me)
    y = fm(ids, fields, values=x)
    ref = local(ids, fields, values=x)
    torch.cuda.synchronize()
    check("forward_equals_local", torch.equal(y.detach(), ref.detach()))
    mv.barrier()
    y.mean().backward()
    torch.cuda.synchronize()
    mv.barrier()
    G = torch.zeros(V, C, dtype=torch.float64)
    touches = torch.zeros(V, dtype=torch.float64)
    for r in range(size):
        ids_r, f_r, x_r = rank_batch(r)
        P = W0.double().cpu().requires_grad_()
        field_aware_factorization_machine_reference(P, ids_r.cpu(), f_r.cpu(), values=x_r.cpu(), num_fields=F,
                                                    num_factors=K).mean().backward()
        G += P.grad
        touches += torch.bincount(ids_r.reshape(-1).cpu(), minlength=V).double()
    got = t.get().view(V, C).double().cpu()
    exp = W0.double().cpu() - LR * G
    # each rank's red.add rounds once, on top of the fp32 rounding of its own gradient (|G| << 1 here)
    tol = 2 ** -23 * (size + 1) * (exp.abs() + LR * G.abs()) + 1e-6 * (touches[:, None] > 0)
    err = ((got - exp).abs() - tol).max().item()
    check("async_sgd_pushes", err <= 0, str(err))
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
