"""Sampled softmax over a MatrixTable sharded across GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_sampled_softmax_check.py

Every rank draws the same candidates for a step. Every rank's forward reads rows from the owners' shards through peer
pointers and must equal, bitwise, the same op over a local single-shard copy of the table. Then every rank pushes its
own gradient (one-sided red.add into the owners, no collective); after a barrier the table must equal
W0 - lr * (sum of every rank's row gradient).
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
from multiverso_b200.ops import PSSampledSoftmax
from multiverso_b200.ops.sampled_softmax import draw_reference

results = {}
V, D, B, S, LR = 20011, 128, 512, 1024, 0.05


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def rank_batch(r):
    g = torch.Generator(device="cuda").manual_seed(100 + r)
    x = torch.randn(B, D, device="cuda", generator=g)
    y = torch.randint(0, V, (B,), device="cuda", generator=g)
    y[::4] = 3                                              # a hot row shared by every rank
    return x, y


def local_table(W):
    """A one-shard table over a local copy, with the sgd updater and no pushes."""
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = V, D, 1, V
    rm.shard_ptrs[0] = W.data_ptr()
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=V, num_col=D, updater=N.UPD_SGD,
                                 is_sparse=False, rt=types.SimpleNamespace(device=W.device))


def main():
    mv.init()
    size, me = mv.size(), mv.rank()
    t = mv.MatrixTable(V, D, "float32", updater="sgd", min_value=-0.1, max_value=0.1, seed=7)
    mv.barrier()
    W0 = t.get().view(V, D).clone()
    ssm = PSSampledSoftmax(t, num_sampled=S, sampler="log_uniform", push_scale=LR, seed=5)
    local = PSSampledSoftmax(local_table(W0), num_sampled=S, sampler="log_uniform", push_scale=None, seed=5)
    cand = ssm.draw(0)
    # the host replay depends on (seed, step) alone: equal to it on every rank means equal across ranks
    check("same_draws_on_every_rank", (cand.cpu().numpy() == draw_reference(ssm._prob, ssm._alias, 5, 0, S)).all())
    x, y = rank_batch(me)
    xr = x.clone().requires_grad_()
    loss = ssm(xr, y)
    with torch.no_grad():
        ref = local(x, y)
    torch.cuda.synchronize()
    check("forward_equals_local", torch.equal(loss.detach(), ref), str((loss.detach() - ref).abs().max().item()))
    mv.barrier()
    loss.mean().backward()
    torch.cuda.synchronize()
    mv.barrier()
    G = torch.zeros(V, D, dtype=torch.float64, device="cuda")
    for r in range(size):
        xr_, yr = rank_batch(r)
        P = W0.double().requires_grad_()
        logsq = torch.log(S * (torch.log((torch.arange(V, device="cuda", dtype=torch.float64) + 2) /
                                         (torch.arange(V, device="cuda", dtype=torch.float64) + 1)) /
                               torch.log(torch.tensor(V + 1.0, dtype=torch.float64))))
        x64 = xr_.double()
        tt = (x64 * P[yr]).sum(1) - logsq[yr]
        s = (x64 @ P[cand].t() - logsq[cand][None, :]).masked_fill(cand[None, :] == yr[:, None], float("-inf"))
        (torch.logsumexp(torch.cat([tt[:, None], s], 1), 1) - tt).mean().backward()
        G += P.grad
    got = t.get().view(V, D).double()
    err = (got - (W0.double() - LR * G)).abs().max().item()
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
