#!/usr/bin/env python
"""Fused embedding bags (emb_bag.cu) against the unfused table path and a local torch EmbeddingBag,
device-timed with CUDA events after warm-up.

Tables: 10M x 128 fp32 (5.1 GB, far larger than L2) and the WordEmbedding shape 1M x 300, sgd updater.
Batches: 16,384 bags of 32 lookups (fixed), or of 1..63 lookups (variable, mean 32); ids uniform or Zipf(1.05)
(the hot rows are the low ids). Arms per workload:

  fused_fwd          mv.ops.embedding_bag (input checks included)
  fused_fwd_bwd      PSEmbedding(table, lr): forward + backward, the coalesced gradient pushed with red.add
  unfused_fwd        table.get_rows(ids) + F.embedding_bag over the gathered rows
  unfused_fwd_bwd    the same + autograd (an L x dim gradient) + table.add_rows of every lookup
  torch_fwd(_bwd)    nn.EmbeddingBag(sparse=True) on a local copy of the weight (+ SGD step): the non-PS bound

Reported: ms per call and gathered bytes per second (lookups x dim x 4 / time). Every line carries the card's
name and power limit. Prints one JSON line per workload; ``--out FILE`` also writes them there.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

import multiverso_b200 as mv
from multiverso_b200.ops import PSEmbedding, embedding_bag

BAGS, MEAN_LEN = 16384, 32


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def batch(V, lengths, dist, g):
    if lengths == "fixed":
        lens = torch.full((BAGS,), MEAN_LEN, device="cuda")
    else:
        lens = torch.randint(1, 2 * MEAN_LEN, (BAGS,), device="cuda", generator=g)
    offsets = torch.cumsum(lens, 0) - lens
    L = int(lens.sum())
    if dist == "uniform":
        ids = torch.randint(0, V, (L,), device="cuda", generator=g)
    else:
        p = torch.arange(1, V + 1, device="cuda", dtype=torch.float64).pow_(-1.05)
        ids = torch.multinomial(p.float(), L, replacement=True, generator=g)
    return ids, offsets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tables", default="10000000x128,1000000x300")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/embedding_bag.py measures the GPU kernels: no CUDA device")
    mv.init()
    card = gpu_info()
    lines = []
    g = torch.Generator(device="cuda").manual_seed(0)
    lr = 1e-3
    for spec in a.tables.split(","):
        V, D = (int(x) for x in spec.split("x"))
        t = mv.MatrixTable(V, D, "float32", updater="sgd", min_value=-0.1, max_value=0.1)
        ref = torch.nn.EmbeddingBag(V, D, mode="sum", sparse=True, device="cuda")
        with torch.no_grad():
            ref.weight.copy_(t.shard.view(V, D))
        sgd = torch.optim.SGD(ref.parameters(), lr=lr)
        layer = PSEmbedding(t, push_scale=lr)
        for lengths in ("fixed", "variable"):
            for dist in ("uniform", "zipf"):
                ids, offsets = batch(V, lengths, dist, g)
                L = ids.numel()
                dout = torch.randn(BAGS, D, device="cuda", generator=g)
                pos = torch.arange(L, device="cuda")

                def unfused(bwd):
                    rows = t.get_rows(ids)
                    if not bwd:
                        return F.embedding_bag(pos, rows, offsets, mode="sum")
                    rows.requires_grad_()
                    F.embedding_bag(pos, rows, offsets, mode="sum").backward(dout)
                    t.add_rows(ids, rows.grad * lr)

                def torch_ref(bwd):
                    y = ref(ids, offsets)
                    if bwd:
                        sgd.zero_grad(set_to_none=True)
                        y.backward(dout)
                        sgd.step()

                arms = {
                    "fused_fwd": lambda: embedding_bag(t, ids, offsets),
                    "fused_fwd_bwd": lambda: layer(ids, offsets).backward(dout),
                    "unfused_fwd": lambda: unfused(False),
                    "unfused_fwd_bwd": lambda: unfused(True),
                    "torch_fwd": lambda: torch_ref(False),
                    "torch_fwd_bwd": lambda: torch_ref(True),
                }
                row = {"gpu": card, "table": [V, D], "bags": BAGS, "lengths": lengths, "ids": dist, "lookups": L,
                       "unique_ids": int(torch.unique(ids).numel())}
                for name, fn in arms.items():
                    ms = timed(fn, a.iters)
                    row[f"{name}_ms"] = round(ms, 4)
                    row[f"{name}_gathered_GBps"] = round(L * D * 4 / ms / 1e6, 1)
                row["fwd_speedup_vs_unfused"] = round(row["unfused_fwd_ms"] / row["fused_fwd_ms"], 2)
                row["fwd_bwd_speedup_vs_unfused"] = round(row["unfused_fwd_bwd_ms"] / row["fused_fwd_bwd_ms"], 2)
                line = json.dumps(row)
                print(line, flush=True)
                lines.append(line)
        del ref, sgd, layer
        t.free()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    mv.shutdown()


if __name__ == "__main__":
    main()
