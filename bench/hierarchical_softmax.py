#!/usr/bin/env python
"""Hierarchical softmax over a MatrixTable (hier_softmax.cu) against the same maths in torch over the gathered rows,
and against PSSampledSoftmax for context, device-timed with CUDA events after warm-up (ms per forward + backward).

Tables (N - 1 inner-node rows) for N = 1M classes at d = 128 and 512 and N = 10M at d = 128, each with the sgd and
the adagrad updater; B = 8192 labels drawn Zipf(1.05), and the Huffman tree built from the same Zipf weights. Arms:

  fused      PSHierarchicalSoftmax(table, counts, push_scale=lr): forward + loss.mean().backward(), input checks
             included
  unfused    get_rows of the unique path nodes, a [B, L_max, d] gather, bmm, logsigmoid + autograd, and one
             coalesced add_rows
  sampled    PSSampledSoftmax(table, 8192, log_uniform) on the same table and batch

Each arm runs --iters steps per repeat; --repeats repeats alternate the arms, and the median, min and max over the
repeats are reported. Also reported: the mean path length, the unique nodes per step, and the logical bytes a fused
step must move (the path rows read once per step, hidden read, the unique node rows pushed) with the rate they imply
at the median fused time: a logical rate, not a measured HBM bandwidth. Every line carries the card's name and
power limit, read in the same run. Prints one JSON line per workload; ``--out FILE`` also writes them there.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.nn.functional as F

import multiverso_b200 as mv
from multiverso_b200.ops import PSHierarchicalSoftmax, PSSampledSoftmax


def timed(fn, iters):
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


def unfused_step(t, hsm, x, y, lr):
    """The op's maths in torch over get_rows of the unique path nodes."""
    ln = hsm.lens[y].to(torch.int64)
    lmax = int(ln.max())
    P = hsm.points[y, :lmax].to(torch.int64)
    s = 1.0 - 2.0 * hsm.codes[y, :lmax].to(torch.float32)
    mask = torch.arange(lmax, device=y.device)[None, :] < ln[:, None]
    P = P.masked_fill(~mask, 0)
    uniq, inv = torch.unique(P, return_inverse=True)
    rows = t.get_rows(uniq).requires_grad_()
    xx = x.detach().requires_grad_()
    z = torch.bmm(rows[inv], xx[:, :, None]).squeeze(2)                  # [B, L_max]
    loss = -(F.logsigmoid(s * z) * mask).sum(1)
    loss.mean().backward()
    t.add_rows(uniq, rows.grad * lr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="1000000x128,1000000x512,10000000x128")
    ap.add_argument("--updaters", default="sgd,adagrad")
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/hierarchical_softmax.py measures the GPU kernels: no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = True
    mv.init()
    card = gpu_info()
    lines = []
    g = torch.Generator(device="cuda").manual_seed(0)
    lr, B = 1e-3, a.batch
    for spec in a.workloads.split(","):
        N, D = (int(v) for v in spec.split("x"))
        w = 1.0 / np.arange(1, N + 1, dtype=np.float64) ** 1.05
        for upd in a.updaters.split(","):
            t = mv.MatrixTable(N - 1, D, "float32", updater=upd, min_value=-0.1, max_value=0.1)
            hsm = PSHierarchicalSoftmax(t, w, push_scale=lr)
            ssm = PSSampledSoftmax(t, num_sampled=8192, sampler="log_uniform", push_scale=lr)
            x = torch.randn(B, D, device="cuda", generator=g, requires_grad=True)
            y = torch.multinomial(torch.from_numpy(w / w.sum()).float().cuda(), B, replacement=True, generator=g)
            ln = hsm.lens[y].to(torch.int64)
            L = int(ln.sum())
            bag = torch.repeat_interleave(torch.arange(B, device="cuda"), ln)
            pos = torch.arange(L, device="cuda") - (torch.cumsum(ln, 0) - ln)[bag]
            U = int(torch.unique(hsm.points[y[bag], pos]).numel())
            arms = {"fused": lambda: hsm(x, y).mean().backward(),
                    "unfused": lambda: unfused_step(t, hsm, x, y, lr),
                    "sampled": lambda: ssm(x, y).mean().backward()}
            for fn in arms.values():                                      # warm-up of every shape
                for _ in range(3):
                    fn()
            times = {k: [] for k in arms}
            for _ in range(a.repeats):
                for k, fn in arms.items():
                    times[k].append(timed(fn, a.iters))
            row = {"gpu": card, "classes": N, "dim": D, "updater": upd, "batch": B,
                   "mean_path_length": round(L / B, 3), "max_path_length": hsm.depth, "unique_nodes": U}
            for k, v in times.items():
                row[f"{k}_ms"] = round(statistics.median(v), 4)
                row[f"{k}_ms_min_max"] = [round(min(v), 4), round(max(v), 4)]
            read, pushed = (L + B) * D * 4, U * D * 4
            row["logical_bytes_read"], row["logical_bytes_pushed"] = read, pushed
            row["logical_GBps_at_fused"] = round((read + pushed) / (row["fused_ms"] * 1e-3) / 1e9, 1)
            row["speedup_vs_unfused"] = round(row["unfused_ms"] / row["fused_ms"], 2)
            line = json.dumps(row)
            print(line, flush=True)
            lines.append(line)
            del hsm, ssm
            x.grad = None
            t.free()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    mv.shutdown()


if __name__ == "__main__":
    main()
