#!/usr/bin/env python
"""Sampled softmax over a MatrixTable (sampled_softmax.cu) against the same maths in torch over the gathered rows, and
against a full softmax, device-timed with CUDA events after warm-up (ms per forward + backward step).

Tables 1M x 128 and 10M x 128 fp32, each with the sgd and the adagrad updater; B = 8192 examples, S in {1024, 8192}
candidates from the log-uniform sampler; labels drawn Zipf(1.05) (the hot rows are the low ids). Arms:

  fused      PSSampledSoftmax(table, S, push_scale=lr): forward + loss.mean().backward(), input checks included
  unfused    the same draws, get_rows of the unique [labels; candidates], the logits as a TF32 matmul, masked
             cross_entropy + autograd, and one coalesced add_rows
  full       PSLinear + F.cross_entropy over every row (1M-row table at B = 1024 only: a [B, 1M] logits matrix,
             a whole-table Get in the backward and a dense whole-table push)

Also reported: the GEMM FLOPs of a step from the shapes (3 products of 2 B S_pad d) and their share of the H100 SXM
data-sheet dense TF32 rate (494.7 TFLOP/s) at the fused time. Every line carries the card's name and power limit.
Prints one JSON line per workload; ``--out FILE`` also writes them there.
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
from multiverso_b200.ops import PSLinear, PSSampledSoftmax

TF32_PEAK = 494.7e12          # H100 SXM5 data sheet, dense TF32 tensor-core FLOP/s


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


def zipf_labels(V, B, g):
    p = torch.arange(1, V + 1, device="cuda", dtype=torch.float64).pow_(-1.05)
    return torch.multinomial(p.float(), B, replacement=True, generator=g)


def unfused_step(t, ssm, x, y, lr):
    """The op's maths in torch over get_rows of the unique rows."""
    cand = ssm.draw(ssm.steps)
    ssm.steps += 1
    B = y.numel()
    uniq, inv = torch.unique(torch.cat([y, cand]), return_inverse=True)
    rows = t.get_rows(uniq).requires_grad_()
    logq = ssm._logq
    log_s = float(ssm._log_s)
    w_y, w_c = rows[inv[:B]], rows[inv[B:]]
    xx = x.detach().requires_grad_()
    tl = (xx * w_y).sum(1) - (log_s + logq[y])
    s = (xx @ w_c.t() - (log_s + logq[cand])[None, :]).masked_fill(cand[None, :] == y[:, None], float("-inf"))
    z = torch.cat([tl[:, None], s], 1)
    F.cross_entropy(z, torch.zeros(B, dtype=torch.int64, device="cuda")).backward()
    t.add_rows(uniq, rows.grad * lr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tables", default="1000000x128,10000000x128")
    ap.add_argument("--updaters", default="sgd,adagrad")
    ap.add_argument("--samples", default="1024,8192")
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/sampled_softmax.py measures the GPU kernels: no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = True
    mv.init()
    card = gpu_info()
    lines = []
    g = torch.Generator(device="cuda").manual_seed(0)
    lr, B = 1e-3, a.batch
    for spec in a.tables.split(","):
        V, D = (int(v) for v in spec.split("x"))
        for upd in a.updaters.split(","):
            t = mv.MatrixTable(V, D, "float32", updater=upd, min_value=-0.1, max_value=0.1)
            x = torch.randn(B, D, device="cuda", generator=g, requires_grad=True)
            y = zipf_labels(V, B, g)
            for S in (int(s) for s in a.samples.split(",")):
                ssm = PSSampledSoftmax(t, num_sampled=S, sampler="log_uniform", push_scale=lr)
                ref = PSSampledSoftmax(t, num_sampled=S, sampler="log_uniform", push_scale=lr)
                row = {"gpu": card, "table": [V, D], "updater": upd, "batch": B, "num_sampled": S,
                       "unique_rows": int(torch.unique(torch.cat([y, ssm.draw(0)])).numel())}
                row["fused_ms"] = round(timed(lambda: ssm(x, y).mean().backward(), a.iters), 4)
                row["unfused_ms"] = round(timed(lambda: unfused_step(t, ref, x, y, lr), a.iters), 4)
                s_pad = (S + 3) // 4 * 4
                flops = 3 * 2 * B * s_pad * D
                row["gemm_gflop"] = round(flops / 1e9, 2)
                row["gemm_share_of_tf32_peak"] = round(flops / (row["fused_ms"] * 1e-3) / TF32_PEAK, 4)
                row["speedup_vs_unfused"] = round(row["unfused_ms"] / row["fused_ms"], 2)
                line = json.dumps(row)
                print(line, flush=True)
                lines.append(line)
                del ssm, ref
            x.grad = None
            t.free()
    # full softmax over every row: PSLinear + cross_entropy, 1M-row table at B = 1024
    V, D, Bf = 1000000, 128, 1024
    if f"{V}x{D}" in a.tables.split(","):
        t = mv.MatrixTable(V, D, "float32", updater="sgd", min_value=-0.1, max_value=0.1)
        lin = PSLinear(t, push_scale=lr)
        x = torch.randn(Bf, D, device="cuda", generator=g, requires_grad=True)
        y = zipf_labels(V, Bf, g)
        ssm = PSSampledSoftmax(t, num_sampled=8192, sampler="log_uniform", push_scale=lr)
        row = {"gpu": card, "table": [V, D], "updater": "sgd", "batch": Bf, "num_sampled": 8192,
               "full_ms": round(timed(lambda: F.cross_entropy(lin(x), y).backward(), a.iters), 4),
               "fused_ms": round(timed(lambda: ssm(x, y).mean().backward(), a.iters), 4)}
        row["speedup_vs_full"] = round(row["full_ms"] / row["fused_ms"], 2)
        line = json.dumps(row)
        print(line, flush=True)
        lines.append(line)
        t.free()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    mv.shutdown()


if __name__ == "__main__":
    main()
