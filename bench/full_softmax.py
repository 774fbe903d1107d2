#!/usr/bin/env python
"""Fused full softmax (mv.ops.full_softmax, topk_cos.cu dot-product form) against the unfused path, device-timed
with CUDA events.

Tables: 1M x 128 and 10M x 128 fp32 MatrixTables (an output layer over a large vocabulary / item set). For B in
{1, 256, 8192} queries and k in {0, 10}, labels given:

  fused     mv.ops.full_softmax: one pass over the table, the [B, N] logits never written
  unfused   gemm_nt over row blocks of the table into a score buffer of at most 2 GB, torch.logsumexp and
            torch.topk per block, merged across blocks (the same maths, the logits through HBM)

Reported per workload: time, the least time of the two bounds (tf32 495 TFLOP/s for 2 B N d flops, HBM 3.35 TB/s
for the table bytes; H100 SXM data sheet) and the fused share of it, naming the bound, and the largest
|lse_fused - lse_unfused|. The GPU name and power limit are read in the same run. Prints one JSON line; ``--out
FILE`` also writes it there.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import full_softmax, gemm_nt

HBM_BPS, TF32_FLOPS = 3.35e12, 495e12
SCORE_BYTES = 2 << 30


def timed(fn, iters, warmup=1):
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


def unfused(W, x, y, k, scores):
    """lse, loss, top-k over row blocks of W [N, d] with a score buffer ``scores`` (flat fp32)."""
    B, N = x.shape[0], W.shape[0]
    blk = max(4, min(N, scores.numel() // max(B, 1)) // 4 * 4)
    lse = torch.full((B,), float("-inf"), device=x.device)
    best_s = torch.empty(B, 0, device=x.device)
    best_i = torch.empty(B, 0, dtype=torch.int64, device=x.device)
    for lo in range(0, N, blk):
        hi = min(N, lo + blk)
        z = gemm_nt(x, W[lo:hi], scores[:B * (hi - lo)].view(B, hi - lo))
        lse = torch.logaddexp(lse, torch.logsumexp(z, 1))
        if k:
            s, i = z.topk(min(k, hi - lo), dim=1)
            best_s, o = torch.cat([best_s, s], 1).topk(k, dim=1)
            best_i = torch.cat([best_i, i + lo], 1).gather(1, o)
    t = (x * W[y]).sum(1)
    return lse, lse - t, best_s, best_i


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", default="1000000,10000000")
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--bs", default="1,256,8192")
    ap.add_argument("--ks", default="0,10")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/full_softmax.py measures the GPU kernel: no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = True
    mv.init()
    d = a.dim
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"gpu": gpu_info(), "dim": d, "results": []}
    scores = torch.empty(SCORE_BYTES // 4, device="cuda")
    for N in [int(v) for v in a.rows.split(",")]:
        t = mv.MatrixTable(N, d, "float32", min_value=-0.1, max_value=0.1)
        W = t.shard.view(N, d)
        torch.cuda.synchronize()
        for B in [int(v) for v in a.bs.split(",")]:
            x = torch.randn(B, d, device="cuda", generator=g)
            y = torch.randint(0, N, (B,), device="cuda", generator=g)
            for k in [int(v) for v in a.ks.split(",")]:
                flops, tbytes = 2.0 * B * N * d, N * d * 4
                t_mma, t_mem = flops / TF32_FLOPS * 1e3, tbytes / HBM_BPS * 1e3
                est = max(t_mma, t_mem) + B * N * 8 / HBM_BPS * 1e3
                iters = max(3, min(50, int(300 / max(est, 0.01))))
                row = {"N": N, "B": B, "k": k}
                row["fused_ms"] = timed(lambda: full_softmax(t, x, y, k=k), iters)
                row["unfused_ms"] = timed(lambda: unfused(W, x, y, k, scores), max(2, iters // 2))
                row["bound"] = "tf32" if t_mma >= t_mem else "hbm"
                row["bound_ms"] = max(t_mma, t_mem)
                row["fused_share_of_bound"] = row["bound_ms"] / row["fused_ms"]
                row["unfused_share_of_bound"] = row["bound_ms"] / row["unfused_ms"]
                row["speedup"] = row["unfused_ms"] / row["fused_ms"]
                r = full_softmax(t, x, y, k=k)
                u = unfused(W, x, y, k, scores)
                row["max_abs_lse_diff"] = (r.lse - u[0]).abs().max().item()
                row["max_abs_loss_diff"] = (r.loss - u[1]).abs().max().item()
                if k:
                    row["topk_ids_equal_rows"] = int((r.ids == u[3]).all(1).sum())
                res["results"].append(row)
                print(json.dumps(row), flush=True)
            del x, y
        t.free()
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    mv.shutdown()


if __name__ == "__main__":
    main()
