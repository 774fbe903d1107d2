#!/usr/bin/env python
"""Training step of the exact full softmax: mv.ops.PSFullSoftmax (fused backward, full_softmax_bwd.cu) against
PSLinear + F.cross_entropy, device-timed with CUDA events.

Workloads: 1M x 128 at B in {1, 256, 1024, 8192}, and 100k x 512 at B = 1024, fp32 sgd MatrixTables. Per workload:

  fused     ms per forward + backward + Add of PSFullSoftmax (hidden requires grad, push_scale set)
  unfused   ms per step of PSLinear + cross_entropy on the same inputs; skipped with a note where its [B, N] logits
            and their gradient would not fit next to the table
  bwd       ms of the fused backward kernels alone (mvb_full_softmax_bwd with dq and dw)

  fwd / add the forward alone and the dense staged Add alone, the parts of the fused step besides the backward

and shares of the tf32 bound (495 TFLOP/s, H100 SXM data sheet): ``useful`` counts 10 B N d flops (the forward, the
two recomputes of the logits and the two products); ``performed`` counts what the kernels execute, with the logits
recomputed once per 128-column output chunk and each product 128 columns wide per chunk:
2 B N d + 2 * chunks * (2 B N d + 2 B N 128). One repetition of each arm after two warm-up calls. The GPU name and
power limit are read in the same run. Prints one JSON line; ``--out FILE`` also writes it.
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
from multiverso_b200.ops.full_softmax import full_softmax, full_softmax_bwd
from multiverso_b200.ops.topk import padded_queries

TF32_FLOPS = 495e12


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.manual_seed(0)
    mv.init()
    dev = torch.device("cuda", 0)
    rows = []
    free = torch.cuda.mem_get_info()[0]
    for N, d, batches in ((1_000_000, 128, (1, 256, 1024, 8192)), (100_000, 512, (1024,))):
        t = mv.MatrixTable(N, d, "float32", updater="sgd", min_value=-0.1, max_value=0.1)
        fsm = mv.ops.PSFullSoftmax(t, push_scale=1e-3)
        lin = mv.ops.PSLinear(t, push_scale=1e-3)
        for B in batches:
            x = torch.randn(B, d, device=dev, requires_grad=True)
            y = torch.randint(0, N, (B,), device=dev)
            row = {"N": N, "d": d, "B": B}

            def fused():
                fsm(x, y).mean().backward()
            row["fused_ms"] = round(timed(fused), 3)
            chunks = (d + 127) // 128
            bwd_flops = 2 * chunks * (2.0 * B * N * d + 2.0 * B * N * 128)
            row["fused_tf32_share_useful"] = round(10.0 * B * N * d / (row["fused_ms"] * 1e-3) / TF32_FLOPS, 4)
            row["fused_tf32_share_performed"] = round((2.0 * B * N * d + bwd_flops) / (row["fused_ms"] * 1e-3)
                                                      / TF32_FLOPS, 4)

            def fwd():
                with torch.no_grad():
                    fsm(x, y)
            row["fwd_ms"] = round(timed(fwd), 3)

            def add():
                t.staging().zero_()
                t.add_async(None, None, staged=True)
            row["add_ms"] = round(timed(add), 3)
            # the unfused arm holds logits, their softmax gradient and the pulled table
            need = 3 * B * N * 4 + N * d * 8
            if need > 0.8 * free:
                row["unfused_ms"] = None
                row["unfused_note"] = f"skipped: needs ~{need / 2**30:.0f} GiB for logits and gradient"
            else:
                def unfused():
                    F.cross_entropy(lin(x), y, reduction="none").mean().backward()
                row["unfused_ms"] = round(timed(unfused), 3)
                row["speedup"] = round(row["unfused_ms"] / row["fused_ms"], 2)
            r = full_softmax(t, x.detach(), y)
            q = padded_queries(x.detach())
            g = torch.full((B,), 1.0 / B, device=dev)
            dq = torch.empty(B, d, device=dev)
            dw = torch.empty(N, d, device=dev)

            def bwd():
                full_softmax_bwd(fsm._rm, q, d, y, r.lse, g, dq, dw, 1e-3)
            row["bwd_ms"] = round(timed(bwd), 3)
            row["bwd_tf32_share_useful"] = round(8.0 * B * N * d / (row["bwd_ms"] * 1e-3) / TF32_FLOPS, 4)
            row["bwd_tf32_share_performed"] = round(bwd_flops / (row["bwd_ms"] * 1e-3) / TF32_FLOPS, 4)
            del dw
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
        del t, fsm, lin
        torch.cuda.empty_cache()
    out = {"bench": "full_softmax_train", "gpu": gpu_info(), "rows": rows}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    mv.shutdown()


if __name__ == "__main__":
    main()
