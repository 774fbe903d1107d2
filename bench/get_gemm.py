#!/usr/bin/env python
"""Fused Get+GEMM (wgmma/TMA, K2-fused) vs the unfused path (P2P Get into HBM, then
cuBLAS TF32 matmul), device-timed, max over ranks.  Y[M x N] = X[M x K] @ W[N x K]^T, W = a
row-sharded MatrixTable (peer HBM when world > 1).  Writes gpurun_out/get_gemm_n<N>.json."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import get_gemm


def timed(fn, iters, world):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    mv.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = torch.tensor([e0.elapsed_time(e1) / iters], dtype=torch.float64, device="cuda")
    if world > 1:
        import torch.distributed as dist
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    mv.barrier()
    return float(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="4096x65536x512,1024x1000000x512,512x1000000x512,8192x16384x1024")
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    mv.init()
    world, rank = mv.size(), mv.rank()
    out = []
    torch.backends.cuda.matmul.allow_tf32 = True
    for shp in a.shapes.split(","):
        M, Nr, K = [int(v) for v in shp.split("x")]
        t = mv.MatrixTable(Nr, K, "float32", min_value=-0.1, max_value=0.1)
        x = torch.randn(M, K, device="cuda")
        y = torch.empty(M, Nr, device="cuda")
        wbuf = torch.empty(Nr * K, device="cuda")
        fused = timed(lambda: get_gemm(t, x, y), a.iters, world)
        from multiverso_b200 import _native
        cfg = int(_native.cuda_lib().mvb_get_gemm_last_config())
        def unfused():
            t.get(wbuf)
            torch.matmul(x, wbuf.view(Nr, K).t(), out=y)
        unf = timed(unfused, a.iters, world)
        get_only = timed(lambda: t.get(wbuf), a.iters, world)
        flops = 2.0 * M * Nr * K
        wbytes = Nr * K * 4
        link_floor = (wbytes * (world - 1) / world / 450e9 * 1e3) if world > 1 else (wbytes / 3350e9 * 1e3)
        out.append({"M": M, "N": Nr, "K": K, "fused_ms": fused, "unfused_get_plus_cublas_ms": unf, "get_only_ms": get_only,
                    "fused_tflops": flops / fused / 1e9, "w_bytes": wbytes, "w_stream_floor_ms": link_floor,
                    "speedup_vs_unfused": unf / fused,
                    "ctas_per_mma": cfg // 1000, "grid": cfg % 1000})
        t.free()
        del x, y, wbuf
    if rank == 0:
        os.makedirs("gpurun_out", exist_ok=True)
        with open(f"gpurun_out/get_gemm_n{world}.json", "w") as f:
            json.dump(out, f, indent=1)
        print(json.dumps(out), flush=True)
    mv.shutdown()


if __name__ == "__main__":
    main()
