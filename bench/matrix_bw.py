#!/usr/bin/env python
"""BASELINE config 2: MatrixTable 1M x 512 fp32 whole-table Get / Add bandwidth, ours (fused
P2P kernels) vs the NCCL comparator, device-timed, max over ranks.  Also config 5's shape
(ArrayTable 4 GB fp32, momentum updater) with --array-gb 4.

    python bench/matrix_bw.py                       (1 GPU)
    torchrun --nproc-per-node 8 bench/matrix_bw.py  (8 GPUs)
Writes gpurun_out/matrix_bw_n<N>.json."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv


def timed(fn, iters, world):
    for _ in range(2):
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
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--cols", type=int, default=512)
    ap.add_argument("--array-gb", type=float, default=0.0)
    ap.add_argument("--updater", default="sgd")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--replica", action="store_true", help="enable the fused Add->Get replica push")
    a = ap.parse_args()
    mv.init(sync=True)
    world, rank = mv.size(), mv.rank()
    if a.array_gb > 0:
        n = int(a.array_gb * (1 << 30) / 4) // (world * 4) * (world * 4)
        table = mv.ArrayTable(n, "float32", updater=a.updater)
        shape = f"ArrayTable {a.array_gb:g} GiB fp32 ({a.updater})"
    else:
        n = a.rows * a.cols
        table = mv.MatrixTable(a.rows, a.cols, "float32", updater=a.updater)
        shape = f"MatrixTable {a.rows}x{a.cols} fp32 ({a.updater})"
    if world > 1 and a.replica:
        table.enable_replica()
        mv.barrier()
    nbytes = n * 4
    out = torch.empty(n, device="cuda")
    opt = mv.AddOption(momentum=0.9, learning_rate=0.01)

    def our_add():
        if world > 1:
            table.staging()            # zero-copy: the producer kernel would write here
            table.wait(table.add_async(None, opt, staged=True))
        else:
            table.wait(table.add_async(out, opt))

    res = {"shape": shape, "n_gpus": world, "bytes": nbytes}
    res["replica"] = bool(world > 1 and a.replica)
    res["ours_add_ms"] = timed(our_add, a.iters, world)
    res["ours_get_ms"] = timed(lambda: table.get(out), a.iters, world)
    def add_get():
        our_add()
        table.get(out)
    res["ours_add_plus_get_ms"] = timed(add_get, a.iters, world)
    if n % world == 0:
        from baseline.nccl_path import NcclDenseTable
        nt = NcclDenseTable(n, a.updater if a.updater in ("sgd", "momentum_sgd", "default") else "sgd")
        delta = torch.full((n,), 1e-3, device="cuda")
        res["nccl_add_ms"] = timed(lambda: nt.add(delta), a.iters, world)
        res["nccl_get_ms"] = timed(lambda: nt.get(out), a.iters, world)
        def nccl_add_get():
            nt.add(delta)
            nt.get(out)
        res["nccl_add_plus_get_ms"] = timed(nccl_add_get, a.iters, world)
        del delta
    link = 450.0   # GB/s per direction per GPU: H100 SXM NVLink 4 (18 links), data-sheet figure
    hbm = 3350.0   # GB/s: H100 SXM HBM3, data-sheet figure
    cross = nbytes * (world - 1) / world
    res["floor_ms"] = (cross / link / 1e6) if world > 1 else (2 * nbytes / hbm / 1e6)
    for k in ("ours_add", "ours_get", "nccl_add", "nccl_get"):
        if k + "_ms" in res:
            res[k + "_gbs"] = nbytes / res[k + "_ms"] / 1e6
            res[k + "_frac_of_floor"] = res["floor_ms"] / res[k + "_ms"]
    if rank == 0:
        os.makedirs("gpurun_out", exist_ok=True)
        tag = ("array" if a.array_gb > 0 else "matrix") + ("_replica" if a.replica else "")
        with open(f"gpurun_out/{tag}_bw_n{world}.json", "w") as f:
            json.dump(res, f, indent=1)
        print(json.dumps(res), flush=True)
    mv.shutdown()


if __name__ == "__main__":
    main()
