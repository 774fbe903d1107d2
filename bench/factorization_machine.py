#!/usr/bin/env python
"""PSFactorizationMachine (fm.cu) against the same maths in torch over the gathered rows, and against PSEmbedding over
the same lookups as the floor, device-timed with CUDA events after warm-up (ms per forward + backward).

Criteo-shaped workloads: B = 8192 bags of 39 lookups, ids drawn Zipf(1.05) over 10M rows, C = k + 1 in {16, 64,
128}, each with the sgd and the rowwise_adagrad updater. Arms:

  fused      PSFactorizationMachine(table, push_scale=lr): forward + y.mean().backward(), input checks included
  unfused    get_rows of the unique ids, the FM in torch with autograd over the [L, C] gather, one coalesced add_rows
  floor      PSEmbedding(table, push_scale=lr) forward + out.mean().backward() over the same lookups: it reads the
             same rows and pushes the same unique rows, so the fused arm cannot beat it by much

Each arm runs --iters steps per repeat; --repeats repeats alternate the arms, and the median, min and max over the
repeats are reported. Also reported: the unique rows per step and the logical bytes a fused step must move (the
looked-up rows read once, the unique rows pushed) with the rate they imply at the median fused time: a logical rate,
not a measured HBM bandwidth. Every line carries the card's name and power limit, read in the same run. Prints one
JSON line per workload; ``--out FILE`` also writes them there.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import PSEmbedding, PSFactorizationMachine
from multiverso_b200.ops.factorization_machine import _fm_y


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


def unfused_step(t, ids, lr):
    """The op's maths in torch over get_rows of the unique ids."""
    B, n = ids.shape
    uniq, inv = torch.unique(ids.reshape(-1), return_inverse=True)
    rows = t.get_rows(uniq).requires_grad_()
    bag = torch.arange(B, device=ids.device).repeat_interleave(n)
    _fm_y(rows[inv], torch.ones(B * n, device=ids.device), bag, B).mean().backward()
    t.add_rows(uniq, rows.grad * lr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--widths", default="16,64,128")
    ap.add_argument("--updaters", default="sgd,rowwise_adagrad")
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--bag", type=int, default=39)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/factorization_machine.py measures the GPU kernels: no CUDA device")
    mv.init()
    card = gpu_info()
    lines = []
    g = torch.Generator(device="cuda").manual_seed(0)
    lr, B, n = 1e-3, a.batch, a.rows
    w = 1.0 / torch.arange(1, n + 1, dtype=torch.float64, device="cuda") ** 1.05
    ids = torch.multinomial((w / w.sum()).float(), B * a.bag, replacement=True, generator=g).view(B, a.bag)
    U = int(torch.unique(ids).numel())
    for C in (int(v) for v in a.widths.split(",")):
        for upd in a.updaters.split(","):
            t = mv.MatrixTable(n, C, "float32", updater=upd, min_value=-0.01, max_value=0.01)
            fm = PSFactorizationMachine(t, push_scale=lr)
            emb = PSEmbedding(t, push_scale=lr)
            arms = {"fused": lambda: fm(ids).mean().backward(),
                    "unfused": lambda: unfused_step(t, ids, lr),
                    "floor": lambda: emb(ids).mean().backward()}
            for fn in arms.values():                                      # warm-up of every shape
                for _ in range(3):
                    fn()
            times = {k: [] for k in arms}
            for _ in range(a.repeats):
                for k, fn in arms.items():
                    times[k].append(timed(fn, a.iters))
            row = {"gpu": card, "rows": n, "C": C, "updater": upd, "batch": B, "bag": a.bag, "unique_rows": U}
            for k, v in times.items():
                row[f"{k}_ms"] = round(statistics.median(v), 4)
                row[f"{k}_ms_min_max"] = [round(min(v), 4), round(max(v), 4)]
            read, pushed = B * a.bag * C * 4, U * C * 4
            row["logical_bytes_read"], row["logical_bytes_pushed"] = read, pushed
            row["logical_GBps_at_fused"] = round((read + pushed) / (row["fused_ms"] * 1e-3) / 1e9, 1)
            row["speedup_vs_unfused"] = round(row["unfused_ms"] / row["fused_ms"], 2)
            row["fused_over_floor"] = round(row["fused_ms"] / row["floor_ms"], 3)
            line = json.dumps(row)
            print(line, flush=True)
            lines.append(line)
            del fm, emb
            t.free()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    mv.shutdown()


if __name__ == "__main__":
    main()
