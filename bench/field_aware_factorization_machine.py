#!/usr/bin/env python
"""PSFieldAwareFactorizationMachine (ffm.cu) against the same maths in torch over the gathered rows, and against
PSEmbedding over the same lookups as the floor, device-timed with CUDA events after warm-up (ms per forward +
backward).

Workloads, ids drawn Zipf(1.05) over 10M rows, tables of width D + 4 (D = F k; a multiple of 4, so every arm runs
over the same table):

  criteo     B = 8192 one-hot bags of F = 39 fields (2-D ids, the field of a lookup is its column), k in {4, 8, 16},
             each with the sgd and the rowwise_adagrad updater
  multi-hot  B = 8192 bags of F = 10 fields holding 1..16 ids each (1-D ids with offsets, about 85 lookups per bag),
             k = 8, sgd

Arms:

  fused      PSFieldAwareFactorizationMachine(table, F, k, push_scale=lr): forward + y.mean().backward(), input
             checks included
  unfused    get_rows of the unique ids, the FFM in torch with autograd over the gathered rows, one coalesced add_rows
  floor      PSEmbedding(table, push_scale=lr) forward + out.mean().backward() over the same lookups: it reads the
             same rows and pushes the same unique rows

Each arm runs --iters steps per repeat; --repeats repeats alternate the arms, and the median, min and max over the
repeats are reported. Also reported: the unique rows per step and the logical bytes a fused step must move (the
looked-up rows read once, H written by the forward and read by the backward, the unique rows pushed) with the rate
they imply at the median fused time: a logical rate, not a measured HBM bandwidth. Every line carries the card's name
and power limit, read in the same run. Prints one JSON line per workload; ``--out FILE`` also writes them there.
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
from multiverso_b200.ops import PSEmbedding, PSFieldAwareFactorizationMachine
from multiverso_b200.ops.embedding import _bag_index
from multiverso_b200.ops.field_aware_factorization_machine import _ffm_y


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


def unfused_step(t, ids, fields, offsets, F, k, lr):
    """The op's maths in torch over get_rows of the unique ids."""
    ids1, f1 = ids.reshape(-1), fields.reshape(-1)
    L = ids1.numel()
    if offsets is None:
        B, n = ids.shape
        bag = torch.arange(B, device=ids.device).repeat_interleave(n)
    else:
        B = offsets.numel()
        bag, _ = _bag_index(offsets, L)
    uniq, inv = torch.unique(ids1, return_inverse=True)
    rows = t.get_rows(uniq).requires_grad_()
    _ffm_y(rows[inv], f1, torch.ones(L, device=ids.device), bag, B, F, k).mean().backward()
    t.add_rows(uniq, rows.grad * lr)


def workloads(a, g, w):
    """(name, F, k, updater, ids, fields, offsets) of every workload."""
    B = a.batch
    ids = torch.multinomial(w, B * 39, replacement=True, generator=g).view(B, 39)
    fields = torch.arange(39, device="cuda").expand(B, 39).contiguous()
    for k in (int(v) for v in a.factors.split(",")):
        for upd in a.updaters.split(","):
            yield "criteo", 39, k, upd, ids, fields, None
    F = 10
    per = torch.randint(1, 17, (B, F), device="cuda", generator=g)                # ids per (bag, field)
    lens = per.sum(1)
    mf = torch.arange(F, device="cuda").expand(B, F).reshape(-1).repeat_interleave(per.reshape(-1))
    mids = torch.multinomial(w, int(lens.sum()), replacement=True, generator=g)
    yield "multi_hot", F, 8, "sgd", mids, mf, torch.cumsum(lens, 0) - lens


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--factors", default="4,8,16")
    ap.add_argument("--updaters", default="sgd,rowwise_adagrad")
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/field_aware_factorization_machine.py measures the GPU kernels: no CUDA device")
    mv.init()
    card = gpu_info()
    lines = []
    g = torch.Generator(device="cuda").manual_seed(0)
    lr, n = 1e-3, a.rows
    w = 1.0 / torch.arange(1, n + 1, dtype=torch.float64, device="cuda") ** 1.05
    w = (w / w.sum()).float()
    for name, F, k, upd, ids, fields, offsets in workloads(a, g, w):
        D = F * k
        C = D + 4
        L = ids.numel()
        U = int(torch.unique(ids).numel())
        t = mv.MatrixTable(n, C, "float32", updater=upd, min_value=-0.01, max_value=0.01)
        ffm = PSFieldAwareFactorizationMachine(t, F, k, push_scale=lr)
        emb = PSEmbedding(t, push_scale=lr)
        arms = {"fused": lambda: ffm(ids, fields, offsets).mean().backward(),
                "unfused": lambda: unfused_step(t, ids, fields, offsets, F, k, lr),
                "floor": lambda: emb(ids, offsets).mean().backward()}
        for fn in arms.values():                                      # warm-up of every shape
            for _ in range(3):
                fn()
        times = {key: [] for key in arms}
        for _ in range(a.repeats):
            for key, fn in arms.items():
                times[key].append(timed(fn, a.iters))
        row = {"gpu": card, "workload": name, "rows": n, "F": F, "k": k, "C": C, "updater": upd,
               "batch": a.batch, "lookups": L, "unique_rows": U}
        for key, v in times.items():
            row[f"{key}_ms"] = round(statistics.median(v), 4)
            row[f"{key}_ms_min_max"] = [round(min(v), 4), round(max(v), 4)]
        read, h, pushed = L * (D + 1) * 4, 2 * L * ((D + 4) // 4 * 4) * 4, U * (D + 1) * 4
        row["logical_bytes_read"], row["logical_bytes_H"], row["logical_bytes_pushed"] = read, h, pushed
        row["logical_GBps_at_fused"] = round((read + h + pushed) / (row["fused_ms"] * 1e-3) / 1e9, 1)
        row["speedup_vs_unfused"] = round(row["unfused_ms"] / row["fused_ms"], 2)
        row["fused_over_floor"] = round(row["fused_ms"] / row["floor_ms"], 3)
        line = json.dumps(row)
        print(line, flush=True)
        lines.append(line)
        del ffm, emb
        t.free()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
    mv.shutdown()


if __name__ == "__main__":
    main()
