#!/usr/bin/env python
"""The embedding-bag collection (emb_bag_coll.cu) against one PSEmbedding per feature plus torch.cat, and against
local torch EmbeddingBags, device-timed with CUDA events after warm-up.

Workloads (16,384 bags per feature, Zipf(1.05) ids: the hot rows are the low ids):

  criteo     26 one-hot features, one table each, dim 64, 26 tables of 10^3 .. 4*10^6 rows (5.4 GB)
  multihot   24 features with bags of 1..20 lookups over 8 tables of dims 32..128; two pairs of features each
             share a 10M x 128 table, the other 20 features are spread over 6 smaller tables

Each workload runs with sgd tables and with adagrad tables. Arms:

  coll_fwd(_bwd)     PSEmbeddingCollection: one fused lookup (+ backward: one coalesced push per table)
  loop_fwd(_bwd)     one PSEmbedding per feature + torch.cat (+ backward)
  torch_fwd(_bwd)    one nn.EmbeddingBag(sparse=True) per table on a local copy of the weights (+ SGD or Adagrad
                     step): the non-PS bound

Reported: ms per call. Every line carries the card's name and power limit. Prints one JSON line per workload and
updater; ``--out FILE`` also writes them there. Nothing else is written.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import EmbeddingBagConfig, PSEmbedding, PSEmbeddingCollection
from multiverso_b200.tables.options import AddOption

BAGS = 16384


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


def workload(name):
    """(tables [(rows, dim)], features [(name, table, max bag length)])."""
    if name == "criteo":
        r = (4e6 / 1e3) ** (1 / 23)
        rows = [4_000_000, 4_000_000] + [int(1e3 * r ** i) for i in range(24)]
        return [(n, 64) for n in rows], [(f"c{i}", i, 1) for i in range(26)]
    tables = [(10_000_000, 128), (10_000_000, 128), (2_000_000, 64), (1_000_000, 96), (500_000, 32),
              (300_000, 128), (100_000, 48), (50_000, 32)]
    feats = [("item", 0, 1), ("history", 0, 20), ("ad", 1, 1), ("ad_history", 1, 20)]
    feats += [(f"s{i}", 2 + i % 6, 1 + (7 * i) % 20) for i in range(20)]
    return tables, feats


def zipf_ids(V, n, g):
    cdf = torch.cumsum(torch.arange(1, V + 1, device="cuda", dtype=torch.float64).pow_(-1.05), 0)
    u = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * cdf[-1]
    return torch.searchsorted(cdf, u).clamp_(max=V - 1)


def run(wl, updater, iters, card, g):
    shapes, feats = workload(wl)
    opt = AddOption(learning_rate=0.1, rho=0.1)
    lr = 1e-3
    tables = [mv.MatrixTable(V, D, "float32", updater=updater, min_value=-0.1, max_value=0.1) for V, D in shapes]
    lengths = torch.stack([torch.randint(1, n + 1, (BAGS,), device="cuda", generator=g) for _, _, n in feats])
    per = [zipf_ids(shapes[t][0], int(lengths[f].sum()), g) for f, (_, t, _) in enumerate(feats)]
    ids = torch.cat(per)
    offs = [torch.cumsum(lengths[f], 0) - lengths[f] for f in range(len(feats))]
    cfgs = [EmbeddingBagConfig(tables[t], [n for n, tt, _ in feats if tt == t], push_scale=lr, option=opt)
            for t in range(len(shapes))]
    ebc = PSEmbeddingCollection(cfgs)
    order = [f for t in range(len(shapes)) for f, (_, tt, _) in enumerate(feats) if tt == t]   # config order
    ids_c = torch.cat([per[f] for f in order])
    len_c = lengths[order]
    per_o, offs_o = [per[f] for f in order], [offs[f] for f in order]
    dim_o = [shapes[feats[f][1]][1] for f in order]
    layers = [PSEmbedding(tables[feats[f][1]], push_scale=lr, option=opt) for f in order]
    dout = torch.randn(BAGS, sum(dim_o), device="cuda", generator=g)
    refs = [torch.nn.EmbeddingBag(V, D, mode="sum", sparse=True, device="cuda") for V, D in shapes]
    params = [r.weight for r in refs]
    topt = torch.optim.SGD(params, lr=lr) if updater == "sgd" else torch.optim.Adagrad(params, lr=lr)

    def loop(bwd):
        y = torch.cat([layer(i, o) for layer, i, o in zip(layers, per_o, offs_o)], 1)
        if bwd:
            y.backward(dout)

    def local(bwd):
        y = torch.cat([refs[feats[f][1]](per[f], offs[f]) for f in order], 1)
        if bwd:
            topt.zero_grad(set_to_none=True)
            y.backward(dout)
            topt.step()

    arms = {
        "coll_fwd": lambda: ebc(ids_c, len_c),
        "coll_fwd_bwd": lambda: ebc(ids_c, len_c).backward(dout),
        "loop_fwd": lambda: loop(False),
        "loop_fwd_bwd": lambda: loop(True),
        "torch_fwd": lambda: local(False),
        "torch_fwd_bwd": lambda: local(True),
    }
    row = {"gpu": card, "workload": wl, "updater": updater, "bags": BAGS, "features": len(feats),
           "tables": len(shapes), "table_GB": round(sum(V * D * 4 for V, D in shapes) / 1e9, 2),
           "lookups": ids.numel()}
    for name, fn in arms.items():
        row[f"{name}_ms"] = round(timed(fn, iters), 4)
    row["fwd_speedup_vs_loop"] = round(row["loop_fwd_ms"] / row["coll_fwd_ms"], 2)
    row["fwd_bwd_speedup_vs_loop"] = round(row["loop_fwd_bwd_ms"] / row["coll_fwd_bwd_ms"], 2)
    row["fwd_bwd_vs_torch"] = round(row["torch_fwd_bwd_ms"] / row["coll_fwd_bwd_ms"], 2)
    del refs, params, topt, layers, ebc
    for t in tables:
        t.free()
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="criteo,multihot")
    ap.add_argument("--updaters", default="sgd,adagrad")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/embedding_bag_collection.py measures the GPU kernels: no CUDA device")
    runs = [(wl, upd) for wl in a.workloads.split(",") for upd in a.updaters.split(",")]
    lines = []
    if len(runs) == 1:
        mv.init()
        lines.append(json.dumps(run(*runs[0], a.iters, gpu_info(), torch.Generator(device="cuda").manual_seed(0))))
        print(lines[-1], flush=True)
        mv.shutdown()
        runs = []
    # one process per workload and updater: each starts with all of its memory and signal-pad channels free
    for wl, upd in runs:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--workloads", wl, "--updaters", upd,
                            "--iters", str(a.iters)], capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit(f"{wl} / {upd} failed:\n{r.stdout[-2000:]}{r.stderr[-4000:]}")
        line = r.stdout.strip().splitlines()[-1]
        print(line, flush=True)
        lines.append(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
