#!/usr/bin/env python
"""HashMatrixTable (hash_rows.cu) on the workloads of bench/embedding_bag_collection.py, device-timed with CUDA events
after warm-up. The Zipf ids of every feature are spread over int64 by hash64, so they are keys, not row ids.

Arms, in ms per call:

  translate_present      one translation of the whole batch (every feature) with every key already present
  translate_first_touch  the same translation starting from an empty index (the index is re-initialised before each
                         timed call, outside the timed interval)
  hash_fwd(_bwd)         PSEmbeddingCollection over hash tables fed keys (+ backward: one push per table)
  dense_fwd(_bwd)        the same collection over dense tables of the workload's shapes fed the pre-mapped row ids
  translate_kernel       GPU time of the lookup kernel alone in translate_present (torch.profiler)
  gather_kernel          GPU time of the collection's forward gather-pool kernel alone in dense_fwd (torch.profiler);
                         translate_below_gather compares these two

Hash tables hold min(rows, 2^21) keys (a batch touches far fewer), so both arms fit on one card with adagrad state.
Every line carries the card's name and power limit. Prints one JSON line per workload and updater; ``--out FILE``
also writes them there. Nothing else is written.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200 import _native as N
from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
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


def kernel_ms(fn, name, iters, warmup=3):
    """GPU time per call of the kernels whose name contains `name` (torch.profiler, CUDA activity): the kernel
    alone, without the host work, other kernels and gaps that an event-timed call includes."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if name in e.key)
    return us / 1e3 / iters


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def workload(name):
    """(tables [(rows, dim)], features [(name, table, max bag length)]), as in bench/embedding_bag_collection.py."""
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


def spread(ids, salt):
    """hash64(id + salt) as int64 (torch int64 arithmetic wraps like uint64)."""
    x = ids + salt * 0x9E3779B9
    for m in (-49064778989728563, -4265267296055464877):    # 0xff51afd7ed558ccd, 0xc4ceb9fe1a85ec53 as int64
        x = x ^ ((x >> 33) & ((1 << 31) - 1))
        x = x * m
    x = x ^ ((x >> 33) & ((1 << 31) - 1))
    return torch.where(x == -(1 << 63), torch.zeros_like(x), x)


def run(wl, updater, arm, iters, card, g):
    shapes, feats = workload(wl)
    opt = AddOption(learning_rate=0.1, rho=0.1)
    lr = 1e-3
    lengths = torch.stack([torch.randint(1, n + 1, (BAGS,), device="cuda", generator=g) for _, _, n in feats])
    order = [f for t in range(len(shapes)) for f, (_, tt, _) in enumerate(feats) if tt == t]     # config order
    per = {f: zipf_ids(shapes[feats[f][1]][0], int(lengths[f].sum()), g) for f in order}
    ids = torch.cat([per[f] for f in order])
    keys = torch.cat([spread(per[f], feats[f][1]) for f in order])
    len_c = lengths[order]
    names = [[n for n, tt, _ in feats if tt == t] for t in range(len(shapes))]
    row = {"gpu": card, "workload": wl, "updater": updater, "bags": BAGS, "features": len(feats),
           "tables": len(shapes), "lookups": ids.numel()}
    dout = torch.randn(BAGS, sum(shapes[feats[f][1]][1] for f in order), device="cuda", generator=g)
    if arm == "dense":
        dense = [mv.MatrixTable(V, D, "float32", updater=updater, min_value=-0.1, max_value=0.1) for V, D in shapes]
        dcoll = PSEmbeddingCollection([EmbeddingBagConfig(t, names[i], push_scale=lr, option=opt)
                                       for i, t in enumerate(dense)])
        row["dense_fwd_ms"] = round(timed(lambda: dcoll(ids, len_c), iters), 4)
        row["gather_kernel_ms"] = round(kernel_ms(lambda: dcoll(ids, len_c), "emb_coll_fwd_kernel", iters), 4)
        row["dense_fwd_bwd_ms"] = round(timed(lambda: dcoll(ids, len_c).backward(dout), iters), 4)
        return row

    hashed = [mv.HashMatrixTable(min(V, 1 << 21), D, updater=updater, min_value=-0.1, max_value=0.1)
              for V, D in shapes]
    hcoll = PSEmbeddingCollection([EmbeddingBagConfig(t, names[i], push_scale=lr, option=opt)
                                   for i, t in enumerate(hashed)])
    rows, status = torch.empty_like(keys), torch.empty(1, dtype=torch.int64, device="cuda")
    seg_end = torch.cumsum(len_c.sum(1), 0)

    def translate():
        hashed[0].lookup_call(keys, rows, status, True, seg_end, hcoll._seg_table, hcoll._d_hash)

    def reinit():
        for t in hashed:
            N.cuda_lib().mvb_hash_rows_init(t._keys_buf.local_ptr, t._ready_buf.local_ptr, t._count_buf.local_ptr,
                                            t.slots, N.stream_ptr())

    first = 0.0
    for _ in range(iters):
        reinit()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        translate()
        e1.record()
        torch.cuda.synchronize()
        first += e0.elapsed_time(e1)
    assert int(status.item()) == 0
    row["distinct_keys"] = sum(t.num_keys() for t in hashed)
    row["translate_first_touch_ms"] = round(first / iters, 4)
    row["translate_present_ms"] = round(timed(translate, iters), 4)
    row["translate_kernel_ms"] = round(kernel_ms(translate, "hash_lookup_kernel", iters), 4)
    row["hash_fwd_ms"] = round(timed(lambda: hcoll(keys, len_c), iters), 4)
    row["hash_fwd_bwd_ms"] = round(timed(lambda: hcoll(keys, len_c).backward(dout), iters), 4)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="criteo,multihot")
    ap.add_argument("--updaters", default="sgd,adagrad")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--arm", choices=["hash", "dense"], default=None,
                    help="run one arm of one workload and updater in this process")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/hash_embedding.py measures the GPU kernels: no CUDA device")
    if a.arm:
        mv.init()
        row = run(a.workloads, a.updaters, a.arm, a.iters, gpu_info(), torch.Generator(device="cuda").manual_seed(0))
        print(json.dumps(row), flush=True)
        mv.shutdown()
        return
    lines = []
    # one process per workload, updater and arm: each starts with all of its memory and signal-pad channels free
    for wl in a.workloads.split(","):
        for upd in a.updaters.split(","):
            row = {}
            for arm in ("hash", "dense"):
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--workloads", wl, "--updaters", upd,
                                    "--arm", arm, "--iters", str(a.iters)], capture_output=True, text=True)
                if r.returncode != 0:
                    raise SystemExit(f"{wl} / {upd} / {arm} failed:\n{r.stdout[-2000:]}{r.stderr[-4000:]}")
                row.update(json.loads(r.stdout.strip().splitlines()[-1]))
            row["translate_below_gather"] = row["translate_kernel_ms"] < row["gather_kernel_ms"]
            lines.append(json.dumps(row))
            print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
