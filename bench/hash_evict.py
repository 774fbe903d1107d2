#!/usr/bin/env python
"""HashMatrixTable access clock and eviction (hash_rows.cu), device-timed after warm-up.

Stamping cost, on the workloads of bench/hash_embedding.py (criteo, multihot; keys spread by hash64), sgd, tables
with track_access off and on, one process per arm, the arms alternating:

  translate_kernel_ms        GPU time of hash_lookup_kernel alone (torch.profiler) in a translation of the whole
                             batch with every key present; "same clock": the stamps are current, so a found key costs
                             a load; "new clock": the clock advances before every call, so every distinct key takes
                             one atomicMax
  fwd_bwd_ms                 PSEmbeddingCollection forward + backward (CUDA events), the clock advancing every step
                             (one fill per table included)

Eviction cost: a table of P = 2^21 slots filled to 7/8 (1 835 008 keys, dim 64) in ten generations stamped 0..9;
evict(older_than=1) removes 10 %, evict(older_than=5) 50 %. Reported per updater (sgd, adagrad): the whole call
(host clock, it ends in a synchronisation), the GPU time of the three eviction kernels (torch.profiler), rows
moved, and the bytes the rebuild must move over the HBM bandwidth of the data sheet (3.35 TB/s).

Every line carries the card's name and power limit. Prints one JSON line per measurement; ``--out FILE`` also
writes them there. Nothing else is written.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
from multiverso_b200.tables.options import AddOption
from hash_embedding import BAGS, gpu_info, kernel_ms, spread, timed, workload, zipf_ids

HBM = 3.35e12


def stamping(wl, track, iters, card, g):
    shapes, feats = workload(wl)
    opt, lr = AddOption(learning_rate=0.1, rho=0.1), 1e-3
    lengths = torch.stack([torch.randint(1, n + 1, (BAGS,), device="cuda", generator=g) for _, _, n in feats])
    order = [f for t in range(len(shapes)) for f, (_, tt, _) in enumerate(feats) if tt == t]
    keys = torch.cat([spread(zipf_ids(shapes[feats[f][1]][0], int(lengths[f].sum()), g), feats[f][1])
                      for f in order])
    len_c = lengths[order]
    names = [[n for n, tt, _ in feats if tt == t] for t in range(len(shapes))]
    dout = torch.randn(BAGS, sum(shapes[feats[f][1]][1] for f in order), device="cuda", generator=g)
    seg_end = torch.cumsum(len_c.sum(1), 0)
    tabs = [mv.HashMatrixTable(min(V, 1 << 21), D, updater="sgd", min_value=-0.1, max_value=0.1,
                               track_access=track) for V, D in shapes]
    coll = PSEmbeddingCollection([EmbeddingBagConfig(t, names[i], push_scale=lr, option=opt)
                                  for i, t in enumerate(tabs)])
    rows, status = torch.empty_like(keys), torch.empty(1, dtype=torch.int64, device="cuda")
    clock = [0]

    def advance():
        if track:
            clock[0] += 1
            for t in tabs:
                t.clock = clock[0]

    def translate(new_clock):
        if new_clock:
            advance()
        tabs[0].lookup_call(keys, rows, status, True, seg_end, coll._seg_table, coll._d_hash)

    def step():
        advance()
        coll(keys, len_c).backward(dout)

    translate(False)
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    row = {"gpu": card, "measure": "stamping", "workload": wl, "track_access": track, "lookups": keys.numel()}
    row["translate_kernel_same_clock_ms"] = round(kernel_ms(lambda: translate(False), "hash_lookup_kernel", iters), 4)
    row["translate_kernel_new_clock_ms"] = round(kernel_ms(lambda: translate(True), "hash_lookup_kernel", iters), 4)
    row["fwd_bwd_ms"] = round(timed(step, iters), 4)
    return row


def eviction(updater, reps, card):
    P, dim, gens = 1 << 21, 64, 10
    n = 7 * P // 8
    keys = spread(torch.arange(n, device="cuda", dtype=torch.int64), 12345)
    assert torch.unique(keys).numel() == n
    gen = torch.arange(n, device="cuda") * gens // n
    out = []
    for rep in range(reps):
        for older_than in (1, 5):
            t = mv.HashMatrixTable(n, dim, updater=updater, min_value=-0.1, max_value=0.1, track_access=True)
            assert t.slots == P
            for c in range(gens):
                t.clock = c
                t.lookup(keys[gen == c])
            assert t.num_keys() == n
            before = t.lookup(keys, insert=False)
            profile = rep == reps - 1
            torch.cuda.synchronize()
            if profile:
                from torch.profiler import ProfilerActivity, profile as prof_ctx
                with prof_ctx(activities=[ProfilerActivity.CUDA]) as prof:
                    t0 = time.perf_counter()
                    removed = t.evict(older_than=older_than)
                    wall = time.perf_counter() - t0
                kern = sum(e.device_time_total for e in prof.key_averages() if "hash_evict" in e.key) / 1e3
            else:
                t0 = time.perf_counter()
                removed = t.evict(older_than=older_than)
                wall = time.perf_counter() - t0
            after = t.lookup(keys, insert=False)
            kept = gen >= older_than
            assert removed == int((~kept).sum()) and bool((after[~kept] == t.zero_row).all())
            moved = int((before[kept] != after[kept]).sum())
            st_bytes = 4 * (dim if t.updater_name == "adagrad" else 0)
            slot = 8 + 4 + 8                                        # key, ready, last_seen
            need = P * (slot + 8) + moved * (2 * (4 * dim + st_bytes + slot) + st_bytes + slot) + \
                removed * (st_bytes + slot)
            row = {"gpu": card, "measure": "evict", "updater": updater, "slots": P, "dim": dim, "keys": n,
                   "removed": removed, "removed_frac": round(removed / n, 3), "rep": rep,
                   "evict_call_ms": round(wall * 1e3, 3), "rows_moved": moved, "bytes": need,
                   "hbm_bound_ms": round(need / HBM * 1e3, 4)}
            if profile:
                row["evict_kernels_ms"] = round(kern, 4)
            out.append(row)
            t.free()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="criteo,multihot")
    ap.add_argument("--updaters", default="sgd,adagrad")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--arm", choices=["off", "on", "evict"], default=None,
                    help="run one arm (one workload or updater) in this process")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/hash_evict.py measures the GPU kernels: no CUDA device")
    if a.arm:
        card = gpu_info()
        mv.init()
        if a.arm == "evict":
            rows = eviction(a.updaters, a.reps, card)
        else:
            rows = [stamping(a.workloads, a.arm == "on", a.iters, card,
                             torch.Generator(device="cuda").manual_seed(0))]
        for r in rows:
            print(json.dumps(r), flush=True)
        mv.shutdown()
        return
    # one process per arm: each starts with all of its memory and signal-pad channels free; the two stamping arms
    # alternate, `reps` times each
    jobs = [(wl, arm) for _ in range(a.reps) for wl in a.workloads.split(",") for arm in ("off", "on")]
    jobs += [(upd, "evict") for upd in a.updaters.split(",")]
    lines = []
    for what, arm in jobs:
        flag = "--updaters" if arm == "evict" else "--workloads"
        r = subprocess.run([sys.executable, os.path.abspath(__file__), flag, what, "--arm", arm, "--iters",
                            str(a.iters), "--reps", str(a.reps)], capture_output=True, text=True)
        if r.returncode != 0:
            raise SystemExit(f"{what} / {arm} failed:\n{r.stdout[-2000:]}{r.stderr[-4000:]}")
        for ln in r.stdout.strip().splitlines():
            if ln.startswith("{"):
                lines.append(ln)
                print(ln, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
