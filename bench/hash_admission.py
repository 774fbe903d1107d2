#!/usr/bin/env python
"""HashMatrixTable count-based admission (hash_rows.cu), admit_after = 1, 2, 4 in one process, the arms alternating.

Workload: keys drawn from Zipf(1.05) over [0, 1e9) (inverse-CDF of the continuous law, floored), spread by hash64;
16 384 bags x 32 lookups per step; dim 64, rowwise_adagrad, capacity 2^23, one GPU, PSEmbedding in training mode.
Every arm sees the same keys in the same order.

  step_ms        one training step (translate + forward + backward + push), CUDA events, after 20 warm-up steps
  count_ms       GPU time of hash_count_keys_kernel per step (torch.profiler, a run of its own)
  lookup_ms      GPU time of hash_lookup_kernel per step
  age_ms         GPU time of the two aging kernels per step
  keys_held      num_keys() after the steps
  zero_share     share of the lookups of the steps that read the zero row (keys not admitted)
  full_at_step   the step whose forward raised "table full" (the arm stops there), or null

Every line carries the card's name and power limit. Prints one JSON line per arm; nothing is written.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import PSEmbedding
from multiverso_b200.tables.options import AddOption
from hash_embedding import gpu_info, kernel_ms, spread

BAGS, PER_BAG, DIM, CAPACITY = 16384, 32, 64, 1 << 23


def zipf_keys(n, g, s=1.05, N=1e9):
    u = torch.rand(n, device="cuda", generator=g, dtype=torch.float64)
    x = ((N ** (1 - s) - 1) * u + 1) ** (1 / (1 - s))            # continuous Zipf on [1, N]
    return spread(x.floor_().to(torch.int64).clamp_(1, int(N)) - 1, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--arms", default="1,2,4")
    args = ap.parse_args()
    card = gpu_info()
    mv.init()
    arms = [int(a) for a in args.arms.split(",")]
    opt = AddOption(learning_rate=0.1)
    tabs = {n: mv.HashMatrixTable(CAPACITY, DIM, updater="rowwise_adagrad", min_value=-0.01, max_value=0.01,
                                  admit_after=n) for n in arms}
    layers = {n: PSEmbedding(t, push_scale=1e-2, option=opt) for n, t in tabs.items()}
    offs = torch.arange(0, BAGS * PER_BAG, PER_BAG, device="cuda")
    dout = torch.randn(BAGS, DIM, device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    g = torch.Generator(device="cuda").manual_seed(7)
    ms = {n: 0.0 for n in arms}
    zeros = {n: 0 for n in arms}
    done = {n: 0 for n in arms}
    full = {n: None for n in arms}
    warm = 20
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

    def step(n, keys):
        layers[n](keys, offs).backward(dout)

    for i in range(args.steps):
        keys = zipf_keys(BAGS * PER_BAG, g)
        for n in arms:
            if full[n] is not None:
                continue
            torch.cuda.synchronize()
            ev[0].record()
            try:
                step(n, keys)
            except RuntimeError as e:
                if "table full" not in str(e):
                    raise
                full[n] = i
                continue
            ev[1].record()
            torch.cuda.synchronize()
            if i >= warm:
                ms[n] += ev[0].elapsed_time(ev[1])
                done[n] += 1
            zeros[n] += int((tabs[n].lookup(keys, insert=False) == tabs[n].zero_row).sum())
    for n in arms:
        keys = zipf_keys(BAGS * PER_BAG, g)
        steps = full[n] if full[n] is not None else args.steps
        if full[n] is not None:                   # time the kernels on keys the full table already holds
            keys = torch.cat([tabs[n].export()[0]] * 2)[:BAGS * PER_BAG]
        kt = {name: kernel_ms(lambda: step(n, keys), name, 5) for name in ("hash_count_keys", "hash_lookup_kernel",
                                                                          "hash_age")}
        print(json.dumps({"bench": "hash_admission", "admit_after": n, "card": card,
                          "step_ms": round(ms[n] / max(done[n], 1), 3), "timed_steps": done[n],
                          "count_ms": round(kt["hash_count_keys"], 4), "lookup_ms": round(kt["hash_lookup_kernel"], 4),
                          "age_ms": round(kt["hash_age"], 4), "keys_held": tabs[n].num_keys(),
                          "slots": tabs[n].S * tabs[n].slots,
                          "zero_share": round(zeros[n] / (max(steps, 1) * BAGS * PER_BAG), 4), "steps": steps,
                          "full_at_step": full[n]}),
              flush=True)
    mv.shutdown()


if __name__ == "__main__":
    main()
