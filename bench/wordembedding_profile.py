#!/usr/bin/env python
"""Where the time of a WordEmbedding training block goes, kernel by kernel.

  python bench/wordembedding_profile.py [--warmup 3] [--blocks 5] [--trace-dir DIR]

Builds the configuration `bench.py` measures (skip-gram, dim 300, vocab 1M, 5 negatives, window 5,
synthetic Zipf corpus of 1M-word blocks, the default deterministic K7), trains the warm-up blocks
untraced, then traces each timed block on its own under torch.profiler with CUDA activities.  Per
block it prints one JSON line: the device time of the deterministic K7 plan (its `sgns_det_plan*`
kernels and the radix sort of its readers, whose kernels carry `sgns_det_plan_reader` in their
names), of its wave kernels (`sgns_det_kernel*`) and of their apply kernels (`sgns_det_apply*`), the
time of every other kernel, and the idle time between kernels inside the block's device span.  The first line names the card,
its power limit and SM clock, read in this process.  Tracing slows the host, so take words/s from
`bench.py`, not from here.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info(torch):
    info = {"name": torch.cuda.get_device_name(), "power_limit_w": None, "sm_clock_mhz": None,
            "sm_clock_max_mhz": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        info["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0
        info["sm_clock_mhz"] = pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
        info["sm_clock_max_mhz"] = pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:   # noqa: BLE001 - fall back to the command-line query
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True)
        f = [x.strip() for x in q.stdout.strip().split(",")]
        if len(f) == 3:
            info["power_limit_w"], info["sm_clock_mhz"], info["sm_clock_max_mhz"] = float(f[0]), float(f[1]), float(f[2])
    return info


def block_profile(prof):
    """Kernel time by group and idle time between kernels, from one traced block."""
    from torch.autograd import DeviceType
    ks = sorted(((e.time_range.start, e.time_range.end, e.name) for e in prof.events()
                 if e.device_type == DeviceType.CUDA and not e.name.startswith("Memcpy")
                 and not e.name.startswith("Memset")), key=lambda k: k[0])
    out = {"det_plan_us": 0.0, "det_kernel_us": 0.0, "det_apply_us": 0.0, "other_kernels_us": 0.0,
           "n_det_plan": 0, "n_det_kernel": 0, "n_det_apply": 0, "n_other": 0}
    for s, e, name in ks:
        if "sgns_det_plan" in name:
            out["det_plan_us"] += e - s
            out["n_det_plan"] += 1
        elif "sgns_det_kernel" in name:
            out["det_kernel_us"] += e - s
            out["n_det_kernel"] += 1
        elif "sgns_det_apply" in name:
            out["det_apply_us"] += e - s
            out["n_det_apply"] += 1
        else:
            out["other_kernels_us"] += e - s
            out["n_other"] += 1
    idle, end = 0.0, None
    for s, e, _ in ks:
        if end is not None and s > end:
            idle += s - end
        end = e if end is None else max(end, e)
    out["idle_between_kernels_us"] = idle
    out["device_span_us"] = (ks[-1][1] - ks[0][0]) if ks else 0.0
    return {k: round(v, 1) if isinstance(v, float) else v for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--block-words", type=int, default=1 << 20)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--trace-dir", default=None, help="also write each block's Chrome trace here")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import multiverso_b200 as mv
    from multiverso_b200.models.wordembedding import (WordEmbedding, WordEmbeddingOption,
                                                      synthetic_zipf_corpus)
    if not torch.cuda.is_available():
        raise SystemExit("wordembedding_profile.py profiles CUDA kernels and needs a GPU")
    mv.init()
    try:
        W, K, B = args.warmup, args.blocks, args.block_words
        # the option values bench.py uses (its default --steps 20 sets total_words)
        opt = WordEmbeddingOption(embeding_size=300, window_size=5, negative_num=5, init_learning_rate=0.025,
                                  sample=0.0, total_words=B * (20 + 3) * 2, epoch=1)
        we = WordEmbedding(opt, args.vocab, seed=1)
        n_blocks = W + K
        corpus = synthetic_zipf_corpus(B * n_blocks, args.vocab, sentence_len=1000, seed=17)
        blocks = torch.from_numpy(corpus).view(n_blocks, B).cuda()
        print(json.dumps({"card": card_info(torch)}), flush=True)
        for i in range(W):
            we.train_block(blocks[i], compute_loss=True)
        torch.cuda.synchronize()
        for i in range(W, n_blocks):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                we.train_block(blocks[i], compute_loss=True)
                torch.cuda.synchronize()
            row = {"block": i - W, "words": int((corpus[i * B:(i + 1) * B] >= 0).sum())}
            row.update(block_profile(prof))
            print(json.dumps(row), flush=True)
            if args.trace_dir:
                os.makedirs(args.trace_dir, exist_ok=True)
                prof.export_chrome_trace(os.path.join(args.trace_dir, f"block{i - W}.pt.trace.json"))
        print(json.dumps({"card_after": card_info(torch)}), flush=True)
    finally:
        mv.shutdown()


if __name__ == "__main__":
    main()
