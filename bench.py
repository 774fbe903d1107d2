#!/usr/bin/env python
"""Headline benchmark: WordEmbedding words/sec (BASELINE.json config 3) + MatrixTable Get/Add GB/s.

  python bench.py --gpus N --steps K --warmup W          (N>1: launched by torch.distributed.run)
  python bench.py --impl reference ...                   (the unmodified reference, if installable)

Config (BASELINE.json): skip-gram, dim=300, vocab=1M, 5 negatives, window 5, synthetic Zipf
corpus, fp32 tables and fp32 math (the reference's dtype), random-init weights.  One step =
one data block of ``--block-words`` corpus words per GPU (weak scaling), trained through the
public WordEmbedding API: RequestParameter -> K7 train kernel -> AddDeltaParameter.
``value`` is device-timed (CUDA events, max over ranks); ``e2e`` adds, per step, the pinned
host->device copy of the block's tokens and a device->host read of the loss.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "wordembedding_words_per_sec"
CONFIG_MODEL = "WordEmbedding skip-gram dim=300 vocab=1M neg=5 window=5 (synthetic Zipf corpus)"


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--block-words", type=int, default=1 << 20)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--negative", type=int, default=5)
    ap.add_argument("--window", type=int, default=5)
    ap.add_argument("--no-table-bw", action="store_true", help="skip the MatrixTable Get/Add sweep")
    ap.add_argument("--metric", default="words", choices=["words", "matrix_bw"],
                    help="words: WordEmbedding words/s (+ MatrixTable Get+Add GB/s as `secondary`); "
                         "matrix_bw: only the MatrixTable 1Mx512 Get+Add GB/s line (BASELINE.json config 2)")
    ap.add_argument("--direct", action="store_true",
                    help="world > 1: K7 trains in the row-sharded tables over NVLink (no block cache); not the default")
    ap.add_argument("--no-pipeline", action="store_true",
                    help="world > 1: train / pull / push strictly one after the other (-is_pipeline 0)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write what they computed (loss, pair count, a fixed sample of "
                         "rows of both embedding tables) as DIR/<name>.npy, so that two builds can be compared")
    return ap.parse_args()


class ClockSampler:
    """SM clocks / throttle reasons sampled DURING the timed region.

    Started before the warm-up, stopped after the timed region; only samples taken inside the timed
    region are reported.  Source: NVML in-process (``pynvml``, the library nvidia-smi itself uses: SM
    clock, max SM clock, clocks-event reasons) every 200 ms, falling back to the recipe's looping
    ``nvidia-smi --query-gpu=... -lms 200`` when pynvml is missing.  Polling is kept sparse on purpose:
    a fast poll / the nvidia-smi loop can stall kernel launches inside device-timed steps.
    BENCH_CLOCK_SAMPLER=smi|nvml|none."""

    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
    # nvmlClocksEventReason* bits
    BITS = {"sw_power_cap": 0x4, "hw_slowdown": 0x8, "sw_thermal_slowdown": 0x20, "hw_thermal_slowdown": 0x40}

    def __init__(self, gpu_index: int = 0, source: str = "smi"):
        self.rows = []          # (monotonic time, sm_mhz, sm_max_mhz, set(reasons))
        self.proc = None
        self.thread = None
        self.gpu = gpu_index
        self.source = os.environ.get("BENCH_CLOCK_SAMPLER", source)
        self.t_begin = self.t_end = None
        self._stop = threading.Event()

    def mark_begin(self):
        self.t_begin = time.monotonic()

    def mark_end(self):
        self.t_end = time.monotonic()

    def start(self):
        if self.source == "none":
            return
        if self.source == "nvml":
            try:
                import pynvml
                pynvml.nvmlInit()
                try:
                    import torch
                    uuid = str(torch.cuda.get_device_properties(self.gpu).uuid)
                    h = pynvml.nvmlDeviceGetHandleByUUID(("GPU-" + uuid).encode() if not uuid.startswith("GPU-") else uuid.encode())
                except Exception:
                    h = pynvml.nvmlDeviceGetHandleByIndex(self.gpu)
                self._nvml, self._h = pynvml, h
                self.thread = threading.Thread(target=self._pump_nvml, daemon=True)
                self.thread.start()
                return
            except Exception:
                self.source = "smi"
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "200",
                 "-i", str(self.gpu)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._pump_smi, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _pump_nvml(self):
        nv, h = self._nvml, self._h
        try:
            mx = float(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))
        except Exception:
            mx = None
        fields = os.environ.get("BENCH_NVML_FIELDS", "both")
        period = float(os.environ.get("BENCH_CLOCK_PERIOD", "0.2"))
        while not self._stop.is_set():
            try:
                sm = float(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)) if fields in ("both", "clock") else 0.0
                mask = int(nv.nvmlDeviceGetCurrentClocksEventReasons(h)) if fields in ("both", "reasons") else 0
                self.rows.append((time.monotonic(), sm, mx, {k for k, b in self.BITS.items() if mask & b}))
            except Exception:
                pass
            self._stop.wait(period)

    def _pump_smi(self):
        for line in self.proc.stdout:
            f = [x.strip() for x in line.strip().split(",")]
            if len(f) < 9:
                continue
            try:
                sm, mx = float(f[1]), float(f[2])
            except ValueError:
                continue
            reasons = {name for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown",
                                                "sw_power_cap"), f[5:9]) if v.lower().startswith("active")}
            self.rows.append((time.monotonic(), sm, mx, reasons))

    def stop(self):
        self._stop.set()
        if self.proc:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=5)
            except Exception:
                self.proc.kill()
        if self.thread is not None:
            self.thread.join(timeout=2)
        if self.thread is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["clock sampler unavailable"], "source": self.source}
        rows = [r for r in self.rows
                if self.t_begin is None or (self.t_begin <= r[0] <= (self.t_end or r[0]) + 0.25)]
        if not rows:                                   # timed region shorter than one sampling period
            rows = self.rows[-2:]
        sm = sorted(r[1] for r in rows)
        mx = [r[2] for r in rows if r[2] is not None]
        reasons = set().union(*[r[3] for r in rows]) if rows else set()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm), "source": self.source}


def run_reference(args) -> None:
    """The reference arm: the UNMODIFIED reference from baseline/_ref through its own CLI."""
    from baseline import reference_arm
    out = reference_arm.run(args)
    if "metric" in out or "unavailable" in out:      # ranks != 0 of a multi-rank run stay silent
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps(out), flush=True)


def main():
    args = parse_args()
    if args.impl == "reference":
        run_reference(args)
        return
    import torch
    import multiverso_b200 as mv
    from multiverso_b200.models.wordembedding import (WordEmbedding, WordEmbeddingOption,
                                                      synthetic_zipf_corpus)

    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world != args.gpus and world > 1:
        args.gpus = world
    if not torch.cuda.is_available():
        # the headline benchmark is a GPU measurement; say so instead of a CUDA traceback
        # (bench/cpu_apps.py measures the CPU plumbing mode)
        if int(os.environ.get("RANK", "0")) == 0:
            print(json.dumps({"metric": "wordembedding_words_per_sec", "value": None, "n_gpus": args.gpus,
                              "unavailable": "no CUDA device in this process; run on an H100"}), flush=True)
        return
    mv.init()
    rank = mv.rank()
    dev = torch.device("cuda", torch.cuda.current_device())
    K, W, B = args.steps, max(args.warmup, 3), args.block_words
    if args.metric == "matrix_bw":
        matrix_bw_main(mv, torch, world, rank, args)
        mv.shutdown()
        return

    opt = WordEmbeddingOption(embeding_size=args.dim, window_size=args.window,
                              negative_num=args.negative, init_learning_rate=0.025, sample=0.0,
                              total_words=B * (K + W) * 2 * world, epoch=1)
    if args.direct:
        os.environ["MVB_WE_MODE"] = "direct"
    we = WordEmbedding(opt, args.vocab, seed=1)

    # synthetic corpus: a distinct block per step and per rank, staged in pinned host memory
    n_blocks = K + W
    corpus = synthetic_zipf_corpus(B * n_blocks, args.vocab, sentence_len=1000, seed=17 + rank)
    pinned = torch.from_numpy(corpus).view(n_blocks, B).pin_memory()
    dev_blocks = pinned.to(dev)               # device-timed arm: tokens already resident
    words_per_block = int((corpus[:B] >= 0).sum())
    tok_dev = torch.empty(B, dtype=torch.int32, device=dev)

    def sync_all():
        torch.cuda.synchronize()
        mv.barrier()
        torch.cuda.synchronize()

    # world > 1: the reference's default pipeline (-is_pipeline 1): block i+1's PrepareData +
    # RequestParameter overlap block i's training, block i's AddDeltaParameter overlaps block i+1's.
    # Every step still issues exactly one prepare+pull, one train and one add-delta.
    pipelined = world > 1 and not args.no_pipeline and we.mode != "direct"
    blocks_list = [dev_blocks[i] for i in range(n_blocks)]        # stable tensor objects

    def step_device(i):
        we.learning_rate = opt.init_learning_rate * max(1e-4, 1.0 - i / (2.0 * n_blocks))
        we.train_block(blocks_list[i], compute_loss=True,
                       next_tokens=blocks_list[(i + 1) % n_blocks] if pipelined else None)

    # ------------------------------------------------------------ device-timed arm
    # the clock sampler (one looping nvidia-smi) is started BEFORE the warm-up so that its start-up
    # (driver enumeration, which can stall kernel launches for milliseconds) is not inside the timed
    # region; only the rows received during the timed region are used, and it is killed after.
    sampler = ClockSampler(torch.cuda.current_device(), source="nvml")
    if rank == 0:
        sampler.start()
    for i in range(W):
        step_device(i)
    sync_all()
    mv.Dashboard.reset()
    launches0 = we.kernel_launches
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler.mark_begin()
    trace_dev = os.environ.get("BENCH_TRACE") == "1" and world > 1
    if trace_dev:
        we.trace = []
    ev0.record()
    for i in range(K):
        step_device(W + i)
    we.flush()                      # pipelined mode: the last block's AddDeltaParameter is part of the K steps
    ev1.record()
    torch.cuda.synchronize()
    sampler.mark_end()
    device_trace = None
    if trace_dev:
        tr, we.trace = we.trace, None
        device_trace = {"k7_ms": [round(a.elapsed_time(b), 3) for a, b in tr],
                        "gap_ms": [round(tr[j][1].elapsed_time(tr[j + 1][0]), 3) for j in range(len(tr) - 1)],
                        "first_start_ms": round(ev0.elapsed_time(tr[0][0]), 3), "tail_ms": round(tr[-1][1].elapsed_time(ev1), 3)}
    ms_local = ev0.elapsed_time(ev1)
    launches = we.kernel_launches - launches0
    sync_all()
    clocks = sampler.stop() if rank == 0 else None
    monitors = mv.Dashboard.snapshot()
    pairs = int(we.pairs.item())
    loss_per_pair = float(we.loss.item()) / max(pairs, 1)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, we, torch)

    # ------------------------------------------------------------ end-to-end arm
    # Through the public API, every step: one H2D copy of a block of inputs from pinned host memory and
    # one D2H read of the step's loss into pinned host memory, consumed on the host.  Both are
    # software-pipelined the way a training loop does it: the loss of step i is read (event wait +
    # float()) while step i+1 runs, and in pipelined mode the block copied during step i is step i+1's.
    we2_steps = K
    we.flush()
    sync_all()
    we._prefetched = None
    E2E_WARM = 2                                     # untimed iterations of the SAME loop (pipeline primed)
    # debugging knobs (never set for a reported number): which part of the e2e loop costs what
    DBG_NO_H2D = os.environ.get("BENCH_E2E_NO_H2D") == "1"
    DBG_NO_D2H = os.environ.get("BENCH_E2E_NO_D2H") == "1"
    DBG_NO_SYNC = os.environ.get("BENCH_E2E_NO_SYNC") == "1"
    tok2 = [tok_dev, torch.empty_like(tok_dev)]
    loss_pin = [torch.zeros(1, dtype=torch.float32).pin_memory() for _ in range(2)]
    loss_ev = [torch.cuda.Event(), torch.cuda.Event()]
    losses_host = []
    copy_stream = torch.cuda.Stream(device=dev)      # the H2D copy of block i+1 runs under block i's training
    main_stream = torch.cuda.current_stream()
    tok2[0].copy_(pinned[W + (-E2E_WARM) % K], non_blocking=True)      # the first warm-up block
    copied = torch.cuda.Event()
    copied.record()
    sync_all()
    step_ev = [torch.cuda.Event(enable_timing=True) for _ in range(we2_steps + 1)]
    done_ev = torch.cuda.Event()                     # end of the previous iteration's work on the main stream
    done_ev.record()
    host_t = []
    t0 = time.perf_counter()
    for i in range(-E2E_WARM, we2_steps):
        if i == 0:
            torch.cuda.synchronize()                 # the primed pipeline (prefetched block, copied tokens) survives this
            if world > 1:
                mv.barrier()
            t0 = time.perf_counter()
            step_ev[0].record()
            done_ev = step_ev[0]
        we.loss.zero_()
        cur, nxt = tok2[i % 2], tok2[(i + 1) % 2]
        cur_copied = copied
        # H2D of one block of inputs per step: block i+1, from pinned host memory, on the copy stream; its
        # buffer was last read by block i-1, i.e. before `done_ev`
        copy_stream.wait_event(done_ev)
        with torch.cuda.stream(copy_stream):
            if not DBG_NO_H2D:
                nxt.copy_(pinned[W + (i + 1) % K], non_blocking=True)
            copied = torch.cuda.Event()
            copied.record(copy_stream)
        main_stream.wait_event(cur_copied)           # this step's tokens are on the device
        if pipelined:
            we.train_block(cur, compute_loss=True, next_tokens=nxt, next_ready=copied)
        else:
            we.train_block(cur, compute_loss=True)
        if not DBG_NO_D2H:
            loss_pin[i % 2].copy_(we.loss, non_blocking=True)    # D2H of the step's result
        loss_ev[i % 2].record()
        if i >= 0:
            step_ev[i + 1].record()
            done_ev = step_ev[i + 1]
            host_t.append(time.perf_counter() - t0)
        else:
            done_ev = torch.cuda.Event()
            done_ev.record()
        if i > 0 and not DBG_NO_SYNC:                            # consume step i-1's loss on the host
            loss_ev[(i - 1) % 2].synchronize()
            losses_host.append(float(loss_pin[(i - 1) % 2]))
    loss_ev[(we2_steps - 1) % 2].synchronize()
    losses_host.append(float(loss_pin[(we2_steps - 1) % 2]))
    torch.cuda.synchronize()
    e2e_s_local = time.perf_counter() - t0
    assert DBG_NO_SYNC or (len(losses_host) == we2_steps and all(l == l for l in losses_host))
    e2e_trace = {"gpu_step_ms": [round(step_ev[i].elapsed_time(step_ev[i + 1]), 2) for i in range(we2_steps)],
                 "host_enqueue_done_ms": [round(t * 1e3, 2) for t in host_t],
                 "total_ms": round(e2e_s_local * 1e3, 2)}
    sync_all()

    # ------------------------------------------------------------ reduce over ranks (max time)
    t = torch.tensor([ms_local, e2e_s_local * 1e3], dtype=torch.float64, device=dev)
    if world > 1:
        import torch.distributed as dist
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_total, e2e_ms_total = float(t[0]), float(t[1])
    total_words = words_per_block * K * world
    value = total_words / (ms_total / 1e3)
    e2e_value = total_words / (e2e_ms_total / 1e3)

    extra = {}
    if not args.no_table_bw:
        extra = table_bandwidth(mv, torch, world)

    if rank == 0:
        out = {
            "metric": METRIC, "value": value, "unit": "words/s", "n_gpus": world, "steps": K,
            "warmup": W, "ms_per_step": ms_total / K, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "dtype": "fp32", "data": "synthetic", "impl": "ours",
            "config": {"model": CONFIG_MODEL, "global_batch": B * world, "seq_len": 1000,
                       "parallelism": (f"dp{world} row-sharded PS tables" + (", pipelined pull/push (-is_pipeline 1)" if pipelined else "")) if world > 1 else "1 GPU (worker+server)",
                       "block_words_per_gpu": B, "l2": "tables 2.4 GB >> 50 MB L2; new token block every step",
                       "pairs_per_word": pairs / max(1, words_per_block * (K + W)),
                       "loss_per_pair": loss_per_pair},
            "clocks": clocks,
            "e2e": {"value": e2e_value, "unit": "words/s", "h2d_bytes_per_step": B * 4,
                    "d2h_bytes_per_step": 4, "ms_per_step": e2e_ms_total / K,
                    "note": "every step: H2D of one block of tokens from pinned host memory (copy stream, the block copied in "
                            "step i is step i+1's) and D2H of the step's loss into pinned host memory, consumed on the host "
                            "during step i+1; 2 untimed warm-up iterations of the same loop"},
            "gpu_launches": launches,
            "extra": dict(extra, monitors_device_arm=monitors, e2e_trace_rank0=e2e_trace,
                          **({"device_trace_rank0": device_trace} if device_trace else {})),
        }
        if "get_plus_add_gbs" in extra:
            # second half of the BASELINE.json metric, same key in the reference arm's line
            out["secondary"] = secondary_block(extra, world)
        print(json.dumps(out), flush=True)
    mv.shutdown()


DUMP_HOT_ROWS = 1024          # the most frequent words of the Zipf corpus: the rows every step updates
DUMP_SAMPLED_ROWS = 16384     # plus a fixed random sample of the rest; 2 tables x ~17k rows x 300 x 4 B = 41 MB


def dump_outputs(out_dir, we, torch):
    """Write what the timed steps hand back to a caller of train_block: the loss and pair
    count summed over all steps so far, and both embedding tables after the last step.  The tables hold vocab x dim floats each, so a
    fixed, seeded set of rows is written (the hottest rows + a uniform sample), capped at 64 MB in all."""
    import numpy as np
    hot = np.arange(min(DUMP_HOT_ROWS, we.V))
    rng = np.random.default_rng(2024)
    ids = np.union1d(hot, rng.choice(we.V, size=min(DUMP_SAMPLED_ROWS, we.V), replace=False))
    ids = ids[:max(1, (60 << 20) // (2 * 4 * we.D))]
    rows = torch.from_numpy(ids).to(we.dev)
    arrays = {"loss_cumulative": we.loss.double(), "pairs_cumulative": we.pairs.double(), "row_ids": rows.double(),
              "input_embedding_rows": we.input_table.get_rows(rows)[:, :we.D].float(),
              "output_embedding_rows": we.output_table.get_rows(rows)[:, :we.D].float()}
    os.makedirs(out_dir, exist_ok=True)
    for name, a in arrays.items():
        np.save(os.path.join(out_dir, name + ".npy"), a.cpu().numpy())


def secondary_block(extra, world):
    return {"metric": "matrix_table_get_plus_add_gbs", "value": extra["get_plus_add_gbs"], "unit": "GB/s",
            "higher_is_better": True, "add_ms": extra["add_ms"], "get_ms": extra["get_ms"],
            "add_gbs": extra["add_gbs"], "get_gbs": extra["get_gbs"], "iters": 5,
            "config": {"table": "MatrixTable 1000000x512 fp32, whole-table Add (sgd updater fused) + whole-table Get",
                       "parallelism": f"{world} GPU(s), row-sharded, fused P2P kernels (no NCCL on the path)",
                       "timing": "CUDA events, max over ranks; 2.05 GB table >> 50 MB L2",
                       "staging": "Add reads the delta from the table's zero-copy symmetric staging buffer "
                                  "(table.staging()); an Add from an ordinary tensor pays one extra local copy"}}


def matrix_bw_main(mv, torch, world, rank, args):
    """`--metric matrix_bw`: BASELINE.json config 2 as the primary line (same JSON contract)."""
    sampler = ClockSampler(torch.cuda.current_device(), source="nvml")
    if rank == 0:
        sampler.start()
    sampler.mark_begin()
    extra = table_bandwidth(mv, torch, world)
    sampler.mark_end()
    clocks = sampler.stop() if rank == 0 else None
    # end to end through the public API: the delta comes from pinned host memory, the pulled table goes back
    # to pinned host memory, every iteration
    rows, cols = 1_000_000, 512
    e2e = None
    try:
        t = mv.MatrixTable(rows, cols, "float32", updater="sgd")
        host_delta = torch.full((rows * cols,), 1e-3).pin_memory()
        host_out = torch.empty(rows * cols).pin_memory()
        dev_delta = torch.empty(rows * cols, device="cuda")
        dev_out = torch.empty(rows * cols, device="cuda")
        n = 3
        for it in range(n + 1):
            if it == 1:
                torch.cuda.synchronize(); mv.barrier()
                import time as _t
                t0 = _t.perf_counter()
            dev_delta.copy_(host_delta, non_blocking=True)
            t.add(dev_delta)
            t.get(dev_out)
            host_out.copy_(dev_out, non_blocking=True)
            torch.cuda.synchronize()
        ms = torch.tensor([(_t.perf_counter() - t0) * 1e3 / n], dtype=torch.float64, device="cuda")
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        e2e = {"value": 2 * rows * cols * 4 / float(ms) / 1e6, "unit": "GB/s", "h2d_bytes_per_step": rows * cols * 4,
               "d2h_bytes_per_step": rows * cols * 4, "ms_per_step": float(ms),
               "note": "delta from pinned host memory (H2D), Add, Get, table back to pinned host memory (D2H): PCIe bound"}
    except Exception as e:   # noqa: BLE001
        e2e = {"error": repr(e)[:200]}
    if rank == 0:
        out = {"metric": "matrix_table_get_plus_add_gbs", "value": extra.get("get_plus_add_gbs"), "unit": "GB/s",
               "n_gpus": world, "steps": 5, "warmup": 2, "ms_per_step": (extra.get("add_ms", 0) + extra.get("get_ms", 0)),
               "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
               "impl": "ours", "config": secondary_block(extra, world)["config"] if "get_plus_add_gbs" in extra else {},
               "clocks": clocks, "e2e": e2e, "gpu_launches": 14, "extra": extra}
        print(json.dumps(out), flush=True)


def table_bandwidth(mv, torch, world):
    """BASELINE config 2: MatrixTable 1M x 512 fp32 whole-table Get and Add (fused updater),
    device-timed, table bytes / time, max over ranks."""
    rows, cols = 1_000_000, 512
    out = {}
    try:
        t = mv.MatrixTable(rows, cols, "float32", updater="sgd")
        nbytes = rows * cols * 4
        delta = t.staging() if world > 1 else torch.full((rows * cols,), 1e-3, device="cuda")
        if world > 1:
            delta.fill_(1e-3)
        buf = torch.empty(rows * cols, device="cuda")
        res = {}
        for name in ("add", "get"):
            for it in range(2):
                (t.add(delta, staged=world > 1) if name == "add" else t.get(buf))
                if world > 1 and name == "add":
                    delta = t.staging()
            torch.cuda.synchronize()
            mv.barrier()
            n = 5
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            handles = []
            for it in range(n):                      # enqueue back to back: device time, not host round trips
                if name == "add":
                    handles.append(t.add_async(delta, staged=world > 1))
                    if world > 1:
                        delta = t.staging()
                else:
                    handles.append(t.get_async(buf)[0])
            e1.record()
            for h in handles:
                t.wait(h)
            torch.cuda.synchronize()
            ms = torch.tensor([e0.elapsed_time(e1) / n], dtype=torch.float64, device="cuda")
            if world > 1:
                import torch.distributed as dist
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
            res[name] = float(ms)
            mv.barrier()
        out = {"matrix_table": f"{rows}x{cols} fp32", "add_ms": res["add"], "get_ms": res["get"],
               "add_gbs": nbytes / res["add"] / 1e6, "get_gbs": nbytes / res["get"] / 1e6,
               "get_plus_add_gbs": 2 * nbytes / (res["add"] + res["get"]) / 1e6}
    except Exception as e:  # the headline metric must still print
        out = {"error": repr(e)[:200]}
    return out


if __name__ == "__main__":
    main()
