#!/usr/bin/env python
"""Fused cosine top-k (topk_cos.cu) against the unfused paths, device-timed with CUDA events.

Table: 1M x 300 fp32 MatrixTable (the word2vec vocabulary / dimension of the reference's WordEmbedding
numbers). For M in {1, 16, 256, 4096, 19544} queries (19,544 = the standard analogy question set), k = 10:

  fused     mv.ops.topk_cosine: one pass over the table, scores never written
  get_gemm  mv.ops.get_gemm into a chunked score buffer (512 queries x 1M), then torch.topk
  get_mm    Get of the whole table, then torch.matmul (tf32) into the same buffer, then torch.topk

(the unfused paths rank raw dot products of pre-normalised rows, which is the cosine ranking). Reported per
M: time, table bytes / time, 2 M V dim / time, and the share of the larger of the two bounds (HBM 3.35 TB/s,
tf32 495 TFLOP/s, H100 SXM data sheet), naming the bound. Then a cross-check of the fused ids against the
unfused ones outside near-ties, and one end-to-end analogy evaluation of 19,544 synthetic questions at
threshold 30,000 and over the whole vocabulary. Prints one JSON line; ``--out FILE`` also writes it there.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.ops import get_gemm, topk_cosine
from multiverso_b200.ops.topk import analogy_queries, take_excluding

HBM_BPS, TF32_FLOPS = 3.35e12, 495e12
SCORE_CHUNK = 512


def timed(fn, iters, warmup=1):
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=300)
    ap.add_argument("--ms", default="1,16,256,4096,19544")
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench/topk_cosine.py measures the GPU kernel: no CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = True
    mv.init()
    V, D, k = a.rows, a.dim, a.k
    t = mv.MatrixTable(V, D, "float32", min_value=-1.0, max_value=1.0)
    W = t.shard.view(V, D)
    W.div_(W.norm(dim=1, keepdim=True))               # unit rows: dot-product ranking == cosine ranking
    torch.cuda.synchronize()
    wbuf = torch.empty(V * D, device="cuda")
    scores = torch.empty(SCORE_CHUNK, V, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(0)
    res = {"gpu": gpu_info(), "table": [V, D], "k": k, "results": []}

    def unfused(q, mode):
        outs, outi = [], []
        if mode == "get_mm":
            t.get(wbuf)
        for lo in range(0, q.shape[0], SCORE_CHUNK):
            qc = q[lo:lo + SCORE_CHUNK]
            y = scores[:qc.shape[0]]
            if mode == "get_gemm":
                get_gemm(t, qc, y)
            else:
                torch.matmul(qc, wbuf.view(V, D).t(), out=y)
            s, i = y.topk(k, dim=1)
            outs.append(s)
            outi.append(i)
        return torch.cat(outs), torch.cat(outi)

    for M in [int(x) for x in a.ms.split(",")]:
        q = torch.randn(M, D, device="cuda", generator=g)
        q = q / q.norm(dim=1, keepdim=True)
        iters = max(2, min(50, int(2000 / max(M, 1) + 2)))
        row = {"M": M}
        row["fused_ms"] = timed(lambda: topk_cosine(t, q, k), iters)
        row["get_gemm_topk_ms"] = timed(lambda: unfused(q, "get_gemm"), max(2, iters // 4))
        row["get_matmul_topk_ms"] = timed(lambda: unfused(q, "get_mm"), max(2, iters // 4))
        tbytes, flops = V * D * 4, 2.0 * M * V * D
        t_mem, t_mma = tbytes / HBM_BPS * 1e3, flops / TF32_FLOPS * 1e3
        for name in ("fused", "get_gemm_topk", "get_matmul_topk"):
            ms = row[f"{name}_ms"]
            row[f"{name}_table_GBps"] = tbytes / ms / 1e6
            row[f"{name}_TFLOPs"] = flops / ms / 1e9
        row["bound"] = "hbm" if t_mem >= t_mma else "tf32"
        row["fused_share_of_bound"] = max(t_mem, t_mma) / row["fused_ms"]
        # cross-check: fused ids against the get_gemm path, outside near-ties (tf32 scores of the unfused
        # path move by ~1e-3 at most)
        fs, fi = topk_cosine(t, q, k)
        us, ui = unfused(q, "get_gemm")
        kth = us[:, -1:]
        ref = (q.double() @ W.double().T) if M <= 256 else None
        agree = (fi.sort(1).values == ui.sort(1).values).all(1)
        ok = agree.clone()
        if ref is not None:
            exact_kth = ref.topk(k, dim=1).values[:, -1:]
            only = ~(fi[:, :, None] == ui[:, None, :]).any(2)
            near = (ref.gather(1, fi) - exact_kth).abs() < 2e-3
            ok = agree | (only <= near).all(1)
        else:
            only = ~(fi[:, :, None] == ui[:, None, :]).any(2)
            ok = agree | (only <= ((fs - kth).abs() < 2e-3)).all(1)
        row["ids_equal_rows"] = int(agree.sum())
        row["ids_agree_outside_near_ties"] = int(ok.sum())
        res["results"].append(row)
        print(json.dumps(row), flush=True)
        del q, fs, fi, us, ui
    # end to end: 19,544 synthetic analogy questions (ids drawn from the first 30,000 words)
    nq = 19544
    ids = torch.randint(0, 30000, (nq, 3), device="cuda", generator=g)
    e2e = {}
    for thr in (30000, V):
        def run():
            qq = analogy_queries(W[ids[:, 0]], W[ids[:, 1]], W[ids[:, 2]])
            s, i = topk_cosine(t, qq, 4, rows=thr)
            return take_excluding(s, i, ids, 1)
        run()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        run()
        torch.cuda.synchronize()
        e2e[f"analogy_{nq}_threshold_{thr}_s"] = time.perf_counter() - t0
    res["end_to_end"] = e2e
    print(json.dumps(e2e), flush=True)
    line = json.dumps(res)
    print(line, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    t.free()
    mv.shutdown()


if __name__ == "__main__":
    main()
