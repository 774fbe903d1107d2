"""Graph walker and DeepWalk / node2vec training throughput on one GPU.

    python bench/graph_embedding.py [--nodes 4000000] [--degree 32] [--length 80] [--blocks 200]

The graph is a seeded Chung-Lu power-law graph generated on the device (expected degrees proportional to
(i + 1)^(-1/(gamma - 1)), gamma = 2.5, scaled to the average degree; nodes * degree / 2 undirected edges whose
endpoints are drawn from that distribution), so nothing is downloaded. Reported, with the GPU's name, power limit
and SM clock read in the same run:

* walker steps/s (CUDA events over several launches after a warm-up, one walk from every node per launch) for
  DeepWalk and for node2vec at (p, q) = (0.25, 4);
* end-to-end tokens/s of walking + training (skip-gram, K = 5, dim 128, window 10, the app's defaults) over
  ``--blocks`` blocks, against training alone on the same blocks walked beforehand; the walker's share is
  1 - train-only time / walk + train time.

Prints one JSON line per measurement.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def chung_lu(n, degree, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.arange(1, n + 1, device=dev, dtype=torch.float64)) ** (-1.0 / 1.5)
    cdf = torch.cumsum(w / w.sum(), 0)
    m = n * degree // 2
    src = torch.searchsorted(cdf, torch.rand(m, device=dev, dtype=torch.float64, generator=g)).clamp(max=n - 1)
    dst = torch.searchsorted(cdf, torch.rand(m, device=dev, dtype=torch.float64, generator=g)).clamp(max=n - 1)
    perm = torch.randperm(n, device=dev, generator=g)          # hubs spread over the id range
    return perm[src], perm[dst]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=4_000_000)
    ap.add_argument("--degree", type=int, default=32)
    ap.add_argument("--length", type=int, default=80)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--blocks", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench/graph_embedding.py needs a GPU")
    import multiverso_b200 as mv
    from multiverso_b200.models.graph_embedding import GraphEmbedding
    from multiverso_b200.models.wordembedding import WordEmbeddingOption
    from multiverso_b200.ops.random_walk import Graph, launch_walks
    dev = torch.device("cuda", 0)
    info = gpu_info()
    src, dst = chung_lu(args.nodes, args.degree, 1, dev)
    g = Graph.from_edges(src, dst, num_nodes=args.nodes)
    del src, dst
    L = args.length
    starts = torch.arange(g.num_nodes, dtype=torch.int32, device=dev)
    out = torch.empty(g.num_nodes, L + 1, dtype=torch.int32, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    for name, p, q in (("deepwalk", 1.0, 1.0), ("node2vec", 0.25, 4.0)):
        launch_walks(g, starts, out, L, p, q, 1, 0, cnt)          # warm-up
        torch.cuda.synchronize()
        cnt.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.iters):
            launch_walks(g, starts, out, L, p, q, 1, (i + 1) * g.num_nodes, cnt)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        steps = int(cnt.item()) - args.iters * g.num_nodes      # transitions: nodes written minus the starts
        print(json.dumps({"bench": "walker", "walk": name, "p": p, "q": q, "nodes": g.num_nodes, "arcs": g.num_arcs,
                          "length": L, "ms_per_launch": ms / args.iters, "steps_per_sec": steps / (ms / 1e3),
                          "gpu": info}), flush=True)
    del out
    mv.init()
    try:
        opt = WordEmbeddingOption(embeding_size=128, window_size=10, negative_num=5, init_learning_rate=0.025)
        ge = GraphEmbedding(g, opt, walk_length=L, walks_per_node=10, seed=1)
        blocks = ge.schedule(1)[:args.blocks]
        bufs = torch.empty(len(blocks), ge.block_walks, L + 1, dtype=torch.int32, device=dev)
        perm = ge.permutation(0, 0)
        we = ge.embedding
        tokens = 0
        for k, (_, e, j, lo, hi) in enumerate(blocks):      # pre-generated walks of the same blocks
            ge.walk_block(perm, e, j, lo, hi, bufs[k])
            tokens += (hi - lo) * (L + 1)
        we.train_block(bufs[0].view(-1))                     # warm-up
        torch.cuda.synchronize()

        def run(walk):
            t0 = time.time()
            for k, (_, e, j, lo, hi) in enumerate(blocks):
                if walk:
                    ge.walk_block(perm, e, j, lo, hi, bufs[k])
                we.train_block(bufs[k][:hi - lo].view(-1), compute_loss=False)
            torch.cuda.synchronize()
            return time.time() - t0
        t_both, t_train = [], []
        for _ in range(2):                                   # alternated, best of two
            t_both.append(run(True))
            t_train.append(run(False))
        tb, tt = min(t_both), min(t_train)
        print(json.dumps({"bench": "end_to_end", "nodes": g.num_nodes, "length": L, "blocks": len(blocks),
                          "walks_per_block": ge.block_walks, "tokens": tokens, "walk_train_tokens_per_sec": tokens / tb,
                          "train_only_tokens_per_sec": tokens / tt, "walker_share": max(0.0, 1 - tt / tb),
                          "gpu": info}), flush=True)
    finally:
        mv.shutdown()


if __name__ == "__main__":
    main()
