"""GraphEmbedding over several GPUs, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tests/mp_graph_embedding_check.py

Every rank's walks for the blocks dealt to it (block b to rank b mod size) must equal random_walks_reference bitwise,
and training a stochastic-block-model graph through the block protocol, with -is_pipeline on and off, must reach the
neighbour-purity threshold of the single-GPU test.
"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import multiverso_b200 as mv
from multiverso_b200.models.graph_embedding import GraphEmbedding
from multiverso_b200.models.wordembedding import WordEmbeddingOption
from multiverso_b200.ops import Graph, random_walks_reference
from test_gpu_graph_embedding import _sbm

results = {}


def check(name, cond, info=""):
    results[name] = bool(cond)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def main():
    mv.init()
    rank, size = mv.rank(), mv.size()
    n, bsize, src, dst, _, _ = _sbm()
    g = Graph.from_edges(src, dst, num_nodes=n)
    for pipeline in (True, False):
        opt = WordEmbeddingOption(embeding_size=64, window_size=5, negative_num=5, init_learning_rate=0.025,
                                  data_block_size=1 << 18, is_pipeline=pipeline)
        ge = GraphEmbedding(g, opt, walk_length=40, walks_per_node=10, p=0.5, q=2.0, seed=3)
        if pipeline:
            mine = [blk for blk in ge.schedule(1) if blk[0] % size == rank]
            check("deal", len(mine) > 1 and all(b % size == rank for b, *_ in mine))
            out = torch.empty(ge.block_walks, ge.L + 1, dtype=torch.int32, device="cuda")
            for b, e, j, lo, hi in mine[:6]:
                perm = ge.permutation(e, j)
                ge.walk_block(perm, e, j, lo, hi, out)
                ref = random_walks_reference(g, perm[lo:hi], ge.L, ge.p, ge.q, ge.seed, ge.first_walk(e, j, lo))
                check(f"walks_{b}", np.array_equal(out[:hi - lo, :ge.L].cpu().numpy(), ref)
                      and bool((out[:hi - lo, ge.L] == -1).all()))
        stats = ge.train()
        _, ids = ge.embedding.most_similar(torch.arange(n), k=10)
        purity = float(((ids.cpu() // bsize) == (torch.arange(n)[:, None] // bsize)).float().mean())
        print(f"[rank {rank}] pipeline={pipeline} purity {purity:.4f} {json.dumps(stats)}", flush=True)
        check(f"purity_pipeline_{pipeline}", purity > 0.85, purity)
        mv.barrier()
    ok = all(results.values())
    print(f"[rank {rank}] {'PASS' if ok else 'FAIL'} {sum(results.values())}/{len(results)}", flush=True)
    mv.shutdown()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
