"""GraphEmbedding: DeepWalk / node2vec node embeddings, random walks on the device fed straight into the skip-gram
trainer (``WordEmbedding``) with node ids as words.

    g, labels = mv.ops.Graph.load("edges.txt")
    ge = GraphEmbedding(g, WordEmbeddingOption(embeding_size=128, window_size=10), walk_length=80,
                        walks_per_node=10, p=1, q=1, seed=1)
    ge.train()
    ge.save_embedding("vec.txt", labels)      # word2vec format keyed by the original labels

**Counts.** The word counts of node v are its (weighted) out-degree: the stationary visit frequencies of a first-order
walk on an undirected graph, i.e. what counting the corpus would give. They set the unigram^0.75 negative distribution
and the hot-row cap. An isolated node has count 0: the alias table gives it probability 0 and it is never drawn as a
negative.

**Dealing.** Pass j (0 <= j < walks_per_node) of epoch e walks every node once, in the order of the permutation
``perm_{e,j}``: the stable ascending argsort of ``hash64(pk + node * 0xBF58476D1CE4E5B9)`` as int64, with
``pk = hash64(hash64(hash64(seed ^ 0xD6E8FEB86659FD93) + e) + j)`` (``hash64`` of ``ops.random_walk``). Walk i of the
pass has the global number ``g = (e * walks_per_node + j) * N + i`` and starts at ``perm_{e,j}[i]``. A pass is cut into
blocks of B walks (the last one shorter), with B (L + 1) about ``data_block_size / 6`` tokens as the word-embedding
app's blocks, and block b (counted over passes and epochs) goes to rank b mod size, as ``BlockLoader`` deals. A
block's rows have the pitch L + 1, so each walk ends in a -1 sentence break and the rows are the trainer's token
block as they are. The corpus is therefore the same at every world size, and each rank's walks are pure functions of
the seed.

**Training.** ``total_words`` = N walks_per_node L sets the learning-rate schedule. The kernel adds each block's node
count to a device counter; the trainer reads it at its periodic word-count sync (every 20 blocks), not once per
block. With ``is_pipeline`` on more than one GPU the next block is walked on a side stream while the current one
trains, and handed over through ``train_block(next_tokens=..., next_ready=...)``.

Memory: the CSR (8 B per node, 4 B per arc, 8 B more per arc when weighted) and two token blocks, besides the
trainer's tables.
"""
from __future__ import annotations

import time
from typing import List, Optional, Tuple

import numpy as np
import torch

from ..ops.random_walk import Graph, _check_walk_args, hash64, hash64_torch, launch_walks
from ..runtime import Runtime
from .wordembedding import WordEmbedding, WordEmbeddingOption

_SYNC_BLOCKS = 20          # word-count sync period of the word-embedding app


class GraphEmbedding:
    """Node embeddings of ``graph`` (a :class:`~multiverso_b200.ops.Graph` on this rank's GPU) trained by skip-gram
    on random walks (see the module docstring). ``embedding`` is the underlying ``WordEmbedding`` (V = N)."""

    def __init__(self, graph: Graph, option: WordEmbeddingOption, walk_length: int = 80, walks_per_node: int = 10,
                 p: float = 1.0, q: float = 1.0, seed: int = 1):
        rt = Runtime.get()
        if rt.backend != "device" or graph.device.type != "cuda":
            raise RuntimeError("GraphEmbedding needs the device backend and a graph on the GPU")
        _check_walk_args(graph, torch.zeros(0, dtype=torch.int32), walk_length, p, q, 0)
        if int(walks_per_node) != walks_per_node or walks_per_node < 1:
            raise ValueError(f"GraphEmbedding: walks_per_node must be a positive integer, got {walks_per_node}")
        counts = graph.degree().to(torch.float64).cpu().numpy()
        if not counts.sum() > 0:
            raise ValueError("GraphEmbedding: the graph has no arcs")
        self.rt, self.graph, self.opt = rt, graph, option
        self.N, self.L, self.walks_per_node = graph.num_nodes, int(walk_length), int(walks_per_node)
        self.p, self.q, self.seed = float(p), float(q), int(seed)
        option.total_words = self.N * self.walks_per_node * self.L
        self.embedding = WordEmbedding(option, self.N, counts, seed=self.seed)
        self.block_walks = max(1, max(1024, int(option.data_block_size) // 6) // (self.L + 1))
        self.dev = self.embedding.dev

    # ------------------------------------------------------------------------------------------------ corpus
    def permutation(self, epoch: int, j: int) -> torch.Tensor:
        """perm_{epoch,j}: the start node of every walk of pass j of the epoch (int64 [N], on the GPU)."""
        s = hash64(np.uint64(self.seed & 0xFFFFFFFFFFFFFFFF) ^ np.uint64(0xD6E8FEB86659FD93))
        with np.errstate(over="ignore"):
            pk = hash64(hash64(s + np.uint64(epoch)) + np.uint64(j))
        nodes = torch.arange(self.N, dtype=torch.int64, device=self.dev)
        key = hash64_torch(nodes * -0x40A7B892E31B1A47 + int(pk.view(np.int64)))    # 0xBF58476D1CE4E5B9 as int64
        return torch.sort(key, stable=True).indices

    def schedule(self, epochs: int) -> List[Tuple[int, int, int, int, int]]:
        """Every block of ``epochs`` epochs in order: (block, epoch, pass, lo, hi), walks [lo, hi) of the pass."""
        out, b = [], 0
        for e in range(epochs):
            for j in range(self.walks_per_node):
                for lo in range(0, self.N, self.block_walks):
                    out.append((b, e, j, lo, min(self.N, lo + self.block_walks)))
                    b += 1
        return out

    def first_walk(self, epoch: int, j: int, lo: int) -> int:
        return (epoch * self.walks_per_node + j) * self.N + lo

    def walk_block(self, perm: torch.Tensor, epoch: int, j: int, lo: int, hi: int, out: torch.Tensor,
                   node_count: Optional[torch.Tensor] = None) -> None:
        """Walks [lo, hi) of pass j into the rows of ``out`` ([>= hi - lo, >= L] int32) on the current stream."""
        starts = perm[lo:hi].to(torch.int32)
        launch_walks(self.graph, starts, out[:hi - lo], self.L, self.p, self.q, self.seed,
                     self.first_walk(epoch, j, lo), node_count)

    # ------------------------------------------------------------------------------------------------ training
    def train(self, epochs: Optional[int] = None) -> dict:
        """Train on this rank's blocks of ``epochs`` (default ``option.epoch``) epochs. Returns this rank's walks,
        tokens (nodes walked), seconds, tokens/s and the walker's share of the GPU time of walking plus training."""
        epochs = int(self.opt.epoch if epochs is None else epochs)
        rank, size = self.rt.rank, max(self.rt.size, 1)
        we, L, dev = self.embedding, self.L, self.dev
        pipelined = bool(self.opt.is_pipeline) and size > 1
        main = torch.cuda.current_stream()
        walker = torch.cuda.Stream(device=dev) if pipelined else main
        bufs = [torch.empty(self.block_walks, L + 1, dtype=torch.int32, device=dev) for _ in range(2)]
        counts = torch.zeros(2, dtype=torch.int64, device=dev)
        total = torch.zeros(1, dtype=torch.int64, device=dev)
        free = [None, None]
        perms = {}
        timing = []
        mine = [blk for blk in self.schedule(epochs) if blk[0] % size == rank]
        t0 = time.time()

        def produce(k):
            _, e, j, lo, hi = mine[k]
            slot = k & 1
            if (e, j) not in perms:
                perms.clear()
                with torch.cuda.stream(walker):
                    perms[(e, j)] = self.permutation(e, j)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            with torch.cuda.stream(walker):
                if free[slot] is not None:
                    walker.wait_event(free[slot])
                counts[slot].zero_()
                ev[0].record(walker)
                self.walk_block(perms[(e, j)], e, j, lo, hi, bufs[slot], counts[slot:slot + 1])
                ev[1].record(walker)
            return bufs[slot][:hi - lo].view(-1), slot, ev

        counted = 0

        def sync_count():
            nonlocal counted
            n = int(total.item())
            we.add_word_count(n - counted)
            counted = n
            we.get_word_count()

        cur = produce(0) if mine else None
        for k in range(len(mine)):
            nxt = produce(k + 1) if k + 1 < len(mine) else None
            tokens, slot, ev = cur
            main.wait_event(ev[1])
            we.update_learning_rate()
            tr = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            tr[0].record(main)
            we.train_block(tokens, compute_loss=(k % 50 == 0),
                           next_tokens=nxt[0] if (pipelined and nxt is not None) else None,
                           next_ready=nxt[2][1] if (pipelined and nxt is not None) else None)
            tr[1].record(main)
            total.add_(counts[slot])
            free[slot] = torch.cuda.Event()
            free[slot].record(main)
            timing.append((ev, tr))
            if (k + 1) % _SYNC_BLOCKS == 0:
                sync_count()
            cur = nxt
        we.flush()
        sync_count()
        torch.cuda.synchronize()
        elapsed = time.time() - t0
        walk_ms = sum(e[0].elapsed_time(e[1]) for e, _ in timing)
        train_ms = sum(t[0].elapsed_time(t[1]) for _, t in timing)
        walks = sum(hi - lo for _, _, _, lo, hi in mine)
        return {"nodes": self.N, "walks": walks, "tokens": counted, "seconds": elapsed,
                "tokens_per_sec": counted / max(elapsed, 1e-9),
                "walk_share": walk_ms / max(walk_ms + train_ms, 1e-9), "rank": rank}

    # ------------------------------------------------------------------------------------------------ results
    def embeddings(self) -> torch.Tensor:
        """The node embeddings [N, D] (the input table)."""
        return self.embedding.embeddings()

    def save_embedding(self, path: str, labels=None, binary: bool = False) -> None:
        """word2vec text / binary format keyed by ``labels[i]`` for node i (default: the node ids); rank 0 only."""
        words = None if labels is None else [str(int(x)) for x in np.asarray(labels)]
        self.embedding.save_embedding(path, words, binary=binary)
