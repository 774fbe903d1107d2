"""The ``graph_embedding`` application: DeepWalk / node2vec node embeddings of an edge-list file.

    python -m multiverso_b200.apps.graph_embedding -graph edges.txt -directed 0 -weighted 0 \
        -walk_length 80 -walks_per_node 10 -p 1 -q 1 -size 128 -window 10 -negative 5 \
        -alpha 0.025 -epoch 1 -output vec.txt -binary 0 -seed 1
    torchrun --nproc-per-node 8 -m multiverso_b200.apps.graph_embedding ...      (8 GPUs)

The word2vec flags mean what they mean for ``wordembedding`` and are parsed the same way (``-cbow``, ``-hs``,
``-use_adagrad``, ``-data_block_size`` and ``-is_pipeline`` pass through); the defaults here are skip-gram with 5
negatives, dim 128 and window 10, which run on the deterministic skip-gram kernel. Every rank reads the edge list,
holds the whole graph on its GPU and walks its share of the blocks (models/graph_embedding.py); rank 0 writes the
embeddings keyed by the file's node labels, which ``wordembedding_eval -neighbours`` reads. Every rank prints one
JSON line with its nodes, walks, tokens, seconds, tokens/s and the walker's share of the GPU time.
"""
from __future__ import annotations

import json
import sys
from typing import List

FLAG_HELP = """-graph <edge list> -directed <0|1> -weighted <0|1> -walk_length <int> -walks_per_node <int>
-p <float> -q <float> -seed <int> -size <int> -window <int> -negative <int> -alpha <float> -epoch <int>
-output <file> -binary <0|1> -cbow <0|1> -hs <0|1> -use_adagrad <0|1> -data_block_size <bytes> -is_pipeline <0|1>"""

# the defaults of this app where they differ from wordembedding's
_DEFAULTS = ["-size", "128", "-window", "10", "-negative", "5"]
_GRAPH_FLAGS = {"-graph": ("graph", str), "-directed": ("directed", lambda v: bool(int(v))),
                "-weighted": ("weighted", lambda v: bool(int(v))), "-walk_length": ("walk_length", int),
                "-walks_per_node": ("walks_per_node", int), "-p": ("p", float), "-q": ("q", float),
                "-seed": ("seed", int)}


def parse_args(argv: List[str]):
    """(WordEmbeddingOption, graph settings dict) of ``-flag value`` pairs; unknown flags are skipped as in
    ``wordembedding``."""
    from .wordembedding import parse_args as we_parse_args
    opt = we_parse_args(_DEFAULTS + list(argv))
    g = dict(graph=None, directed=False, weighted=False, walk_length=80, walks_per_node=10, p=1.0, q=1.0, seed=1)
    i = 0
    while i < len(argv):
        if argv[i] in _GRAPH_FLAGS and i + 1 < len(argv):
            name, conv = _GRAPH_FLAGS[argv[i]]
            g[name] = conv(argv[i + 1])
            i += 2
        else:
            i += 1
    return opt, g


def run(argv: List[str]) -> dict:
    import torch
    opt, g = parse_args(argv)
    if not g["graph"]:
        print("usage: graph_embedding " + FLAG_HELP)
        return {}
    if not torch.cuda.is_available():
        raise SystemExit("graph_embedding needs a CUDA GPU: the walker and the trainer run on the device "
                         "(there is no CPU implementation of this application)")
    import multiverso_b200 as mv
    from ..models.graph_embedding import GraphEmbedding
    from ..ops.random_walk import Graph
    from ..utils import Log
    mv.init()
    rank = mv.rank()
    graph, labels = Graph.load(g["graph"], directed=g["directed"], weighted=g["weighted"])
    Log.info("graph %d nodes, %d arcs, dim %d, walks %d x %d nodes, p %g q %g", graph.num_nodes, graph.num_arcs,
             opt.embeding_size, g["walks_per_node"], g["walk_length"], g["p"], g["q"])
    ge = GraphEmbedding(graph, opt, walk_length=g["walk_length"], walks_per_node=g["walks_per_node"], p=g["p"],
                        q=g["q"], seed=g["seed"])
    stats = ge.train()
    mv.barrier()
    if opt.output_file:
        ge.save_embedding(opt.output_file, labels, binary=opt.output_binary)
        mv.runtime.Runtime.get().host_barrier()
    print(json.dumps(stats), flush=True)
    mv.shutdown()
    return stats


if __name__ == "__main__":
    run(sys.argv[1:])
