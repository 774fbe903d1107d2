"""Probe: do the register-path row kernels co-reside with the persistent K7 CTAs?  (1 GPU)
Times a row pull alone, and the same pull launched ~300 us after K7 started on another stream."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import multiverso_b200 as mv  # noqa: E402
from multiverso_b200 import _native as N  # noqa: E402
from multiverso_b200.models.wordembedding import WordEmbedding, WordEmbeddingOption, synthetic_zipf_corpus  # noqa: E402

mv.init()
V, D = 1_000_000, 300
we = WordEmbedding(WordEmbeddingOption(embeding_size=D, window_size=5, negative_num=5, init_learning_rate=0.025), V)
toks = torch.from_numpy(synthetic_zipf_corpus(1 << 20, V, 1000, seed=3)).cuda()
t = we.output_table
k = 600_000
ids = torch.arange(0, k, dtype=torch.int32, device="cuda")
cache = torch.empty(k, D, device="cuda"); old = torch.empty(k, D, device="cuda")
lib = N.cuda_lib()
side = torch.cuda.Stream()
main = torch.cuda.current_stream()


def pull(ctas_per_sm):
    lib.mvb_rows_pull(t._rowmap, 4, ids, None, k, cache, old, D, ctas_per_sm, torch.cuda.current_stream().cuda_stream)


for ctas_per_sm in (1, 2):
    for _ in range(2):
        pull(ctas_per_sm)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); pull(ctas_per_sm); e1.record(); torch.cuda.synchronize()
    alone = e0.elapsed_time(e1)
    we.train_block(toks); torch.cuda.synchronize()
    k0, k1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    k0.record(main)
    we.train_block(toks)
    k1.record(main)
    with torch.cuda.stream(side):
        side.wait_event(k0)
        torch.cuda._sleep(600_000)          # ~300 us: K7 is running by now
        s0.record(side); pull(ctas_per_sm); s1.record(side)
    torch.cuda.synchronize()
    print(f"{ctas_per_sm} CTAs/SM: pull alone {alone:.2f} ms, under K7 {s0.elapsed_time(s1):.2f} ms, K7 {k0.elapsed_time(k1):.2f} ms, "
          f"pull end - K7 start {k0.elapsed_time(s1):.2f} ms, carveout={os.environ.get('MVB_SIDE_CARVEOUT', '-')}", flush=True)
mv.shutdown()
