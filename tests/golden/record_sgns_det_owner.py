#!/usr/bin/env python
"""Records tests/golden/sgns_det_owner.json: the exact result of the deterministic skip-gram kernel
(`mvb_sgns_train_det`) on seeded cases of many waves each, as SHA-256 digests of both tables after
training plus the loss bits and pair count.

  python tests/golden/record_sgns_det_owner.py [OUT]

The cases span the mix of rows a wave reads once (written in place by their reader) and rows it reads
more than once (summed in the fixed-point accumulator): large and uniform vocabularies where nearly every
row has one reader, a small hot vocabulary where none has, block-cache slots with padded rows, partial
lanes, the widest window with 7 negatives, sentence breaks on CTA slice boundaries and a block split over
two calls.  Column 3 of both tables starts at -0.0: its deltas are exactly zero, so any write of an
unchanged element flips the sign bit.  Digests depend on the wave size, which follows from the GPU's SM
count and shared memory: they were recorded on an H100 SXM (132 SMs).
"""
from __future__ import annotations

import hashlib
import json
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

# breaks on, just before and just after the boundaries of 20-centre slices
_SLICE_BREAKS = sorted({b for s in range(0, 16000, 140) for b in (s - 1, s, s + 1) if b >= 0})

CASES = {
    # most rows of a wave have one reader; the Zipf head has many
    "zipf_v200k": dict(V=200_000, D=300, LD=300, W=5, K=5, n_tok=24000, tokens="zipf", neg="alias",
                       maps=False, scales=True),
    # almost every row has one reader, input rows at slice interiors included; uniform negatives
    "uniform_v1m": dict(V=1_000_000, D=300, LD=300, W=5, K=5, n_tok=16000, tokens="uniform", neg="pool",
                        maps=False, scales=False, breaks=_SLICE_BREAKS),
    # no row has one reader
    "hot_v40": dict(V=40, D=300, LD=300, W=5, K=5, n_tok=8000, tokens="uniform", neg="alias",
                    maps=False, scales=True),
    # block-cache slots and padded rows
    "maps_ld320_v100k": dict(V=100_000, D=300, LD=320, W=5, K=5, n_tok=16000, tokens="uniform", neg="alias",
                             maps=True, scales=False),
    # rows of an odd number of floats (partial lanes), padded
    "dim37_v100k": dict(V=100_000, D=37, LD=40, W=5, K=5, n_tok=16000, tokens="zipf", neg="alias",
                        maps=False, scales=True),
    # the widest rows and window, 7 negatives: slices of 6 centres
    "dim512_w15_k7": dict(V=100_000, D=512, LD=512, W=15, K=7, n_tok=8000, tokens="zipf", neg="alias",
                          maps=False, scales=True),
    # one block in two calls: every call starts with no reader counts (the first call's last wave has an even
    # index, so counts it left behind would sit where the second call's first wave looks)
    "zipf_v200k_2calls": dict(V=200_000, D=300, LD=300, W=5, K=5, n_tok=24000, tokens="zipf", neg="alias",
                              maps=False, scales=True, calls=(0, 7000, 24000)),
}


def make_case(name: str) -> dict:
    """Device tensors and sampler of a case: tokens, tables (initial state), maps, scales, negatives."""
    import numpy as np
    import torch
    from multiverso_b200.models.wordembedding import synthetic_zipf_corpus
    c = CASES[name]
    V, D, LD = c["V"], c["D"], c["LD"]
    g = torch.Generator().manual_seed(23)
    if c["tokens"] == "zipf":
        tl = torch.from_numpy(synthetic_zipf_corpus(c["n_tok"], V, 1000, seed=7))
    else:
        tl = torch.randint(0, V, (c["n_tok"],), generator=g).to(torch.int32)
        tl[500::501] = -1
    for b in c.get("breaks", ()):
        tl[b] = -1
    base_in = (torch.rand(V, D, generator=g) - 0.5) * 0.4
    base_out = (torch.rand(V, D, generator=g) - 0.5) * 0.4
    base_in[:, 3] = -0.0
    base_out[:, 3] = -0.0
    w_in, w_out = torch.full((V, LD), 7.0), torch.full((V, LD), -7.0)   # pad columns keep these
    m = None
    if c["maps"]:
        perm = torch.randperm(V, generator=g)
        w_in[perm, :D], w_out[perm, :D] = base_in, base_out
        m = perm.to(torch.int32)
    else:
        w_in[:, :D], w_out[:, :D] = base_in, base_out
    prob = alias = pool = None
    if c["neg"] == "pool":
        pool = torch.randperm(V, generator=g).to(torch.int32)
    else:
        # unigram^0.75 alias table built on the host (Vose), so negatives follow the corpus like training does
        t = tl.numpy()
        counts = np.bincount(t[t >= 0], minlength=V).astype(np.float64) + 1.0
        p = counts ** 0.75
        p *= V / p.sum()
        prob, alias = np.ones(V, dtype=np.float32), np.arange(V, dtype=np.int32)
        small, large = [i for i in range(V) if p[i] < 1], [i for i in range(V) if p[i] >= 1]
        while small and large:
            s, l_ = small.pop(), large.pop()
            prob[s], alias[s] = p[s], l_
            p[l_] -= 1 - p[s]
            (small if p[l_] < 1 else large).append(l_)
        prob, alias = torch.from_numpy(prob), torch.from_numpy(alias)
    s_in = 0.5 + torch.rand(V, generator=g)
    s_out = 0.5 + torch.rand(V, generator=g)
    return dict(c=c, tokens=tl, w_in=w_in, w_out=w_out, map=m, prob=prob, alias=alias, pool=pool,
                s_in=s_in if c["scales"] else None, s_out=s_out if c["scales"] else None,
                lr=2e-2, seed=0x5EED)


def train(case: dict):
    """Runs the case through `mvb_sgns_train_det` on the GPU: (w_in, w_out, pairs, loss) on the host."""
    import torch
    from multiverso_b200 import _native as N
    c = case["c"]
    dev = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in case.items()}
    out = torch.zeros(2, dtype=torch.int64, device="cuda")
    cuts = c.get("calls", (0, c["n_tok"]))
    for s, e in zip(cuts[:-1], cuts[1:]):
        toks = dev["tokens"][s:e]
        a = N.Sgns()
        a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
        a.w_in, a.w_out = dev["w_in"].data_ptr(), dev["w_out"].data_ptr()
        a.dim, a.ld, a.window, a.negative = c["D"], c["LD"], c["W"], c["K"]
        a.lr, a.seed, a.vocab = case["lr"], case["seed"] + s, c["V"]
        if dev["pool"] is not None:
            a.neg_pool, a.neg_pool_size = dev["pool"].data_ptr(), dev["pool"].numel()
        else:
            a.alias_prob, a.alias_idx = dev["prob"].data_ptr(), dev["alias"].data_ptr()
        a.map_in, a.map_out = N.ptr(dev["map"]), N.ptr(dev["map"])
        if dev["s_in"] is not None:
            a.scale_in, a.scale_out = dev["s_in"].data_ptr(), dev["s_out"].data_ptr()
        a.pair_count, a.loss_sum = out.data_ptr(), out.data_ptr() + 8
        rc = N.cuda_lib().mvb_sgns_train_det(a, N.stream_ptr())
        assert rc == 0, rc
    torch.cuda.synchronize()
    o = out.cpu()
    return dev["w_in"].cpu(), dev["w_out"].cpu(), int(o[0]), o[1:].view(torch.float32)[0].item()


def run_case(name: str) -> dict:
    w_in, w_out, pairs, loss = train(make_case(name))
    loss_bits = struct.unpack("<I", struct.pack("<f", loss))[0]
    return {"in_sha256": hashlib.sha256(w_in.numpy().tobytes()).hexdigest(),
            "out_sha256": hashlib.sha256(w_out.numpy().tobytes()).hexdigest(),
            "loss_bits": f"{loss_bits:08x}", "pairs": pairs}


def main():
    import torch
    import multiverso_b200 as mv
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                  "sgns_det_owner.json")
    mv.init()
    try:
        res = {"card": torch.cuda.get_device_name(),
               "cases": {name: run_case(name) for name in CASES}}
    finally:
        mv.shutdown()
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(res, indent=1, sort_keys=True))


if __name__ == "__main__":
    main()
