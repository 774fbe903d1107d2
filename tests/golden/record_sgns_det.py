#!/usr/bin/env python
"""Records tests/golden/sgns_det_parent.json: the exact result of the deterministic skip-gram kernel
(`mvb_sgns_train_det`) on three seeded multi-wave cases, as SHA-256 digests of both tables after
training plus the loss bits and pair count.

  python tests/golden/record_sgns_det.py [OUT]

The digests depend on the wave size, which follows from the GPU's SM count and shared memory:
they were recorded on an H100 SXM (132 SMs).  `tests/test_gpu_sgns_det_tiles.py` runs the same
cases through `run_case` and asserts equality, so any change to the kernel that alters a single bit
of the result fails there.
"""
from __future__ import annotations

import hashlib
import json
import os
import struct
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

CASES = {
    # Zipf tokens: hot rows are contexts / outputs of many centres of one wave; per-word step scales
    "zipf_v5000": dict(V=5000, D=300, LD=300, W=5, K=5, n_tok=20000, zipf=True, maps=False, scales=True),
    # a block cache: id -> slot maps and padded rows
    "maps_ld320": dict(V=3000, D=300, LD=320, W=5, K=5, n_tok=20000, zipf=False, maps=True, scales=False),
    # the largest rows and window, 7 negatives
    "dim512_w15": dict(V=4000, D=512, LD=512, W=15, K=7, n_tok=8000, zipf=True, maps=False, scales=True),
}


def run_case(name: str) -> dict:
    import numpy as np
    import torch
    from multiverso_b200 import _native as N
    from multiverso_b200.models.wordembedding import synthetic_zipf_corpus
    c = CASES[name]
    V, D, LD = c["V"], c["D"], c["LD"]
    g = torch.Generator().manual_seed(11)
    if c["zipf"]:
        tl = torch.from_numpy(synthetic_zipf_corpus(c["n_tok"], V, 1000, seed=5))
    else:
        tl = torch.randint(0, V, (c["n_tok"],), generator=g).to(torch.int32)
        tl[200::201] = -1
    toks = tl.cuda()
    base_in = ((torch.rand(V, D, generator=g) - 0.5) * 0.4)
    base_out = ((torch.rand(V, D, generator=g) - 0.5) * 0.4)
    w_in, w_out = torch.zeros(V, LD), torch.zeros(V, LD)
    m = None
    if c["maps"]:
        perm = torch.randperm(V, generator=g)
        w_in[perm, :D], w_out[perm, :D] = base_in, base_out
        m = perm.to(torch.int32).cuda()
    else:
        w_in[:, :D], w_out[:, :D] = base_in, base_out
    w_in, w_out = w_in.cuda(), w_out.cuda()
    # unigram^0.75 alias table built on the host (Vose), so negatives follow the corpus like training does
    counts = np.bincount(tl.numpy()[tl.numpy() >= 0], minlength=V).astype(np.float64) + 1.0
    p = counts ** 0.75
    p *= V / p.sum()
    prob, alias = np.ones(V, dtype=np.float32), np.arange(V, dtype=np.int32)
    small, large = [i for i in range(V) if p[i] < 1], [i for i in range(V) if p[i] >= 1]
    while small and large:
        s, l_ = small.pop(), large.pop()
        prob[s], alias[s] = p[s], l_
        p[l_] -= 1 - p[s]
        (small if p[l_] < 1 else large).append(l_)
    prob_d, alias_d = torch.from_numpy(prob).cuda(), torch.from_numpy(alias).cuda()
    s_in = (0.5 + torch.rand(V, generator=g)).cuda()
    s_out = (0.5 + torch.rand(V, generator=g)).cuda()
    out = torch.zeros(2, dtype=torch.int64, device="cuda")
    a = N.Sgns()
    a.tokens, a.n_tokens, a.w_in, a.w_out = toks.data_ptr(), toks.numel(), w_in.data_ptr(), w_out.data_ptr()
    a.dim, a.ld, a.window, a.negative, a.lr, a.seed = D, LD, c["W"], c["K"], 2e-2, 0x5EED
    a.vocab, a.alias_prob, a.alias_idx = V, prob_d.data_ptr(), alias_d.data_ptr()
    a.map_in, a.map_out = N.ptr(m), N.ptr(m)
    if c["scales"]:
        a.scale_in, a.scale_out = s_in.data_ptr(), s_out.data_ptr()
    a.pair_count, a.loss_sum = out.data_ptr(), out.data_ptr() + 8
    rc = N.cuda_lib().mvb_sgns_train_det(a, N.stream_ptr())
    assert rc == 0, rc
    torch.cuda.synchronize()
    o = out.cpu()
    loss_bits = struct.unpack("<I", struct.pack("<f", o[1:].view(torch.float32)[0].item()))[0]
    return {"in_sha256": hashlib.sha256(w_in.cpu().numpy().tobytes()).hexdigest(),
            "out_sha256": hashlib.sha256(w_out.cpu().numpy().tobytes()).hexdigest(),
            "loss_bits": f"{loss_bits:08x}", "pairs": int(o[0])}


def main():
    import torch
    import multiverso_b200 as mv
    out_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                  "sgns_det_parent.json")
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
