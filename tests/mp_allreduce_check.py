"""``parallel.aggregate`` over real peers, launched with torchrun (one rank per GPU):

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tests/mp_allreduce_check.py

tests/test_gpu_allreduce_kernels.py pins the kernels on one GPU; this script covers the host logic above them:
the size thresholds that pick a kernel, staging growth, tensors in symmetric memory, unaligned views and the
channel epochs of calls mixed back to back. Every rank regenerates every rank's seeded data, so each checks its own
result against the exact rank-order sum (that file's ``_model``) bit for bit wherever a P2P kernel runs, and
against the f32 bound plus equal bits on all ranks where the sum may be taken in the switch (``rank_ordered``).
"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import multiverso_b200 as mv
from multiverso_b200.parallel import aggregate, symm_tensor
from multiverso_b200.parallel.collectives import FUSED_BYTES, TWO_SHOT_BYTES
from test_gpu_allreduce_kernels import _bytes, _data, _model

results = {}
_seed = [0]


def check(name, cond, info=""):
    results[name] = bool(cond) and results.get(name, True)
    if not cond:
        print(f"[rank {mv.rank()}] FAIL {name} {info}", flush=True)


def rank_ordered(dtype, nbytes, algo):
    """Whether ``aggregate`` promises the rank-order sum for this call. It does wherever a P2P kernel runs. An f32
    message beyond the fused path goes to the NVLS kernel when ``algo`` is "nvls", or "auto" on four or more ranks,
    and the platform has multicast memory; the switch adds in its own order."""
    if dtype != torch.float32 or (algo in ("auto", "fused") and nbytes <= FUSED_BYTES):
        return True
    return not (algo == "nvls" or (algo == "auto" and mv.size() >= 4))


def run(name, dtype, n, algo="auto", into=None, lead=0):
    """Aggregate fresh data of n elements and check the result. ``into``: a tensor to reduce in (a view of symmetric
    memory); otherwise a new tensor, cut ``lead`` elements into its allocation. A rank-ordered call must equal the
    exact model bit for bit. One that may add in the switch must lie within the f32 bound of the fp64 sum and leave
    the same bits on every rank: the int64 sum of the result's bits, taken with the rank-ordered integer two-shot,
    equals W times the local bits on every rank only if all ranks hold the same."""
    _seed[0] += 1
    W = mv.size()
    x = _data(dtype, W, n, seed=_seed[0])
    exp = _model(x)
    if into is None:
        into = torch.empty(lead + n, dtype=dtype, device="cuda")[lead:]
    into.copy_(x[mv.rank()].cuda())
    out = aggregate(into, algo=algo)
    torch.cuda.synchronize()
    got = into.cpu()
    what = f"dtype {dtype} n {n} algo {algo}"
    check(name, out.data_ptr() == into.data_ptr(), what + ": result is not the argument")
    if rank_ordered(dtype, n * into.element_size(), algo):
        es = into.element_size()
        bad = (_bytes(got).view(n, es) != _bytes(exp).view(n, es)).any(1).nonzero().view(-1)
        check(name, len(bad) == 0, f"{what}: {len(bad)} elements differ from the exact sum, first {bad[:4].tolist()}")
        return
    x64 = x.double()
    err = (got.double() - x64.sum(0)).abs()
    check(name, bool((err <= W * 2.0 ** -24 * x64.abs().sum(0)).all()), f"{what}: off the fp64 sum by {err.max().item()}")
    bits = into.view(torch.int32).to(torch.int64)
    total = aggregate(bits.clone(), algo="twoshot")
    check(name, torch.equal(total, W * bits), what + ": ranks hold different bits")


def main():
    mv.init()
    W = mv.size()
    f32 = torch.float32
    # every algorithm, every element type, on both sides of the fused threshold and of the two-shot threshold
    for dtype in (torch.float32, torch.float64, torch.int32, torch.int64, torch.int8):
        es = torch.empty(0, dtype=dtype).element_size()
        for algo in ("auto", "fused", "oneshot", "twoshot"):
            for nbytes in (FUSED_BYTES - 8, FUSED_BYTES, FUSED_BYTES + 8):
                run(f"{algo}_at_fused_threshold", dtype, nbytes // es, algo)
        for algo in ("oneshot", "twoshot"):
            for nbytes in (TWO_SHOT_BYTES - 8, TWO_SHOT_BYTES, TWO_SHOT_BYTES + 8):
                run(f"{algo}_at_twoshot_threshold", dtype, nbytes // es, algo)
        for n in (1, 7, 16 // es * W + 1):
            run("small", dtype, n)
    for nbytes in (FUSED_BYTES - 4, FUSED_BYTES + 4):
        run("f32_next_to_fused_threshold", f32, nbytes // 4)
    # staging grows at least twice (release and re-allocate), then a smaller message runs in the larger staging
    for n in (300_001, 700_003, 1_500_007, 400_001):
        run("staging_growth", f32, n)
        run("staging_growth", f32, n + 2, "twoshot")
        run("staging_growth", torch.int8, 4 * n + 3, "twoshot")
    # results that do not start on a 16-byte boundary, above the fused path's size
    for algo in ("auto", "oneshot", "twoshot"):
        run(f"unaligned_{algo}", f32, 300_000, algo, lead=1)
        run(f"unaligned_{algo}", torch.float64, 200_001, algo, lead=1)
        for lead in (1, 4, 8):
            run(f"unaligned_{algo}", torch.int8, 1_200_005, algo, lead=lead)
    # symmetric memory: reduced in place at offset 0 and at a 16-byte multiple, through the staging at 4 bytes;
    # mixed with staged and fused calls so that the channels' epochs interleave
    zs = symm_tensor(600_011, f32)
    for it in range(3):
        for lead in (0, 4, 1):
            for algo in ("auto", "twoshot"):
                run(f"symm_views_{algo}", f32, zs.numel() - lead, algo, into=zs[lead:])
            run("symm_views_mixed", f32, 300_001 + it, "twoshot")
            run("symm_views_mixed", torch.int32, 1000 + it)
    # 50 fused calls back to back with changing data and sizes: the two staging halves alternate
    for it in range(50):
        run("fused_back_to_back", (f32, torch.int32, torch.float64)[it % 3], (1, 5, 1000, 4099, 100_000)[it % 5])
    # NVLS forced (or its two-shot fallback where the platform has no multicast memory)
    run("nvls_or_fallback", f32, 1_200_003, "nvls")
    mv.barrier()
    mv.shutdown()


if __name__ == "__main__":
    t0 = time.time()
    try:
        main()
    except Exception:
        import traceback
        traceback.print_exc()
        results["exception"] = False
    rank = int(os.environ.get("RANK", "0"))
    ok = all(results.values()) and len(results) > 0
    print(f"[rank {rank}] {'PASS' if ok else 'FAIL'} {json.dumps(results)} ({time.time() - t0:.1f}s)", flush=True)
    sys.exit(0 if ok else 1)
