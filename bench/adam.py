"""adagrad, rowwise_adagrad, adam and ftrl: row Adds, an embedding-collection training step and whole-table Adds.

    python bench/adam.py [--iters 20] [--out FILE]

Workloads (fp32, one GPU):

* ``add_rows``: the unique ids of a 1M-lookup Zipf(1.05) batch over a 4M-row table of 64 or 128 columns, added with
  ``MatrixTable.add_rows`` (the owner-side row Add every embedding layer's backward takes on a stateful table);
* ``collection_step``: forward + backward of a ``PSEmbeddingCollection`` of two tables (4M x 128 shared by two
  features, 1M x 64), batch 4096, 20 ids per bag and feature, Zipf ids;
* ``whole_add``: ``MatrixTable.add`` of a 65536 x 1024 delta (the fused Add);
* ``whole_add_1d``: ``ArrayTable.add`` of a 16M-element delta (the fused Add on rows of one element: adam runs a
  thread per row there and forms its two fp64 bias factors per element);
* ``state_bytes``: the updater state per GPU of the 4M x 128 table.

Times are CUDA-event times over ``--iters`` calls after three warm-up calls, the median of three windows; each line
names the card and its power limit, read in the same run. Words moved per element of a whole-table Add: adagrad
reads the delta, the row and its state and writes both (5); rowwise_adagrad reads the delta twice and the row and
writes the row (4, plus one accumulator read and write per row); adam reads the delta, the row, m and v and writes
the last three (7, plus one step count read and write per row); ftrl reads the delta, the row, z and n and writes
the last three (7). The AddOption is lr 0.05, rho 0.1, momentum 0.9 and lambda 0.1 (adam's beta1 is momentum; ftrl's
alpha, lambda1 and lambda2 are rho, lambda and momentum; the other updaters ignore what they do not use).
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

UPDATERS = ["adagrad", "rowwise_adagrad", "adam", "ftrl"]
WORDS = {"adagrad": 5, "rowwise_adagrad": 4, "adam": 7, "ftrl": 7}
ROW_STATE = ("rowwise_adagrad", "adam")        # one state word per row, read and written


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(3):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) / iters)
    return sorted(out)[1]


def zipf_ids(V, n, g):
    """n ids in [0, V) with P(id k) ~ 1 / (k + 1)^1.05."""
    cdf = torch.cumsum(torch.arange(1, V + 1, device="cuda", dtype=torch.float64).pow_(-1.05), 0)
    u = torch.rand(n, device="cuda", generator=g, dtype=torch.float64) * cdf[-1]
    return torch.searchsorted(cdf, u).clamp_(max=V - 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench/adam.py measures on a GPU"
    import multiverso_b200 as mv
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    mv.init()
    card = gpu_info()
    g = torch.Generator(device="cuda").manual_seed(1)
    opt = mv.AddOption(learning_rate=0.05, rho=0.1, momentum=0.9, lambda_=0.1)
    lines = []

    def state_bytes(*tables):
        return sum(s.numel() * 4 for t in tables for s in t.state)

    def emit(row):
        row["gpu"] = card
        lines.append(json.dumps(row))
        print(lines[-1], flush=True)

    V = 4 << 20
    for dim in (64, 128):
        ids = torch.unique(zipf_ids(V, 1 << 20, g))
        vals = torch.randn(ids.numel(), dim, device="cuda", generator=g) * 0.01
        for upd in UPDATERS:
            t = mv.MatrixTable(V, dim, "float32", updater=upd)
            ms = timed(lambda: t.add_rows(ids, vals, opt), a.iters)
            emit({"bench": "add_rows", "updater": upd, "rows": int(ids.numel()), "dim": dim, "ms": round(ms, 4),
                  "state_bytes": state_bytes(t)})
            t.free()
            del t
            torch.cuda.empty_cache()

    B, L = 4096, 20
    for upd in UPDATERS:
        t1 = mv.MatrixTable(V, 128, "float32", updater=upd, min_value=-0.1, max_value=0.1)
        t2 = mv.MatrixTable(1 << 20, 64, "float32", updater=upd, min_value=-0.1, max_value=0.1)
        ebc = PSEmbeddingCollection([EmbeddingBagConfig(t1, ["a", "b"], option=opt),
                                     EmbeddingBagConfig(t2, ["c"], option=opt)])
        ids = torch.cat([zipf_ids(V, B * L, g), zipf_ids(V, B * L, g), zipf_ids(1 << 20, B * L, g)])
        lengths = torch.full((3, B), L, device="cuda")
        dout = torch.randn(B, 128 + 128 + 64, device="cuda", generator=g)
        ms = timed(lambda: ebc(ids, lengths).backward(dout), a.iters)
        emit({"bench": "collection_step", "updater": upd, "batch": B, "bag": L, "ms": round(ms, 4),
              "state_bytes": state_bytes(t1, t2)})
        t1.free(), t2.free()
        del t1, t2, ebc
        torch.cuda.empty_cache()

    R, Cc = 65536, 1024
    d = torch.randn(R * Cc, device="cuda", generator=g) * 0.01
    for upd in UPDATERS:
        t = mv.MatrixTable(R, Cc, "float32", updater=upd)
        ms = timed(lambda: t.add(d, opt), a.iters)
        gb = R * Cc * 4 * WORDS[upd] / 1e9
        emit({"bench": "whole_add", "updater": upd, "shape": [R, Cc], "ms": round(ms, 4),
              "gbps_counted": round(gb / (ms / 1e3), 1), "state_bytes": state_bytes(t)})
        t.free()
        del t
        torch.cuda.empty_cache()

    n = 16 << 20
    d = torch.randn(n, device="cuda", generator=g) * 0.01
    for upd in UPDATERS:
        t = mv.ArrayTable(n, "float32", updater=upd)
        ms = timed(lambda: t.add(d, opt), a.iters)
        gb = n * 4 * (WORDS[upd] + (2 if upd in ROW_STATE else 0)) / 1e9
        emit({"bench": "whole_add_1d", "updater": upd, "size": n, "ms": round(ms, 4),
              "gbps_counted": round(gb / (ms / 1e3), 1), "state_bytes": state_bytes(t)})
        t.free()
        del t
        torch.cuda.empty_cache()

    for upd in UPDATERS:
        t = mv.MatrixTable(V, 128, "float32", updater=upd)
        emit({"bench": "state_bytes", "updater": upd, "table": [V, 128], "state_bytes": state_bytes(t),
              "table_bytes": V * 128 * 4})
        t.free()
        del t
        torch.cuda.empty_cache()
    mv.shutdown()
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
