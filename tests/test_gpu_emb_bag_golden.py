"""The embedding-bag kernels (csrc/cuda/emb_bag.cu, emb_bag_coll.cu) bit for bit against recorded results.

The kernels are deterministic by design (fixed summation order, one epilogue per unique row), so a fixed input gives
the same bytes on every run, grid and SM count. Inputs come from fixed seeds on the CPU; every result is hashed with
SHA-256 and compared with tests/golden/emb_bag_digests.json, which also holds each result's float64 sum to tell a
rounding drift from a broken kernel. Covered: every register class on both paths (1..4 float4 per lane: dims up to
128, 129..256, 257..384 and above; column slabs above 512 on the single table), sum / mean / per-sample weights with
empty bags, Zipf ids whose hot runs span many backward chunks (the merge pass), the push and the compact epilogues,
the per-sample-weight gradient, and a collection with mixed dims and shared tables.

Record the file on an H100 with ``python tests/test_gpu_emb_bag_golden.py --write [PATH]``."""
import argparse
import hashlib
import json
import os
import sys
import types

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "emb_bag_digests.json")
DIMS = [4, 30, 64, 200, 300, 512, 1000]     # register classes 1, 1, 1, 2, 3, 4, 4 (two slabs)
MODES = [("sum", False), ("sum", True), ("mean", False)]


def _lengths(g, n, max_len):
    lens = torch.randint(0, max_len + 1, (n,), generator=g)
    lens[::7] = 0                                                   # empty bags
    return lens


def _zipf(g, V, L):
    """Zipf(1.1) ids: id 0 alone is about a tenth of the lookups, so its run spans many 256-lookup chunks."""
    p = torch.arange(1, V + 1, dtype=torch.float64).pow_(-1.1)
    return torch.multinomial(p, L, replacement=True, generator=g)


def _table(g, V, dim, S, gap=5):
    """A V x dim table with a padded row pitch (padding holds garbage) as S shards at separate places of one
    buffer: (row map, buffer, function reading the rows back)."""
    from multiverso_b200 import _native as N
    pitch = (dim + 3) // 4 * 4 + 4
    W = torch.randn(V, pitch, generator=g)
    W[:, dim:] = 1e6
    buf = torch.full((V + S * gap, pitch), 1e3)
    rm = N.RowMap()
    rps = V // S
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = V, pitch, S, rps
    spans = []
    for s in range(S):
        lo, hi = s * rps, (V if s == S - 1 else (s + 1) * rps)
        buf[lo + (s + 1) * gap:hi + (s + 1) * gap] = W[lo:hi]
        spans.append((lo + (s + 1) * gap, hi - lo))
    buf = buf.cuda()
    for s, (at, _) in enumerate(spans):
        rm.shard_ptrs[s] = buf[at].data_ptr()
    return rm, buf, lambda: torch.cat([buf[a:a + k, :dim] for a, k in spans])


class _Capture(types.SimpleNamespace):
    """A table handle whose compact pushes are recorded instead of applied."""

    def add_rows_async(self, uniq, grads, option=None):
        self.pushed.append((uniq.clone(), grads.clone()))


def _single(res):
    from multiverso_b200 import _native as N
    from multiverso_b200.ops.embedding import _fwd_device, _psw_grad_device, _push_device
    for dim in DIMS:
        for m, (mode, weighted) in enumerate(MODES):
            name = f"single/d{dim}/{mode}{'_psw' if weighted else ''}"
            g = torch.Generator().manual_seed(10 * dim + m)
            V, B = 5003, 600
            lens = _lengths(g, B, 40)
            offsets = (torch.cumsum(lens, 0) - lens).cuda()
            ids = _zipf(g, V, int(lens.sum())).cuda()
            psw = torch.rand(ids.numel(), generator=g).cuda() if weighted else None
            dout = torch.randn(B, dim, generator=g).cuda()
            rm, buf, back = _table(g, V, dim, 3)
            res[name + "/fwd"] = _fwd_device(rm, dim, ids, offsets, psw, mode)
            res[name + "/psw_grad"] = _psw_grad_device(rm, dim, ids, offsets, mode, dout)
            sgd = types.SimpleNamespace(updater=N.UPD_SGD, is_sparse=False, num_col=rm.num_col)
            _push_device(sgd, rm, dim, ids, offsets, psw, mode, dout, 0.5, None)
            res[name + "/push"] = back()
            ada = _Capture(updater=N.UPD_ADAGRAD, is_sparse=False, num_col=rm.num_col, pushed=[])
            _push_device(ada, rm, dim, ids, offsets, psw, mode, dout, 0.5, None)
            (uniq, grads), = ada.pushed
            res[name + "/compact_uniq"], res[name + "/compact_grads"] = uniq, grads
            torch.cuda.synchronize()


def _collection(res):
    """Dims 4, 30, 64, 256, 300 and 512 (every register class); three tables shared by two features each; push and
    compact tables."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    for weighted in (False, True):
        name = f"coll/{'psw' if weighted else 'nopsw'}"
        g = torch.Generator().manual_seed(77 + weighted)
        dims, rows = [4, 30, 64, 300, 512, 256], [900, 5003, 7001, 3001, 1201, 4001]
        upd = [N.UPD_SGD, N.UPD_SGD, N.UPD_ADAGRAD, N.UPD_MOMENTUM, N.UPD_DEFAULT, N.UPD_ADAGRAD]
        modes = ["sum"] * 6 if weighted else ["mean", "sum", "mean", "sum", "sum", "mean"]
        feats = [["a"], ["b1", "b2"], ["c"], ["d1", "d2"], ["e"], ["f1", "f2"]]
        tab = [0, 1, 1, 2, 3, 3, 4, 5, 5]
        keep, cfgs = [], []
        for t, (V, dim) in enumerate(zip(rows, dims)):
            rm, buf, back = _table(g, V, dim, 1 + t % 3)
            table = _Capture(_rowmap=rm, dtype=torch.float32, num_row=V, num_col=dim, updater=upd[t], is_sparse=False,
                             rt=types.SimpleNamespace(device=torch.device("cuda", 0)), pushed=[])
            keep.append((buf, back, table))
            cfgs.append(EmbeddingBagConfig(table, feats[t], push_scale=0.25, mode=modes[t]))
        ebc = PSEmbeddingCollection(cfgs)
        B = 500
        lengths = torch.stack([_lengths(g, B, 30) for _ in tab])
        ids = torch.cat([_zipf(g, rows[t], int(n)) for t, n in zip(tab, lengths.sum(1))]).cuda()
        psw = torch.rand(ids.numel(), generator=g).cuda().requires_grad_() if weighted else None
        dout = torch.randn(B, ebc.out_dim, generator=g).cuda()
        out = ebc(ids, lengths.cuda(), psw)
        out.backward(dout)
        torch.cuda.synchronize()
        res[name + "/fwd"] = out.detach()
        if weighted:
            res[name + "/psw_grad"] = psw.grad
        for t, (buf, back, table) in enumerate(keep):
            if table.pushed:
                (uniq, grads), = table.pushed
                res[f"{name}/t{t}/compact_uniq"], res[f"{name}/t{t}/compact_grads"] = uniq, grads
            else:
                res[f"{name}/t{t}/push"] = back()


def results():
    res = {}
    _single(res)
    _collection(res)
    return {k: {"sha256": hashlib.sha256(v.contiguous().cpu().numpy().tobytes()).hexdigest(),
                "sum": float(v.double().sum())} for k, v in res.items()}


def test_bitwise_equal_to_recorded():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    with open(GOLDEN) as f:
        want = json.load(f)
    got = results()
    assert sorted(got) == sorted(want)
    bad = [f"{k}: sum {got[k]['sum']!r}, recorded {want[k]['sum']!r}" for k in want
           if got[k]["sha256"] != want[k]["sha256"]]
    assert not bad, "\n".join(bad)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--write", nargs="?", const=GOLDEN, metavar="PATH", help="record the digests (default: %(const)s)")
    a = ap.parse_args()
    r = results()
    if a.write:
        os.makedirs(os.path.dirname(os.path.abspath(a.write)), exist_ok=True)
        with open(a.write, "w") as f:
            json.dump(r, f, indent=1, sort_keys=True)
            f.write("\n")
    print(f"{len(r)} results" + (f" written to {a.write}" if a.write else ""))
