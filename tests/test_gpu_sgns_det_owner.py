"""The deterministic skip-gram kernel (`mvb_sgns_train_det`) over many waves, where a row that one reader of a
wave reads alone is written in place by that reader and every other row goes through the fixed-point
accumulator and the apply.

Every wave but the first of a call runs both paths, so these cases span several waves.  Their exact bits
(tables, loss, pair count) must match digests recorded from the accumulator-only kernel
(tests/golden/record_sgns_det_owner.py), and two of them are checked against an fp64 model of the wave
schedule in which every read sees the tables as the previous wave left them."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
M64 = (1 << 64) - 1


def _recorder():
    spec = importlib.util.spec_from_file_location("record_sgns_det_owner",
                                                  os.path.join(GOLDEN, "record_sgns_det_owner.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _sm132():
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip("digests and wave sizes are those of a 132-SM H100")


@pytest.mark.parametrize("case", ["zipf_v200k", "uniform_v1m", "hot_v40", "maps_ld320_v100k", "dim37_v100k",
                                  "dim512_w15_k7", "zipf_v200k_2calls"])
def test_sgns_det_owner_bits_match_recorded(mv_device, case):
    with open(os.path.join(GOLDEN, "sgns_det_owner.json")) as f:
        want = json.load(f)["cases"][case]
    _sm132()
    assert _recorder().run_case(case) == want


def _hash64(x):
    x = x.astype(np.uint64)
    x ^= x >> np.uint64(33); x *= np.uint64(0xff51afd7ed558ccd)
    x ^= x >> np.uint64(33); x *= np.uint64(0xc4ceb9fe1a85ec53)
    x ^= x >> np.uint64(33)
    return x


def _model(case, wave):
    """fp64 model of the wave schedule: (w_in, w_out) after training, and the rows any wave read."""
    c = case["c"]
    V, D, W, K, lr, seed = c["V"], c["D"], c["W"], c["K"], case["lr"], case["seed"]
    tl = case["tokens"].numpy().astype(np.int64)
    n = len(tl)
    m = case["map"].numpy().astype(np.int64) if case["map"] is not None else np.arange(V)
    si = case["s_in"].double().numpy() if case["s_in"] is not None else np.ones(V)
    so = case["s_out"].double().numpy() if case["s_out"] is not None else np.ones(V)
    IN, OUT = case["w_in"][:, :D].double(), case["w_out"][:, :D].double()     # by table row
    read_in, read_out = np.zeros(V, dtype=bool), np.zeros(V, dtype=bool)
    with np.errstate(over="ignore"):
        pos = np.arange(n, dtype=np.uint64)
        prng = _hash64(np.uint64(seed) ^ ((pos + np.uint64(1)) * np.uint64(0x9E3779B97F4A7C15)))
        hw = W - (prng >> np.uint64(16)) % np.uint64(W)
        negs = np.full((n, K), -1, dtype=np.int64)
        for k in range(1, K + 1):
            r = _hash64(prng ^ np.uint64((k * 0xD6E8FEB86659FD93) & M64))
            if case["pool"] is not None:
                pool = case["pool"].numpy().astype(np.int64)
                t = pool[((r >> np.uint64(8)) % np.uint64(len(pool))).astype(np.int64)]
            else:
                idx = ((r >> np.uint64(32)) % np.uint64(V)).astype(np.int64)
                u = (r & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(1.0 / 16777216.0)
                prob, alias = case["prob"].numpy(), case["alias"].numpy().astype(np.int64)
                t = np.where(u < prob[idx], idx, alias[idx])
            negs[:, k - 1] = np.where(t == tl, -1, t)
    for p0 in range(0, n, wave):
        cr, cw, orow, ow, lab = [], [], [], [], []
        for p in range(p0, min(p0 + wave, n)):
            if tl[p] < 0:
                continue
            ctxs = []
            for sgn in (-1, 1):
                for d in range(1, int(hw[p]) + 1):
                    q = p + sgn * d
                    if q < 0 or q >= n or tl[q] < 0:
                        break
                    ctxs.append(tl[q])
            outs = [(tl[p], 1.0)] + [(t, 0.0) for t in negs[p] if t >= 0]
            for x in ctxs:
                for (o, label) in outs:
                    cw.append(x); ow.append(o); lab.append(label)
        cw, ow = np.array(cw, dtype=np.int64), np.array(ow, dtype=np.int64)
        cr, orow = torch.from_numpy(m[cw]), torch.from_numpy(m[ow])
        read_in[m[cw]] = True
        read_out[m[ow]] = True
        h, o = IN[cr], OUT[orow]
        g = (torch.tensor(lab, dtype=torch.float64) - torch.sigmoid((h * o).sum(1))) * lr
        d_in = torch.zeros_like(IN).index_add_(0, cr, (g * torch.from_numpy(si[cw]))[:, None] * o)
        d_out = torch.zeros_like(OUT).index_add_(0, orow, (g * torch.from_numpy(so[ow]))[:, None] * h)
        IN += d_in
        OUT += d_out
    return IN, OUT, read_in, read_out


@pytest.mark.parametrize("case", ["zipf_v200k", "maps_ld320_v100k"])
def test_sgns_det_owner_matches_wave_model(mv_device, case):
    """Tables after training against the fp64 wave model (the bounds of test_gpu_sgns_det_tiles); rows no wave
    read and the pad columns keep their bits, and so does the -0.0 column, whose deltas are all zero."""
    from multiverso_b200 import _native as N
    _sm132()
    rec = _recorder()
    cs = rec.make_case(case)
    c = cs["c"]
    D = c["D"]
    wave = N.cuda_lib().mvb_sgns_win_inflight(D, c["K"], c["W"])
    assert c["n_tok"] > 3 * wave
    w_in, w_out, _, _ = rec.train(cs)
    IN, OUT, read_in, read_out = _model(cs, wave)
    for got, init, ref, read in ((w_in, cs["w_in"], IN, read_in), (w_out, cs["w_out"], OUT, read_out)):
        assert torch.equal(got[:, D:].view(torch.int32), init[:, D:].view(torch.int32))
        assert torch.equal(got[:, 3].view(torch.int32), init[:, 3].view(torch.int32))
        unread = torch.from_numpy(~read)
        assert 0 < int(unread.sum()) < c["V"]
        assert torch.equal(got[unread].view(torch.int32), init[unread].view(torch.int32))
        d_got, d_ref = got[:, :D].double() - init[:, :D].double(), ref - init[:, :D].double()
        err = float(torch.linalg.norm(d_got - d_ref) / torch.linalg.norm(d_ref))
        assert err < 1e-4, err
