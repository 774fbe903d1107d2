"""The plan of the deterministic skip-gram kernel (`mvb_sgns_train_det`) at its edges, and its scratch memory.

Before its first wave a call plans the whole block: every position's input row, every centre's output rows and
window, and one reader per (wave, table, row) read, sorted by that key to find the rows a wave reads once (written
in place by their reader) and the rows it shares (summed in a compact accumulator, one slot per shared row).
These tests run blocks whose plan is unusual -- shorter than one wave, a short last wave, no reader at all, sort
keys wider than 32 bits -- against the fp64 wave model of test_gpu_sgns_det_owner.py, and check that rows no wave
read keep their bits.  A subprocess checks that the scratch of a 1M-word block at the shape `bench.py` trains
stays under 1 GB."""
import importlib.util
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _wave(D, K, W):
    from multiverso_b200 import _native as N
    return N.cuda_lib().mvb_sgns_win_inflight(D, K, W)


def _case(tokens, rows, D, W=5, K=5, V=None, word_map=None, pool=None, scales=True, seed=0x5EED):
    """A case in the layout of tests/golden/record_sgns_det_owner.py: `rows` table rows, words [0, V)."""
    V = rows if V is None else V
    g = torch.Generator().manual_seed(rows + D)
    w_in = ((torch.rand(rows, D, generator=g) - 0.5) * 0.4)
    w_out = ((torch.rand(rows, D, generator=g) - 0.5) * 0.4)
    s_in, s_out = 0.5 + torch.rand(V, generator=g), 0.5 + torch.rand(V, generator=g)
    c = dict(V=V, D=D, LD=D, W=W, K=K, n_tok=len(tokens))
    return dict(c=c, tokens=torch.as_tensor(tokens, dtype=torch.int32), w_in=w_in, w_out=w_out,
                map=None if word_map is None else torch.as_tensor(word_map, dtype=torch.int32),
                prob=None, alias=None, pool=torch.as_tensor(pool, dtype=torch.int32),
                s_in=s_in if scales else None, s_out=s_out if scales else None, lr=2e-2, seed=seed)


def _check(case, wave):
    rec = _load("record_sgns_det_owner", os.path.join(HERE, "golden", "record_sgns_det_owner.py"))
    model = _load("sgns_det_owner_model", os.path.join(HERE, "test_gpu_sgns_det_owner.py"))
    D = case["c"]["D"]
    init_in, init_out = case["w_in"].clone(), case["w_out"].clone()
    w_in, w_out, pairs, loss = rec.train(case)
    IN, OUT, read_in, read_out = model._model(case, wave)
    for got, init, ref, read in ((w_in, init_in, IN, read_in), (w_out, init_out, OUT, read_out)):
        unread = torch.from_numpy(~read[:got.shape[0]])      # the model marks the table rows it read
        assert 0 < int(unread.sum()) < got.shape[0]
        assert torch.equal(got[unread].view(torch.int32), init[unread].view(torch.int32))
        d_got, d_ref = got[:, :D].double() - init[:, :D].double(), ref - init[:, :D].double()
        err = float(torch.linalg.norm(d_got - d_ref) / torch.linalg.norm(d_ref))
        assert err < 1e-4, err
    assert pairs > 0 and loss > 0


def test_sgns_det_plan_block_shorter_than_a_wave(mv_device):
    V, D = 4096, 64
    wave = _wave(D, 5, 5)
    g = np.random.default_rng(1)
    toks = g.integers(0, V - 16, 1000)
    toks[::97] = -1
    assert len(toks) < wave
    _check(_case(toks, V, D, pool=list(range(V - 16, V))), wave)


def test_sgns_det_plan_short_last_wave(mv_device):
    """Two full waves and one of 37 centres; 500 words, so most rows are shared by many readers."""
    V, D = 600, 100
    wave = _wave(D, 5, 5)
    g = np.random.default_rng(2)
    toks = g.integers(0, 500, 2 * wave + 37)
    toks[250::251] = -1
    _check(_case(toks, V, D, pool=g.integers(0, 500, 50)), wave)


def test_sgns_det_plan_only_sentence_breaks(mv_device):
    """No centre trains: no reader, an empty list of shared rows in every wave, tables and counters untouched."""
    V, D = 4096, 300
    wave = _wave(D, 5, 5)
    case = _case(np.full(wave + 100, -1), V, D, pool=list(range(16)))
    rec = _load("record_sgns_det_owner", os.path.join(HERE, "golden", "record_sgns_det_owner.py"))
    init_in, init_out = case["w_in"].clone(), case["w_out"].clone()
    w_in, w_out, pairs, loss = rec.train(case)
    assert torch.equal(w_in.view(torch.int32), init_in.view(torch.int32))
    assert torch.equal(w_out.view(torch.int32), init_out.view(torch.int32))
    assert pairs == 0 and loss == 0.0


def test_sgns_det_plan_keys_wider_than_32_bits(mv_device):
    """Sort keys (wave, table, row) = (2 wave + table) * vocab + row beyond 2^32: 8.4M words and 257 waves.
    The words are mapped to 40k cache slots of 4 floats, so the tables and the fp64 model stay small."""
    V, rows, D = 8_400_000, 40_000, 4
    wave = _wave(D, 5, 5)
    n_waves = 257
    assert (n_waves - 1) * 2 * V >= 1 << 32
    g = np.random.default_rng(3)
    words = g.choice(V, rows, replace=False)
    word_map = np.full(V, -1, dtype=np.int64)
    word_map[words] = g.permutation(rows)
    toks = words[g.integers(0, 30_000, (n_waves - 1) * wave + 11)]
    toks[400::401] = -1
    _check(_case(toks, rows, D, V=V, word_map=word_map, pool=words[:5000], scales=False), wave)


_MEMORY = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
import multiverso_b200 as mv
from multiverso_b200 import _native as N
from multiverso_b200.models.wordembedding import synthetic_zipf_corpus
mv.init()
try:
    V, D, n = 1_000_000, 300, 1 << 20
    w_in = (torch.rand(V, D, device="cuda") - 0.5) / D
    w_out = torch.zeros(V, D, device="cuda")
    toks = torch.from_numpy(synthetic_zipf_corpus(n, V, 1000, seed=5)).cuda()
    pool = torch.randint(0, V, (1 << 20,), dtype=torch.int32, device="cuda")
    out = torch.zeros(2, dtype=torch.int64, device="cuda")
    a = N.Sgns()
    a.tokens, a.n_tokens, a.w_in, a.w_out = toks.data_ptr(), n, w_in.data_ptr(), w_out.data_ptr()
    a.dim, a.ld, a.window, a.negative, a.lr, a.seed, a.vocab = D, D, 5, 5, 0.025, 1, V
    a.neg_pool, a.neg_pool_size = pool.data_ptr(), pool.numel()
    a.pair_count, a.loss_sum = out.data_ptr(), out.data_ptr() + 8
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    rc = N.cuda_lib().mvb_sgns_train_det(a, N.stream_ptr())
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    print(json.dumps({"rc": rc, "drop": free0 - free1, "pairs": int(out[0])}))
finally:
    mv.shutdown()
"""


def test_sgns_det_plan_scratch_under_1gb():
    """The first call of a process allocates the scratch: at vocab 1M, dim 300 and 1M tokens the device's free
    memory drops by less than 1 GB (a dense accumulator over the vocabulary took 4.85 GB)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    r = subprocess.run([sys.executable, "-c", _MEMORY, ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["rc"] == 0 and res["pairs"] > 0
    assert res["drop"] < 1 << 30, res
