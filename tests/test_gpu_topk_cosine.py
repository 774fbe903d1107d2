"""Fused cosine top-k kernel (csrc/cuda/topk_cos.cu) against fp64, over multi-shard row maps, its tie /
edge-row rules, the WordEmbedding search API and the evaluation CLI on the GPU."""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

TOL = 1e-5


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _fp64_cos(W, Q, rows):
    dim = Q.shape[1]
    Wd = W[:rows, :dim].double()
    wn = Wd.norm(dim=1)
    Wu = Wd / torch.where(wn > 0, wn, torch.ones_like(wn))[:, None]
    Qd = Q.double()
    return (Qd / Qd.norm(dim=1, keepdim=True)) @ Wu.T


def _check(W, Q, k, rows, s, i):
    """Scores within TOL of the fp64 cosine of the returned ids; the id set is the fp64 top-k except for rows
    within TOL of the k-th score; scores descend, equal scores with ascending ids; missing slots -1 / -inf."""
    C = _fp64_cos(W, Q, rows).cpu()
    s, i = s.cpu(), i.cpu()
    kk = min(k, rows)
    assert (i[:, kk:] == -1).all() and torch.isinf(s[:, kk:]).all() and (s[:, kk:] < 0).all()
    assert not torch.isnan(s).any()
    got = i[:, :kk]
    assert (got >= 0).all() and (got < rows).all()
    ref = C.gather(1, got)
    assert (s[:, :kk].double() - ref).abs().max().item() < TOL
    sd, si = s[:, :kk], i[:, :kk]
    assert (sd[:, 1:] <= sd[:, :-1]).all()
    tie = sd[:, 1:] == sd[:, :-1]
    assert (si[:, 1:][tie] > si[:, :-1][tie]).all()
    vals, _ = C.topk(kk, dim=1)
    kth = vals[:, -1:]
    for m in range(Q.shape[0]):
        ref_set = set(torch.nonzero(C[m] > kth[m] + TOL).view(-1).tolist())
        near = set(torch.nonzero((C[m] - kth[m]).abs() <= TOL).view(-1).tolist())
        g = set(got[m].tolist())
        assert ref_set <= g, m
        assert g <= ref_set | near, m


@pytest.mark.parametrize("M,rows,dim,k", [(1, 1000, 300, 10), (77, 100000, 300, 40), (300, 65537, 128, 64),
                                          (130, 257, 100, 1), (4, 5, 300, 10)])
def test_topk_matches_fp64(cuda, M, rows, dim, k):
    from multiverso_b200.ops import TOPK_MAX, topk_cosine
    assert TOPK_MAX == 64
    g = torch.Generator(device=cuda).manual_seed(M + rows)
    pitch = (dim + 3) // 4 * 4
    W = torch.randn(rows, pitch, device=cuda, generator=g)
    W[:, dim:] = 0
    Q = torch.randn(M, dim, device=cuda, generator=g)
    s, i = topk_cosine(W, Q, k)
    _check(W, Q, k, rows, s, i)


def test_topk_padded_pitch_and_row_limit(cuda):
    from multiverso_b200.ops import topk_cosine
    g = torch.Generator(device=cuda).manual_seed(5)
    W = torch.randn(5000, 320, device=cuda, generator=g)
    W[:, 300:] = 1e6 * torch.rand(5000, 20, device=cuda, generator=g)     # padding garbage must not count
    Q = torch.randn(33, 300, device=cuda, generator=g)
    for rows in (None, 1037):                                            # 1037 ends inside a 128-row tile
        n = 5000 if rows is None else rows
        s, i = topk_cosine(W, Q, 20, rows=rows)
        _check(W, Q, 20, n, s, i)
        assert (i < n).all()


def _shard_call(W, Q, k, S, gap=37):
    """The same data as S shards at separate places of one buffer, ``gap`` rows of garbage between them:
    reference rows_per_server rule, the last shard takes the remainder. A kernel that addressed a row of
    shard s > 0 from any base but its own would read the garbage."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops.topk import _topk_device
    n, pitch = W.shape
    rps = n // S
    buf = torch.full((n + S * gap, pitch), 1e3, device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, rps
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
    out = _topk_device(rm, pitch, Q, k, None)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("n", [100003, 1003])
def test_topk_sharded_bitwise_equal(cuda, n):
    from multiverso_b200.ops import topk_cosine
    g = torch.Generator(device=cuda).manual_seed(n)
    W = torch.randn(n, 300, device=cuda, generator=g)
    Q = torch.randn(140, 300, device=cuda, generator=g)
    s1, i1 = topk_cosine(W, Q, 16)
    for S in (3, 8):
        s, i = _shard_call(W, Q, 16, S)
        assert torch.equal(i, i1) and torch.equal(s, s1), S


@pytest.mark.parametrize("nproc", [2, 4])
def test_topk_peer_shards_multi_gpu(nproc):
    """The table sharded over 2 / 4 GPUs (tests/mp_topk_check.py under torchrun): W tiles by TMA from peer HBM,
    candidate rows re-read through peer pointers; bitwise equal to a local single-shard search."""
    import os
    import subprocess
    import sys
    if not torch.cuda.is_available() or torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 200 + nproc
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "mp_topk_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail


def test_topk_query_chunks(cuda):
    """More queries than one kernel call takes: every chunk, the short last one included, gives what a call of
    its own gives."""
    from multiverso_b200.ops import topk_cosine
    from multiverso_b200.ops.topk import _Q_CHUNK
    g = torch.Generator(device=cuda).manual_seed(21)
    W = torch.randn(20000, 64, device=cuda, generator=g)
    for M in (_Q_CHUNK + 1, _Q_CHUNK + 3584):
        Q = torch.randn(M, 64, device=cuda, generator=g)
        s, i = topk_cosine(W, Q, 10)
        s2, i2 = topk_cosine(W, Q[_Q_CHUNK:], 10)
        assert torch.equal(s[_Q_CHUNK:], s2) and torch.equal(i[_Q_CHUNK:], i2)
        _check(W, Q[:300], 10, 20000, s[:300], i[:300])


def test_topk_deterministic_duplicates_zero_rows(cuda):
    from multiverso_b200.ops import topk_cosine
    g = torch.Generator(device=cuda).manual_seed(9)
    W = torch.randn(20000, 64, device=cuda, generator=g)
    W[12345] = W[77]
    Q = torch.randn(500, 64, device=cuda, generator=g)
    Q[0] = W[77]
    a = topk_cosine(W, Q, 10)
    b = topk_cosine(W, Q, 10)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert a[1][0, :2].tolist() == [77, 12345] and a[0][0, 0] == a[0][0, 1]
    Z = torch.randn(5, 32, device=cuda, generator=g)
    Z[1] = 0
    Z[3] = 0
    s, i = topk_cosine(Z, torch.randn(3, 32, device=cuda, generator=g), 10)
    assert not torch.isnan(s).any()
    assert (s[i == 1] == 0).all() and (s[i == 3] == 0).all() and (i[:, :5] >= 0).all()
    assert (i[:, 5:] == -1).all() and torch.isinf(s[:, 5:]).all()


def test_topk_errors(cuda):
    from multiverso_b200.ops import topk_cosine
    W = torch.randn(100, 32, device=cuda)
    Q = torch.randn(2, 32, device=cuda)
    for bad_k in (0, 65):
        with pytest.raises(ValueError):
            topk_cosine(W, Q, bad_k)
    with pytest.raises(TypeError):
        topk_cosine(W, Q.double(), 3)
    with pytest.raises(ValueError):
        topk_cosine(W, torch.randn(2, 33, device=cuda), 3)               # wrong dim
    with pytest.raises(ValueError):
        topk_cosine(torch.randn(100, 30, device=cuda), torch.randn(2, 30, device=cuda), 3)   # pitch % 4
    with pytest.raises(ValueError):
        topk_cosine(W, Q.cpu(), 3)


def test_topk_on_matrix_table(mv_device):
    from multiverso_b200.ops import topk_cosine, topk_cosine_reference
    mv = mv_device
    t = mv.MatrixTable(3000, 64, "float32", min_value=-1.0, max_value=1.0)
    W = t.get().view(3000, 64).clone()
    Q = torch.randn(50, 64, device="cuda")
    s, i = topk_cosine(t, Q, 12, rows=2900)
    rs, ri = topk_cosine_reference(W.cpu(), Q.cpu(), 12, rows=2900)
    assert torch.equal(i.cpu(), ri)
    assert (s.cpu() - rs).abs().max() < TOL


# ------------------------------------------------------------------------------------------ model API
def _we(mv, V, D, **kw):
    from multiverso_b200.models.wordembedding import WordEmbedding, WordEmbeddingOption
    opt = WordEmbeddingOption(embeding_size=D, window_size=2, negative_num=5, init_learning_rate=0.05, **kw)
    return WordEmbedding(opt, vocab_size=V, word_counts=np.ones(V))


def test_model_search_planted(mv_device):
    from multiverso_b200.ops.topk import analogy_queries, take_excluding, topk_cosine_reference
    we = _we(mv_device, 2000, 64)
    rng = np.random.default_rng(1)
    E = rng.normal(size=(2000, 64)).astype(np.float32)
    r = rng.normal(size=64).astype(np.float32)
    E[1000:1020] = E[0:20] + r + 0.05 * rng.normal(size=(20, 64)).astype(np.float32)   # capital_i = country_i + r
    we.input_table.shard.view(2000, 64).copy_(torch.from_numpy(E))
    Et = torch.from_numpy(E)
    ids = torch.arange(0, 40)
    s, i = we.most_similar(ids, k=10)
    rs, ri = topk_cosine_reference(Et, Et[ids], 11)
    rs, ri = take_excluding(rs, ri, ids[:, None], 10)
    assert torch.equal(i.cpu(), ri) and (s.cpu() - rs).abs().max() < TOL
    a, b, c = torch.zeros(19, dtype=torch.int64), torch.full((19,), 1000), torch.arange(1, 20)
    s, i = we.analogy(a, b, c, k=3)
    rs, ri = topk_cosine_reference(Et, analogy_queries(Et[a], Et[b], Et[c]), 6)
    rs, ri = take_excluding(rs, ri, torch.stack([a, b, c], 1), 3)
    assert torch.equal(i.cpu(), ri) and (s.cpu() - rs).abs().max() < TOL
    assert i[:, 0].cpu().tolist() == list(range(1001, 1020))
    assert we.most_similar(ids[:2], k=63)[1].shape == (2, 63)
    assert we.analogy(a[:2], b[:2], c[:2], k=61)[1].shape == (2, 61)
    with pytest.raises(ValueError, match=r"most_similar: k must be in \[1, 63\], got 64"):
        we.most_similar(ids, k=64)
    with pytest.raises(ValueError, match=r"analogy: k must be in \[1, 61\], got 62"):
        we.analogy(a, b, c, k=62)


def test_model_most_similar_after_training(mv_device):
    """The paired corpus of test_gpu_apps (w(2i) is always followed by w(2i+1)), skip-gram: the partner
    must rank among the 10 nearest words for a clear majority of pairs."""
    V = 500
    we = _we(mv_device, V, 64)
    rng = np.random.default_rng(0)
    sents = []
    for _ in range(3000):
        base = rng.integers(0, V // 2, size=12) * 2
        sents.append(np.stack([base, base + 1], 1).reshape(-1))
        sents.append([-1])
    toks = torch.from_numpy(np.concatenate(sents).astype(np.int32)).cuda()
    for _ in range(4):
        we.train_block(toks)
    torch.cuda.synchronize()
    even = torch.arange(0, V, 2)
    _, i = we.most_similar(even, k=10)
    hit = (i.cpu() == (even + 1)[:, None]).any(1).float().mean().item()
    print(f"partner within top-10: {hit:.3f}")
    assert hit >= 0.9, hit                 # 1.000 on one H100


# ------------------------------------------------------------------------------------------ CLI
@pytest.mark.parametrize("binary", [0, 1])
def test_eval_cli_gpu_equals_host(cuda, tmp_path, binary, capsys):
    from multiverso_b200.apps import wordembedding_eval as ev
    from test_topk_cosine_cpu import check_planted_result, planted_fixture
    fx, exp = planted_fixture(str(tmp_path), bool(binary))
    argv = ["-vectors", fx["vectors"], "-binary", str(binary), "-analogy", fx["analogy"],
            "-similarity", fx["similarity"]]
    gpu = ev.run(argv + ["-device", "cuda"])
    host = ev.run(argv + ["-device", "cpu"])
    check_planted_result(gpu, exp)
    assert gpu.pop("device") == "cuda" and host.pop("device") == "cpu"
    assert json.dumps(gpu, sort_keys=True) == json.dumps(host, sort_keys=True)
    nb = ["-neighbours", "country1,capital2,x7", "-k", "8"]
    g = ev.run(argv[:4] + nb + ["-device", "cuda"])["neighbours"]
    h = ev.run(argv[:4] + nb + ["-device", "cpu"])["neighbours"]
    for w in g:
        assert [x[0] for x in g[w]] == [x[0] for x in h[w]]
        assert np.allclose([x[1] for x in g[w]], [x[1] for x in h[w]], atol=1e-5)
