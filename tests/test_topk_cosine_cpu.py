"""CPU tier of the cosine top-k search and the word-vector evaluation tool: the vector-file parser on files
written by build/bin/wordembedding, the question / similarity parsers, Spearman against scipy, the host
implementation of ``topk_cosine`` against numpy brute force, and the CLI's JSON on planted embeddings."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def planted_fixture(d, binary=False, seed=0):
    """Vectors where capital_i = country_i + r + small noise among random distractors, an analogy file with
    a planted section, a section whose answers are random distractors and out-of-vocabulary lines, and a
    similarity file whose scores are a monotone function of the vectors' cosines.
    Returns (paths, expected) with the exact counts the CLI must report."""
    rng = np.random.default_rng(seed)
    D, P, X = 48, 20, 300
    r = rng.normal(size=D)
    country = rng.normal(size=(P, D))
    capital = country + r + 0.05 * rng.normal(size=(P, D))
    distract = rng.normal(size=(X, D))
    words = [f"country{i}" for i in range(P)] + [f"capital{i}" for i in range(P)] + [f"x{j}" for j in range(X)]
    vecs = np.concatenate([country, capital, distract]).astype(np.float32)
    vpath = os.path.join(d, "vec.bin" if binary else "vec.txt")
    with open(vpath, "wb") as f:
        f.write(f"{len(words)} {D}\n".encode())
        for w, v in zip(words, vecs):
            if binary:
                f.write(w.encode() + b" " + v.tobytes() + b"\n")
            else:
                f.write((w + " " + " ".join(f"{x:.6f}" for x in v) + "\n").encode())
    if not binary:                                       # the values as the file holds them
        vecs = np.array([[f"{x:.6f}" for x in v] for v in vecs]).astype(np.float32)
    qpath = os.path.join(d, "questions.txt")
    n_planted = n_random = n_oov = 0
    with open(qpath, "w") as f:
        f.write(": capital-planted\n")
        for i in range(P):
            for j in range(P):
                if i != j:
                    f.write(f"country{i} capital{i} country{j} capital{j}\n")
                    n_planted += 1
        f.write(": random\n")
        for i in range(1, P):
            f.write(f"country0 capital0 country{i} x{int(rng.integers(X))}\n")
            n_random += 1
        for i in range(5):
            f.write(f"country{i} capital{i} nosuchword{i} capital0\n")
            n_oov += 1
    spath = os.path.join(d, "pairs.txt")
    pairs = set()
    while len(pairs) < 60:
        a, b = rng.integers(len(words), size=2)
        if a != b:
            pairs.add((int(a), int(b)))
    with open(spath, "w") as f:
        f.write("# word1 word2 human score\n")
        for a, b in sorted(pairs):
            va, vb = vecs[a].astype(np.float64), vecs[b].astype(np.float64)
            c = va @ vb / (np.linalg.norm(va) * np.linalg.norm(vb))
            f.write(f"{words[a]} {words[b]} {np.exp(3 * c):.12f}\n")
        f.write("nosuchword capital0 5.0   # out of vocabulary\n")
    expected = dict(planted=n_planted, random=n_random, oov=n_oov, pairs=len(pairs), pairs_skipped=1)
    return dict(vectors=vpath, analogy=qpath, similarity=spath, words=words, vecs=vecs), expected


def check_planted_result(res, exp):
    an = res["analogy"]
    assert an["sections"]["capital-planted"] == {"correct": exp["planted"], "seen": exp["planted"], "accuracy": 1.0}
    assert an["sections"]["random"]["correct"] == 0 and an["sections"]["random"]["seen"] == exp["random"]
    assert an["seen"] == exp["planted"] + exp["random"] and an["skipped"] == exp["oov"]
    assert an["correct"] == exp["planted"]
    sim = res["similarity"]
    assert sim["pairs"] == exp["pairs"] and sim["skipped"] == exp["pairs_skipped"]
    assert abs(sim["spearman"] - 1.0) < 1e-12


# ------------------------------------------------------------------------------------------ parsers
@pytest.fixture(scope="module")
def native_vectors(tmp_path_factory):
    from multiverso_b200 import _build
    _build.build_host()
    d = tmp_path_factory.mktemp("vec")
    corpus = d / "corpus.txt"
    rng = np.random.default_rng(0)
    with open(corpus, "w") as f:
        for _ in range(2000):
            f.write(" ".join(f"t{rng.integers(4)}w{w}" for w in rng.integers(20, size=8)) + "\n")
    out = {}
    for binary in (0, 1):
        path = str(d / f"vec{binary}")
        r = subprocess.run([os.path.join(ROOT, "build", "bin", "wordembedding"), "-train_file", str(corpus),
                            "-output", path, "-size", "20", "-epoch", "1", "-threads", "1", "-min_count", "1",
                            "-binary", str(binary)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, r.stderr[-2000:]
        out[binary] = path
    return out


@pytest.mark.parametrize("binary", [0, 1])
def test_load_vectors_native_files(native_vectors, binary):
    from multiverso_b200.apps.wordembedding_eval import load_vectors
    from test_native_apps import load_embeddings
    words, vecs = load_vectors(native_vectors[binary], bool(binary))
    ref_words, ref = load_embeddings(native_vectors[binary], bool(binary))
    assert words == ref_words and vecs.dtype == np.float32
    np.testing.assert_array_equal(vecs, ref)
    assert vecs.shape == (80, 20)


def test_load_vectors_rejects_short_lines(tmp_path):
    from multiverso_b200.apps.wordembedding_eval import load_vectors
    p = tmp_path / "bad.txt"
    p.write_text("2 3\na 1 2 3\nb 1 2\n")
    with pytest.raises(ValueError):
        load_vectors(str(p), False)


def test_question_and_pair_parsers(tmp_path):
    from multiverso_b200.apps.wordembedding_eval import read_pairs, read_questions
    q = tmp_path / "q.txt"
    q.write_text(": capital-common-countries\nAthens Greece Baghdad Iraq\n\n: family\nboy girl brother sister\n"
                 "bad line\n")
    assert read_questions(str(q)) == [("capital-common-countries", ["Athens", "Greece", "Baghdad", "Iraq"]),
                                      ("family", ["boy", "girl", "brother", "sister"])]
    s = tmp_path / "s.txt"
    s.write_text("# Word 1\tWord 2\tHuman (mean)\nlove\tsex\t6.77\ntiger cat 7.35  # trailing\n\nshort 1\n")
    assert read_pairs(str(s)) == [("love", "sex", 6.77), ("tiger", "cat", 7.35)]


def test_spearman_matches_scipy_with_ties():
    from scipy.stats import spearmanr
    from multiverso_b200.apps.wordembedding_eval import spearman
    rng = np.random.default_rng(3)
    for _ in range(20):
        n = int(rng.integers(3, 60))
        x = rng.integers(0, 6, size=n).astype(float)         # many ties
        y = x + rng.normal(size=n) * rng.random()
        y[rng.random(n) < 0.3] = 1.0
        ref = spearmanr(x, y).statistic
        got = spearman(x, y)
        if np.isnan(ref):
            assert np.isnan(got)
        else:
            assert abs(got - ref) < 1e-12, (got, ref)
    assert np.isnan(spearman([1.0], [2.0]))


# ------------------------------------------------------------------------------------------ host top-k
def _brute(W, Q, k, rows):
    """numpy fp64 brute force with the (score desc, id asc) order; zero rows score 0."""
    dim = Q.shape[1]
    Wd = W[:rows, :dim].astype(np.float64)
    wn = np.linalg.norm(Wd, axis=1)
    Wu = Wd / np.where(wn > 0, wn, 1)[:, None]
    Qd = Q.astype(np.float64)
    Qu = Qd / np.linalg.norm(Qd, axis=1, keepdims=True)
    S = Qu @ Wu.T
    ids = np.full((len(Q), k), -1)
    sc = np.full((len(Q), k), -np.inf)
    for m in range(len(Q)):
        o = np.lexsort((np.arange(rows), -S[m]))[:k]
        ids[m, :len(o)] = o
        sc[m, :len(o)] = S[m, o]
    return sc, ids


@pytest.mark.parametrize("n,pitch,dim,k,rows", [(1000, 32, 32, 10, None), (257, 104, 100, 40, None),
                                                 (5, 300, 300, 10, None), (3000, 68, 64, 64, 1777)])
def test_host_topk_matches_bruteforce(n, pitch, dim, k, rows):
    from multiverso_b200.ops import topk_cosine
    rng = np.random.default_rng(n)
    W = rng.normal(size=(n, pitch)).astype(np.float32)
    W[:, dim:] = 1e6                                     # padding columns never count
    W[3] = 0.0                                           # a zero row scores 0
    Q = rng.normal(size=(13, dim)).astype(np.float32)
    if n > 11:
        W[7] = W[11]                                     # duplicates: both come back, the smaller id first
        Q[0] = W[11, :dim]
    s, i = topk_cosine(torch.from_numpy(W), torch.from_numpy(Q), k, rows=rows)
    rs, ri = _brute(W, Q, k, n if rows is None else rows)
    np.testing.assert_array_equal(i.numpy(), ri)
    np.testing.assert_allclose(s.numpy(), rs, atol=1e-5)
    if n > 11:
        assert list(i[0, :2].numpy()) == [7, 11]
    if k >= n:
        assert s[:, n:].isinf().all() and (i[:, n:] == -1).all()
        assert (s[i == 3] == 0).all()


def test_host_topk_tie_rule_and_chunks():
    from multiverso_b200.ops import topk_cosine_reference
    W = np.tile(np.eye(4, dtype=np.float32), (50, 1))         # 50 copies of every direction
    Q = np.eye(4, dtype=np.float32)[[2]]
    s, i = topk_cosine_reference(torch.from_numpy(W), torch.from_numpy(Q), 10, row_chunk=7)
    assert i[0].tolist() == [2 + 4 * j for j in range(10)] and (s == 1).all()


def test_host_topk_errors():
    from multiverso_b200.ops import topk_cosine
    W = torch.randn(10, 8)
    with pytest.raises(ValueError):
        topk_cosine(W, torch.randn(2, 8), 0)
    with pytest.raises(ValueError):
        topk_cosine(W, torch.randn(2, 8), 65)
    with pytest.raises(TypeError):
        topk_cosine(W, torch.randn(2, 8, dtype=torch.float64), 3)
    with pytest.raises(ValueError):
        topk_cosine(W, torch.randn(2, 9), 3)
    with pytest.raises(ValueError):
        topk_cosine(W, torch.randn(2, 8), 3, rows=11)


# ------------------------------------------------------------------------------------------ CLI
@pytest.mark.parametrize("binary", [0, 1])
def test_eval_cli_planted_host(tmp_path, binary, capsys):
    from multiverso_b200.apps import wordembedding_eval as ev
    fx, exp = planted_fixture(str(tmp_path), bool(binary))
    res = ev.run(["-vectors", fx["vectors"], "-binary", str(binary), "-analogy", fx["analogy"],
                  "-similarity", fx["similarity"], "-neighbours", "country3,nosuchword", "-k", "5",
                  "-device", "cpu"])
    line = [l for l in capsys.readouterr().out.splitlines() if l.startswith("{")]
    assert json.loads(line[-1]) == json.loads(json.dumps(res))
    check_planted_result(res, exp)
    assert res["vectors"] == len(fx["words"]) and res["device"] == "cpu"
    nb = res["neighbours"]
    assert nb["nosuchword"] is None and len(nb["country3"]) == 5
    assert nb["country3"][0][0] == "capital3"            # capital3 = country3 + r: nearest after itself


def test_eval_cli_threshold_skips(tmp_path):
    from multiverso_b200.apps import wordembedding_eval as ev
    fx, exp = planted_fixture(str(tmp_path))
    # the first 30 words: country0..19 and capital0..9; questions using capital10..19 are skipped
    res = ev.run(["-vectors", fx["vectors"], "-analogy", fx["analogy"], "-threshold", "30", "-device", "cpu"])
    an = res["analogy"]
    kept = sum(1 for i in range(20) for j in range(20) if i != j and i < 10 and j < 10)
    assert an["sections"]["capital-planted"]["seen"] == kept
    assert an["sections"]["capital-planted"]["correct"] == kept
    assert an["skipped"] == exp["oov"] + exp["planted"] - kept + exp["random"]


def test_eval_cli_usage(capsys):
    from multiverso_b200.apps import wordembedding_eval as ev
    assert ev.run([]) == {}
    assert "usage" in capsys.readouterr().out
    with pytest.raises(SystemExit):
        ev.run(["-vectorz", "x"])


def test_eval_cli_neighbours_k_limit(tmp_path):
    from multiverso_b200.apps import wordembedding_eval as ev
    fx, _ = planted_fixture(str(tmp_path))
    base = ["-vectors", fx["vectors"], "-neighbours", "country3", "-device", "cpu"]
    assert len(ev.run(base + ["-k", "63"])["neighbours"]["country3"]) == 63
    with pytest.raises(ValueError, match=r"k must be in \[1, 63\], got 64"):
        ev.run(base + ["-k", "64"])
