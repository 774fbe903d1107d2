"""The Huffman encoder of hierarchical softmax (`MVA_HuffmanBuild`, csrc/host/applib/wordembedding_data.cpp)
and the integer frequencies `HuffmanTables` gives it, against an exact-integer `heapq` Huffman.

Huffman trees are not unique under ties, but their cost sum(freq * len) is: every check of optimality
compares that cost, and the tree itself is checked for what the kernels rely on (root-first paths from
inner node V-2, prefix-free codes, inner-node ids in [0, V-1), two children per inner node with codes 0 / 1)."""
import ctypes as C
import heapq

import numpy as np
import pytest

MAX_CODE = 64


def _build(freq, max_code=MAX_CODE):
    from multiverso_b200.apps._applib import lib
    freq = np.ascontiguousarray(np.asarray(freq, dtype=np.int64))
    V = len(freq)
    P = np.full((V, max_code), -7, dtype=np.int32)
    Cd = np.full((V, max_code), -7, dtype=np.int8)
    lens = np.full(V, -7, dtype=np.int32)
    rc = lib().MVA_HuffmanBuild(freq.ctypes.data_as(C.c_void_p), V, max_code, P.ctypes.data_as(C.c_void_p),
                                Cd.ctypes.data_as(C.c_void_p), lens.ctypes.data_as(C.c_void_p))
    return rc, P, Cd, lens


def _optimal_cost(freq):
    """sum(freq * len) of a Huffman code = the sum of all merged weights, in exact Python integers."""
    h = [int(f) for f in freq]
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        s = heapq.heappop(h) + heapq.heappop(h)
        cost += s
        heapq.heappush(h, s)
    return cost


def _check_tree(freq, rc, P, Cd, lens):
    V = len(freq)
    assert rc == int(lens.max()) and (lens >= 0).all()
    assert sum(int(f) * int(n) for f, n in zip(freq, lens)) == _optimal_cost(freq)
    if V == 1:
        assert lens[0] == 0
        return
    assert (lens >= 1).all()
    codes = ["".join(str(int(b)) for b in Cd[w, :lens[w]]) for w in range(V)]
    s = sorted(codes)
    assert all(not s[i + 1].startswith(s[i]) for i in range(V - 1)), "codes are not prefix-free"
    child = {}                                   # (inner node, branch code) -> child (inner node or ("leaf", w))
    for w in range(V):
        n = int(lens[w])
        pts, cds = P[w, :n], Cd[w, :n]
        assert pts[0] == V - 2, "path does not start at the root"
        assert ((pts >= 0) & (pts < V - 1)).all() and np.isin(cds, (0, 1)).all()
        for d in range(n):
            nxt = int(pts[d + 1]) if d + 1 < n else ("leaf", w)
            assert child.setdefault((int(pts[d]), int(cds[d])), nxt) == nxt, "inner node with two children on one branch"
    # all V - 1 inner nodes appear, each with exactly a 0-child and a 1-child
    assert sorted(child) == [(i, b) for i in range(V - 1) for b in (0, 1)]


def _zipf(V, total):
    w = 1.0 / np.arange(1, V + 1)
    return np.maximum(np.round(w / w.sum() * total), 1).astype(np.int64)


def _freqs(kind, V, rng):
    if kind == "random":
        return rng.integers(1, 10 ** 6, size=V)
    if kind == "zipf":
        return _zipf(V, 10 ** 7)
    if kind == "uniform":
        return np.full(V, 5, dtype=np.int64)
    if kind == "tied":                                   # few distinct values, many ties between leaves and sums
        return rng.choice(np.array([1, 2, 3, 4, 8], dtype=np.int64), size=V)
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["random", "zipf", "uniform", "tied"])
@pytest.mark.parametrize("V", [1, 2, 3, 4, 5, 17, 64, 1000, 5000])
def test_huffman_build_is_an_optimal_prefix_tree(kind, V):
    freq = _freqs(kind, V, np.random.default_rng(V))
    rc, P, Cd, lens = _build(freq)
    _check_tree(freq, rc, P, Cd, lens)


def test_huffman_build_v1_and_v2():
    rc, _, _, lens = _build([42])
    assert rc == 0 and lens[0] == 0
    rc, P, Cd, lens = _build([3, 9])
    assert rc == 1 and list(lens) == [1, 1] and P[0, 0] == P[1, 0] == 0 and sorted(Cd[:, 0]) == [0, 1]


def test_huffman_tables_one_word_has_one_column():
    """A builder return of 0 (one word, empty code) still gives tables of width max_code = 1."""
    from multiverso_b200.models.wordembedding import HuffmanTables
    h = HuffmanTables(np.array([5.0]), "cpu")
    assert h.max_code == 1 and h.points.shape == (1, 1) and h.codes.shape == (1, 1) and int(h.lens[0]) == 0
    h = HuffmanTables(np.array([5.0, 7.0]), "cpu")
    assert h.max_code == 1 and h.points.shape == (2, 1) and sorted(h.lens.tolist()) == [1, 1]


def test_huffman_build_rejects_codes_longer_than_max_code():
    """42 Fibonacci frequencies make a chain: the two rarest words sit 41 levels deep."""
    fib = [1, 1]
    while len(fib) < 42:
        fib.append(fib[-1] + fib[-2])
    rc, P, Cd, lens = _build(fib, max_code=41)
    assert rc == 41 and sorted(lens.tolist())[-2:] == [41, 41]
    _check_tree(fib, rc, P, Cd, lens)
    assert _build(fib, max_code=40)[0] == -1
    assert _build(fib[:41], max_code=40)[0] == 40


def _cost(counts, lens):
    return sum(int(c) * int(n) for c, n in zip(counts, lens))


def test_huffman_tables_optimal_for_large_integer_counts():
    """Zipf counts over 5000 words totalling 3e11: the code lengths must be optimal for the counts
    themselves (scaling them by 1e9 would overflow the encoder's int64 frequencies)."""
    from multiverso_b200.models.wordembedding import HuffmanTables
    counts = _zipf(5000, 3 * 10 ** 11)
    h = HuffmanTables(counts.astype(np.float64), "cpu")
    assert _cost(counts, h.lens.numpy()) == _optimal_cost(counts)


def test_huffman_frequencies_stay_below_the_int64_limit():
    from multiverso_b200.models.wordembedding import HuffmanTables
    w = 1.0 / np.arange(1, 5001)
    f = HuffmanTables.int_frequencies(w)                      # fractional weights: scaled by 1e9
    assert f.dtype == np.int64 and f[0] == 10 ** 9 and np.array_equal(f, np.floor(w * 1e9))
    assert np.array_equal(HuffmanTables.int_frequencies(np.array([0.0, 3.0, 7.0])), [1, 3, 7])   # whole counts as they are
    for big in (w * 1e12, np.round(w * 1e19)):               # totals above 2^62, fractional and whole
        f = HuffmanTables.int_frequencies(big)
        assert (f >= 1).all() and sum(int(x) for x in f) < 2 ** 62
        assert _cost(f, HuffmanTables(big, "cpu").lens.numpy()) == _optimal_cost(f)
