"""Count-based admission of a HashMatrixTable (csrc/cuda/hash_rows.cu) as an exact numpy model, checked without a
GPU: the counter indexes, per-occurrence counts of keys that hold no slot, the estimate, aging at W / 2 and per-call
admission; that the sketch never under-counts and is exact without collisions; and the argument refusals that need
no device. tests/test_gpu_hash_admission.py compares the kernels bitwise with `SketchModel`."""
import numpy as np
import pytest

M64 = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15
INT64_MIN = -(1 << 63)


def hash64_np(x):
    """MurmurHash3's 64-bit finaliser (hash64 of mvb_common.cuh) on a uint64 array."""
    x = np.asarray(x, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xFF51AFD7ED558CCD)
        x ^= x >> np.uint64(33)
        x *= np.uint64(0xC4CEB9FE1A85EC53)
        x ^= x >> np.uint64(33)
    return x


def cells(keys, W):
    """[4, n] flat counter indexes of int64 `keys` in one server's sketch: row r at r W +
    ((hash64(key + (r + 1) GOLD) >> 32) & (W - 1))."""
    k = np.asarray(keys, dtype=np.int64).view(np.uint64)
    out = np.empty((4, k.size), np.int64)
    with np.errstate(over="ignore"):
        for r in range(4):
            h = hash64_np(k + np.uint64(((r + 1) * GOLD) & M64))
            out[r] = r * W + ((h >> np.uint64(32)) & np.uint64(W - 1)).astype(np.int64)
    return out


class SketchModel:
    """S servers' sketches (uint32 counters [S, 4 W], uint64 totals [S]) and the keys that hold a slot.

    ``call(keys)`` is one inserting lookup: every occurrence of a key that holds no slot adds 1 to its 4 counters and
    to its owner's total; then every such key whose estimate (the minimum of its counters) is >= n gets a slot; then
    each server whose total reached R = W / 2 has its counters and total shifted right by the smallest k that takes
    the total below R. Returns the set of keys admitted by the call."""

    def __init__(self, S, W, n):
        self.S, self.W, self.n, self.R = S, W, n, W // 2
        self.counters = np.zeros((S, 4 * W), np.int64)
        self.total = np.zeros(S, np.int64)
        self.held = set()

    def owner(self, keys):
        return np.remainder(np.asarray(keys, np.int64), self.S)

    def estimate(self, keys):
        keys = np.asarray(keys, np.int64)
        c = cells(keys, self.W)
        s = self.owner(keys)
        return np.min(np.stack([self.counters[s, c[r]] for r in range(4)]), 0)

    def count(self, keys):
        keys = np.asarray(keys, np.int64)
        keys = keys[(keys != INT64_MIN) & ~np.isin(keys, np.fromiter(self.held, np.int64, len(self.held)))]
        if keys.size:
            c, s = cells(keys, self.W), self.owner(keys)
            for r in range(4):
                np.add.at(self.counters, (s, c[r]), 1)
            np.add.at(self.total, s, 1)

    def admit(self, keys):
        cand = np.unique(np.asarray(keys, np.int64))
        cand = cand[(cand != INT64_MIN) & ~np.isin(cand, np.fromiter(self.held, np.int64, len(self.held)))]
        new = set(cand[self.estimate(cand) >= self.n].tolist()) if cand.size else set()
        self.held |= new
        return new

    def age(self):
        for s in range(self.S):
            if self.total[s] >= self.R:
                k = 1
                while self.total[s] >> k >= self.R:
                    k += 1
                self.counters[s] >>= k
                self.total[s] >>= k

    def call(self, keys):
        self.count(keys)
        new = self.admit(keys)
        self.age()
        return new


def _scalar_cell(key, r, W):
    x = ((key & M64) + (r + 1) * GOLD) & M64
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & M64
    x ^= x >> 33
    return r * W + ((x >> 32) & (W - 1))


def test_counter_indexes():
    keys = [0, 1, -1, 5, INT64_MIN + 1, (1 << 63) - 1, 123456789012345, -987654321]
    for W in (2, 64, 1 << 20, 1 << 31):
        c = cells(keys, W)
        for i, k in enumerate(keys):
            assert [int(c[r, i]) for r in range(4)] == [_scalar_cell(k, r, W) for r in range(4)]
        assert ((c >= np.arange(4)[:, None] * W) & (c < (np.arange(4)[:, None] + 1) * W)).all()
    # independent of the probe home (low bits of hash64(key)) and of the owner (key mod S)
    rng = np.random.default_rng(0)
    ks = rng.integers(-(1 << 62), 1 << 62, 200000)
    W = 64
    home = (hash64_np(ks.view(np.uint64)) & np.uint64(W - 1)).astype(np.int64)
    c0 = cells(ks, W)[0]
    assert abs(np.corrcoef(home, c0)[0, 1]) < 0.01
    for r in range(4):
        hist = np.bincount(cells(ks[ks % 8 == 3], W)[r] - r * W, minlength=W)
        assert hist.min() > 0.8 * hist.mean()


def test_counts_missing_occurrences_only():
    m = SketchModel(S=3, W=64, n=3)
    m.held = {30}
    m.count([7, 7, 7, 30, 30, 8, INT64_MIN])
    assert m.total.tolist() == [0, 3, 1]                    # 7 (x3) and 8 (x1); held 30 and INT64_MIN count nothing
    assert int(m.estimate([7])[0]) >= 3 and int(m.estimate([8])[0]) >= 1
    assert m.counters.sum() == 4 * 4


def test_per_call_admission():
    m = SketchModel(S=1, W=1 << 12, n=3)
    assert m.call([11]) == set()                              # count 1
    assert m.call([11, 11]) == {11}                           # n - 2 = 1 seen twice: admitted in that call
    assert m.call([11, 11]) == set() and m.total[0] == 3      # held keys count nothing
    assert m.call([12, 13, 13, 13]) == {13}
    assert m.call([14] * 5) == {14}                           # one call reaching n alone


def test_aging_at_half_width():
    m = SketchModel(S=2, W=16, n=1000)
    keys = [2 * i for i in range(7)]                          # all on server 0
    m.call(keys)
    assert m.total.tolist() == [7, 0]
    before = m.counters.copy()
    m.call([100])                                             # total 8 = R: shifted by 1
    assert m.total.tolist() == [4, 0]
    c = before.copy()
    c[0, cells([100], 16)[:, 0]] += 1
    assert np.array_equal(m.counters, c >> 1)
    m2 = SketchModel(S=1, W=16, n=1000)
    m2.call([5] * 40)                                         # 40 -> 40 >> 3 = 5 < 8: one step of k = 3
    assert m2.total[0] == 5 and int(m2.estimate([5])[0]) == 5


def _zipf_stream(rng, n_keys, n):
    p = 1.0 / np.arange(1, n_keys + 1) ** 1.05
    ids = rng.choice(n_keys, n, p=p / p.sum())
    return (hash64_np(ids.astype(np.uint64)) >> np.uint64(1)).astype(np.int64)


def test_never_under_counts_and_exact_without_collisions():
    rng = np.random.default_rng(1)
    for W, exact in ((256, False), (1 << 22, True)):
        # nothing is admitted, so every key keeps counting; exact per-key counts are aged with the same decisions
        m = SketchModel(S=1, W=W, n=1 << 30)
        stream = _zipf_stream(rng, 120, 3000)
        per_key = {}
        for call in np.array_split(stream, 30):
            m.count(call)
            for k in call.tolist():
                per_key[k] = per_key.get(k, 0) + 1
            if m.total[0] >= m.R:
                shift = 1
                while m.total[0] >> shift >= m.R:
                    shift += 1
                per_key = {k: v >> shift for k, v in per_key.items()}
            m.age()
        keys = np.array(sorted(per_key), np.int64)
        est = m.estimate(keys)
        if exact:
            assert all(len(set(cells(keys, W)[r].tolist())) == keys.size for r in range(4))
        exact_counts = np.array([per_key[k] for k in keys.tolist()])
        assert (est >= exact_counts).all()
        if exact:
            assert np.array_equal(est, exact_counts)


def test_over_count_rate_at_half_load():
    """Mean counter load 1/2 (W / 2 distinct keys counted once): a key never seen reads >= 1 with probability close
    to (1 - e^-1/2)^4 = 2.4 %."""
    rng = np.random.default_rng(2)
    W = 1 << 14
    m = SketchModel(S=1, W=W, n=1 << 30)
    m.count(rng.integers(0, 1 << 62, W // 2))
    fresh = rng.integers(-(1 << 62), 0, 50000)
    rate = float((m.estimate(fresh) >= 1).mean())
    assert 0.015 < rate < 0.035, rate


def test_argument_refusals():
    from multiverso_b200.tables.device import check_admit_after
    for ok in (1, 2, 3, (1 << 31) - 1):
        check_admit_after(ok)
    for bad, exc in ((0, ValueError), (-2, ValueError), (1 << 31, ValueError), (2.0, TypeError), ("3", TypeError),
                     (True, TypeError), (None, TypeError)):
        with pytest.raises(exc, match="admit_after"):
            check_admit_after(bad)


def test_refusals_before_the_backend():
    import torch
    if torch.cuda.is_available():
        pytest.skip("the host backend is chosen only without a CUDA device")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.init()
    try:
        with pytest.raises(ValueError, match="admit_after"):
            mv.HashMatrixTable(10, 4, admit_after=0)
        with pytest.raises(TypeError, match="admit_after"):
            mv.HashMatrixTable(10, 4, admit_after=2.5)
        with pytest.raises(NotImplementedError, match="device backend"):
            mv.HashMatrixTable(10, 4, admit_after=3)
    finally:
        mv.shutdown()
        mv.FLAGS.reset()
