"""The placement rule of a HashMatrixTable eviction (mvb_hash_rows_evict, csrc/cuda/hash_rows.cu) as a numpy model,
checked without a GPU on crafted index states: clusters that wrap from slot P - 1 to slot 0, runs of refused and
marked slots, and indexes without an empty slot. The GPU tests compare the kernel bitwise with `rebuild`."""
import numpy as np
import pytest

M64 = (1 << 64) - 1
EMPTY = -(1 << 63)
READY, REFUSED, MARKED = 1, 2, 3


def hash64(x):
    """MurmurHash3's 64-bit finaliser (mix64 of mvb_common.cuh) on a Python int."""
    x &= M64
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & M64
    return x ^ (x >> 33)


def home(key, P):
    return hash64(int(key)) & (P - 1)


def rebuild(keys, ready, last_seen, older_than=None):
    """One server's index after an eviction. A slot is a victim when it holds a key and is marked (3), refused (2)
    or, with `older_than`, live with last_seen < older_than. Returns (keys, ready, last_seen, origin, removed):
    origin[j] is the old slot whose row and state are now at slot j (-1: empty), removed the live keys removed.

    Clusters (maximal runs of non-empty slots, cut before anything changes) are walked from their first slot: a
    victim is cleared, a survivor moves to the first empty slot probing from its home, or stays. Without an empty
    slot, the lowest victim is first deleted by backward shifting (Knuth's Algorithm R), and the index is walked as
    one cluster starting after the last hole."""
    keys, ready, ls = np.array(keys, np.int64), np.array(ready, np.int32), np.array(last_seen, np.int64)
    P = keys.size
    mask = P - 1
    origin = np.where(keys != EMPTY, np.arange(P), -1)
    if older_than is not None:
        ready[(keys != EMPTY) & (ready == READY) & (ls < older_than)] = MARKED
    removed = int(((keys != EMPTY) & (ready == MARKED)).sum())
    full = keys != EMPTY
    starts = [j for j in range(P) if full[j] and not full[j - 1]]

    def clear(j):
        keys[j], ready[j], ls[j], origin[j] = EMPTY, 0, 0, -1

    def move(to, fr):
        keys[to], ready[to], ls[to], origin[to] = keys[fr], ready[fr], ls[fr], origin[fr]
        clear(fr)

    if not starts:
        victims = [j for j in range(P) if ready[j] != READY]
        if victims:
            hole = j = victims[0]
            clear(hole)
            while True:
                j = (j + 1) & mask
                if keys[j] == EMPTY:
                    break
                h = home(keys[j], P)
                stays = (hole < h <= j) if hole <= j else (h > hole or h <= j)
                if not stays:
                    move(hole, j)
                    hole = j
            starts = [(hole + 1) & mask]
    for x in starts:
        while keys[x & mask] != EMPTY:
            j = x & mask
            if ready[j] != READY:
                clear(j)
            else:
                h = home(keys[j], P)
                for d in range((j - h) & mask):
                    if keys[(h + d) & mask] == EMPTY:
                        move((h + d) & mask, j)
                        break
            x += 1
    return keys, ready, ls, origin, removed


def keys_with_home(P, rng, want_homes):
    """Distinct int64 keys (never INT64_MIN), one per requested home slot."""
    pool = {}
    out = []
    for h in want_homes:
        while not pool.get(h):
            k = int(rng.integers(-(1 << 63) + 1, (1 << 63) - 1))
            pool.setdefault(home(k, P), []).append(k)
        out.append(pool[h].pop())
    return out


def craft(P, n, rng, refused=0.1, marked=0.1, homes=None):
    """A valid linear-probing index of n keys in P slots, inserted one by one at the first empty slot of their
    chain, with random ready states and stamps. `homes`: the home slot of each key (default random)."""
    homes = rng.integers(0, P, n) if homes is None else homes
    ks = keys_with_home(P, rng, [int(h) for h in homes])
    keys = np.full(P, EMPTY, np.int64)
    ready = np.zeros(P, np.int32)
    for k in ks:
        j = home(k, P)
        while keys[j] != EMPTY:
            j = (j + 1) & (P - 1)
        keys[j] = k
        u = rng.random()
        ready[j] = REFUSED if u < refused else MARKED if u < refused + marked else READY
    ls = np.where(keys != EMPTY, rng.integers(0, 10, P), 0).astype(np.int64)
    return keys, ready, ls


def wrapping_homes(P, n, rng):
    """Homes crowded just below P - 1, so the chains wrap into slot 0."""
    return (P - 1 - rng.integers(0, max(P // 8, 2), n)) % P


def check(keys0, ready0, ls0, older_than, out):
    """Invariants of a rebuild: exactly the survivors remain, each with its stamp, reachable from its home without
    an empty slot on the way, and (cluster case) never further from its home than before."""
    keys, ready, ls, origin, removed = out
    P = keys0.size
    live0 = (keys0 != EMPTY) & (ready0 == READY)
    aged = live0 & (ls0 < older_than) if older_than is not None else np.zeros(P, bool)
    survive = live0 & ~aged
    assert removed == int((live0 & ~survive).sum()) + int(((keys0 != EMPTY) & (ready0 == MARKED)).sum())
    assert sorted(keys[keys != EMPTY].tolist()) == sorted(keys0[survive].tolist())
    assert bool((ready[keys != EMPTY] == READY).all()) and bool((ready[keys == EMPTY] == 0).all())
    assert bool((ls[keys == EMPTY] == 0).all()) and bool((origin[keys == EMPTY] == -1).all())
    occ = np.nonzero(keys != EMPTY)[0]
    assert np.array_equal(keys[occ], keys0[origin[occ]]) and np.array_equal(ls[occ], ls0[origin[occ]])
    had_empty = bool((keys0 == EMPTY).any())
    for j in occ:
        h = home(keys[j], P)
        for d in range((j - h) & (P - 1)):
            assert keys[(h + d) & (P - 1)] != EMPTY, (j, h, d)
        if had_empty:
            assert (j - h) % P <= (origin[j] - h) % P


@pytest.mark.parametrize("P", [2, 4, 32, 64, 256, 1024])
@pytest.mark.parametrize("load", [0.3, 0.7, 0.875])
def test_random_indexes(P, load):
    rng = np.random.default_rng(P * 1000 + int(load * 100))
    for trial in range(6):
        n = max(1, int(P * load))
        keys, ready, ls = craft(P, n, rng, homes=wrapping_homes(P, n, rng) if trial % 2 else None)
        for older_than in (None, 0, 3, 10):
            check(keys, ready, ls, older_than, rebuild(keys, ready, ls, older_than))


@pytest.mark.parametrize("P", [64, 512])
def test_wrapping_cluster_with_victims(P):
    rng = np.random.default_rng(P)
    n = P // 2
    keys, ready, ls = craft(P, n, rng, homes=wrapping_homes(P, n, rng))
    assert keys[P - 1] != EMPTY and keys[0] != EMPTY                      # a cluster crosses P - 1 -> 0
    out = rebuild(keys, ready, ls, 2)
    check(keys, ready, ls, 2, out)
    assert (out[3][out[0] != EMPTY] != np.nonzero(out[0] != EMPTY)[0]).any()   # something moved


@pytest.mark.parametrize("P", [2, 16, 128, 1024])
def test_no_empty_slot(P):
    """Every slot taken (the state refused inserts leave behind in a small table): the index is still rebuilt."""
    rng = np.random.default_rng(P + 7)
    for trial in range(8):
        keys, ready, ls = craft(P, P, rng, refused=0.15, marked=0.05,
                                homes=wrapping_homes(P, P, rng) if trial % 2 else None)
        assert not (keys == EMPTY).any()
        ready[rng.integers(0, P)] = REFUSED                                    # at least one victim
        for older_than in (None, 4):
            check(keys, ready, ls, older_than, rebuild(keys, ready, ls, older_than))
    keys, ready, ls = craft(P, P, rng, refused=0, marked=0)                    # no victim at all: nothing changes
    out = rebuild(keys, ready, ls)
    assert np.array_equal(out[0], keys) and np.array_equal(out[3], np.arange(P)) and out[4] == 0


def test_runs_of_victims_and_unmoved_prefix():
    """A survivor with no victim before it in its cluster keeps its slot; a run of victims is cleared."""
    P = 64
    rng = np.random.default_rng(5)
    keys, ready, ls = craft(P, 40, rng, refused=0, marked=0, homes=np.full(40, 10))
    assert np.array_equal(np.nonzero(keys != EMPTY)[0], np.arange(10, 50))
    ready[20:26] = MARKED
    ready[26:28] = REFUSED
    out = rebuild(keys, ready, ls)
    check(keys, ready, ls, None, out)
    assert np.array_equal(out[3][10:20], np.arange(10, 20))                  # before the first victim: in place
    assert np.array_equal(out[3][20:42], np.arange(28, 50))                  # the rest shifts back over the run
    assert bool((out[0][42:] == EMPTY).all()) and out[4] == 6
