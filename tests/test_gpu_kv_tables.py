"""The KVTable's shards (csrc/cuda/kv.cu) and the key-addressed shards of the application tables (csrc/cuda/keys.cu)
on the GPU, against exact models over S servers emulated on one device.

KV: one dict per server; key k lives on server k mod S (Python's % is the kernel's owner_of) and its probe chain
starts at hash64(k) & (cap - 1). Values are chosen so that every order of the atomic adds gives the exact sum, and
results are compared bitwise. Besides values, every check reads the raw shards: each live key is stored once, on its
owner, at a slot reachable from its start slot without crossing an empty slot (wrapping at cap), and no empty slot
holds a value. The cases cover the keys at the ends of the int64 range, a Zipf head raced for by thousands of lanes
at first touch, chains that wrap from the last slot to slot 0, the rehash into a larger table, a full table, the
reserved key INT64_MIN, and KVTable growth for one batch larger than the table and for a checkpoint load.

Key tables: a float64 model of [size, width] values and the touched set, over the range partition of
tables/custom.py, with every shard and bitmap between guard bands that must keep their sentinel."""
import io

import numpy as np
import pytest
import torch

from test_gpu_hash_embedding import _spread, _zipf
from test_gpu_w2v_generic import _hash64

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SPECIAL = [0, -1, -7, INT64_MAX, INT64_MIN + 1, 1 << 62, -(1 << 62)]
VTYPES = {"f32": torch.float32, "f64": torch.float64, "i32": torch.int32, "i64": torch.int64}
# value = units * scale; the unit bound for a key added `reps` times keeps every partial sum exact (below 2^24
# units for fp32, 2^53 for fp64) and in range (2^31 for int32, 2^62 for int64, so int64 values reach 2^62)
SCALE = {"f32": 2.0 ** -10, "f64": 2.0 ** -30, "i32": 1, "i64": 1}


def _unit_bound(vt, reps):
    return {"f32": min(2 ** 10 - 1, 2 ** 24 // reps), "f64": min(2 ** 40, 2 ** 53 // reps),
            "i32": min(1000, 2 ** 31 // reps - 1), "i64": 2 ** 62 // reps}[vt]


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _lib():
    from multiverso_b200 import _native as N
    return N, N.cuda_lib()


def _s64(c):
    return c - (1 << 64) if c >= 1 << 63 else c


_C1, _C2, _LO31 = _s64(0xff51afd7ed558ccd), _s64(0xc4ceb9fe1a85ec53), (1 << 31) - 1


def _mix64(x):
    """hash64 of an int64 tensor, elementwise (wrapping products, logical shifts)."""
    x = x ^ ((x >> 33) & _LO31)
    x = x * _C1
    x = x ^ ((x >> 33) & _LO31)
    x = x * _C2
    return x ^ ((x >> 33) & _LO31)


def _start(keys, cap):
    return _mix64(keys) & (cap - 1)


def _units(vt, n, reps, g, dev):
    """n signed value units, at most _unit_bound(vt, reps) in magnitude and never 0 (int64: at least half of it)."""
    K = _unit_bound(vt, reps)
    lo = K // 2 if vt == "i64" else 1
    mag = torch.randint(lo, K + 1, (n,), generator=g, device=dev)
    sign = torch.randint(0, 2, (n,), generator=g, device=dev) * 2 - 1
    return mag * sign


def _as(vt, units):
    if vt in ("f32", "f64"):
        return (units.double() * SCALE[vt]).to(VTYPES[vt])
    return units.to(VTYPES[vt])


def _max_reps(*key_batches):
    _, counts = torch.unique(torch.cat(key_batches), return_counts=True)
    return int(counts.max())


class _KV:
    """S emulated servers of a KVTable on one GPU: S separately allocated (keys, values) shards of `cap` slots, each
    set up by mvb_kv_init, and the descriptor over them that KVDeviceTable builds over the peer mapping."""

    def __init__(self, S, cap, vt, shards=None):
        N, lib = _lib()
        dev = torch.device("cuda", 0)
        self.S, self.cap, self.vt = S, cap, vt
        self.code = N.dtype_code(VTYPES[vt])
        if shards is None:
            shards = []
            for _ in range(S):
                k = torch.empty(cap, dtype=torch.int64, device=dev)
                lib.mvb_kv_init(k, cap, N.stream_ptr())
                shards.append((k, torch.zeros(cap, dtype=VTYPES[vt], device=dev)))
        self.shards = shards
        kv = N.KV()
        kv.vtype, kv.nservers, kv.capacity = self.code, S, cap
        for s, (k, v) in enumerate(shards):
            kv.keys[s], kv.vals[s] = k.data_ptr(), v.data_ptr()
        self.kv = kv
        self.err = torch.zeros(1, dtype=torch.int32, device=dev)

    def add(self, keys, vals):
        N, lib = _lib()
        lib.mvb_kv_add(self.kv, keys, vals, keys.numel(), self.err, N.stream_ptr())

    def get(self, keys):
        N, lib = _lib()
        out = torch.full((keys.numel(),), 99, dtype=VTYPES[self.vt], device=keys.device)
        lib.mvb_kv_get(self.kv, keys, out, keys.numel(), N.stream_ptr())
        return out

    def dump(self, s):
        N, lib = _lib()
        k, v = self.shards[s]
        ok, ov = torch.empty_like(k), torch.empty_like(v)
        cnt = torch.full((1,), -1, dtype=torch.int64, device=k.device)
        lib.mvb_kv_dump(self.code, k, v, self.cap, ok, ov, cnt, N.stream_ptr())
        n = int(cnt.item())
        return ok[:n], ov[:n]

    def count(self, s):
        N, lib = _lib()
        out = torch.full((1,), -1, dtype=torch.int64, device="cuda")
        lib.mvb_kv_count(self.shards[s][0], self.cap, out, N.stream_ptr())
        return int(out.item())

    def error(self):
        e = int(self.err.item())
        self.err.zero_()
        return e

    def rehash(self, factor):
        """Every shard re-inserted into a new shard of factor x cap slots (growth of KVDeviceTable)."""
        N, lib = _lib()
        ncap, shards = self.cap * factor, []
        for k, v in self.shards:
            nk = torch.empty(ncap, dtype=torch.int64, device=k.device)
            nv = torch.zeros(ncap, dtype=v.dtype, device=v.device)
            lib.mvb_kv_init(nk, ncap, N.stream_ptr())
            lib.mvb_kv_rehash(self.code, k, v, self.cap, nk, nv, ncap, self.err, N.stream_ptr())
            shards.append((nk, nv))
        new = _KV(self.S, ncap, self.vt, shards)
        new.err = self.err
        return new

    def snapshot(self):
        return [(k.clone(), v.clone()) for k, v in self.shards]


class _Model:
    """The reference KVTable's servers: one dict per server, key -> sum of value units."""

    def __init__(self, S):
        self.S = S
        self.shards = [{} for _ in range(S)]

    def add(self, keys, units):
        uk, inv = torch.unique(keys, return_inverse=True)
        tot = torch.zeros(uk.numel(), dtype=torch.int64, device=keys.device).index_add_(0, inv, units)
        for k, t in zip(uk.tolist(), tot.tolist()):
            d = self.shards[k % self.S]
            d[k] = d.get(k, 0) + t

    def keys(self):
        return sorted(k for d in self.shards for k in d)

    def units(self, keys):
        return [self.shards[k % self.S].get(k, 0) for k in keys]


def _check_kv(kv, model):
    """The shards hold exactly the model, each key once on its owner at a reachable slot; dump, count and get agree."""
    dev, vt, cap = kv.shards[0][0].device, kv.vt, kv.cap
    assert kv.error() == 0
    for s, (K, V) in enumerate(kv.shards):
        want = sorted(model.shards[s])
        want_k = torch.tensor(want, dtype=torch.int64, device=dev)
        want_v = _as(vt, torch.tensor(model.units(want), dtype=torch.int64, device=dev))
        occ = K != INT64_MIN
        assert kv.count(s) == len(want) == int(occ.sum())
        assert not bool((V[~occ] != 0).any()), f"server {s}: an empty slot holds a value"
        # every stored key once, on its owner, with the model's value
        sk, order = torch.sort(K[occ])
        assert torch.equal(sk, want_k), f"server {s}: stored keys differ from the model (duplicates or losses)"
        assert torch.equal(V[occ][order], want_v), f"server {s}: values differ from the model"
        assert bool((torch.remainder(sk, kv.S) == s).all())
        # reachable: no empty slot in [start, slot) of any key, cyclically (prefix sums over the doubled table)
        j = occ.nonzero().view(-1)
        st = _start(K[j], cap)
        dist = (j - st) & (cap - 1)
        empty = (~occ).long()
        E = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(torch.cat([empty, empty]), 0)])
        assert bool((E[st + dist] == E[st]).all()), f"server {s}: a key sits behind an empty slot of its chain"
        # the dump is the shard's content, complete
        dk, dv = kv.dump(s)
        dk, o2 = torch.sort(dk)
        assert torch.equal(dk, want_k) and torch.equal(dv[o2], want_v)
    allk = model.keys()
    if allk:
        keys = torch.tensor(allk, dtype=torch.int64, device=dev)
        want = _as(vt, torch.tensor(model.units(allk), dtype=torch.int64, device=dev))
        assert torch.equal(kv.get(keys), want)


def _candidates(n, S, dev):
    """n distinct keys spread over the int64 range (hash64 is a bijection), INT64_MIN left out."""
    c = _mix64(torch.arange(n, dtype=torch.int64, device=dev) + 1000 * S)
    return c[c != INT64_MIN]


def _cap_for(keys, S, load):
    per = int(torch.bincount(torch.remainder(keys, S), minlength=S).max())
    return 1 << max(4, int(np.ceil(np.log2(per / load + 1))))


def test_mix64_model_matches_hash64(cuda):
    keys = torch.tensor(SPECIAL + [INT64_MIN] + _spread(200, 5), dtype=torch.int64, device=cuda)
    got = _mix64(keys).tolist()
    assert got == [_s64(_hash64(k)) for k in keys.tolist()]


@pytest.mark.parametrize("vt", list(VTYPES))
@pytest.mark.parametrize("S", [1, 3, 8])
def test_special_keys_and_zipf(cuda, S, vt):
    """Keys at the ends of the int64 range and spread over all of it; a Zipf batch of 10^6 entries whose head key
    (0) is raced for by thousands of lanes at first touch, then a second batch onto the stored keys."""
    g = torch.Generator(device=cuda).manual_seed(10 * S + len(vt))
    pool = torch.tensor(SPECIAL + _spread(30000, S), dtype=torch.int64, device=cuda)
    kv, model = _KV(S, _cap_for(pool, S, 0.75), vt), _Model(S)
    k1 = pool[_zipf(pool.numel(), 1_000_000, g, cuda)]
    assert int((k1 == 0).sum()) > 5000
    k1 = torch.cat([pool[:len(SPECIAL)], k1])
    k2 = pool[torch.randint(0, pool.numel(), (200_000,), generator=g, device=cuda)]
    reps = _max_reps(k1, k2)
    u = _units(vt, k1.numel() + k2.numel(), reps, g, cuda)
    for k, uu in ((k1, u[:k1.numel()]), (k2, u[k1.numel():])):
        kv.add(k, _as(vt, uu))
        model.add(k, uu)
        _check_kv(kv, model)
    missing = torch.tensor(_spread(2000, 10**6 + S), dtype=torch.int64, device=cuda)
    missing = missing[~torch.isin(missing, pool)]
    assert bool((kv.get(missing) == 0).all())


def _wrap_table(S, vt, cuda, cap=1024):
    """Per server: 64 keys whose chain starts at the last slot and 8 at each of the four slots before it, plus 24
    starting at slots 0..3, added 1-8 times each in one shuffled launch: the chains wrap to slot 0 under contention."""
    g = torch.Generator(device=cuda).manual_seed(S * 7 + cap)
    cand = _candidates(1 << 22, S, cuda)
    st, own = _start(cand, cap), torch.remainder(cand, S)
    picked = []
    for s in range(S):
        for slot, n in [(cap - 1, 64)] + [(cap - d, 8) for d in range(2, 6)] + [(d, 6) for d in range(4)]:
            hit = cand[(st == slot) & (own == s)]
            assert hit.numel() >= n
            picked.append(hit[:n])
    keys = torch.cat(picked)
    rep = torch.randint(1, 9, (keys.numel(),), generator=g, device=cuda)
    batch = keys.repeat_interleave(rep)
    batch = batch[torch.randperm(batch.numel(), generator=g, device=cuda)]
    u = _units(vt, batch.numel(), 16, g, cuda)         # test_rehash adds the batch twice
    kv, model = _KV(S, cap, vt), _Model(S)
    kv.add(batch, _as(vt, u))
    model.add(batch, u)
    return kv, model, batch, u


@pytest.mark.parametrize("vt", list(VTYPES))
@pytest.mark.parametrize("S", [1, 3, 8])
def test_collision_chains_wrap(cuda, S, vt):
    kv, model, _, _ = _wrap_table(S, vt, cuda)
    _check_kv(kv, model)
    cap = kv.cap
    for K, _ in kv.shards:
        # 96 keys start in the last 5 slots: at least 91 of them wrapped to the front of the table
        j = (K != INT64_MIN).nonzero().view(-1)
        assert int(((_start(K[j], cap) >= cap - 5) & (j < cap - 5)).sum()) >= 91


@pytest.mark.parametrize("factor", [2, 4])
@pytest.mark.parametrize("vt", list(VTYPES))
@pytest.mark.parametrize("S", [1, 3, 8])
def test_rehash(cuda, S, vt, factor):
    """Growth re-inserts every shard, the key in its last slot included, into a table of factor x the capacity;
    the new table then takes the same batch again."""
    kv, model, batch, u = _wrap_table(S, vt, cuda)
    assert all(int(K[kv.cap - 1]) != INT64_MIN for K, _ in kv.shards)
    big = kv.rehash(factor)
    _check_kv(big, model)
    big.add(batch, _as(vt, u))
    model.add(batch, u)
    _check_kv(big, model)


@pytest.mark.parametrize("vt", list(VTYPES))
def test_full_table(cuda, vt):
    """20 distinct keys into 16 slots in one launch: error 5001, and exactly 16 keys stored, each once, with its
    value; the others read 0. An error flag, not a fault."""
    g = torch.Generator(device=cuda).manual_seed(16)
    keys = torch.tensor(SPECIAL + _spread(13, 16), dtype=torch.int64, device=cuda)[:20]
    assert torch.unique(keys).numel() == 20
    u = _units(vt, 20, 1, g, cuda)
    kv = _KV(1, 16, vt)
    kv.add(keys, _as(vt, u))
    assert kv.error() == 5001
    stored = kv.shards[0][0]
    assert kv.count(0) == 16 and torch.unique(stored).numel() == 16 and bool(torch.isin(stored, keys).all())
    model = _Model(1)
    sel = torch.isin(keys, stored)
    model.add(keys[sel], u[sel])
    _check_kv(kv, model)
    assert bool((kv.get(keys[~sel]) == 0).all())


@pytest.mark.parametrize("vt", list(VTYPES))
@pytest.mark.parametrize("S", [1, 3])
def test_int64_min_is_not_a_key(cuda, S, vt):
    """INT64_MIN marks empty slots. Adding it sets error 5003 and changes no slot; a key whose chain starts where
    INT64_MIN's would gets exactly its own value; get(INT64_MIN) reads 0."""
    g = torch.Generator(device=cuda).manual_seed(S)
    cap = 64
    kv, model = _KV(S, cap, vt), _Model(S)
    k0 = torch.tensor(_spread(40, 3), dtype=torch.int64, device=cuda)
    u0 = _units(vt, k0.numel(), 1, g, cuda)
    kv.add(k0, _as(vt, u0))
    model.add(k0, u0)
    bad = torch.tensor([INT64_MIN], device=cuda)
    cand = _candidates(1 << 20, S, cuda)
    twin = cand[(_start(cand, cap) == int(_start(bad, cap))) & (torch.remainder(cand, S) == INT64_MIN % S)]
    twin = twin[~torch.isin(twin, k0)][:1]
    assert twin.numel() == 1
    before = kv.snapshot()
    u_bad, u_twin = _units(vt, 2, 1, g, cuda)
    kv.add(bad, _as(vt, u_bad.view(1)))
    torch.cuda.synchronize()
    after_bad, err_bad = kv.snapshot(), kv.error()
    kv.add(twin, _as(vt, u_twin.view(1)))
    model.add(twin, u_twin.view(1))
    assert torch.equal(kv.get(twin), _as(vt, u_twin.view(1))), "the twin key took the value added for INT64_MIN"
    assert torch.equal(kv.get(bad), torch.zeros(1, dtype=VTYPES[vt], device=cuda))
    assert err_bad == 5003
    assert all(torch.equal(a, b) for x, y in zip(before, after_bad) for a, b in zip(x, y))
    _check_kv(kv, model)
    # in a batch: the other keys are added
    k3 = torch.tensor([5, INT64_MIN, -5, INT64_MIN], dtype=torch.int64, device=cuda)
    u3 = _units(vt, 4, 1, g, cuda)
    kv.add(k3, _as(vt, u3))
    assert kv.error() == 5003
    model.add(k3[[0, 2]], u3[[0, 2]])
    _check_kv(kv, model)


# ---------------------------------------------------------------------------------------------- KVTable (table level)
def _table_dict(t):
    """The table's content through its checkpoint writer: {key: value}."""
    buf = io.BytesIO()
    t.store(buf)
    raw = buf.getvalue()
    n = int(np.frombuffer(raw[:8], np.int64)[0])
    keys = np.frombuffer(raw[8:8 + 8 * n], np.int64)
    vals = np.frombuffer(raw[8 + 8 * n:], torch.empty((), dtype=t.vdtype).numpy().dtype)
    assert vals.size == n
    return dict(zip(keys.tolist(), vals.tolist()))


def test_one_batch_larger_than_the_table(mv_device):
    """A single-process add of 5000 new keys into 1024 slots grows the table first."""
    mv = mv_device
    from multiverso_b200.runtime import Runtime
    kv = mv.KVTable("int64", "float32", capacity=1024)
    keys = torch.tensor(_spread(5000, 42)[:5000], dtype=torch.int64)
    assert keys.numel() == 5000
    vals = (torch.arange(5000, dtype=torch.float64) - 2500).mul_(2.0 ** -10).float()
    kv.add(keys, vals)
    assert torch.equal(kv.get(keys).cpu(), vals)
    assert kv.live_keys() == 5000 and kv.capacity >= 2 * 5000
    Runtime.get().check_watchdog()
    kv.add(keys, vals)                                  # the same keys again: no new slots
    assert torch.equal(kv.get(keys).cpu(), 2 * vals) and kv.live_keys() == 5000


@pytest.mark.parametrize("vdtype", ["float32", "int64"])
def test_checkpoint_into_a_small_table(mv_device, tmp_path, vdtype):
    """A table grown to 50 000 keys, saved and loaded into a fresh table of 1024 slots: the same dict."""
    mv = mv_device
    kv = mv.KVTable("int64", vdtype, capacity=1024)
    g = torch.Generator().manual_seed(1)
    keys = torch.tensor(_spread(50000, 9)[:50000], dtype=torch.int64)
    assert keys.numel() == 50000
    for lo in range(0, 50000, 5000):
        k = keys[lo:lo + 5000]
        if vdtype == "float32":
            v = torch.randint(-1023, 1024, (k.numel(),), generator=g).double().mul_(2.0 ** -10).float()
        else:
            v = torch.randint(1 << 59, 1 << 60, (k.numel(),), generator=g) * (1 - 2 * (torch.arange(k.numel()) % 2))
        kv.add(k, v)
        kv.add(k[:700], v[:700])
    want = _table_dict(kv)
    assert len(want) == 50000 and kv.capacity >= 2 * 50000
    mv.save_table(kv, str(tmp_path / "kv"))
    fresh = mv.KVTable("int64", vdtype, capacity=1024)
    mv.load_table(fresh, str(tmp_path / "kv"))
    assert _table_dict(fresh) == want and fresh.capacity >= 2 * 50000
    got = fresh.get(keys).cpu()
    assert got.tolist() == [want[k] for k in keys.tolist()]


def test_kvtable_rejects_int64_min(mv_device):
    mv = mv_device
    from multiverso_b200.runtime import Runtime
    from multiverso_b200.utils.log import FatalError
    kv = mv.KVTable("int64", "float64")
    kv.add([3, INT64_MIN, -3], [1.0, 2.0, 4.0])
    torch.cuda.synchronize()
    with pytest.raises(FatalError, match="kv-bad-key"):
        Runtime.get().check_watchdog()
    Runtime.get().check_watchdog()                      # the flag is cleared
    assert kv.get([3, -3, INT64_MIN]).tolist() == [1.0, 4.0, 0.0]
    assert kv.live_keys() == 2 and _table_dict(kv) == {3: 1.0, -3: 4.0}


# ------------------------------------------------------------------------------------------------------- key tables
SENTINEL = 0x5A5A5A5B          # int32 bits of the guard bands (bit 0 set: a bitmap read past its end shows)
GUARD = 40                     # 4-byte words around each region


class _KeyMap:
    """S emulated servers of a SparseDeviceTable on one GPU, partitioned as tables/custom.py does: per = size // S,
    the last server takes the remainder, per = 1 and servers from `size` on empty when size < S. Every shard
    (len_s x width fp32) and every touched bitmap (ceil(len_s / 32) words) lies in one buffer between guard bands
    holding SENTINEL."""

    def __init__(self, size, S, width, dev):
        N, _ = _lib()
        self.size, self.S, self.width = size, S, width
        if size >= S:
            self.per = size // S
            self.lo = [s * self.per for s in range(S)]
            self.hi = [(s + 1) * self.per for s in range(S)]
            self.hi[-1] = size
        else:
            self.per = 1
            self.lo = [min(s, size) for s in range(S)]
            self.hi = [min(s + 1, size) for s in range(S)]
        lens = [h - l for l, h in zip(self.lo, self.hi)]
        regions = [n * width for n in lens] + [(n + 31) // 32 for n in lens]
        self.at, pos = [], GUARD
        for n in regions:
            self.at.append(pos)
            pos += n + GUARD
        self.mem = torch.full((pos,), SENTINEL, dtype=torch.int32, device=dev)
        for a, n in zip(self.at, regions):
            self.mem[a:a + n] = 0
        self.regions = regions
        base = self.mem.data_ptr()
        m = N.KeyMap()
        m.size, m.per_server, m.nservers, m.width = size, self.per, S, width
        for s in range(S):
            m.shard_ptrs[s] = base + 4 * self.at[s]
            m.touched_ptrs[s] = base + 4 * self.at[S + s]
        self.m = m

    def add(self, keys, vals, sign):
        N, lib = _lib()
        lib.mvb_keys_add(self.m, keys, vals, keys.numel(), sign, N.stream_ptr())

    def get(self, keys):
        N, lib = _lib()
        out = torch.full((keys.numel(), self.width), 99.0, device=keys.device)
        lib.mvb_keys_get(self.m, keys, out, keys.numel(), N.stream_ptr())
        return out

    def collect(self, cap):
        """(count, keys[:min(count, cap)], values) and the output buffers' guard bands."""
        N, lib = _lib()
        dev = self.mem.device
        ok = torch.full((cap + GUARD,), SENTINEL, dtype=torch.int64, device=dev)
        ov = torch.full(((cap + GUARD) * self.width,), SENTINEL, dtype=torch.int32, device=dev)
        cnt = torch.full((1,), -1, dtype=torch.int64, device=dev)
        lib.mvb_keys_collect(self.m, ok, ov.view(torch.float32), cnt, cap, N.stream_ptr())
        n = int(cnt.item())
        w = min(n, cap)
        return n, ok[:w], ov.view(torch.float32)[:w * self.width].view(w, self.width), ok[cap:], ov[cap * self.width:]

    def touched(self):
        """The set of keys whose touched bit is set, and whether any bit past a shard's last key is set."""
        bits, stray = set(), False
        for s in range(self.S):
            a, nw = self.at[self.S + s], self.regions[self.S + s]
            words = self.mem[a:a + nw].cpu().numpy().view(np.uint32)
            flat = np.unpackbits(words.view(np.uint8), bitorder="little")
            n = self.hi[s] - self.lo[s]
            bits |= {self.lo[s] + int(i) for i in np.flatnonzero(flat[:n])}
            stray |= bool(flat[n:].any())
        return bits, stray

    def guards_intact(self):
        ends = [0] + [a + n for a, n in zip(self.at, self.regions)]
        starts = self.at + [self.mem.numel()]
        return all(bool((self.mem[e:b] == SENTINEL).all()) for e, b in zip(ends, starts))


def _edge_keys(km):
    """Per server: its first key, local 1, 31, 32, 33 and its last key (the remainder server's last is size - 1)."""
    out = []
    for lo, hi in zip(km.lo, km.hi):
        out += [k for k in (lo, lo + 1, lo + 31, lo + 32, lo + 33, hi - 1) if lo <= k < hi]
    return out


@pytest.mark.parametrize("width", [1, 2, 16])
@pytest.mark.parametrize("size", [1, 5, 31, 32, 33, 1000, 100003])
@pytest.mark.parametrize("S", [1, 2, 3, 8])
def test_key_tables(cuda, S, size, width):
    """Two adds (sign +1, then -1) with repeated keys and out-of-range keys; get, the touched bits and collect
    (with and without room for every touched key) against the dense model; the guard bands keep their sentinel."""
    g = torch.Generator(device=cuda).manual_seed(S * 1000 + size * 17 + width)
    km = _KeyMap(size, S, width, cuda)
    model = np.zeros((size, width), np.float64)
    touched = set()
    invalid = [-1, size, size + 1000, INT64_MIN, INT64_MAX]
    edges = _edge_keys(km)
    for sign, n_rand in ((1.0, min(size // 2 + 1, 5000)), (-1.0, min(size // 3 + 1, 3000))):
        rnd = torch.randint(0, size, (n_rand,), generator=g, device=cuda)
        k = torch.cat([torch.tensor(edges[::2] if sign > 0 else edges[1::2], dtype=torch.int64, device=cuda), rnd,
                       rnd[:n_rand // 4], torch.tensor(invalid, dtype=torch.int64, device=cuda)])
        k = k[torch.randperm(k.numel(), generator=g, device=cuda)]
        # dyadic values: multiples of 2^-8 below 2^4 in magnitude, so any sum of up to 2^12 of them is exact in fp32
        v = torch.randint(-(1 << 12) + 1, 1 << 12, (k.numel(), width), generator=g, device=cuda).double() * 2.0 ** -8
        km.add(k, v.float().contiguous(), sign)
        kk, vv = k.cpu().numpy(), v.cpu().numpy()
        ok = (kk >= 0) & (kk < size)
        np.add.at(model, kk[ok], sign * vv[ok])
        touched |= set(kk[ok].tolist())
    torch.cuda.synchronize()
    want = torch.from_numpy(model.astype(np.float32)).to(cuda)
    q = torch.arange(size, device=cuda) if size <= 1000 else torch.cat(
        [torch.tensor(edges, device=cuda), torch.randint(0, size, (5000,), generator=g, device=cuda)])
    assert torch.equal(km.get(q), want[q])
    assert bool((km.get(torch.tensor(invalid, device=cuda)) == 0).all())
    bits, stray = km.touched()
    assert bits == touched and not stray
    n, ck, cv, kguard, vguard = km.collect(size + 7)
    assert n == len(touched) and ck.numel() == n
    assert sorted(ck.tolist()) == sorted(touched)
    assert torch.equal(cv, want[ck])
    assert bool((kguard == SENTINEL).all()) and bool((vguard == SENTINEL).all())
    if len(touched) >= 2:
        cap = len(touched) // 2
        n, ck, cv, kguard, vguard = km.collect(cap)
        assert n == len(touched) and ck.numel() == cap               # the full count, only cap entries written
        assert torch.unique(ck).numel() == cap and set(ck.tolist()) <= touched
        assert torch.equal(cv, want[ck])
        assert bool((kguard == SENTINEL).all()) and bool((vguard == SENTINEL).all())
    assert km.guards_intact()
