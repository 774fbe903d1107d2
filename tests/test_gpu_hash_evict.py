"""HashMatrixTable eviction and access clock on the GPU (csrc/cuda/hash_rows.cu).

* mvb_hash_rows_evict on S = 1, 3, 8 emulated servers with crafted indexes (wrapping clusters, runs of refused and
  marked slots, no empty slot) and state slabs laid out like adagrad, rowwise_adagrad and a two-array updater:
  keys, ready flags and stamps bitwise equal to the numpy model of tests/test_hash_evict_cpu.py, rows and every
  state slab moved bitwise, freed slots with zero state, the zero row and the memory between shards untouched.
* Stamping: the largest clock of the inserting lookups that touched a key, nothing from lookups that do not insert.
* The table: evict after training with PSEmbedding / PSEmbeddingCollection, a training run with periodic evictions
  bitwise equal to a dense twin whose evicted rows are reset, capacity recovery, checkpoints."""
import io
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_hash_embedding import _init_model, _spread, _zipf
from test_hash_evict_cpu import EMPTY, MARKED, READY, REFUSED, craft, rebuild, wrapping_homes

pytestmark = pytest.mark.gpu

INT64_MIN = -(1 << 63)
GUARD = 7.25


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


class _Servers:
    """S emulated servers of P slots on one GPU: index arrays, stamps, a row shard and `nst` state arrays of
    `n_slabs` slabs per server, each placed between guard values."""

    def __init__(self, S, P, dim, nst, n_slabs, srow, track=True):
        from multiverso_b200 import _native as N
        dev = torch.device("cuda", 0)
        self.S, self.P, self.dim, self.nst, self.n_slabs, self.srow = S, P, dim, nst, n_slabs, srow
        self.keys = torch.full((S, P), EMPTY, dtype=torch.int64, device=dev)
        self.ready = torch.zeros(S, P, dtype=torch.int32, device=dev)
        self.count = torch.zeros(S, 2, dtype=torch.int64, device=dev)
        self.ls = torch.zeros(S, P + 1, dtype=torch.int64, device=dev)
        self.clock = torch.zeros(1, dtype=torch.int64, device=dev)
        self.gap = 8
        self.rows = torch.full((S, P + 1 + 2 * self.gap, dim), GUARD, device=dev)
        self.stride = (P + 1) * srow + 12                                   # slabs apart, guard values between
        self.state = torch.full((S, max(nst, 1), n_slabs * self.stride + 16), GUARD, device=dev)
        h = N.HashRows()
        h.nservers, h.slots = S, P
        h.map.num_row, h.map.num_col, h.map.nservers, h.map.rows_per_server = S * P + 1, dim, S, P if S > 1 else P + 1
        for s in range(S):
            h.map.shard_ptrs[s] = self.rows[s, self.gap].data_ptr()
            h.keys[s], h.ready[s], h.count[s] = self.keys[s].data_ptr(), self.ready[s].data_ptr(), self.count[s].data_ptr()
            if track:
                h.last_seen[s] = self.ls[s].data_ptr()
        h.clock = self.clock.data_ptr() if track else None
        h.init, h.lo, h.hi, h.seed = N.HASH_INIT_UNIFORM, -0.5, 0.5, 3
        self.h = h
        self.d = torch.frombuffer(bytearray(h), dtype=torch.uint8).to(dev)

    def shard(self, s):
        return self.rows[s, self.gap:self.gap + self.P]

    def slab(self, s, a, k):
        return self.state[s, a, k * self.stride:k * self.stride + self.P * self.srow].view(self.P, self.srow)

    def evict(self, s, older_than=None):
        from multiverso_b200 import _native as N
        counts = torch.empty(2, dtype=torch.int64, device="cuda")
        work = torch.empty(self.P // 2 + 2, dtype=torch.int64, device="cuda")
        st = [self.state[s, a, 0:].data_ptr() if a < self.nst else None for a in range(2)]
        N.cuda_lib().mvb_hash_rows_evict(self.h, s, INT64_MIN if older_than is None else older_than, st[0], st[1],
                                         self.n_slabs, self.stride, self.srow, counts, work, N.stream_ptr())
        return counts.tolist()

    def lookup(self, keys, insert=True):
        from multiverso_b200 import _native as N
        rows, status = torch.empty_like(keys), torch.zeros(1, dtype=torch.int64, device=keys.device)
        a = N.HashLookup()
        a.tables, a.keys, a.n, a.insert = self.d.data_ptr(), keys.data_ptr(), keys.numel(), int(insert)
        a.rows, a.status, a.timeout_s = rows.data_ptr(), status.data_ptr(), 30.0
        N.cuda_lib().mvb_hash_rows_lookup(a, N.stream_ptr())
        return rows, int(status.item())


LAYOUTS = {"adagrad": (1, 3, None), "rowwise_adagrad": (1, 3, 1), "two_arrays": (2, 2, None), "sgd": (0, 1, None)}


@pytest.mark.parametrize("S", [1, 3, 8])
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_rebuild_matches_model(cuda, S, layout):
    nst, n_slabs, srow = LAYOUTS[layout]
    dim = 16
    rng = np.random.default_rng(S * 31 + len(layout))
    for P, case in ((64, "wrap"), (1024, "random"), (128, "full"), (32, "full")):
        e = _Servers(S, P, dim, nst, n_slabs, srow or dim)
        before = []
        for s in range(S):
            n = P if case == "full" else int(P * 0.8)
            homes = wrapping_homes(P, n, rng) if case != "random" else None
            keys, ready, ls = craft(P, n, rng, refused=0.08, marked=0.08, homes=homes)
            if case == "full":
                ready[rng.integers(0, P)] = REFUSED
            e.keys[s] = torch.from_numpy(keys).to(cuda)
            e.ready[s] = torch.from_numpy(ready).to(cuda)
            e.ls[s, :P] = torch.from_numpy(ls).to(cuda)
            e.count[s, 0] = int((ready == READY).sum()) + int((ready == MARKED).sum())  # marked keys were live
            e.shard(s).copy_(torch.randn(P, dim, device=cuda))
            for a in range(nst):
                for k in range(n_slabs):
                    sl = e.slab(s, a, k)
                    sl.copy_(torch.rand(P, sl.shape[1], device=cuda) + 1)
                    sl[torch.from_numpy(keys == EMPTY).to(cuda)] = 0                  # empty slots hold zero state
            before.append((keys, ready, ls))
        rows0, state0, count0 = e.rows.clone(), e.state.clone(), e.count.clone()
        older_than = 5 if case != "random" else None
        for s in range(S):
            keys, ready, ls = before[s]
            want_k, want_r, want_ls, origin, removed = rebuild(keys, ready, ls, older_than)
            removed_k, moved = e.evict(s, older_than)
            assert removed_k == removed
            assert np.array_equal(e.keys[s].cpu().numpy(), want_k), (P, case, s)
            assert np.array_equal(e.ready[s].cpu().numpy(), want_r)
            assert np.array_equal(e.ls[s, :P].cpu().numpy(), want_ls) and int(e.ls[s, P]) == 0
            assert int(e.count[s, 0]) == int(count0[s, 0]) - removed and int(e.count[s, 1]) == int(count0[s, 1])
            occ = torch.from_numpy(np.nonzero(want_k != EMPTY)[0]).to(cuda)
            src = torch.from_numpy(origin[want_k != EMPTY]).to(cuda)
            if case != "full":                                                 # each survivor moved at most once
                assert moved == int((origin[want_k != EMPTY] != np.nonzero(want_k != EMPTY)[0]).sum())
            assert torch.equal(e.shard(s)[occ], rows0[s, e.gap:e.gap + P][src])
            free = torch.from_numpy(want_k == EMPTY).to(cuda)
            for a in range(nst):
                for k in range(n_slabs):
                    old = state0[s, a, k * e.stride:k * e.stride + P * e.slab(s, a, k).shape[1]].view(P, -1)
                    assert torch.equal(e.slab(s, a, k)[occ], old[src])
                    assert bool((e.slab(s, a, k)[free] == 0).all())
            # outside the P slots nothing changed: the zero row (last server), guards, the state between slabs
            assert torch.equal(e.rows[s, :e.gap], rows0[s, :e.gap]) and torch.equal(e.rows[s, e.gap + P:],
                                                                                   rows0[s, e.gap + P:])
            for a in range(nst):
                for k in range(n_slabs):
                    lo, hi = k * e.stride + P * e.slab(s, a, k).shape[1], (k + 1) * e.stride
                    assert torch.equal(e.state[s, a, lo:hi], state0[s, a, lo:hi])
                assert torch.equal(e.state[s, a, n_slabs * e.stride:], state0[s, a, n_slabs * e.stride:])
        if S == 1:                                                           # the lookup kernel finds every survivor
            ks = e.keys[0][e.keys[0] != EMPTY]
            rows, st = e.lookup(ks, insert=False)
            assert st == 0 and torch.equal(e.keys[0][rows], ks)


def test_rebuild_argument_codes(cuda):
    from multiverso_b200 import _native as N
    e = _Servers(1, 64, 8, 1, 1, 8, track=False)
    lib = N.cuda_lib()
    counts = torch.empty(2, dtype=torch.int64, device=cuda)
    work = torch.empty(40, dtype=torch.int64, device=cuda)
    st = e.state[0, 0].data_ptr()

    def code(h, server=0, older=INT64_MIN, n_slabs=1, stride=e.stride, srow=8):
        try:
            lib.mvb_hash_rows_evict(h, server, older, st, None, n_slabs, stride, srow, counts, work, N.stream_ptr())
            return 0
        except N.NativeError as err:
            return int(str(err).split("rc=")[1].split(":")[0])

    assert code(e.h) == 0
    assert code(e.h, server=1) == -1 and code(e.h, server=-1) == -1
    assert code(e.h, older=5) == -5                                          # no last_seen
    assert code(e.h, n_slabs=0) == -6 and code(e.h, srow=0) == -6 and code(e.h, n_slabs=2, stride=8) == -6
    for field, val, rc in (("slots", 48, -4), ("nservers", 0, -3), ("nservers", 9, -3)):
        h = N.HashRows.from_buffer_copy(e.h)
        setattr(h, field, val)
        assert code(h) == rc, field
    h = N.HashRows.from_buffer_copy(e.h)
    h.map.rows_per_server = 0
    assert code(h) == N.BAD_ROW_MAP
    h.map.rows_per_server, h.map.num_col = 65, 6
    assert code(h) == N.BAD_ROW_MAP


def test_stamping(cuda):
    """A Zipf batch whose head key repeats thousands of times, inserted under several clocks: each key's stamp is the
    largest clock of the inserting lookups that touched it; lookups that do not insert leave every stamp alone."""
    S, P = 3, 1 << 12
    e = _Servers(S, P, 8, 0, 1, 8)
    g = torch.Generator(device=cuda).manual_seed(5)
    pool = torch.tensor(_spread(6000, 17), dtype=torch.int64, device=cuda)
    want = {}
    for clock in (3, 1, 7, 5, 2):
        e.clock.fill_(clock)
        n = 200_000 if clock != 2 else 1000
        keys = pool[_zipf(pool.numel(), n, g, cuda)]
        if clock == 3:
            assert (keys == pool[0]).sum().item() > 5000
        _, st = e.lookup(keys)
        assert st == 0
        for k in torch.unique(keys).tolist():
            want[k] = max(want.get(k, clock), clock)
    uk = torch.tensor(sorted(want), dtype=torch.int64, device=cuda)
    rows, _ = e.lookup(uk, insert=False)

    def stamps():
        return e.ls[:, :P].reshape(-1)[rows].tolist()

    assert stamps() == [want[k] for k in uk.tolist()]
    e.clock.fill_(100)
    e.lookup(uk, insert=False)                                              # reads stamp nothing
    assert stamps() == [want[k] for k in uk.tolist()]
    e.lookup(uk[:10])                                                       # an inserting lookup of present keys does
    assert stamps()[:10] == [100] * 10 and stamps()[10:] == [want[k] for k in uk.tolist()[10:]]
    # an untracked descriptor takes the path without stamps
    u = _Servers(S, P, 8, 0, 1, 8, track=False)
    r1, st = u.lookup(uk)
    assert st == 0 and bool((u.ls == 0).all())
    r2, _ = u.lookup(uk, insert=False)
    assert torch.equal(r1, r2)


def _state_rows(t, rows):
    if not t.state:
        return torch.zeros(0)
    st = t.state[0]
    if t.updater_name == "rowwise_adagrad":
        return st[rows]
    return st[:t.my_len].view(-1, t.num_col)[rows]


@pytest.mark.parametrize("updater", ["sgd", "adagrad", "rowwise_adagrad"])
def test_evict_after_training(mv_device, updater):
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbedding, PSEmbeddingCollection, embedding_bag
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(3)
    dim = 32
    t = mv.HashMatrixTable(3000, dim, updater=updater, min_value=-0.5, max_value=0.5, seed=11, track_access=True)
    opt = AddOption(learning_rate=0.5, rho=0.1)
    old = torch.tensor(_spread(1200, 61), dtype=torch.int64, device="cuda")
    new = torch.tensor(_spread(800, 62), dtype=torch.int64, device="cuda")
    t.clock = 0
    ids = old[torch.randint(0, old.numel(), (3000,), generator=g, device="cuda")]
    PSEmbedding(t, push_scale=0.1, option=opt)(ids, torch.arange(0, 3000, 3, device="cuda")).backward(
        torch.randn(1000, dim, device="cuda", generator=g))
    t.clock = 1
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["a", "b"], push_scale=0.1, option=opt)])
    both = torch.cat([new, old[:100]])
    lengths = torch.full((2, both.numel() // 2), 1, dtype=torch.int64, device="cuda")
    ebc(both, lengths).backward(torch.randn(both.numel() // 2, 2 * dim, device="cuda", generator=g))
    torch.cuda.synchronize()
    seen_old = torch.unique(ids)
    idle = seen_old[~torch.isin(seen_old, both)]
    keep = torch.unique(both)
    assert t.clock == 1 and bool((t.last_seen(idle) == 0).all()) and bool((t.last_seen(keep) == 1).all())
    assert bool((t.last_seen(torch.tensor(_spread(5, 99), device="cuda")) == -1).all())
    n0 = t.num_keys()
    k0, v0 = t.export()
    s0 = _state_rows(t, t.lookup(keep, insert=False))
    assert t.evict(older_than=1) == idle.numel()
    assert t.num_keys() == n0 - idle.numel()
    k1, v1 = t.export()
    assert torch.equal(k1, keep) and torch.equal(v1, v0[torch.searchsorted(k0, keep)])
    assert torch.equal(_state_rows(t, t.lookup(keep, insert=False)), s0)
    assert bool((t.last_seen(keep) == 1).all()) and bool((t.last_seen(idle) == -1).all())
    assert bool((t.get(idle) == 0).all())
    # evicted keys come back as new keys
    t.clock = 2
    rows = t.lookup(idle)
    assert np.array_equal(t.get(idle).cpu().numpy(), _init_model(idle.tolist(), 11, -0.5, 0.5, dim))
    assert bool((_state_rows(t, rows) == 0).all()) and bool((t.last_seen(idle) == 2).all())
    # the collection built before the evict still trains, on the keys' new rows
    out = ebc(both, lengths)
    assert torch.equal(out[:, :dim], embedding_bag(t, both[:lengths.shape[1]],
                                                   torch.arange(lengths.shape[1], device="cuda")))
    before = t.get(keep)
    out.backward(torch.ones_like(out))
    torch.cuda.synchronize()
    assert not torch.equal(t.get(keep), before)
    # only listed keys, on top of an age rule that removes nothing
    assert t.evict(older_than=0, keys=torch.cat([keep[:7], torch.tensor([INT64_MIN, 12345], device="cuda")])) == 7
    assert bool((t.get(keep[:7]) == 0).all()) and t.num_keys() == n0 - 7


@pytest.mark.parametrize("updater", ["sgd", "adagrad"])
def test_periodic_evictions_against_dense_twin(mv_device, updater):
    """Training with an eviction every third step is bitwise a dense table (key i at row i) whose rows and state are
    reset to a new key's when the hash table evicts the key. Every step has at most 256 lookups, so each row's
    gradient is summed in lookup order whatever its row id."""
    from multiverso_b200.ops import PSEmbedding
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(9)
    dim, K = 16, 300
    keys = torch.tensor(_spread(K, 71), dtype=torch.int64, device="cuda")
    h = mv.HashMatrixTable(400, dim, updater=updater, min_value=-1, max_value=1, seed=5, track_access=True)
    d = mv.MatrixTable(K, dim, "float32", updater=updater)
    init = torch.from_numpy(_init_model(keys.tolist(), 5, -1, 1, dim)).cuda()
    d.shard.view(K, dim).copy_(init)
    opt = AddOption(learning_rate=0.5, rho=0.1)
    total = 0
    for step in range(12):
        h.clock = step
        lens = torch.randint(0, 6, (40,), generator=g, device="cuda")
        pos = _zipf(K, int(lens.sum()), g, "cuda")
        offs = torch.cumsum(lens, 0) - lens
        dout = torch.randn(40, dim, device="cuda", generator=g)
        yh = PSEmbedding(h, push_scale=0.3, option=opt)(keys[pos], offs)
        yd = PSEmbedding(d, push_scale=0.3, option=opt)(pos, offs)
        assert torch.equal(yh, yd), step
        yh.backward(dout)
        yd.backward(dout)
        if step % 3 == 2:
            ls = h.last_seen(keys)
            gone = (ls >= 0) & (ls < step - 1)
            total += int(gone.sum())
            assert h.evict(older_than=step - 1) == int(gone.sum())
            d.shard.view(K, dim)[gone] = init[gone]
            if updater == "adagrad":
                d.state[0][:d.my_len].view(K, dim)[gone] = 0
        torch.cuda.synchronize()
        present = h.lookup(keys, insert=False) != h.zero_row
        assert torch.equal(h.get(keys)[present], d.get_rows(torch.arange(K, device="cuda"))[present]), step
    assert total > 0


def test_capacity_recovery(mv_device):
    mv = mv_device
    t = mv.HashMatrixTable(100, 8, updater="sgd", min_value=-1, max_value=1)
    first = torch.tensor(_spread(100, 3), dtype=torch.int64, device="cuda")
    t.lookup(first)
    more = torch.tensor(_spread(20, 4), dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match="table full"):
        t.lookup(more)
    assert t.num_keys() == 112
    refused = t.lookup(more, insert=False) == t.zero_row
    assert int(refused.sum()) == 8
    keep = torch.cat([first[50:], more[~refused]])
    vals = t.get(keep)
    assert t.evict(keys=first[:50]) == 50                                    # refused slots go too, uncounted
    assert t.num_keys() == 62 and torch.equal(t.get(keep), vals) and bool((t.get(first[:50]) == 0).all())
    fresh = torch.tensor(_spread(42, 5), dtype=torch.int64, device="cuda")
    t.lookup(torch.cat([fresh, more[refused]]))                              # no "table full" any more
    assert t.num_keys() == 112 and torch.equal(t.get(keep), vals)
    with pytest.raises(ValueError, match="track_access"):
        t.evict(older_than=3)
    with pytest.raises(ValueError, match="track_access"):
        t.clock = 4
    with pytest.raises(ValueError, match="track_access"):
        t.last_seen(first)
    assert t.evict() == 0 and t.num_keys() == 112


def test_checkpoint(mv_device):
    from multiverso_b200.ops import PSEmbedding
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(4)
    keys = torch.tensor(_spread(500, 81), dtype=torch.int64, device="cuda")
    for track in (False, True):
        a = mv.HashMatrixTable(700, 16, updater="adagrad", min_value=-1, max_value=1, track_access=track)
        for clock in range(3):
            if track:
                a.clock = clock
            ids = keys[torch.randint(0, 500, (600,), generator=g, device="cuda")]
            PSEmbedding(a, push_scale=0.1, option=AddOption(learning_rate=0.5))(
                ids, torch.arange(0, 600, 2, device="cuda")).backward(torch.randn(300, 16, device="cuda", generator=g))
        torch.cuda.synchronize()
        buf = io.BytesIO()
        a.store(buf)
        today = a.my_len * 4 + sum(st.numel() * 4 for st in a.state) + a.slots * 12
        assert len(buf.getvalue()) == today + (a.slots * 8 if track else 0)
        b = mv.HashMatrixTable(700, 16, updater="adagrad", min_value=-1, max_value=1, track_access=track)
        buf.seek(0)
        b.load(buf)
        ka, va = a.export()
        kb, vb = b.export()
        assert torch.equal(ka, kb) and torch.equal(va, vb)
        if track:
            assert torch.equal(b.last_seen(ka), a.last_seen(ka)) and len(set(a.last_seen(ka).tolist())) == 3
            c = mv.HashMatrixTable(700, 16, updater="adagrad", track_access=True)
            short = io.BytesIO(buf.getvalue()[:today])
            with pytest.raises(ValueError, match="last-seen"):
                c.load(short)


@pytest.mark.parametrize("nproc", [2, 4])
def test_hash_evict_multi_gpu(nproc):
    """Ranks erase keys owned by peers and stamp the same keys at different clocks; after a collective evict every
    rank's get is bitwise equal (tests/mp_hash_evict_check.py under torchrun)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 900 + nproc
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_hash_evict_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
