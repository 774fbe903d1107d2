"""HashMatrixTable on the GPU (csrc/cuda/hash_rows.cu): one row per distinct key inside its owner's range under a
Zipf batch on 1, 3 and 8 emulated shards, initial rows bitwise equal to a numpy model of the init formula, results
that do not depend on which slot a key got, PSEmbedding and PSEmbeddingCollection over hash tables bitwise equal to
the same calls over dense tables holding the same rows at remapped ids, the capacity limit, eval mode and
checkpoints."""
import io
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from test_gpu_w2v_generic import M64, _hash64

pytestmark = pytest.mark.gpu

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
SPECIAL = [0, -1, -7, 5, 1 << 62, -(1 << 62), INT64_MAX, INT64_MIN + 1]


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _spread(n, salt=0):
    """n distinct int64 keys spread over the whole range (hash64 of 0..n-1), signs included."""
    ks = {_hash64(i * 7919 + salt) for i in range(n)}
    ks = [k - (1 << 64) if k >= 1 << 63 else k for k in ks]
    return [k for k in ks if k != INT64_MIN]


def _zipf(n_keys, n, g, dev):
    cdf = torch.cumsum(torch.arange(1, n_keys + 1, device=dev, dtype=torch.float64).pow_(-1.1), 0)
    u = torch.rand(n, device=dev, generator=g, dtype=torch.float64) * cdf[-1]
    return torch.searchsorted(cdf, u).clamp_(max=n_keys - 1)


class _Index:
    """S emulated servers of a hash index on one GPU: S sets of (keys, ready, count, shard) pointers, the shards at
    separate places with garbage between them."""

    def __init__(self, S, P, dim, lo=-0.5, hi=0.5, seed=3, gap=5):
        from multiverso_b200 import _native as N
        dev = torch.device("cuda", 0)
        self.S, self.P, self.dim = S, P, dim
        self.keys = torch.empty(S, P, dtype=torch.int64, device=dev)
        self.ready = torch.empty(S, P, dtype=torch.int32, device=dev)
        self.count = torch.empty(S, 2, dtype=torch.int64, device=dev)
        rps = P if S > 1 else P + 1
        self.buf = torch.full((S * (P + 1 + gap), dim), 1e3, device=dev)
        h = N.HashRows()
        h.nservers, h.slots = S, P
        h.map.num_row, h.map.num_col, h.map.nservers, h.map.rows_per_server = S * P + 1, dim, S, rps
        self.spans = []
        for s in range(S):
            at = s * (P + 1 + gap) + gap
            n = P + 1 if s == S - 1 else P
            self.buf[at:at + n] = 0
            h.map.shard_ptrs[s] = self.buf[at].data_ptr()
            h.keys[s], h.ready[s], h.count[s] = self.keys[s].data_ptr(), self.ready[s].data_ptr(), self.count[s].data_ptr()
            N.cuda_lib().mvb_hash_rows_init(self.keys[s], self.ready[s], self.count[s], P, N.stream_ptr())
            self.spans.append((at, n))
        h.init, h.lo, h.hi, h.seed = N.HASH_INIT_UNIFORM, lo, hi, seed
        self.h = h
        self.d = torch.frombuffer(bytearray(h), dtype=torch.uint8).to(dev)

    def lookup(self, keys, insert=True):
        from multiverso_b200 import _native as N
        rows, status = torch.empty_like(keys), torch.zeros(1, dtype=torch.int64, device=keys.device)
        a = N.HashLookup()
        a.tables, a.keys, a.n, a.insert = self.d.data_ptr(), keys.data_ptr(), keys.numel(), int(insert)
        a.rows, a.status, a.timeout_s = rows.data_ptr(), status.data_ptr(), 30.0
        N.cuda_lib().mvb_hash_rows_lookup(a, N.stream_ptr())
        return rows, int(status.item())

    def num_keys(self):
        from multiverso_b200 import _native as N
        out = torch.empty(1, dtype=torch.int64, device="cuda")
        N.cuda_lib().mvb_hash_rows_count(self.h, out, N.stream_ptr())
        return int(out.item())

    def table(self):
        return torch.cat([self.buf[a:a + n] for a, n in self.spans])


def _init_model(keys, seed, lo, hi, dim):
    """Rows of new keys: lo + u (hi - lo), u = (hash64(hash64(key ^ seed) + c) >> 40) 2^-24, rounded fp32 ops."""
    out = np.empty((len(keys), dim), np.float32)
    lo32, d32 = np.float32(lo), np.float32(hi) - np.float32(lo)
    for i, k in enumerate(keys):
        h0 = _hash64((k & M64) ^ seed)
        for c in range(dim):
            u = np.float32(_hash64(h0 + c) >> 40) * np.float32(2.0 ** -24)
            out[i, c] = lo32 + u * d32
    return out


@pytest.mark.parametrize("S", [1, 3, 8])
def test_lookup_zipf_one_row_per_key(cuda, S):
    g = torch.Generator(device=cuda).manual_seed(S)
    pool = SPECIAL + _spread(30000, S)
    per = np.bincount([k % S for k in pool], minlength=S).max()
    P = 1 << int(np.ceil(np.log2(per * 8 / 7 + 1)))
    idx = _Index(S, P, 8)
    pool_t = torch.tensor(pool, dtype=torch.int64, device=cuda)
    keys = pool_t[_zipf(len(pool), 1_000_000, g, cuda)]
    assert (keys == pool_t[0]).sum().item() > 5000                     # the head key (0) thousands of times
    rows, st = idx.lookup(keys)
    assert st == 0
    uk, inv = torch.unique(keys, return_inverse=True)
    first = torch.full((uk.numel(),), -1, dtype=torch.int64, device=cuda).scatter_(0, inv, rows)
    assert torch.equal(first[inv], rows)                                  # every occurrence: the same row
    assert torch.unique(first).numel() == uk.numel()                      # distinct keys: distinct rows
    owner = torch.remainder(uk, S)
    assert bool(((first >= owner * P) & (first < (owner + 1) * P)).all())
    assert idx.num_keys() == uk.numel()
    rows2, st = idx.lookup(keys)                                          # later calls: the same rows, no insert
    assert st == 0 and torch.equal(rows2, rows) and idx.num_keys() == uk.numel()
    missing = torch.tensor(_spread(500, 10**6 + S), dtype=torch.int64, device=cuda)
    missing = missing[~torch.isin(missing, uk)]
    r, st = idx.lookup(torch.cat([missing, uk[:100]]), insert=False)
    assert st == 0 and bool((r[:missing.numel()] == S * P).all()) and torch.equal(r[missing.numel():], first[:100])
    assert idx.num_keys() == uk.numel()
    _, st = idx.lookup(torch.tensor([5, INT64_MIN], device=cuda))
    assert st >> 40 == 3                                                   # INT64_MIN is never inserted
    assert idx.num_keys() == uk.numel()
    # rows hold the model's initial values; the zero row stays zero
    W = idx.table()
    some = uk[torch.randperm(uk.numel(), generator=g, device=cuda)[:64]]
    want = _init_model(some.tolist() + SPECIAL, 3, -0.5, 0.5, 8)
    sel = torch.cat([first[torch.searchsorted(uk, some)], first[torch.searchsorted(uk, torch.tensor(SPECIAL,
                                                                                                   device=cuda))]])
    assert np.array_equal(W[sel].cpu().numpy(), want)
    assert bool((W[S * P] == 0).all())


def test_initial_values(mv_device):
    mv = mv_device
    keys = torch.tensor(SPECIAL + _spread(300, 77), dtype=torch.int64)
    t = mv.HashMatrixTable(1000, 36, min_value=-0.25, max_value=0.75, seed=12345)
    got = t.get(keys.cuda())
    assert bool((got == 0).all())                                         # get inserts nothing
    t.lookup(keys)
    assert t.num_keys() == keys.numel()
    assert np.array_equal(t.get(keys).cpu().numpy(), _init_model(keys.tolist(), 12345, -0.25, 0.75, 36))
    c = mv.HashMatrixTable(100, 8, init_value=0.375)
    c.lookup(keys[:50])
    assert bool((c.get(keys[:50]) == 0.375).all())
    with pytest.raises(ValueError, match="INT64_MIN"):
        c.lookup(torch.tensor([1, INT64_MIN]))
    assert c.num_keys() == 50


def _bags(keys, B, g):
    n = keys.numel()
    lens = torch.randint(0, 9, (B,), generator=g, device="cuda")
    lens[::5] = 0
    pos = torch.randint(0, n, (int(lens.sum()),), generator=g, device="cuda")
    return keys[pos], torch.cumsum(lens, 0) - lens


def test_slot_independence(mv_device):
    """Two tables whose keys arrived in different orders (small P: probe chains cross): get and a PSEmbedding forward
    give the same bits per key; so does an sgd step whose lookups fit one backward chunk (256), where every row's
    gradient is summed in lookup order. Over more lookups, the pieces of a row's gradient are grouped by where its
    run falls in the row-sorted lookups, which depends on the slots: the rows agree to fp32 rounding."""
    from multiverso_b200.ops import PSEmbedding
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(8)
    keys = torch.tensor(_spread(110, 5), dtype=torch.int64, device="cuda")
    a = mv.HashMatrixTable(110, 16, updater="sgd", min_value=-1, max_value=1, seed=9)
    b = mv.HashMatrixTable(110, 16, updater="sgd", min_value=-1, max_value=1, seed=9)
    assert a.slots == 128
    ra = a.lookup(keys)
    b.lookup(keys.flip(0))
    rb = b.lookup(keys)
    assert not torch.equal(ra, rb)                                         # different slots for some keys
    assert torch.equal(a.get(keys), b.get(keys))
    for B, exact in ((40, True), (400, False)):
        ids, offs = _bags(keys, B, g)
        assert (ids.numel() <= 256) == exact
        psw = torch.rand(ids.numel(), device="cuda", generator=g)
        dout = torch.randn(B, 16, device="cuda", generator=g)
        outs = []
        for t in (a, b):
            y = PSEmbedding(t, push_scale=0.3)(ids, offs, psw)
            y.backward(dout)
            outs.append(y.detach())
        torch.cuda.synchronize()
        assert torch.equal(outs[0], outs[1])
        if exact:
            assert torch.equal(a.get(keys), b.get(keys))
        else:
            torch.testing.assert_close(a.get(keys), b.get(keys), rtol=1e-6, atol=1e-6)


def _dense_twin(mv, h, keys, updater):
    """A dense MatrixTable of K = len(keys) rows holding h's row of keys[i] at row remap[i], the rank of that row
    among the keys' rows (ids remapped in the same order, so a backward sorts the lookups of both tables alike).
    Returns (table, remap)."""
    K = keys.numel()
    remap = torch.empty(K, dtype=torch.int64, device="cuda")
    remap[torch.argsort(h.lookup(keys, insert=False))] = torch.arange(K, device="cuda")
    d = mv.MatrixTable(K, h.num_col, "float32", updater=updater)
    vals = h.get(keys)
    d.shard.view(K, h.num_col)[remap] = vals
    assert torch.equal(d.get_rows(remap), vals)
    return d, remap


@pytest.mark.parametrize("mode,weighted,updater", [("sum", False, "sgd"), ("mean", False, "sgd"),
                                                   ("sum", True, "sgd"), ("sum", True, "adagrad")])
def test_against_dense_table(mv_device, mode, weighted, updater):
    from multiverso_b200.ops import PSEmbedding
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(21)
    keys = torch.tensor(sorted(_spread(3000, 44) + SPECIAL), dtype=torch.int64, device="cuda")
    h = mv.HashMatrixTable(4000, 64, updater=updater, min_value=-0.1, max_value=0.1)
    h.lookup(keys)
    d, remap = _dense_twin(mv, h, keys, updater)
    lens = torch.randint(0, 30, (3000,), generator=g, device="cuda")
    lens[::9] = 0
    pos = _zipf(keys.numel(), int(lens.sum()), g, "cuda")                      # key positions
    offs = torch.cumsum(lens, 0) - lens
    psw = torch.rand(pos.numel(), device="cuda", generator=g) if weighted else None
    dout = torch.randn(3000, 64, device="cuda", generator=g)
    opt = AddOption(learning_rate=0.5, rho=0.1)
    yh = PSEmbedding(h, push_scale=0.2, option=opt, mode=mode)(keys[pos], offs, psw)
    yd = PSEmbedding(d, push_scale=0.2, option=opt, mode=mode)(remap[pos], offs, psw)
    assert torch.equal(yh, yd)
    yh.backward(dout)
    yd.backward(dout)
    torch.cuda.synchronize()
    rows = h.lookup(keys, insert=False)
    assert torch.equal(h.get(keys), d.get_rows(remap))
    if updater == "adagrad":
        sh, sd = h.state[0][:h.my_len].view(-1, 64), d.state[0][:d.my_len].view(-1, 64)
        assert torch.equal(sh[rows], sd[remap]) and bool(sh.abs().sum() > 0)
        assert bool((sh[h.zero_row] == 0).all())
    assert bool((h.get_rows(torch.tensor([h.zero_row], device="cuda")) == 0).all())


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def _kernels(fn, name):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if name in e.name)


def test_collection_mixed_tables(mv_device):
    """A dense table, a hash table shared by two features and a second hash table: the same bits as the collection
    over dense twins fed remapped ids, and the dense feature the same bits as the collection without hash tables."""
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection, embedding_bag
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(31)
    B = 700
    ka = torch.tensor(sorted(_spread(2000, 1) + SPECIAL), dtype=torch.int64, device="cuda")
    kb = torch.tensor(sorted(_spread(500, 2)), dtype=torch.int64, device="cuda")
    dense = mv.MatrixTable(900, 32, "float32", updater="sgd", min_value=-1, max_value=1)
    dense2 = mv.MatrixTable(900, 32, "float32", updater="sgd")
    dense2.add_rows(torch.arange(900, device="cuda"), -dense.get().view(900, 32))
    ha = mv.HashMatrixTable(2100, 64, updater="sgd", min_value=-0.5, max_value=0.5)
    hb = mv.HashMatrixTable(600, 16, updater="sgd", init_value=0.25)
    lengths = torch.randint(0, 12, (4, B), generator=g, device="cuda")
    n = lengths.sum(1).tolist()
    pa = [torch.randint(0, ka.numel(), (n[1],), generator=g, device="cuda"),
          torch.randint(0, ka.numel(), (n[2],), generator=g, device="cuda")]
    pa[0][::3] = 0                                                               # a shared hot key
    pb = torch.randint(0, kb.numel(), (n[3],), generator=g, device="cuda")
    d_ids = torch.randint(0, 900, (n[0],), generator=g, device="cuda")
    keys = torch.cat([d_ids, ka[pa[0]], ka[pa[1]], kb[pb]])
    dout = torch.randn(B, 32 + 128 + 16, device="cuda", generator=g)
    cfg = [EmbeddingBagConfig(dense, ["d"], push_scale=0.1), EmbeddingBagConfig(ha, ["x", "y"], push_scale=0.1),
           EmbeddingBagConfig(hb, ["z"], push_scale=0.1, mode="mean")]
    ebc = PSEmbeddingCollection(cfg)
    assert _kernels(lambda: ebc(keys, lengths), "hash_lookup") == 1                 # one translation per call
    ha.lookup(ka), hb.lookup(kb)                                                      # every key now has a row
    (tw_a, ma), (tw_b, mb) = _dense_twin(mv, ha, ka, "sgd"), _dense_twin(mv, hb, kb, "sgd")
    twin = PSEmbeddingCollection([EmbeddingBagConfig(dense2, ["d"], push_scale=0.1),
                                  EmbeddingBagConfig(tw_a, ["x", "y"], push_scale=0.1),
                                  EmbeddingBagConfig(tw_b, ["z"], push_scale=0.1, mode="mean")])
    out_list = []
    assert _syncs(lambda: out_list.append(ebc(keys, lengths))) == 1                  # one host read per forward
    out = out_list[0]
    ref = twin(torch.cat([d_ids, ma[pa[0]], ma[pa[1]], mb[pb]]), lengths)
    assert torch.equal(out, ref)
    only_dense = PSEmbeddingCollection([EmbeddingBagConfig(dense, ["d"], push_scale=None)])
    assert torch.equal(out[:, :32], only_dense(d_ids, lengths[:1]))
    parts = ebc.split(out)
    starts = [0] + torch.cumsum(lengths.sum(1), 0).tolist()
    for f, name in ((1, "x"), (2, "y"), (3, "z")):
        t = ha if f < 3 else hb
        ref_f = embedding_bag(t, keys[starts[f]:starts[f + 1]], torch.cumsum(lengths[f], 0) - lengths[f],
                              mode="mean" if f == 3 else "sum")
        assert torch.equal(parts[name], ref_f), name
    out.backward(dout)
    ref.backward(dout)
    torch.cuda.synchronize()
    assert torch.equal(ha.get(ka), tw_a.get_rows(ma))
    assert torch.equal(hb.get(kb), tw_b.get_rows(mb))
    assert torch.equal(dense.get(), dense2.get())


def test_capacity(mv_device):
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbedding, PSEmbeddingCollection, embedding_bag
    mv = mv_device
    t = mv.HashMatrixTable(100, 8, updater="sgd", min_value=-1, max_value=1)
    assert t.slots == 128
    first = torch.tensor(_spread(100, 3), dtype=torch.int64, device="cuda")
    rows = t.lookup(first)
    vals = t.get(first)
    more = torch.tensor(_spread(20, 4), dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match=r"table full on server 0 \(at most 112 keys"):
        t.lookup(more)
    assert t.num_keys() == 112
    with pytest.raises(RuntimeError, match="table full"):
        t.lookup(torch.tensor(_spread(5, 5), dtype=torch.int64, device="cuda"))
    assert torch.equal(t.lookup(first), rows) and torch.equal(t.get(first), vals)
    t.add(first, torch.ones(100, 8, device="cuda"))
    assert torch.equal(t.get(first), vals - 1)
    assert t.num_keys() == 112
    # the 8 keys of `more` that were refused are missing, not errors, for every lookup that does not insert
    got = t.lookup(more, insert=False)
    refused = got == t.zero_row
    assert int(refused.sum()) == 8
    admitted = t.get(more)
    assert bool((admitted[refused] == 0).all()) and bool((admitted[~refused] != 0).any())
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["m"], push_scale=0.1)]).eval()
    y = ebc(more, torch.ones(1, 20, dtype=torch.int64, device="cuda"))
    assert torch.equal(y, admitted)
    assert torch.equal(PSEmbedding(t, push_scale=0.1).eval()(more, torch.arange(20, device="cuda")), admitted)
    assert torch.equal(embedding_bag(t, more, torch.arange(20, device="cuda")), admitted)
    with pytest.raises(RuntimeError, match="table full"):                    # inserting them still is
        PSEmbedding(t, push_scale=0.1)(more, torch.arange(20, device="cuda"))
    assert t.num_keys() == 112


def test_malformed_lengths_insert_nothing(mv_device):
    """The collection translates before it checks the lengths; lengths that would hand keys to the wrong table
    insert nothing, and the checks raise."""
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    mv = mv_device
    h = mv.HashMatrixTable(500, 8, updater="sgd")
    d = mv.MatrixTable(100, 8, "float32", updater="sgd")
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(d, ["d"]), EmbeddingBagConfig(h, ["h"])])
    ids = torch.tensor([1, 2, 3, 10**12, -5], device="cuda")
    for lengths, msg in (([[2], [2]], "lengths sum to 4"), ([[6], [-1]], "non-negative")):
        with pytest.raises(ValueError, match=msg):
            ebc(ids, torch.tensor(lengths, device="cuda"))
        assert h.num_keys() == 0
    ebc(ids, torch.tensor([[3], [2]], device="cuda"))
    assert h.num_keys() == 2


def test_eval_mode(mv_device):
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbedding, PSEmbeddingCollection, embedding_bag
    mv = mv_device
    t = mv.HashMatrixTable(500, 16, updater="sgd", min_value=-1, max_value=1)
    known = torch.tensor(_spread(50, 6), dtype=torch.int64, device="cuda")
    t.lookup(known)
    before = t.get(known)
    new = torch.tensor(_spread(50, 7), dtype=torch.int64, device="cuda")
    ids = torch.stack([known[:20], new[:20]], 1).reshape(-1)                       # bag b: (known b, new b)
    offs = torch.arange(0, 40, 2, device="cuda")
    layer = PSEmbedding(t, push_scale=0.1).eval()
    y = layer(ids, offs)
    assert t.num_keys() == 50
    assert torch.equal(y, t.get(known[:20]))                                       # the new keys add zeros
    assert torch.equal(y, embedding_bag(t, ids, offs))
    with pytest.raises(RuntimeError, match="eval mode"):
        y.sum().backward()
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["a"], push_scale=0.1)]).eval()
    yc = ebc(ids, torch.full((1, 20), 2, device="cuda"))
    assert torch.equal(yc, y) and t.num_keys() == 50
    with pytest.raises(RuntimeError, match="eval-mode"):
        yc.sum().backward()
    assert torch.equal(t.get(known), before)                                       # nothing was pushed
    with pytest.raises(TypeError, match="whole-table"):
        t.get_async()


def test_checkpoint_round_trip(mv_device):
    from multiverso_b200.ops import PSEmbedding
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(41)
    keys = torch.tensor(_spread(800, 8), dtype=torch.int64, device="cuda")
    a = mv.HashMatrixTable(1000, 32, updater="adagrad", min_value=-1, max_value=1, seed=4)
    ids, offs = _bags(keys, 300, g)
    PSEmbedding(a, push_scale=0.1, option=AddOption(learning_rate=0.5, rho=0.1))(ids, offs).backward(
        torch.randn(300, 32, device="cuda", generator=g))
    torch.cuda.synchronize()
    buf = io.BytesIO()
    a.store(buf)
    b = mv.HashMatrixTable(1000, 32, updater="adagrad", min_value=-1, max_value=1, seed=4)
    buf.seek(0)
    b.load(buf)
    n = a.num_keys()
    assert b.num_keys() == n and n == torch.unique(ids).numel()
    ka, va = a.export()
    kb, vb = b.export()
    assert torch.equal(ka, kb) and torch.equal(va, vb)
    assert torch.equal(b.lookup(ka, insert=True), a.lookup(ka, insert=False))
    assert b.num_keys() == n
    assert torch.equal(b.state[0], a.state[0]) and bool(b.state[0].abs().sum() > 0)


@pytest.mark.parametrize("nproc", [2, 4])
def test_hash_embedding_multi_gpu(nproc):
    """All ranks insert overlapping keys at once (tests/mp_hash_embedding_check.py under torchrun): one row per key,
    num_keys the size of the union, every rank's get bitwise equal, async sgd pushes land as init - lr * sum."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 800 + nproc
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_hash_embedding_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
