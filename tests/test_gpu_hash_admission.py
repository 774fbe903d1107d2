"""Count-based admission of a HashMatrixTable on the GPU (csrc/cuda/hash_rows.cu, the push_rows bound of
csrc/cuda/emb_bag.cu / emb_bag_coll.cu): sketch counters and totals bitwise equal to the numpy model of
tests/test_hash_admission_cpu.py on 1, 3 and 8 emulated servers under Zipf calls with aging, admit_after=1 equal to
the table without the argument, PSEmbedding and PSEmbeddingCollection training that pushes nothing for keys not
admitted, the calls that count nothing, add / table full / evict / checkpoints, and the new error codes."""
import io

import numpy as np
import pytest
import torch

from test_gpu_hash_embedding import _kernels, _spread, _syncs, _zipf
from test_hash_admission_cpu import SketchModel

pytestmark = pytest.mark.gpu

INT64_MIN = -(1 << 63)


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


class _Index:
    """S emulated servers of a hash index with admission on one GPU (as test_gpu_hash_embedding builds them)."""

    def __init__(self, S, P, dim, n):
        from multiverso_b200 import _native as N
        dev = torch.device("cuda", 0)
        self.S, self.P = S, P
        self.keys = torch.empty(S, P, dtype=torch.int64, device=dev)
        self.ready = torch.empty(S, P, dtype=torch.int32, device=dev)
        self.count = torch.empty(S, 2, dtype=torch.int64, device=dev)
        self.sketch = torch.zeros(S, 4 * P, dtype=torch.int32, device=dev)
        self.total = torch.zeros(S, 2, dtype=torch.int64, device=dev)
        self.age = torch.zeros(8, dtype=torch.int32, device=dev)
        rps = P if S > 1 else P + 1
        self.buf = torch.zeros(S * (P + 1), dim, device=dev)
        h = N.HashRows()
        h.nservers, h.slots = S, P
        h.map.num_row, h.map.num_col, h.map.nservers, h.map.rows_per_server = S * P + 1, dim, S, rps
        for s in range(S):
            h.map.shard_ptrs[s] = self.buf[s * P].data_ptr()
            h.keys[s], h.ready[s], h.count[s] = self.keys[s].data_ptr(), self.ready[s].data_ptr(), self.count[s].data_ptr()
            h.sketch[s], h.total[s] = self.sketch[s].data_ptr(), self.total[s].data_ptr()
            N.cuda_lib().mvb_hash_rows_init(self.keys[s], self.ready[s], self.count[s], P, N.stream_ptr())
        h.init, h.init_value = N.HASH_INIT_CONST, 0.5
        h.age, h.width, h.admit_after = self.age.data_ptr(), P, n
        self.h = h
        self.d = torch.frombuffer(bytearray(h), dtype=torch.uint8).to(dev)

    def lookup(self, keys, insert=True):
        from multiverso_b200 import _native as N
        rows, status = torch.empty_like(keys), torch.zeros(1, dtype=torch.int64, device=keys.device)
        a = N.HashLookup()
        a.tables, a.keys, a.n, a.insert = self.d.data_ptr(), keys.data_ptr(), keys.numel(), int(insert)
        a.rows, a.status, a.timeout_s, a.admit = rows.data_ptr(), status.data_ptr(), 30.0, int(insert)
        lib = N.cuda_lib()
        lib.mvb_hash_rows_lookup(a, N.stream_ptr())
        if insert:
            lib.mvb_hash_rows_age(self.h, N.stream_ptr())
        return rows, int(status.item())

    def held(self):
        k = self.keys.view(-1)
        return set(k[k != INT64_MIN].tolist())


@pytest.mark.parametrize("S", [1, 3, 8])
def test_sketch_matches_model(cuda, S):
    """Zipf calls with keys repeated within a warp and across warps, P small enough that aging fires several times:
    after every call the counters and totals are bitwise the model's, the keys holding slots are the model's, and
    every occurrence of a key in the call got the same row (the zero row when not admitted)."""
    P, n = 512, 3
    idx = _Index(S, P, 8, n)
    model = SketchModel(S, P, n)
    g = torch.Generator(device=cuda).manual_seed(100 + S)
    pool = torch.tensor(_spread(250 * S, S), dtype=torch.int64, device=cuda)
    aged = 0
    for call in range(24):
        keys = pool[_zipf(pool.numel(), 700, g, cuda)]
        keys[:64] = keys[0]                                   # one key over two whole warps
        before = model.total.copy()
        new = model.call(keys.cpu().numpy())
        aged += int((model.total < before).sum())
        rows, st = idx.lookup(keys)
        assert st == 0
        assert np.array_equal(idx.sketch.cpu().numpy().view(np.uint32).astype(np.int64), model.counters), call
        assert idx.total[:, 0].tolist() == model.total.tolist(), call
        assert idx.held() == model.held, call
        uk, inv = torch.unique(keys, return_inverse=True)
        first = torch.full((uk.numel(),), -1, dtype=torch.int64, device=cuda).scatter_(0, inv, rows)
        assert torch.equal(first[inv], rows)
        adm = torch.tensor([k in model.held for k in uk.tolist()], device=cuda)
        assert bool((first[~adm] == S * P).all()) and bool((first[adm] < S * P).all())
        assert new <= set(uk.tolist())
    assert aged >= S + 2
    # non-inserting lookups count nothing and admit nothing
    sk = idx.sketch.clone()
    rows, st = idx.lookup(pool, insert=False)
    assert st == 0 and torch.equal(idx.sketch, sk) and idx.held() == model.held


def _train(t, steps, g, pool, B=200, psw=False, mode="sum", push_scale=0.05):
    from multiverso_b200.ops import PSEmbedding
    layer = PSEmbedding(t, push_scale=push_scale, mode=mode)
    outs = []
    for _ in range(steps):
        lens = torch.randint(0, 12, (B,), generator=g, device="cuda")
        keys = pool[_zipf(pool.numel(), int(lens.sum()), g, "cuda")]
        w = torch.rand(keys.numel(), generator=g, device="cuda") if psw else None
        y = layer(keys, torch.cumsum(lens, 0) - lens, w)
        y.backward(torch.randn(B, t.num_col, generator=g, device="cuda"))
        outs.append(y.detach())
    torch.cuda.synchronize()
    return outs


def test_admit_after_one_is_the_plain_table(mv_device):
    """The same kernel launches, rows and values as the table built without the argument. Keys are inserted one per
    call first, so both tables give every key the same slot (within a call, slots follow arrival order)."""
    mv = mv_device
    pool = torch.tensor(_spread(600, 1), dtype=torch.int64, device="cuda")
    names = []
    res = []
    for kw in ({}, {"admit_after": 1}):
        t = mv.HashMatrixTable(1000, 16, updater="sgd", min_value=-0.1, max_value=0.1, **kw)
        for i in range(pool.numel()):
            t.lookup(pool[i:i + 1])
        g = torch.Generator(device="cuda").manual_seed(5)
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            outs = _train(t, 6, g, pool, psw=True)
        names.append(sorted(e.name for e in prof.events() if "anonymous namespace" in e.name))   # this library's
        res.append((outs, t.lookup(pool, insert=False), t.get(pool), t.shard.clone()))
    assert names[0] and names[0] == names[1] and not any("count_keys" in n or "hash_age" in n for n in names[0])
    (o0, r0, g0, s0), (o1, r1, g1, s1) = res
    assert all(torch.equal(a, b) for a, b in zip(o0, o1))
    assert torch.equal(r0, r1) and torch.equal(g0, g1) and torch.equal(s0, s1)


@pytest.mark.parametrize("updater", ["sgd", "rowwise_adagrad", "adam"])
@pytest.mark.parametrize("weighted", [False, True])
def test_training_against_dense_twin(mv_device, updater, weighted):
    """admit_after=3 over 20 steps: the forward and every admitted row bitwise equal to a dense MatrixTable of the
    same rows fed the same slot ids, with the lookups not admitted given weight 0; the zero row stays zero; host
    reads per forward / backward as with admission off."""
    from multiverso_b200.ops import PSEmbedding
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    opt = AddOption(learning_rate=0.1, rho=0.05, momentum=0.9) if updater == "adam" else \
        AddOption(learning_rate=0.5)
    h = mv.HashMatrixTable(8000, 32, updater=updater, admit_after=3)
    off = mv.HashMatrixTable(8000, 32, updater=updater)
    d = mv.MatrixTable(h.num_row, 32, "float32", updater=updater)
    assert d.shard.numel() == h.shard.numel()
    pool = torch.tensor(_spread(6000, 9), dtype=torch.int64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(17)
    zr = torch.tensor([h.zero_row], device="cuda")
    lh, ld, lo = (PSEmbedding(t, push_scale=0.05, option=opt) for t in (h, d, off))
    not_admitted = 0
    for step in range(20):
        B = 300
        lens = torch.randint(0, 16, (B,), generator=g, device="cuda")
        offs = torch.cumsum(lens, 0) - lens
        keys = pool[_zipf(pool.numel(), int(lens.sum()), g, "cuda")]
        w = torch.rand(keys.numel(), generator=g, device="cuda") if weighted else None
        dout = torch.randn(B, 32, generator=g, device="cuda")
        out = []
        n_h = _syncs(lambda: out.append(lh(keys, offs, w)))
        n_off = _syncs(lambda: out.append(lo(keys, offs, w)))
        assert n_h == n_off == 1
        yh = out[0]
        rows = h.lookup(keys, insert=False)                   # one rank: the rows of the forward
        mask = (rows != h.zero_row).float()
        not_admitted += int((mask == 0).sum())
        yd = ld(rows, offs, mask * w if weighted else mask)
        assert torch.equal(yh, yd), step
        assert _syncs(lambda: yh.backward(dout)) == _syncs(lambda: out[1].backward(dout))
        yd.backward(dout)
        torch.cuda.synchronize()
        held = torch.unique(rows[rows != h.zero_row])
        assert torch.equal(h.get_rows(held), d.get_rows(held)), step
        assert bool((h.get_rows(zr) == 0).all()), step
    assert not_admitted > 100
    for a, b in zip(h.state, d.state):                        # the admitted rows' updater state too
        ra = a[:h.zero_row * (a.numel() // h.num_row)] if a.numel() else a
        assert ra.numel() == 0 or bool(ra.abs().sum() > 0)


def test_mean_bags_against_fp64(mv_device):
    from multiverso_b200.ops import PSEmbedding
    mv = mv_device
    h = mv.HashMatrixTable(2000, 16, updater="sgd", admit_after=3, min_value=-0.5, max_value=0.5)
    pool = torch.tensor(_spread(3000, 4), dtype=torch.int64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(3)
    layer, lr = PSEmbedding(h, push_scale=0.3, mode="mean"), 0.3
    for step in range(20):
        B = 200
        lens = torch.randint(0, 10, (B,), generator=g, device="cuda")
        offs = torch.cumsum(lens, 0) - lens
        keys = pool[_zipf(pool.numel(), int(lens.sum()), g, "cuda")]
        dout = torch.randn(B, 16, generator=g, device="cuda")
        y = layer(keys, offs)
        rows = h.lookup(keys, insert=False)
        W0 = h.shard.view(-1, 16).double().clone()
        bag = torch.repeat_interleave(torch.arange(B, device="cuda"), lens)
        ref = torch.zeros(B, 16, dtype=torch.float64, device="cuda").index_add_(0, bag, W0[rows])
        ref /= lens.clamp(min=1)[:, None].double()
        torch.testing.assert_close(y.double(), ref, rtol=1e-5, atol=1e-6)
        y.backward(dout)
        torch.cuda.synchronize()
        grad = torch.zeros_like(W0).index_add_(0, rows, dout.double()[bag] / lens.double()[bag][:, None])
        grad[h.zero_row] = 0
        torch.testing.assert_close(h.shard.view(-1, 16).double(), W0 - lr * grad, rtol=1e-5, atol=1e-6)
        assert bool((h.shard.view(-1, 16)[h.zero_row] == 0).all())


def test_collection_mixed_tables(mv_device):
    """An admission hash table, a plain hash table and a dense table in one collection: each feature equals
    PSEmbedding over a twin of its table, the tables end equal, and neither zero row is pushed to."""
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbedding, PSEmbeddingCollection
    mv = mv_device

    def tables():
        return (mv.HashMatrixTable(2000, 16, updater="sgd", admit_after=3, min_value=-1, max_value=1),
                mv.HashMatrixTable(1000, 8, updater="rowwise_adagrad", min_value=-1, max_value=1),
                mv.MatrixTable(500, 12, "float32", updater="adam"))

    ha, hb, d = tables()
    ta, tb, td = tables()
    td.shard.copy_(d.shard)
    from multiverso_b200.tables.options import AddOption
    opt = AddOption(learning_rate=0.1, rho=0.05, momentum=0.9)
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(ha, ["a1", "a2"], push_scale=0.1),
                                 EmbeddingBagConfig(hb, ["b"], push_scale=0.1, option=AddOption(learning_rate=0.5)),
                                 EmbeddingBagConfig(d, ["d"], push_scale=0.1, option=opt)])
    la = PSEmbedding(ta, push_scale=0.1)
    lb = PSEmbedding(tb, push_scale=0.1, option=AddOption(learning_rate=0.5))
    ld = PSEmbedding(td, push_scale=0.1, option=opt)
    pa = torch.tensor(_spread(2500, 1), dtype=torch.int64, device="cuda")
    pb = torch.tensor(_spread(900, 2), dtype=torch.int64, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(8)
    B = 150
    for step in range(8):
        lengths = torch.randint(0, 9, (4, B), generator=g, device="cuda")
        n = lengths.sum(1).tolist()
        ka = pa[_zipf(pa.numel(), n[0] + n[1], g, "cuda")]
        kb = pb[_zipf(pb.numel(), n[2], g, "cuda")]
        kd = torch.randint(0, 500, (n[3],), generator=g, device="cuda")
        dout = torch.randn(B, 16 + 16 + 8 + 12, generator=g, device="cuda")
        y = ebc(torch.cat([ka, kb, kd]), lengths)
        # features a1 and a2 over one table: the single-table twin sees them as one call of 2B bags
        la_lens = torch.cat([lengths[0], lengths[1]])
        ya = la(ka, torch.cumsum(la_lens, 0) - la_lens)
        yb = lb(kb, torch.cumsum(lengths[2], 0) - lengths[2])
        yd = ld(kd, torch.cumsum(lengths[3], 0) - lengths[3])
        parts = ebc.split(y)
        # which slot a key gets depends on arrival order, and with it the grouping of a row's gradient pieces over
        # backward chunks: hash features agree to fp32 rounding, the dense one bit for bit
        for name, ref in (("a1", ya[:B]), ("a2", ya[B:]), ("b", yb)):
            torch.testing.assert_close(parts[name], ref, rtol=1e-5, atol=1e-6)
        assert torch.equal(parts["d"], yd), step
        y.backward(dout)
        ya.backward(torch.cat([dout[:, :16], dout[:, 16:32]], 0))
        yb.backward(dout[:, 32:40])
        yd.backward(dout[:, 40:])
        torch.cuda.synchronize()
        assert torch.equal(_sketch(ha), _sketch(ta)), step                        # the same counts and admissions
        assert torch.equal(ha.lookup(pa, insert=False) == ha.zero_row, ta.lookup(pa, insert=False) == ta.zero_row)
        torch.testing.assert_close(ha.get(pa), ta.get(pa), rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(hb.get(pb), tb.get(pb), rtol=1e-5, atol=1e-6)
        assert torch.equal(d.shard, td.shard), step
        for t in (ha, hb):
            assert bool((t.shard.view(-1, t.num_col)[t.zero_row] == 0).all())
    assert ha.num_keys() == ta.num_keys() and 0 < ha.num_keys() < torch.unique(pa).numel()


def _sketch(t):
    return t._sketch_buf.tensor(torch.uint8).clone()


def test_calls_that_count_nothing(mv_device):
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbedding, PSEmbeddingCollection, embedding_bag
    mv = mv_device
    t = mv.HashMatrixTable(500, 8, updater="sgd", admit_after=2, track_access=True)
    d = mv.MatrixTable(100, 8, "float32", updater="sgd")
    keys = torch.tensor(_spread(40, 3), dtype=torch.int64, device="cuda")
    t.lookup(keys[:10])                                        # counted once each, not admitted
    assert t.num_keys() == 0
    s0 = _sketch(t)
    assert int(s0.view(torch.int64)[-1]) == 10                 # the total
    offs = torch.arange(0, 40, 4, device="cuda")
    PSEmbedding(t, push_scale=0.1).eval()(keys, offs)
    embedding_bag(t, keys, offs)
    t.get(keys)
    t.lookup(keys, insert=False)
    t.last_seen(keys)
    PSEmbeddingCollection([EmbeddingBagConfig(t, ["h"])]).eval()(keys, torch.full((1, 10), 4, device="cuda"))
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(d, ["d"]), EmbeddingBagConfig(t, ["h"])])
    ids = torch.cat([torch.tensor([1, 2, 3], device="cuda"), keys[:10]])
    for lengths, msg in (([[2], [10]], "lengths sum to 12"), ([[14], [-1]], "non-negative")):
        with pytest.raises(ValueError, match=msg):
            ebc(ids, torch.tensor(lengths, device="cuda"))
    torch.cuda.synchronize()
    assert torch.equal(_sketch(t), s0) and t.num_keys() == 0
    ebc(ids, torch.tensor([[3], [10]], device="cuda"))        # the second sighting admits the 10 keys
    assert t.num_keys() == 10


def _estimates(t, keys):
    """The table's current estimates of `keys` (one server), read from its sketch with the model's indexes."""
    from test_hash_admission_cpu import cells
    c = _sketch(t)[:16 * t.slots].view(torch.int32).cpu().numpy().view(np.uint32).astype(np.int64)
    return c[cells(keys.cpu().numpy(), t.slots)].min(0)


def test_add_full_evict_and_checkpoint(mv_device):
    mv = mv_device
    t = mv.HashMatrixTable(1000, 8, updater="sgd", admit_after=2, track_access=True)
    k = torch.tensor(_spread(300, 5), dtype=torch.int64, device="cuda")
    t.add(k[:20], torch.ones(20, 8, device="cuda"))           # first sighting: values dropped
    assert t.num_keys() == 0 and bool((t.shard == 0).all())
    t.add(k[:20], torch.ones(20, 8, device="cuda"))           # second: admitted, then added
    assert t.num_keys() == 20 and bool((t.get(k[:20]) == -1).all())
    assert bool((t.shard.view(-1, 8)[t.zero_row] == 0).all())
    # evict: a removed key comes back as soon as its remaining estimate reaches n (here it is still >= 2)
    t.clock = 5
    t.lookup(k[:20])
    t.lookup(k[20:30])                                        # counted once: not admitted, not stamped
    assert t.num_keys() == 20
    assert t.evict(older_than=6) == 20 and t.num_keys() == 0
    assert bool((_estimates(t, k[:20]) >= 2).all())
    t.lookup(k[:30])
    assert t.num_keys() == 30
    # checkpoint: a resumed table counts and admits exactly like the uninterrupted one
    buf = io.BytesIO()
    t.store(buf)
    u = mv.HashMatrixTable(1000, 8, updater="sgd", admit_after=2, track_access=True)
    buf.seek(0)
    u.load(buf)
    assert torch.equal(_sketch(u), _sketch(t)) and u.num_keys() == t.num_keys()
    more = torch.tensor(_spread(600, 6), dtype=torch.int64, device="cuda")
    for x in (more[:300], more[100:400], more[:500], more):
        assert torch.equal(t.lookup(x) == t.zero_row, u.lookup(x) == u.zero_row)
        assert torch.equal(_sketch(u), _sketch(t)) and u.num_keys() == t.num_keys()
    for kw in ({}, {"admit_after": 3}):
        w = mv.HashMatrixTable(1000, 8, updater="sgd", track_access=True, **kw)
        buf.seek(0)
        with pytest.raises(ValueError, match="admit"):
            w.load(buf)
    plain = mv.HashMatrixTable(1000, 8, updater="sgd", track_access=True)
    b2 = io.BytesIO()
    plain.store(b2)
    b2.seek(0)
    with pytest.raises(ValueError, match="admission sketch"):
        u.load(b2)


def test_table_full(mv_device):
    """An admitted key that meets a full server raises "table full" as without admission; a key not admitted there
    reads zeros without an error."""
    mv = mv_device
    f = mv.HashMatrixTable(100, 8, updater="sgd", admit_after=2)
    k = torch.tensor(_spread(400, 7), dtype=torch.int64, device="cuda")
    with pytest.raises(RuntimeError, match=r"table full on server 0 \(at most 112 keys"):
        f.lookup(torch.cat([k[:150], k[:150]]))              # every key seen twice in the call: all admitted
    assert f.num_keys() == 112
    est = _estimates(f, k[150:])
    fresh = k[150:][torch.from_numpy(est == 0).cuda()][:5]   # one more sighting leaves them below 2
    assert fresh.numel() == 5
    rows = f.lookup(fresh)
    assert bool((rows == f.zero_row).all()) and f.num_keys() == 112


def test_push_rows_bound(cuda):
    """mvb_embedding_bag_bwd with push_rows: 0 is today's backward bit for bit; a bound leaves the rows at and above
    it out of n_unique and the compact output, and every other row's gradient is bitwise unchanged."""
    from multiverso_b200 import _native as N
    lib = N.cuda_lib()
    g = torch.Generator(device=cuda).manual_seed(2)
    R, dim, L, B = 300, 20, 5000, 400
    W = torch.randn(R, 20, generator=g, device=cuda)
    ids = torch.randint(0, R, (L,), generator=g, device=cuda)
    ids[::7] = R - 1
    ids[::11] = R - 2
    offs = torch.sort(torch.randint(0, L, (B,), generator=g, device=cuda))[0]
    offs[0] = 0
    psw = torch.rand(L, generator=g, device=cuda)
    dout = torch.randn(B, 20, generator=g, device=cuda)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = R, 20, 1, R
    rm.shard_ptrs[0] = W.data_ptr()
    sid, perm = torch.sort(ids, stable=True)
    nb = lib.mvb_embedding_bag_scratch_bytes(L, dim)
    scratch = torch.empty(nb, dtype=torch.uint8, device=cuda)

    def run(push_rows):
        a = N.EmbBag()
        a.wmap, a.dim, a.ids, a.L, a.offsets, a.B = rm, dim, sid.data_ptr(), L, offs.data_ptr(), B
        a.psw, a.dout, a.ldd, a.perm = psw.data_ptr(), dout.data_ptr(), 20, perm.data_ptr()
        a.scratch, a.scratch_bytes, a.epilogue, a.scale = scratch.data_ptr(), nb, N.EMB_COMPACT, 0.5
        a.push_rows = push_rows
        nu = torch.empty(1, dtype=torch.int64, device=cuda)
        a.n_unique = nu.data_ptr()
        lib.mvb_embedding_bag_bwd(a, N.stream_ptr())
        U = int(nu.item())
        grads = torch.full((U, 20), 7.0, device=cuda)
        uniq = torch.full((U,), -5, dtype=torch.int64, device=cuda)
        a.grads, a.ldg, a.uniq = grads.data_ptr(), 20, uniq.data_ptr()
        lib.mvb_embedding_bag_bwd(a, N.stream_ptr())
        return U, grads, uniq

    U0, g0, u0 = run(0)
    assert U0 == torch.unique(ids).numel() and torch.equal(u0, torch.unique(ids))
    for bound, drop in ((R - 1, 1), (R - 2, 2), (R + 5, 0)):
        U, gb, ub = run(bound)
        assert U == U0 - drop and torch.equal(ub, u0[:U]) and torch.equal(gb, g0[:U]), bound
    # the fused push: rows below the bound get bitwise today's push, the rows above none
    for bound in (0, R - 2):
        Wp = W.clone()
        rmp = N.RowMap.from_buffer_copy(rm)
        rmp.shard_ptrs[0] = Wp.data_ptr()
        a = N.EmbBag()
        a.wmap, a.dim, a.ids, a.L, a.offsets, a.B = rmp, dim, sid.data_ptr(), L, offs.data_ptr(), B
        a.psw, a.dout, a.ldd, a.perm = psw.data_ptr(), dout.data_ptr(), 20, perm.data_ptr()
        a.scratch, a.scratch_bytes, a.epilogue, a.scale, a.push_rows = scratch.data_ptr(), nb, N.EMB_PUSH, 0.5, bound
        lib.mvb_embedding_bag_bwd(a, N.stream_ptr())
        torch.cuda.synchronize()
        if bound == 0:
            W_all = Wp
        else:
            assert torch.equal(Wp[:bound], W_all[:bound]) and torch.equal(Wp[bound:], W[bound:])


def test_age_error_codes(cuda):
    from multiverso_b200 import _native as N
    idx = _Index(2, 64, 8, 3)
    lib = N.cuda_lib()

    def code(h):
        try:
            lib.mvb_hash_rows_age(h, N.stream_ptr())
            return 0
        except N.NativeError as err:
            return int(str(err).split("rc=")[1].split(":")[0])

    assert code(idx.h) == 0
    cases = [("nservers", 0, -3), ("nservers", 9, -3), ("slots", 48, -4), ("admit_after", 1, -7),
             ("admit_after", 0, -7), ("width", 48, -8), ("width", 1, -8), ("width", 1 << 32, -8), ("age", None, -9)]
    for field, val, rc in cases:
        h = N.HashRows.from_buffer_copy(idx.h)
        setattr(h, field, val)
        assert _kernels(lambda: code(h), "hash_") == 0 and code(h) == rc, field
    for arr in ("sketch", "total"):
        h = N.HashRows.from_buffer_copy(idx.h)
        getattr(h, arr)[1] = None
        assert _kernels(lambda: code(h), "hash_") == 0 and code(h) == -9, arr


@pytest.mark.parametrize("nproc", [2, 4])
def test_hash_admission_multi_gpu(nproc):
    """Ranks count shared keys into sketches that peers own; afterwards every rank's get agrees
    (tests/mp_hash_admission_check.py under torchrun)."""
    import os
    import subprocess
    import sys
    if not torch.cuda.is_available() or torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 1000 + nproc
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_hash_admission_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
