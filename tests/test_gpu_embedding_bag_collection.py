"""PSEmbeddingCollection on the GPU (csrc/cuda/emb_bag_coll.cu): each feature bitwise equal to embedding_bag over its
table, multi-shard row maps, a shared table pushed as one PSEmbedding call over the features' bags, independence of
the tables, one stateful step per row, determinism, host synchronisations and launch counts."""
import os
import subprocess
import sys
import types
import warnings

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _jagged(nrows, B, max_len, g, dev, empty_feature=None, zipf_head=None):
    """ids / lengths in the jagged layout: some empty bags, optionally a feature with no lookups at all and a hot id
    that makes up about 40 % of every feature's lookups."""
    F = len(nrows)
    lengths = torch.randint(0, max_len + 1, (F, B), generator=g, device=dev)
    lengths[:, ::7] = 0
    if empty_feature is not None:
        lengths[empty_feature] = 0
    parts = []
    for f, n in enumerate(nrows):
        ids = torch.randint(0, n, (int(lengths[f].sum()),), generator=g, device=dev)
        if zipf_head is not None:
            ids[torch.rand(ids.numel(), generator=g, device=dev) < 0.4] = zipf_head
        parts.append(ids)
    return torch.cat(parts), lengths


def _feature(ids, lengths, f):
    """(ids, offsets) of feature f, as embedding_bag takes them."""
    starts = [0] + torch.cumsum(lengths.sum(1), 0).tolist()
    return ids[starts[f]:starts[f + 1]], torch.cumsum(lengths[f], 0) - lengths[f], (starts[f], starts[f + 1])


def _sharded(W, S, gap=37):
    """W as S shards at separate places of one buffer with garbage rows between them (reference rows_per_server
    rule, the last shard takes the remainder), and a function reading the table back."""
    from multiverso_b200 import _native as N
    n, pitch = W.shape
    rps = n // S
    buf = torch.full((n + S * gap, pitch), 1e3, device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, rps
    spans = []
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
        spans.append((at, hi - lo))
    return rm, buf, lambda: torch.cat([buf[a:a + k] for a, k in spans])


def _fake_table(rm, updater, num_row, num_col):
    """A MatrixTable handle over an explicit row map: what the collection reads of a device table."""
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=num_row, num_col=num_col, updater=updater,
                                 is_sparse=False, rt=types.SimpleNamespace(device=torch.device("cuda", 0)))


@pytest.mark.parametrize("weighted", [False, True])
def test_forward_bitwise_mixed_dims(cuda, weighted):
    """Dims 4, 30, 64, 300 and 512 in one collection (a shared table, empty bags, a feature with no lookups):
    every feature's columns equal embedding_bag over its table bit for bit."""
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection, embedding_bag
    g = torch.Generator(device=cuda).manual_seed(1)
    dims, rows = [4, 30, 64, 300, 512], [900, 5000, 70000, 3000, 1200]
    Ws = []
    for n, d in zip(rows, dims):
        W = torch.randn(n, (d + 3) // 4 * 4 + 4, device=cuda, generator=g)
        W[:, d:] = 1e6                                                   # pitch padding must never count
        Ws.append(W[:, :d])
    modes = ["sum"] * 5 if weighted else ["mean", "sum", "mean", "sum", "sum"]
    feats = [["a"], ["b1", "b2"], ["c"], ["d", "d2", "d3"], ["e"]]
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(W, f, push_scale=None, mode=m)
                                 for W, f, m in zip(Ws, feats, modes)])
    tab = [0, 1, 1, 2, 3, 3, 3, 4]
    B = 333
    ids, lengths = _jagged([rows[t] for t in tab], B, 40, g, cuda, empty_feature=5)
    psw = torch.rand(ids.numel(), device=cuda, generator=g) if weighted else None
    out = ebc(ids, lengths, psw)
    assert out.shape == (B, sum(dims[t] for t in tab))
    for f, (name, part) in enumerate(ebc.split(out).items()):
        i, o, (lo, hi) = _feature(ids, lengths, f)
        ref = embedding_bag(Ws[tab[f]], i, o, None if psw is None else psw[lo:hi], modes[tab[f]])
        assert torch.equal(part, ref), name
    assert (ebc.split(out)["d2"] == 0).all()
    empty = ebc(torch.zeros(0, dtype=torch.int64, device=cuda), torch.zeros(len(tab), 0, dtype=torch.int64))
    assert empty.shape == (0, out.shape[1])


def _collection_step(tables, feats, modes, ids, lengths, dout, psw=None, scale=0.5):
    """Forward + fused sgd backward of a collection over (row map, back, dim) tables."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    cfgs = [EmbeddingBagConfig(_fake_table(rm, N.UPD_SGD, nrow, dim), f, push_scale=scale, mode=m)
            for (rm, nrow, dim), f, m in zip(tables, feats, modes)]
    ebc = PSEmbeddingCollection(cfgs)
    out = ebc(ids, lengths, psw)
    out.backward(dout)
    torch.cuda.synchronize()
    return out.detach()


@pytest.mark.parametrize("S", [3, 8])
def test_sharded_bitwise_equal(cuda, S):
    g = torch.Generator(device=cuda).manual_seed(11)
    Wa, Wb = torch.randn(10007, 64, device=cuda, generator=g), torch.randn(4001, 300, device=cuda, generator=g)
    ids, lengths = _jagged([10007, 10007, 4001], 900, 50, g, cuda, zipf_head=5)
    dout = torch.randn(900, 64 + 64 + 300, device=cuda, generator=g)
    res = []
    for nshards in (1, S):
        (ra, _, ba), (rb, _, bb) = _sharded(Wa, nshards, 0 if nshards == 1 else 37), \
            _sharded(Wb, nshards, 0 if nshards == 1 else 37)
        out = _collection_step([(ra, 10007, 64), (rb, 4001, 300)], [["x", "y"], ["z"]], ["sum", "mean"], ids, lengths,
                               dout)
        res.append((out, ba(), bb()))
    for a, b in zip(*res):
        assert torch.equal(a, b)


def test_shared_table_equals_stacked_psembedding(cuda):
    """sgd: the table two features share ends bitwise equal to one PSEmbedding call over both features' bags
    stacked; the unrelated table does not change that."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops.embedding import _fwd_device, _push_device
    g = torch.Generator(device=cuda).manual_seed(3)
    Wa, Wu = torch.randn(20000, 128, device=cuda, generator=g), torch.randn(500, 32, device=cuda, generator=g)
    ids, lengths = _jagged([500, 20000, 20000], 2048, 30, g, cuda, zipf_head=9)
    psw = torch.rand(ids.numel(), device=cuda, generator=g)
    dout = torch.randn(2048, 32 + 256, device=cuda, generator=g)
    (ru, keep_u, _), (ra, keep_a, back) = _sharded(Wu, 1, 0), _sharded(Wa, 1, 0)   # the buffers stay alive
    out = _collection_step([(ru, 500, 32), (ra, 20000, 128)], [["u"], ["q", "t"]], ["sum", "sum"], ids, lengths, dout,
                           psw)
    got = back()
    # one PSEmbedding call: the two features' bags one after the other
    i1, o1, (lo1, hi1) = _feature(ids, lengths, 1)
    i2, o2, (lo2, hi2) = _feature(ids, lengths, 2)
    sids, soff = torch.cat([i1, i2]), torch.cat([o1, o2 + i1.numel()])
    sdout = torch.cat([dout[:, 32:160], dout[:, 160:]]).contiguous()
    spsw = psw[lo1:hi2].contiguous()
    rm, _, back2 = _sharded(Wa, 1, 0)
    ref = _fwd_device(rm, 128, sids, soff, spsw, "sum")
    table = types.SimpleNamespace(updater=N.UPD_SGD, is_sparse=False, num_col=128)
    _push_device(table, rm, 128, sids, soff, spsw, "sum", sdout, 0.5, None)
    torch.cuda.synchronize()
    assert torch.equal(out[:, 32:], torch.cat([ref[:2048], ref[2048:]], 1))
    assert torch.equal(got, back2())


def test_unrelated_table_leaves_others_unchanged(cuda):
    """Adding a table (and its lookups) to a collection changes no other table's output or pushed rows."""
    g = torch.Generator(device=cuda).manual_seed(4)
    Wx, Wa, Wb = (torch.randn(n, d, device=cuda, generator=g) for n, d in ((3000, 64), (9000, 64), (7000, 256)))
    idx, lx = _jagged([3000], 1500, 25, g, cuda)
    ids, lengths = _jagged([9000, 9000, 7000], 1500, 25, g, cuda, zipf_head=2)
    dout = torch.randn(1500, 64 + 64 + 256, device=cuda, generator=g)
    dx = torch.randn(1500, 64, device=cuda, generator=g)
    (ra, _, ba), (rb, _, bb) = _sharded(Wa, 1, 0), _sharded(Wb, 1, 0)
    out1 = _collection_step([(ra, 9000, 64), (rb, 7000, 256)], [["a1", "a2"], ["b"]], ["mean", "sum"], ids, lengths,
                            dout)
    r1 = (ba(), bb())
    (rx, keep_x, _), (ra, _, ba), (rb, _, bb) = _sharded(Wx, 1, 0), _sharded(Wa, 1, 0), _sharded(Wb, 1, 0)
    out2 = _collection_step([(rx, 3000, 64), (ra, 9000, 64), (rb, 7000, 256)], [["x"], ["a1", "a2"], ["b"]],
                            ["sum", "mean", "sum"], torch.cat([idx, ids]), torch.cat([lx, lengths]),
                            torch.cat([dx, dout], 1))
    assert torch.equal(out2[:, 64:], out1)
    assert torch.equal(ba(), r1[0]) and torch.equal(bb(), r1[1])


@pytest.mark.parametrize("updater", ["momentum_sgd", "adagrad"])
def test_stateful_one_step_per_row(mv_device, updater):
    """A table shared by two features under a stateful updater: one step per touched row with the gradient summed
    over both features (fp64 expectation); a second table gets its own step."""
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    V, dim, scale = 2000, 32, 0.1
    t = mv.MatrixTable(V, dim, "float32", updater=updater, min_value=-1.0, max_value=1.0)
    t2 = mv.MatrixTable(300, 16, "float32", updater=updater, min_value=-1.0, max_value=1.0)
    W0, W20 = t.get().view(V, dim).double(), t2.get().view(300, 16).double()
    g = torch.Generator(device="cuda").manual_seed(2)
    B = 300
    lengths = torch.full((3, B), 20, device="cuda")
    ids = torch.cat([torch.randint(0, 40, (6000,), device="cuda", generator=g),     # heavy duplicates, shared rows
                     torch.randint(0, 40, (6000,), device="cuda", generator=g),
                     torch.randint(0, 300, (6000,), device="cuda", generator=g)])
    dout = torch.randn(B, 2 * dim + 16, device="cuda", generator=g)
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["q", "k"], push_scale=scale, option=opt),
                                 EmbeddingBagConfig(t2, ["o"], push_scale=scale, option=opt)])
    ebc(ids, lengths).backward(dout)
    torch.cuda.synchronize()
    bag = torch.arange(6000, device="cuda") // 20

    def expect(W, V, idl, douts):
        G = torch.zeros(V, W.shape[1], dtype=torch.float64, device="cuda")
        for i, d in zip(idl, douts):
            G.index_add_(0, i, d.double()[bag])
        G *= scale
        touched = torch.unique(torch.cat(idl))
        exp, gt = W.clone(), G[touched]
        if updater == "momentum_sgd":
            exp[touched] -= (1.0 - 0.9) * gt
        else:
            gn = gt / 0.5
            exp[touched] -= 0.2 * torch.rsqrt(gn * gn + 1e-6) * gn
        return exp

    for got, exp in ((t.get().view(V, dim).double(), expect(W0, V, [ids[:6000], ids[6000:12000]],
                                                           [dout[:, :dim], dout[:, dim:2 * dim]])),
                     (t2.get().view(300, 16).double(), expect(W20, 300, [ids[12000:]], [dout[:, 2 * dim:]]))):
        assert (got - exp).abs().max().item() < 1e-4 * max(1.0, exp.abs().max().item())


def test_deterministic_zipf_head(cuda):
    """One id is about 40 % of 400k lookups of two features over one table: its run spans hundreds of chunks."""
    g = torch.Generator(device=cuda).manual_seed(5)
    W = torch.randn(50000, 128, device=cuda, generator=g)
    ids, lengths = _jagged([50000, 50000], 8192, 48, g, cuda, zipf_head=17)
    assert (ids == 17).float().mean() >= 0.3 and ids.numel() > 300000
    dout = torch.randn(8192, 256, device=cuda, generator=g)
    runs = []
    for _ in range(2):
        rm, _, back = _sharded(W, 1, 0)
        out = _collection_step([(rm, 50000, 128)], [["a", "b"]], ["mean"], ids, lengths, dout)
        runs.append((out, back()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    assert not torch.equal(runs[0][1], W)


def _syncs(fn):
    """Synchronising torch calls made by fn (torch's sync debug mode in 'warn')."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def test_host_syncs(mv_device):
    """1 per forward, however many features; 0 per sgd backward; 1 per backward with compact tables."""
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(6)
    sgd = [mv.MatrixTable(1000 + 100 * i, 64, "float32", updater="sgd") for i in range(6)]
    ada = mv.MatrixTable(800, 32, "float32", updater="adagrad")
    ids, lengths = _jagged([1000, 1000, 1100, 1200, 1300, 1400, 1500], 512, 6, g, "cuda")
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(sgd[0], ["f0", "f1"], push_scale=0.1)] +
                                [EmbeddingBagConfig(t, [f"g{i}"], push_scale=0.1) for i, t in enumerate(sgd[1:])])
    ebc(ids, lengths).sum().backward()                     # warm-up
    out = []
    assert _syncs(lambda: out.append(ebc(ids, lengths))) == 1
    assert _syncs(lambda: out[0].sum().backward()) == 0
    ids2, l2 = _jagged([800, 1000], 512, 6, g, "cuda")
    ebc2 = PSEmbeddingCollection([EmbeddingBagConfig(ada, ["a"], push_scale=0.1),
                                  EmbeddingBagConfig(sgd[0], ["s"], push_scale=0.1)])
    ebc2(ids2, l2).sum().backward()
    y = ebc2(ids2, l2)
    assert _syncs(lambda: y.sum().backward()) == 1


def _coll_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "emb_coll" in e.name)


def test_launch_count_independent_of_features(cuda):
    """The collection's own kernels per forward + backward: the same for 4 and for 64 features (and tables)."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    g = torch.Generator(device=cuda).manual_seed(7)
    counts = []
    for F in (4, 64):
        keep = [_sharded(torch.randn(500, 64, device=cuda, generator=g), 1, 0) for _ in range(F)]
        ebc = PSEmbeddingCollection([EmbeddingBagConfig(_fake_table(rm, N.UPD_SGD, 500, 64), [f"f{i}"],
                                                        push_scale=0.1) for i, (rm, _, _) in enumerate(keep)])
        ids, lengths = _jagged([500] * F, 256, 3, g, cuda)
        ebc(ids, lengths).sum().backward()
        counts.append(_coll_kernels(lambda: ebc(ids, lengths).sum().backward()))
    assert counts[0] == counts[1] == 6, counts        # forward; keys, count, scan, main and merge


def test_errors_raise_without_launching(mv_device):
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection
    t = mv_device.MatrixTable(100, 32, "float32", updater="sgd")
    t2 = mv_device.MatrixTable(5000, 32, "float32", updater="sgd")
    ebc = PSEmbeddingCollection([EmbeddingBagConfig(t, ["a"]), EmbeddingBagConfig(t2, ["b"])])
    cases = [
        (torch.tensor([1, 200, 3], device="cuda"), torch.tensor([[2], [1]], device="cuda"), r"feature 'a'.*\[0, 100\)"),
        (torch.tensor([1, 2, 3], device="cuda"), torch.tensor([[2], [2]], device="cuda"), "lengths sum to 4"),
        (torch.tensor([1, 2, 3], device="cuda"), torch.tensor([[4], [-1]], device="cuda"), "non-negative"),
    ]
    for ids, lengths, msg in cases:
        def call():
            with pytest.raises(ValueError, match=msg):
                ebc(ids, lengths)
        assert _coll_kernels(call) == 0
    t30 = mv_device.MatrixTable(100, 30, "float32")
    with pytest.raises(ValueError, match="must be a multiple of 4"):
        PSEmbeddingCollection([EmbeddingBagConfig(t30, ["a"])])


@pytest.mark.parametrize("nproc", [2, 4])
def test_collection_peer_shards_multi_gpu(nproc):
    """Tables sharded over 2 / 4 GPUs (tests/mp_embedding_collection_check.py under torchrun): forward bitwise equal to
    local single-shard copies; async sgd pushes from every rank land as W0 - lr * sum of the rank gradients."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 600 + nproc
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_embedding_collection_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
