"""Embedding-bag kernels (csrc/cuda/emb_bag.cu) against fp64, over multi-shard row maps, their determinism with
Zipf-head ids, and PSEmbedding's pushes into sgd / momentum / AdaGrad / is_sparse tables."""
import types

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 1e-5


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _bags(V, B, n_max, g, dev, zipf_head=None):
    """Variable-length bags (some empty); with zipf_head, that id makes up about 40 % of the lookups."""
    lens = torch.randint(0, n_max + 1, (B,), generator=g, device=dev)
    lens[::7] = 0
    lens[1::11] = 1
    offsets = torch.cumsum(lens, 0) - lens
    L = int(lens.sum())
    ids = torch.randint(0, V, (L,), generator=g, device=dev)
    if zipf_head is not None:
        ids[torch.rand(L, generator=g, device=dev) < 0.4] = zipf_head
    return ids, offsets


def _fp64(W, dim, ids, offsets, psw, mode):
    """(fp64 result, fp64 sum of |terms|) per output element."""
    Wd = W[:, :dim].double()
    p = None if psw is None else psw.double()
    ref = F.embedding_bag(ids, Wd, offsets, mode=mode, per_sample_weights=p)
    mag = F.embedding_bag(ids, Wd.abs(), offsets, mode=mode, per_sample_weights=None if p is None else p.abs())
    return ref, mag


def _close(out, ref, mag):
    err = (out.double() - ref).abs()
    assert (err <= TOL * mag + 1e-30).all(), (err / mag.clamp_min(1e-30)).max().item()


@pytest.mark.parametrize("dim", [4, 16, 64, 128, 300, 1000])
@pytest.mark.parametrize("mode,weighted", [("sum", False), ("sum", True), ("mean", False)])
def test_forward_matches_fp64(cuda, dim, mode, weighted):
    from multiverso_b200.ops import embedding_bag
    g = torch.Generator(device=cuda).manual_seed(dim)
    W = torch.randn(5000, dim, device=cuda, generator=g)
    ids, offsets = _bags(5000, 700, 40, g, cuda)
    psw = torch.rand(ids.numel(), device=cuda, generator=g) if weighted else None
    out = embedding_bag(W, ids, offsets, psw, mode)
    assert out.shape == (700, dim)
    _close(out, *_fp64(W, dim, ids, offsets, psw, mode))
    empty = torch.diff(offsets, append=torch.tensor([ids.numel()], device=cuda)) == 0
    assert empty.any() and (out[empty] == 0).all()


def test_forward_padded_pitch_long_bag_and_2d(cuda):
    from multiverso_b200.ops import embedding_bag
    g = torch.Generator(device=cuda).manual_seed(3)
    W = torch.randn(20000, 320, device=cuda, generator=g)
    W[:, 300:] = 1e6                                               # padding columns must never count
    ids = torch.randint(0, 20000, (100000 + 50,), device=cuda, generator=g)
    offsets = torch.tensor([0, 0, 10, 100010, 100010], device=cuda)   # empty, 10, one bag of 10^5, empty, 40
    for mode in ("sum", "mean"):
        out = embedding_bag(W[:, :300], ids, offsets, mode=mode)
        _close(out, *_fp64(W, 300, ids, offsets, None, mode))
    ids2 = torch.randint(0, 20000, (64, 24), device=cuda, generator=g, dtype=torch.int32)
    out = embedding_bag(W[:, :300], ids2, mode="mean")
    _close(out, *_fp64(W, 300, ids2.long().view(-1), torch.arange(0, 64 * 24, 24, device=cuda), None, "mean"))


def _sharded(W, S, gap=37):
    """W as S shards at separate places of one buffer with garbage rows between them (reference
    rows_per_server rule, the last shard takes the remainder), and a function reading the table back."""
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


def _single(W):
    rm, buf, back = _sharded(W, 1, gap=0)
    return rm, buf, back


def _step(rm, dim, ids, offsets, psw, mode, dout, updater, is_sparse=False, num_col=None):
    """Forward + fused backward push over an explicit row map, the table handle faked."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops.embedding import _fwd_device, _push_device
    out = _fwd_device(rm, dim, ids, offsets, psw, mode)
    table = types.SimpleNamespace(updater=updater, is_sparse=is_sparse, num_col=num_col or rm.num_col)
    assert updater in (N.UPD_DEFAULT, N.UPD_SGD)
    _push_device(table, rm, dim, ids, offsets, psw, mode, dout, 0.5, None)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("dim", [64, 300, 1000])
def test_sharded_bitwise_equal(cuda, dim):
    from multiverso_b200 import _native as N
    g = torch.Generator(device=cuda).manual_seed(11)
    V = 10007
    W = torch.randn(V, dim, device=cuda, generator=g)
    ids, offsets = _bags(V, 900, 60, g, cuda, zipf_head=5)
    psw = torch.rand(ids.numel(), device=cuda, generator=g)
    dout = torch.randn(900, dim, device=cuda, generator=g)
    rm, _, back = _single(W)
    out1 = _step(rm, dim, ids, offsets, psw, "sum", dout, N.UPD_SGD)
    W1 = back()
    for S in (3, 8):
        rm, _, back = _sharded(W, S)
        out = _step(rm, dim, ids, offsets, psw, "sum", dout, N.UPD_SGD)
        assert torch.equal(out, out1), S
        assert torch.equal(back(), W1), S


def test_deterministic_zipf_head(cuda):
    """One id is about 40 % of 400k lookups: its run spans hundreds of backward chunks (the split path)."""
    from multiverso_b200 import _native as N
    g = torch.Generator(device=cuda).manual_seed(5)
    V, dim = 50000, 128
    W = torch.randn(V, dim, device=cuda, generator=g)
    ids, offsets = _bags(V, 16384, 48, g, cuda, zipf_head=17)
    assert (ids == 17).float().mean() >= 0.3
    dout = torch.randn(16384, dim, device=cuda, generator=g)
    runs = []
    for _ in range(2):
        rm, _, back = _single(W)
        out = _step(rm, dim, ids, offsets, None, "mean", dout, N.UPD_DEFAULT)
        runs.append((out, back()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    # the pushed rows equal the fp64 coalesced gradient
    bag = torch.repeat_interleave(torch.arange(16384, device=cuda),
                                  torch.diff(offsets, append=torch.tensor([ids.numel()], device=cuda)))
    lens = torch.bincount(bag, minlength=16384).double()
    contrib = dout.double()[bag] / lens[bag][:, None]
    G = torch.zeros(V, dim, dtype=torch.float64, device=cuda).index_add_(0, ids, contrib)
    mag = torch.zeros(V, dim, dtype=torch.float64, device=cuda).index_add_(0, ids, contrib.abs())
    delta = runs[0][1].double() - W.double()
    assert ((delta - 0.5 * G).abs() <= 1e-5 * 0.5 * mag + 2e-6 * W.double().abs() + 1e-30).all()


def test_sgd_step_equals_embeddingbag(mv_device):
    from multiverso_b200.ops import PSEmbedding
    mv = mv_device
    V, dim, lr = 3000, 64, 0.05
    t = mv.MatrixTable(V, dim, "float32", updater="sgd", min_value=-1.0, max_value=1.0)
    W0 = t.get().view(V, dim).clone()
    g = torch.Generator(device="cuda").manual_seed(1)
    ids, offsets = _bags(V, 500, 30, g, "cuda")
    psw = torch.rand(ids.numel(), device="cuda", generator=g)
    target = torch.randn(500, dim, device="cuda", generator=g)
    layer = PSEmbedding(t, push_scale=lr)
    ((layer(ids, offsets, psw) - target) ** 2).sum().backward()
    torch.cuda.synchronize()
    ref = torch.nn.EmbeddingBag(V, dim, mode="sum", sparse=True).cuda()
    with torch.no_grad():
        ref.weight.copy_(W0)
    ((ref(ids, offsets, per_sample_weights=psw) - target) ** 2).sum().backward()
    torch.optim.SGD(ref.parameters(), lr=lr).step()
    exp = ref.weight.detach()
    assert ((t.get().view(V, dim) - exp).abs() <= 1e-5 * exp.abs().clamp_min(1.0)).all()


@pytest.mark.parametrize("updater", ["momentum_sgd", "adagrad"])
def test_stateful_one_step_per_unique_row(mv_device, updater):
    """Heavy duplicates: each touched row gets exactly one updater step with its coalesced gradient."""
    from multiverso_b200.ops import PSEmbedding
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    V, dim, scale = 2000, 32, 0.1
    t = mv.MatrixTable(V, dim, "float32", updater=updater, min_value=-1.0, max_value=1.0)
    W0 = t.get().view(V, dim).double()
    g = torch.Generator(device="cuda").manual_seed(2)
    ids = torch.randint(0, 40, (6000,), device="cuda", generator=g)      # ~150 lookups per touched row
    offsets = torch.arange(0, 6000, 20, device="cuda")
    dout = torch.randn(300, dim, device="cuda", generator=g)
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    layer = PSEmbedding(t, push_scale=scale, option=opt)
    y = layer(ids, offsets)
    y.backward(dout)
    torch.cuda.synchronize()
    bag = torch.arange(6000, device="cuda") // 20
    G = torch.zeros(V, dim, dtype=torch.float64, device="cuda").index_add_(0, ids, dout.double()[bag]) * scale
    exp = W0.clone()
    touched = torch.unique(ids)
    gt = G[touched]
    if updater == "momentum_sgd":
        s0 = (1.0 - 0.9) * gt                          # s0 = m s0 + (1 - m) g from s0 = 0
        exp[touched] -= s0
    else:
        gn = gt / 0.5
        s0 = gn * gn
        exp[touched] -= 0.2 * torch.rsqrt(s0 + 1e-6) * gn
    got = t.get().view(V, dim).double()
    assert (got - exp).abs().max().item() < 1e-4 * max(1.0, exp.abs().max().item())
    untouched = torch.ones(V, dtype=torch.bool, device="cuda")
    untouched[touched] = False
    assert torch.equal(got[untouched], W0[untouched])


def test_psw_grad_equals_autograd(cuda):
    from multiverso_b200.ops import embedding_bag
    g = torch.Generator(device=cuda).manual_seed(8)
    for dim in (16, 300):
        W = torch.randn(4000, dim, device=cuda, generator=g)
        ids, offsets = _bags(4000, 300, 30, g, cuda)
        p = torch.rand(ids.numel(), device=cuda, generator=g).requires_grad_()
        dout = torch.randn(300, dim, device=cuda, generator=g)
        embedding_bag(W, ids, offsets, p).backward(dout)
        p2 = p.detach().double().requires_grad_()
        F.embedding_bag(ids, W.double(), offsets, mode="sum", per_sample_weights=p2).backward(dout.double())
        mag = (dout.double()[torch.repeat_interleave(torch.arange(300, device=cuda), torch.diff(
            offsets, append=torch.tensor([ids.numel()], device=cuda)))].abs() * W.double()[ids].abs()).sum(1)
        assert ((p.grad.double() - p2.grad).abs() <= TOL * mag + 1e-30).all()


def test_is_sparse_stale_rows(mv_device):
    from multiverso_b200.ops import PSEmbedding
    mv = mv_device
    t = mv.MatrixTable(1000, 16, "float32", updater="sgd", is_sparse=True)
    t.get_stale()                                       # first pull: everything
    ids = torch.tensor([5, 9, 5, 700, 9, 9, 42], device="cuda")
    PSEmbedding(t, push_scale=0.1)(ids, torch.tensor([0, 3], device="cuda")).sum().backward()
    torch.cuda.synchronize()
    stale, rows = t.get_stale()
    assert stale.tolist() == [5, 9, 42, 700]
    assert (rows == -0.1 * torch.tensor([2.0, 3.0, 1.0, 1.0], device="cuda")[:, None]).all()


def test_device_errors(mv_device):
    from multiverso_b200.ops import PSEmbedding, embedding_bag
    W = torch.randn(100, 30, device="cuda")
    with pytest.raises(ValueError, match="must be a multiple of 4"):
        embedding_bag(W, torch.tensor([1, 2], device="cuda"), torch.tensor([0], device="cuda"))
    t = mv_device.MatrixTable(100, 30, "float32")
    with pytest.raises(ValueError, match="must be a multiple of 4"):
        PSEmbedding(t)(torch.tensor([1, 2], device="cuda"), torch.tensor([0], device="cuda"))
    t = mv_device.MatrixTable(100, 32, "float32")
    with pytest.raises(ValueError, match=r"ids must be in \[0, 100\)"):
        PSEmbedding(t)(torch.tensor([1, 100], device="cuda"), torch.tensor([0], device="cuda"))


@pytest.mark.parametrize("nproc", [2, 4])
def test_embedding_peer_shards_multi_gpu(nproc):
    """The table sharded over 2 / 4 GPUs (tests/mp_embedding_check.py under torchrun): forward bitwise equal to a
    local single-shard copy; async sgd pushes from every rank land as W0 - lr * sum of the rank gradients."""
    import os
    import subprocess
    import sys
    if not torch.cuda.is_available() or torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 400 + nproc
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_embedding_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
