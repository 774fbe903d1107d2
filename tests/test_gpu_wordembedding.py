"""K7 numerics vs a plain PyTorch fp32 reference of the same sample schedule, plus
convergence checks for every mode (skip-gram / CBOW x NS / HS, AdaGrad)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _sig(x):
    return 1.0 / (1.0 + torch.exp(-x))


@pytest.mark.parametrize("D,K,hogwild", [(64, 8, 0), (200, 8, 0), (300, 8, 0), (512, 8, 0), (300, 5, 1)])
def test_sgns_fast_kernel_matches_reference(mv_device, D, K, hogwild):
    """The Hogwild kernels through the default dispatch: K = 8 runs the register kernel (one
    instantiation per row width: D 64 / 200 / 300 / 512), hogwild = 1 the window kernel.
    window=1 (no random shrink) and a one-word negative pool make the sample schedule
    deterministic: centre p trains (ctx p-1 -> p) then (ctx p+1 -> p), each with K draws of
    the pool word evaluated on pre-update rows. All words distinct, so cross-warp coupling
    is only through red.add accumulation: warps may or may not observe each other's updates
    (Hogwild), an O(lr^2) effect, so the test uses a small lr and compares the UPDATES with a
    relative tolerance (a wrong sign / missing term would be off by >= 100%)."""
    from multiverso_b200 import _native as N
    V, lr = 64, 1e-3
    torch.manual_seed(0)
    w_in = (torch.rand(V, D, device="cuda") - 0.5) * 0.2
    w_out = (torch.rand(V, D, device="cuda") - 0.5) * 0.2
    toks = torch.tensor([3, 9, 27, 5, -1, 11, 2, -1, 40], dtype=torch.int32, device="cuda")
    pool = torch.tensor([63], dtype=torch.int32, device="cuda")
    ref_in, ref_out = w_in.double().cpu().clone(), w_out.double().cpu().clone()
    i0, o0 = ref_in.clone(), ref_out.clone()
    tl = toks.cpu().tolist()
    for p, c in enumerate(tl):
        if c < 0:
            continue
        crow = o0[c].clone()
        for q in (p - 1, p + 1):
            if q < 0 or q >= len(tl) or tl[q] < 0:
                continue
            h = i0[tl[q]]
            herr = torch.zeros(D, dtype=torch.float64)
            g = (1 - _sig(h @ crow)) * lr
            herr += g * crow
            ref_out[c] += g * h
            crow = crow + g * h
            nrow = o0[63]
            gn = (0 - _sig(h @ nrow)) * lr
            herr += K * gn * nrow
            ref_out[63] += K * gn * h
            ref_in[tl[q]] += herr
    a = N.Sgns()
    loss = torch.zeros(1, device="cuda")
    pairs = torch.zeros(1, dtype=torch.int64, device="cuda")
    a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
    a.w_in, a.w_out, a.dim, a.ld = w_in.data_ptr(), w_out.data_ptr(), D, D
    a.window, a.negative, a.lr = 1, K, lr
    a.vocab, a.neg_pool, a.neg_pool_size = V, pool.data_ptr(), 1
    a.seed, a.loss_sum, a.pair_count = 1234, loss.data_ptr(), pairs.data_ptr()
    a.hogwild = hogwild
    N.cuda_lib().mvb_sgns_train(a, N.stream_ptr())
    torch.cuda.synchronize()
    assert int(pairs.item()) == 8
    d_in, d_out = w_in.double().cpu() - i0, w_out.double().cpu() - o0
    r_in, r_out = ref_in - i0, ref_out - o0
    assert r_in.abs().max() > 1e-5 and r_out.abs().max() > 1e-5
    e_in = ((d_in - r_in).norm() / r_in.norm()).item()
    e_out = ((d_out - r_out).norm() / r_out.norm()).item()
    assert e_in < 0.05 and e_out < 0.05, (e_in, e_out)
    assert float(loss.item()) > 0


@pytest.mark.parametrize("mode", ["sg_ns", "cbow_ns", "sg_hs", "cbow_hs", "sg_ns_adagrad", "sg_ns_d100", "sg_ns_k8", "sg_ns_win"])
def test_wordembedding_loss_decreases(mv_device, mode):
    from multiverso_b200.models.wordembedding import (WordEmbedding, WordEmbeddingOption,
                                                      synthetic_zipf_corpus)
    V = 2000
    opt = WordEmbeddingOption(embeding_size=100 if mode.endswith("d100") else 64, window_size=5,
                              negative_num=8 if mode.endswith("k8") else 5,
                              cbow="cbow" in mode, hs="hs" in mode, use_adagrad="adagrad" in mode,
                              init_learning_rate=0.025 if "hs" in mode else 0.05)
    we = WordEmbedding(opt, V)
    we.hogwild = mode.endswith("win")
    # a learnable corpus: word 2i is always followed by word 2i+1
    rng = np.random.default_rng(0)
    base = rng.integers(0, V // 2, size=40000) * 2
    toks = np.stack([base, base + 1], 1).reshape(-1).astype(np.int32)
    toks[100::101] = -1
    toks = torch.from_numpy(toks).cuda()
    losses = []
    for it in range(6):
        we.loss.zero_(); we.pairs.zero_()
        we.train_block(toks)
        torch.cuda.synchronize()
        losses.append(float(we.loss.item()) / max(int(we.pairs.item()), 1))
    assert losses[-1] < losses[0] * 0.9, losses
    emb = we.embeddings()
    assert torch.isfinite(emb).all()


def test_default_kernel_is_deterministic(mv_device):
    """The default K7 gives the same tables, loss and pair count on every run of the same input
    (Zipf corpus: hot rows are updated by many positions of the same wave)."""
    from multiverso_b200.models.wordembedding import (WordEmbedding, WordEmbeddingOption,
                                                      synthetic_zipf_corpus)
    V = 5000
    toks = torch.from_numpy(synthetic_zipf_corpus(200000, V, 1000, seed=3)).cuda()
    runs = []
    for _ in range(2):
        we = WordEmbedding(WordEmbeddingOption(embeding_size=300, window_size=5, negative_num=5), V, seed=1)
        for _ in range(2):
            we.train_block(toks)
        torch.cuda.synchronize()
        runs.append((we.input_table.get().clone(), we.output_table.get().clone(), we.loss.item(), we.pairs.item()))
    (i0, o0, l0, p0), (i1, o1, l1, p1) = runs
    assert p0 == p1 and p0 > 0 and l0 == l1
    assert torch.equal(i0, i1) and torch.equal(o0, o1)


def test_default_kernel_is_deterministic_at_dim_50(mv_device):
    """A row width that is not a multiple of 4 also runs on the deterministic waves."""
    from multiverso_b200.models.wordembedding import (WordEmbedding, WordEmbeddingOption,
                                                      synthetic_zipf_corpus)
    V = 5000
    toks = torch.from_numpy(synthetic_zipf_corpus(200000, V, 1000, seed=3)).cuda()
    runs = []
    for _ in range(2):
        we = WordEmbedding(WordEmbeddingOption(embeding_size=50, window_size=5, negative_num=5), V, seed=1)
        for _ in range(2):
            we.train_block(toks)
        torch.cuda.synchronize()
        runs.append((we.input_table.get().clone(), we.output_table.get().clone(), we.loss.item(), we.pairs.item(),
                     we.kernel_launches))
    (i0, o0, l0, p0, k0), (i1, o1, l1, p1, k1) = runs
    assert p0 == p1 and p0 > 0 and l0 == l1 and k0 == k1 and k0 >= 4     # two launches per wave
    assert torch.equal(i0, i1) and torch.equal(o0, o1) and not torch.equal(i0, torch.zeros_like(i0))


@pytest.mark.parametrize("dim,pad", [(37, 0), (37, 3), (50, 0), (50, 14), (300, 0)])
def test_dispatch_runs_the_deterministic_kernel_at_any_width(mv_device, dim, pad):
    """`mvb_sgns_train` sends skip-gram + NS (hogwild = 0) to the deterministic waves at any dim <= 512 and any
    row pitch: the same bits as a direct `mvb_sgns_train_det` call, and two launches per wave (the generic
    kernel would make one)."""
    from multiverso_b200 import _native as N
    V, ld = 3000, dim + pad
    g = torch.Generator().manual_seed(dim + pad)
    toks = torch.randint(0, V, (20000,), generator=g).to(torch.int32)
    toks[200::201] = -1
    toks = toks.cuda()
    prob, alias = torch.ones(V, device="cuda"), torch.arange(V, dtype=torch.int32, device="cuda")
    base = [torch.zeros(V, ld) for _ in range(2)]
    for b in base:
        b[:, :dim] = (torch.rand(V, dim, generator=g) - 0.5) * 0.4

    def run(fn):
        w_in, w_out = base[0].cuda(), base[1].cuda()
        a, out = N.Sgns(), torch.zeros(2, dtype=torch.int64, device="cuda")
        a.tokens, a.n_tokens, a.w_in, a.w_out = toks.data_ptr(), toks.numel(), w_in.data_ptr(), w_out.data_ptr()
        a.dim, a.ld, a.window, a.negative, a.lr, a.seed = dim, ld, 5, 5, 1e-2, 77
        a.vocab, a.alias_prob, a.alias_idx = V, prob.data_ptr(), alias.data_ptr()
        a.pair_count, a.loss_sum = out.data_ptr(), out.data_ptr() + 8
        getattr(N.cuda_lib(), fn)(a, N.stream_ptr())
        launches = N.cuda_lib().mvb_sgns_last_launches()
        torch.cuda.synchronize()
        return w_in, w_out, out.cpu(), launches

    i1, o1, r1, n1 = run("mvb_sgns_train")
    i2, o2, r2, n2 = run("mvb_sgns_train_det")
    assert n1 == n2 and n1 >= 2 and n1 % 2 == 0
    assert torch.equal(r1, r2) and r1[0] > 0
    assert torch.equal(i1, i2) and torch.equal(o1, o2) and not torch.equal(i1.cpu(), base[0])
    assert (i1[:, dim:] == 0).all() and (o1[:, dim:] == 0).all()


M64 = (1 << 64) - 1


def _hash64(x):
    x &= M64
    x ^= x >> 33; x = (x * 0xff51afd7ed558ccd) & M64
    x ^= x >> 33; x = (x * 0xc4ceb9fe1a85ec53) & M64
    x ^= x >> 33
    return x


@pytest.mark.parametrize("n_tok,dim", [(60, 300), (1500, 300), (700, 64), (400, 200)])
def test_sgns_window_kernel_matches_schedule(mv_device, n_tok, dim):
    """The window-batched K7 against a plain fp64 re-implementation of ITS sample
    schedule: per centre p the hash RNG gives the window shrink and K pool draws shared by the
    position's contexts; scores on pre-update rows; input delta sum_k g_ck out_k, output delta
    sum_c g_ck in_c.  All tokens are distinct and the pool words are not tokens, so rows only couple
    through reduce-add accumulation (exact) and Hogwild visibility (O(lr^2)).  1500 tokens span 24
    CTAs: the range ends (halo of 2W virtual centres, ring hand-over) are covered."""
    _check_schedule("mvb_sgns_train_win", n_tok, dim, 2e-2)


@pytest.mark.parametrize("n_tok,dim", [(60, 300), (1500, 300), (700, 64), (400, 200)])
def test_sgns_det_kernel_matches_schedule(mv_device, n_tok, dim):
    """The deterministic K7 against the same fp64 schedule.  These blocks fit in one wave, whose reads
    all see the initial rows exactly as the reference does, so the match is tight."""
    _check_schedule("mvb_sgns_train_det", n_tok, dim, 1e-4)


def _check_schedule(fn, n_tok, dim, tol):
    from multiverso_b200 import _native as N
    V, D, K, W, lr, seed = 4096, dim, 5, 5, 1e-4, 0xC0FFEE
    g = torch.Generator().manual_seed(1)
    w_in = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()
    w_out = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()
    ids = torch.randperm(V - 16, generator=g)[:n_tok].tolist()
    tl = list(ids)
    for b in range(37, n_tok, 53):
        tl[b] = -1
    pool_l = list(range(V - 16, V - 9))                       # 7 pool words, never tokens
    toks = torch.tensor(tl, dtype=torch.int32, device="cuda")
    pool = torch.tensor(pool_l, dtype=torch.int32, device="cuda")
    s_in, s_out = 0.5 + torch.rand(V, generator=g), 0.5 + torch.rand(V, generator=g)   # hot-row step scales
    i0, o0 = w_in.double().cpu(), w_out.double().cpu()
    ref_in, ref_out = i0.clone(), o0.clone()
    n_pairs = 0
    for p, c in enumerate(tl):
        if c < 0:
            continue
        prng = _hash64(seed ^ (((p + 1) * 0x9E3779B97F4A7C15) & M64))
        hw = W - ((prng >> 16) % W)
        ctxs = []
        for sgn in (-1, 1):
            for d in range(1, hw + 1):
                q = p + sgn * d
                if q < 0 or q >= n_tok or tl[q] < 0:
                    break
                ctxs.append(tl[q])
        outs = [(c, 1.0)]
        for k in range(1, K + 1):
            r = _hash64(prng ^ ((k * 0xD6E8FEB86659FD93) & M64))
            t = pool_l[(r >> 8) % len(pool_l)]
            if t != c:
                outs.append((t, 0.0))
        for x in ctxs:
            h = i0[x]
            for (o, label) in outs:
                gk = (label - _sig(h @ o0[o])) * lr
                ref_in[x] += gk * s_in[x].item() * o0[o]
                ref_out[o] += gk * s_out[o].item() * h
            n_pairs += 1
    a = N.Sgns()
    loss = torch.zeros(1, device="cuda")
    pairs = torch.zeros(1, dtype=torch.int64, device="cuda")
    a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
    a.w_in, a.w_out, a.dim, a.ld = w_in.data_ptr(), w_out.data_ptr(), D, D
    a.window, a.negative, a.lr = W, K, lr
    a.vocab, a.neg_pool, a.neg_pool_size = V, pool.data_ptr(), len(pool_l)
    a.seed, a.loss_sum, a.pair_count = seed, loss.data_ptr(), pairs.data_ptr()
    si, so = s_in.cuda(), s_out.cuda()
    a.scale_in, a.scale_out = si.data_ptr(), so.data_ptr()
    getattr(N.cuda_lib(), fn)(a, N.stream_ptr())
    torch.cuda.synchronize()
    assert int(pairs.item()) == n_pairs
    d_in, d_out = w_in.double().cpu() - i0, w_out.double().cpu() - o0
    r_in, r_out = ref_in - i0, ref_out - o0
    e_in = ((d_in - r_in).norm() / r_in.norm()).item()
    e_out = ((d_out - r_out).norm() / r_out.norm()).item()
    assert e_in < tol and e_out < tol, (e_in, e_out)
    # rows that are neither tokens nor pool words are untouched
    untouched = torch.ones(V, dtype=torch.bool)
    untouched[[t for t in tl if t >= 0] + pool_l] = False
    assert d_in[untouched].abs().max() == 0 and d_out[untouched].abs().max() == 0
    assert float(loss.item()) > 0


def test_sgns_window_kernel_maps_and_ld(mv_device):
    """Block mode of the window kernel: rows live in a compact cache addressed through id -> slot maps
    (world > 1) and rows are padded (ld > dim); result must equal the identity-mapped run on the same
    data (same seed => same schedule) up to Hogwild noise."""
    from multiverso_b200 import _native as N
    V, D, LD, K, W, lr, seed = 3000, 300, 320, 5, 5, 1e-3, 77
    g = torch.Generator().manual_seed(3)
    n_tok = 4000
    tl = torch.randint(0, V, (n_tok,), generator=g).to(torch.int32)
    tl[200::201] = -1
    toks = tl.cuda()
    prob = torch.ones(V, device="cuda")
    alias = torch.arange(V, dtype=torch.int32, device="cuda")
    base_in = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()
    base_out = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()

    def run(w_in, w_out, ld, map_in, map_out):
        a = N.Sgns()
        pairs = torch.zeros(1, dtype=torch.int64, device="cuda")
        a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
        a.w_in, a.w_out, a.dim, a.ld = w_in.data_ptr(), w_out.data_ptr(), D, ld
        a.window, a.negative, a.lr = W, K, lr
        a.vocab, a.alias_prob, a.alias_idx = V, prob.data_ptr(), alias.data_ptr()
        a.map_in, a.map_out = N.ptr(map_in), N.ptr(map_out)
        a.seed, a.pair_count = seed, pairs.data_ptr()
        N.cuda_lib().mvb_sgns_train_win(a, N.stream_ptr())
        torch.cuda.synchronize()
        return int(pairs.item())

    a_in, a_out = base_in.clone(), base_out.clone()
    n1 = run(a_in, a_out, D, None, None)
    perm = torch.randperm(V, generator=g).cuda()                 # id -> slot
    c_in = torch.zeros(V, LD, device="cuda"); c_out = torch.zeros(V, LD, device="cuda")
    c_in[perm, :D] = base_in; c_out[perm, :D] = base_out
    m = perm.to(torch.int32)
    n2 = run(c_in, c_out, LD, m, m)
    assert n1 == n2 and n1 > 0
    d1_in, d1_out = a_in - base_in, a_out - base_out
    d2_in, d2_out = c_in[perm, :D] - base_in, c_out[perm, :D] - base_out
    assert (c_in[:, D:] == 0).all() and (c_out[:, D:] == 0).all()      # padding never written
    e_in = ((d1_in - d2_in).norm() / d1_in.norm()).item()
    e_out = ((d1_out - d2_out).norm() / d1_out.norm()).item()
    assert e_in < 5e-2 and e_out < 5e-2, (e_in, e_out)


def test_sgns_det_kernel_maps_and_ld(mv_device):
    """Deterministic K7 over several waves on a cache through id -> slot maps with padded rows (ld > dim):
    same schedule and arithmetic, so it equals the identity-mapped run exactly; the padding is never written."""
    from multiverso_b200 import _native as N
    V, D, LD = 3000, 300, 320
    g = torch.Generator().manual_seed(3)
    toks = torch.randint(0, V, (20000,), generator=g).to(torch.int32)
    toks[200::201] = -1
    toks = toks.cuda()
    prob, alias = torch.ones(V, device="cuda"), torch.arange(V, dtype=torch.int32, device="cuda")
    base = [((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda() for _ in range(2)]

    def run(w_in, w_out, m):
        a, out = N.Sgns(), torch.zeros(2, dtype=torch.int64, device="cuda")
        a.tokens, a.n_tokens, a.w_in, a.w_out = toks.data_ptr(), toks.numel(), w_in.data_ptr(), w_out.data_ptr()
        a.dim, a.ld, a.window, a.negative, a.lr, a.seed = D, w_in.stride(0), 5, 5, 1e-2, 77
        a.vocab, a.alias_prob, a.alias_idx, a.map_in, a.map_out = V, prob.data_ptr(), alias.data_ptr(), N.ptr(m), N.ptr(m)
        a.pair_count, a.loss_sum = out.data_ptr(), out.data_ptr() + 8
        N.cuda_lib().mvb_sgns_train_det(a, N.stream_ptr())
        return out.cpu()

    a_in, a_out = base[0].clone(), base[1].clone()
    r1 = run(a_in, a_out, None)
    perm = torch.randperm(V, generator=g).cuda()                 # id -> slot
    c_in, c_out = torch.zeros(V, LD, device="cuda"), torch.zeros(V, LD, device="cuda")
    c_in[perm, :D], c_out[perm, :D] = base[0], base[1]
    r2 = run(c_in, c_out, perm.to(torch.int32))
    assert torch.equal(r1, r2) and r1[0] > 0 and r1[1] != 0       # pairs, loss (float bits)
    assert torch.equal(c_in[perm, :D], a_in) and torch.equal(c_out[perm, :D], a_out)
    assert (c_in[:, D:] == 0).all() and (c_out[:, D:] == 0).all() and not torch.equal(a_in, base[0])


def test_direct_mode_declines_what_the_window_kernel_does_not_cover(mv_device):
    """Direct mode (nservers > 1) runs on the window kernel alone.  With dim 516 it declines, and the call
    raises without touching either table instead of running a kernel that ignores the peer shards."""
    from multiverso_b200 import _native as N
    V, D = 64, 516
    g = torch.Generator().manual_seed(5)
    w_in = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()
    w_out = ((torch.rand(V, D, generator=g) - 0.5) * 0.4).cuda()
    i0, o0 = w_in.clone(), w_out.clone()
    toks = torch.randint(0, V, (500,), generator=g).to(torch.int32).cuda()
    prob, alias = torch.ones(V, device="cuda"), torch.arange(V, dtype=torch.int32, device="cuda")
    a = N.Sgns()
    a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
    a.w_in, a.w_out, a.dim, a.ld = w_in.data_ptr(), w_out.data_ptr(), D, D
    a.window, a.negative, a.lr, a.seed = 5, 5, 0.05, 11
    a.vocab, a.alias_prob, a.alias_idx = V, prob.data_ptr(), alias.data_ptr()
    a.nservers, a.rows_per_server = 2, V // 2
    for s_ in range(2):                                   # the two halves of one table as the two shards
        a.w_in_peers[s_], a.w_out_peers[s_] = w_in[s_ * V // 2].data_ptr(), w_out[s_ * V // 2].data_ptr()
    with pytest.raises(N.NativeError):
        N.cuda_lib().mvb_sgns_train(a, N.stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(w_in, i0) and torch.equal(w_out, o0)


def test_synthetic_corpus_shape():
    from multiverso_b200.models.wordembedding import synthetic_zipf_corpus
    c = synthetic_zipf_corpus(10000, 1000, sentence_len=100)
    assert c.shape == (10000,) and c.max() < 1000 and (c == -1).sum() == 99
