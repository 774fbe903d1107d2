"""PSFieldAwareFactorizationMachine on the GPU (csrc/cuda/ffm.cu): y and the pushed row gradient (fused red.add and
compact) against fp64 within the bounds derived in the op's docstring, up to the widest D + 1 = 1021 and with a bag
longer than one shared-memory tile; bitwise equality with fp64 on exactly representable operands; F = 1 against
PSFactorizationMachine; bitwise equality over runs, shards and tile sizes; the no-grad forward; one updater step per
touched row for sgd, adagrad, rowwise_adagrad, adam and ftrl; HashMatrixTable insertion, eval mode and admission;
host synchronisations; a planted FFM trained end to end; errors raised without a launch."""
import types
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _sharded(W, S, gap=37):
    """W [n, C] as S shards of a row pitch round4(C) at separate places of one buffer with NaN rows between them
    (reference rows_per_server rule, the last shard takes the remainder), and a function reading the table back."""
    from multiverso_b200 import _native as N
    n, C = W.shape
    pitch = (C + 3) // 4 * 4
    rps = n // S
    buf = torch.full((n + S * gap, pitch), float("nan"), device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, rps
    spans = []
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo, :C] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
        spans.append((at, hi - lo))
    return rm, buf, lambda: torch.cat([buf[a:a + k, :C] for a, k in spans])


def _fake_table(rm, num_row, num_col, updater=None):
    """A MatrixTable handle over an explicit row map: what the op reads of a device table."""
    from multiverso_b200 import _native as N
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=num_row, num_col=num_col,
                                 updater=N.UPD_DEFAULT if updater is None else updater, is_sparse=False,
                                 rt=types.SimpleNamespace(device=torch.device("cuda", 0)))


def _zipf_ids(n, L, gen, s=1.05):
    w = torch.from_numpy(1.0 / np.arange(1, n + 1) ** s).cuda()
    return torch.multinomial(w / w.sum(), L, replacement=True, generator=gen)


def _batch(n, B, F, gen, long_bag=600, max_len=40):
    """Zipf ids in bags of 0..max_len lookups: bag 0 empty, bag 1 one lookup, bag 2 long_bag lookups (many per
    field); random fields; signed values."""
    lens = torch.randint(0, max_len + 1, (B,), device="cuda", generator=gen)
    lens[0], lens[1], lens[2] = 0, 1, long_bag
    L = int(lens.sum())
    ids = _zipf_ids(n, L, gen)
    fields = torch.randint(0, F, (L,), device="cuda", generator=gen)
    x = torch.randn(L, device="cuda", generator=gen)
    return ids, fields, torch.cumsum(lens, 0) - lens, x


def _reference(W, ids, fields, offsets, x, g, F, k):
    """fp64 y, its bound, the row gradient G of sum(g * y), its bound (the op's docstring), and H."""
    n = W.shape[0]
    D = F * k
    B, L = offsets.numel(), ids.numel()
    dev = W.device
    lens = torch.diff(offsets, append=torch.tensor([L], device=dev))
    bag = torch.repeat_interleave(torch.arange(B, device=dev), lens)
    R = W.double()[ids][:, :D + 1]
    V = R[:, :D].reshape(L, F, k)
    xd, gd = x.double(), g.double()
    H = torch.zeros(L * F, k, dtype=torch.float64, device=dev)
    A = torch.zeros(L * F, k, dtype=torch.float64, device=dev)
    for d in range(1, int(lens.max())):
        j = torch.nonzero(bag[:-d] == bag[d:]).view(-1)
        l = j + d
        for p, q in ((j, l), (l, j)):            # H_p[f_q] += x_p x_q V_q[f_p]
            t = (xd[p] * xd[q])[:, None] * V[q, fields[p]]
            H.index_add_(0, p * F + fields[q], t)
            A.index_add_(0, p * F + fields[q], t.abs())
    H, A = H.view(L, D), A.view(L, D)
    same = torch.zeros(B * F, dtype=torch.float64, device=dev).index_add_(
        0, bag * F + fields, torch.ones(L, dtype=torch.float64, device=dev)).view(B, F)
    njf = same[bag] - torch.nn.functional.one_hot(fields, F).double()           # [L, F]
    njc = njf.repeat_interleave(k, 1)                                          # [L, D]
    H = torch.cat([H, xd[:, None]], 1)
    zeros = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)        # noqa: E731
    lin = zeros(B).index_add_(0, bag, xd * R[:, D])
    y = lin + 0.5 * zeros(B).index_add_(0, bag, (H[:, :D] * R[:, :D]).sum(1))
    nq = (D + 4) // 4
    Nb = 4 * torch.ceil(lens.double() * nq / 256)
    Lam = zeros(B).index_add_(0, bag, (xd * R[:, D]).abs())
    Q = zeros(B).index_add_(0, bag, ((njc + Nb[bag][:, None] + 13) * A * R[:, :D].abs()).sum(1))
    tol_y = U * ((Nb + 12) * Lam + 0.5 * Q + y.abs())
    gb = gd[bag]
    G = zeros(n, D + 1).index_add_(0, ids, gb[:, None] * H)
    m = torch.bincount(ids, minlength=n).double()
    Ae = torch.cat([(njc + 1) * A, zeros(L, 1)], 1)
    tol_G = U * zeros(n, D + 1).index_add_(0, ids, gb.abs()[:, None] * Ae) \
        + (2 * m + 4)[:, None] * U * zeros(n, D + 1).index_add_(0, ids, (gb[:, None] * H).abs())
    return y, tol_y, G, tol_G, torch.unique(ids), H


def _run(W, ids, fields, offsets, x, g, F, k, S=1, updater=None, push_scale=1.0):
    """One forward + backward over a fake table of S shards: (y, table after, compact pushes)."""
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine
    rm, keep, back = _sharded(W, S, 0 if S == 1 else 37)
    t = _fake_table(rm, W.shape[0], W.shape[1], updater)
    pushes = []
    t.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    ffm = PSFieldAwareFactorizationMachine(t, F, k, push_scale=push_scale)
    y = ffm(ids, fields, offsets, x)
    (y * g).sum().backward()
    torch.cuda.synchronize()
    return y.detach(), back(), pushes


def _assert_within(got, exp, tol, what):
    err = (got.double() - exp).abs()
    assert (err <= tol).all(), (what, (err / tol.clamp_min(1e-300)).max().item())


@pytest.mark.parametrize("F,k,extra", [(1, 4, 0), (3, 4, 3), (5, 8, 0), (39, 4, 3), (16, 16, 7), (255, 4, 3)])
def test_matches_fp64(cuda, F, k, extra):
    """B = 1024 bags over 5000 Zipf rows (the hottest row's run crosses many 256-lookup chunks), with an empty, a
    one-lookup and a 600-lookup bag (longer than one shared-memory tile at every D here, many lookups per field):
    y against fp64, the row gradient from a default table with push_scale = 1 (fused red.add) and from the compact
    push of an adagrad table. Columns past D hold NaN: they are never read."""
    from multiverso_b200 import _native as N
    gen = torch.Generator(device=cuda).manual_seed(F * 100 + k)
    n, B, D = 5000, 1024, F * k
    W = torch.randn(n, D + 1 + extra, device=cuda, generator=gen) / (F * k) ** 0.5
    W[:, D + 1:] = float("nan")
    ids, fields, offsets, x = _batch(n, B, F, gen)
    assert int(torch.bincount(ids).max()) > 2 * 256
    g = torch.randn(B, device=cuda, generator=gen)
    y, after, _ = _run(W, ids, fields, offsets, x, g, F, k)
    y_r, tol_y, G, tol_G, touched, _ = _reference(W, ids, fields, offsets, x, g, F, k)
    assert y[0] == 0
    _assert_within(y, y_r, tol_y, f"y F={F} k={k}")
    d = after[:, :D + 1].double() - W[:, :D + 1].double()
    _assert_within(d, G, tol_G + U * (W[:, :D + 1].double() + G).abs(), f"fused F={F} k={k}")
    assert after[:, D + 1:].isnan().all()
    keep = torch.ones(n, dtype=torch.bool, device=cuda)
    keep[touched] = False
    assert torch.equal(after[keep, :D + 1], W[keep, :D + 1])
    y2, after2, pushes = _run(W, ids, fields, offsets, x, g, F, k, updater=N.UPD_ADAGRAD)
    assert torch.equal(y2, y) and torch.equal(after2.nan_to_num(), W.nan_to_num()) and len(pushes) == 1
    uid, vals = pushes[0]
    assert torch.equal(uid, touched) and vals.shape == (touched.numel(), W.shape[1])
    _assert_within(vals[:, :D + 1], G[uid], tol_G[uid], f"compact F={F} k={k}")
    assert not vals[:, D + 1:].any()


def test_exact_operands_are_bitwise_fp64(cuda):
    """Rows in {-1/4, 0, 1/4}, values and g in {+-1/2, +-1}: every product and partial sum is a multiple of 2^-7 far
    below 2^17, so fp32 is exact in any order, and y, the compact G and the table after a fused push with
    push_scale = 1/2 equal fp64 bit for bit."""
    from multiverso_b200 import _native as N
    gen = torch.Generator(device=cuda).manual_seed(5)
    n, B, F, k = 3000, 512, 6, 4
    D = F * k
    W = torch.randint(-1, 2, (n, D + 1), device=cuda, generator=gen).float() / 4
    ids, fields, offsets, _ = _batch(n, B, F, gen)
    L = ids.numel()
    pm = lambda s: (torch.randint(0, 2, s, device=cuda, generator=gen) * 2 - 1).float()     # noqa: E731
    x = pm((L,)) / 2 ** torch.randint(0, 2, (L,), device=cuda, generator=gen).float()
    g = pm((B,)) / 2 ** torch.randint(0, 2, (B,), device=cuda, generator=gen).float()
    y_r, _, G, _, touched, _ = _reference(W, ids, fields, offsets, x, g, F, k)
    y, after, _ = _run(W, ids, fields, offsets, x, g, F, k, push_scale=0.5)
    assert torch.equal(y.double(), y_r)
    assert torch.equal(after.double(), W.double() + 0.5 * G)
    _, _, pushes = _run(W, ids, fields, offsets, x, g, F, k, updater=N.UPD_ADAGRAD, push_scale=0.5)
    uid, vals = pushes[0]
    assert torch.equal(uid, touched) and torch.equal(vals.double(), 0.5 * G[uid])


def test_one_field_matches_the_factorization_machine(cuda):
    """F = 1 is the FM with C = k + 1: y and the fused push of both layers over the same table agree within the sum
    of their bounds (the FM's from its docstring)."""
    from multiverso_b200.ops import PSFactorizationMachine
    gen = torch.Generator(device=cuda).manual_seed(8)
    n, B, k = 4000, 1024, 12
    C = k + 1
    W = torch.randn(n, C, device=cuda, generator=gen) / C ** 0.5
    ids, _, offsets, x = _batch(n, B, 1, gen)
    fields = torch.zeros_like(ids)
    g = torch.randn(B, device=cuda, generator=gen)
    y, after, _ = _run(W, ids, fields, offsets, x, g, 1, k)
    y_r, tol_y, G, tol_G, _, _ = _reference(W, ids, fields, offsets, x, g, 1, k)
    rm, buf, back = _sharded(W, 1, 0)
    fm = PSFactorizationMachine(_fake_table(rm, n, C))
    yf = fm(ids, offsets, x)
    (yf * g).sum().backward()
    torch.cuda.synchronize()
    # the FM's bounds (factorization_machine.py)
    L = ids.numel()
    lens = torch.diff(offsets, append=torch.tensor([L], device=cuda))
    bag = torch.repeat_interleave(torch.arange(B, device=cuda), lens)
    Wd, xd, gd = W.double(), x.double(), g.double()
    R = Wd[ids]
    z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=cuda)          # noqa: E731
    S = z(B, C).index_add_(0, bag, xd[:, None] * R)
    A = z(B, C).index_add_(0, bag, (xd[:, None] * R).abs())
    q = z(B).index_add_(0, bag, xd ** 2 * (R[:, :k] ** 2).sum(1))
    ss, nb, P = (S[:, :k] ** 2).sum(1), lens.double(), (A[:, :k] ** 2).sum(1)
    tol_fm = U * ((nb + 5) * (A[:, k] + P) + 9 * ss + (nb + 7) * q + 0.5 * (ss - q).abs() + y_r.abs())
    Sp = S.clone()
    Sp[:, k] = 1
    vp = R.clone()
    vp[:, k] = 0
    gx = gd[bag] * xd
    m = torch.bincount(ids, minlength=n).double()
    Ae = A.clone()
    Ae[:, k] = 0
    tol_Gfm = U * z(n, C).index_add_(0, ids, gx.abs()[:, None] * (nb[bag][:, None] + 5) * Ae[bag]) \
        + (2 * m + 4)[:, None] * U * (z(n, C).index_add_(0, ids, gx.abs()[:, None] * Sp[bag].abs())
                                      + z(n, C).index_add_(0, ids, (gd[bag].abs() * xd ** 2)[:, None] * vp.abs()))
    _assert_within(y, yf.detach().double(), tol_y + tol_fm, "y vs fm")
    tol_push = U * (Wd + G).abs()
    _assert_within(after.double() - Wd, back().double() - Wd, tol_G + tol_Gfm + 2 * tol_push, "G vs fm")


def _outputs(W, ids, fields, offsets, x, g, F, k, S, updater=None, max_len=None):
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine
    rm, keep, back = _sharded(W, S, 0 if S == 1 else 37)
    t = _fake_table(rm, W.shape[0], W.shape[1], updater)
    pushes = []
    t.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    ffm = PSFieldAwareFactorizationMachine(t, F, k)
    lens = torch.diff(offsets, append=torch.tensor([ids.numel()], device=ids.device))
    ml = int(lens.max()) if max_len is None else max_len
    yl, h = ffm._launch(ids, offsets, fields.int(), x, ml, grad=True)
    y = ffm(ids, fields, offsets, x)
    (y * g).sum().backward()
    torch.cuda.synchronize()
    out = [y.detach(), yl, h, back()]
    for p in pushes:
        out += list(p)
    return out


@pytest.mark.parametrize("F,k", [(8, 4), (20, 12)])
def test_bitwise_over_shards_runs_and_tiles(cuda, F, k):
    """y, H, the table after the push and the compact pushes are bitwise the same over 1 / 2 / 3 / 8 shards, over
    repeated runs, and over the shared-memory tile (sized by the longest bag, or by the kernel alone)."""
    from multiverso_b200 import _native as N
    gen = torch.Generator(device=cuda).manual_seed(9)
    n, B = 100003, 2048
    W = torch.randn(n, F * k + 1, device=cuda, generator=gen) * 0.1
    ids, fields, offsets, x = _batch(n, B, F, gen)
    g = torch.randn(B, device=cuda, generator=gen)
    for updater in (None, N.UPD_ADAGRAD):
        ref = _outputs(W, ids, fields, offsets, x, g, F, k, 1, updater)
        for shards, ml in ((1, None), (2, None), (3, None), (8, None), (1, 0), (1, 7), (3, 1)):
            got = _outputs(W, ids, fields, offsets, x, g, F, k, shards, updater, ml)
            assert len(got) == len(ref)
            for i, (a, b) in enumerate(zip(ref, got)):
                assert torch.equal(a, b), (updater, shards, ml, i)


def test_no_grad_forward_is_bitwise_the_training_forward(cuda):
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine
    n, F, k = 5000, 10, 8
    gen = torch.Generator(device=cuda).manual_seed(1)
    rm, keep, back = _sharded(torch.randn(n, F * k + 1, device=cuda, generator=gen), 1, 0)
    ffm = PSFieldAwareFactorizationMachine(_fake_table(rm, n, F * k + 1), F, k, push_scale=None)
    ids, fields, offsets, x = _batch(n, 300, F, gen)
    with torch.no_grad():
        ev = ffm(ids, fields, offsets, x)
    tr = ffm(ids, fields, offsets, x)
    assert ev.grad_fn is None and tr.grad_fn is not None and torch.equal(ev, tr.detach())
    ids2 = ids[:600].view(20, 30)                                  # 2-D bags equal 1-D bags with offsets
    f2 = fields[:600].view(20, 30)
    with torch.no_grad():
        assert torch.equal(ffm(ids2, f2), ffm(ids[:600], fields[:600], torch.arange(0, 600, 30, device=cuda)))


@pytest.mark.parametrize("updater", ["sgd", "adagrad", "rowwise_adagrad", "adam", "ftrl"])
def test_updaters_step_once_per_touched_row(mv_device, updater):
    """The real table after one backward equals a twin given the recorded coalesced gradient through add_rows;
    touched rows changed, untouched ones did not, and adam counted exactly one step per touched row."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    n, F, k, B, scale = 3000, 6, 8, 1024, 0.1
    C = F * k + 4
    kw = dict(min_value=-0.5, max_value=0.5, seed=11)
    t = mv.MatrixTable(n, C, "float32", updater=updater, **kw)
    twin = mv.MatrixTable(n, C, "float32", updater=updater, **kw)
    W0 = t.get().view(n, C).clone()
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    gen = torch.Generator(device="cuda").manual_seed(3)
    ids, fields, offsets, x = _batch(n, B, F, gen, long_bag=300)
    rm, keep, _ = _sharded(W0, 1, 0)
    rec, pushes = _fake_table(rm, n, C, N.UPD_ADAGRAD), []
    rec.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone()))
    PSFieldAwareFactorizationMachine(rec, F, k, push_scale=scale, option=opt)(ids, fields, offsets, x).mean() \
        .backward()
    PSFieldAwareFactorizationMachine(t, F, k, push_scale=scale, option=opt)(ids, fields, offsets, x).mean() \
        .backward()
    torch.cuda.synchronize()
    assert len(pushes) == 1
    uniq, grads = pushes[0]
    twin.wait(twin.add_rows_async(uniq, grads, opt))
    torch.cuda.synchronize()
    got = t.get().view(n, C)
    assert torch.equal(got, twin.get().view(n, C))
    touched = torch.zeros(n, dtype=torch.bool, device="cuda")
    touched[uniq] = True
    assert torch.equal(got[~touched], W0[~touched])
    assert ((got - W0).abs().max(1).values[touched] > 0).float().mean() > 0.9
    if updater == "adam":
        rows = t.my_len // t.num_col
        steps = t.state[1][t.state_stride:t.state_stride + rows]
        assert torch.equal(steps, touched.to(steps.dtype))


def _spread(n, seed):
    rng = np.random.default_rng(seed)
    return rng.choice(np.arange(1, 1 << 40, 7919), n, replace=False)


def test_hash_table_insert_eval_and_admission(mv_device):
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine
    from multiverso_b200.ops import field_aware_factorization_machine_reference as ref
    mv = mv_device
    F, k = 3, 4
    D = F * k
    kw = dict(num_fields=F, num_factors=k)
    # training mode inserts the missing keys; y is the FFM of the rows they got
    t = mv.HashMatrixTable(1000, D + 4, updater="sgd", min_value=-0.5, max_value=0.5, seed=3)
    keys = torch.tensor(_spread(300, 1), dtype=torch.int64, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(2)
    bags = keys[torch.randint(0, 300, (64, 8), device="cuda", generator=gen)]
    fields = torch.randint(0, F, (64, 8), device="cuda", generator=gen)
    ffm = PSFieldAwareFactorizationMachine(t, F, k, push_scale=0.1)
    y = ffm(bags, fields)
    uk, inv = torch.unique(bags, return_inverse=True)
    assert t.num_keys() == uk.numel()
    assert torch.allclose(y.double(), ref(t.get(uk), inv, fields, **kw), rtol=1e-5, atol=1e-5)
    y.sum().backward()
    # eval mode: new keys read the zero row and are not inserted; a backward after it raises
    known = uk[:20]
    before = t.get(known)
    new = torch.tensor(_spread(20, 9), dtype=torch.int64, device="cuda") + 3
    pairs = torch.stack([known, new], 1)                                       # bag b: (known b, new b)
    pf = torch.tensor([[0, 1]] * 20, device="cuda")
    ffm.eval()
    ye = ffm(pairs, pf)
    assert t.num_keys() == uk.numel()
    exp = ref(before, torch.arange(20, device="cuda")[:, None], pf[:, :1], **kw)
    assert torch.allclose(ye.double(), exp, rtol=0, atol=1e-6)
    with pytest.raises(RuntimeError, match="eval mode"):
        ye.sum().backward()
    with torch.no_grad():
        assert torch.equal(ffm(pairs, pf), ye.detach())
    assert torch.equal(t.get(known), before)
    # admit_after=3: keys seen fewer than 3 times add nothing to y and are not pushed; the zero row stays zero
    h = mv.HashMatrixTable(1000, D + 4, updater="sgd", admit_after=3, min_value=-0.5, max_value=0.5, seed=4)
    adm = torch.tensor(_spread(32, 5), dtype=torch.int64, device="cuda")
    for _ in range(4):
        h.lookup(adm)
    assert bool((h.lookup(adm, insert=False) != h.zero_row).all())
    fresh = torch.tensor(_spread(32, 6), dtype=torch.int64, device="cuda") + 1
    fa = PSFieldAwareFactorizationMachine(h, F, k, push_scale=0.5)
    w_adm = h.get(adm)
    yh = fa(torch.stack([adm, fresh, fresh.flip(0)], 1), torch.tensor([[0, 1, 2]] * 32, device="cuda"))
    assert bool((h.lookup(fresh, insert=False) == h.zero_row).all())
    exp = ref(w_adm, torch.arange(32, device="cuda")[:, None], torch.zeros(32, 1, dtype=torch.int64, device="cuda"),
              **kw)
    assert torch.allclose(yh.double(), exp, rtol=0, atol=1e-6)
    yh.sum().backward()
    torch.cuda.synchronize()
    assert bool((h.shard.view(-1, D + 4)[h.zero_row] == 0).all())
    # the admitted key's partners are zero rows: its factor gradient is 0, its linear weight moved by -0.5
    assert torch.allclose(h.get(adm)[:, D], w_adm[:, D] - 0.5, atol=1e-6)
    assert torch.equal(h.get(adm)[:, :D], w_adm[:, :D])


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


def test_host_syncs_and_empty_batch(mv_device):
    """1 per forward (the id, offset and field checks), 0 per sgd backward, 1 per compact (adagrad) backward; an
    empty batch after a full call pushes nothing."""
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine
    mv = mv_device
    n, F, k = 4000, 4, 4
    C = F * k + 4
    g = torch.Generator(device="cuda").manual_seed(6)
    ids, fields, offsets, x = _batch(n, 512, F, g, long_bag=50)
    for updater, want in (("sgd", 0), ("adagrad", 1)):
        t = mv.MatrixTable(n, C, "float32", updater=updater, min_value=-0.5, max_value=0.5)
        ffm = PSFieldAwareFactorizationMachine(t, F, k, push_scale=0.1)
        ffm(ids, fields, offsets, x).mean().backward()                 # warm-up
        out = []
        assert _syncs(lambda: out.append(ffm(ids, fields, offsets, x))) == 1
        assert _syncs(lambda: out[0].mean().backward()) == want, updater
        torch.cuda.synchronize()
        before = t.get().clone()
        e = torch.zeros(0, dtype=torch.int64, device="cuda")
        y = ffm(e, e, e)
        assert y.shape == (0,)
        y.sum().backward()
        y = ffm(e, e, torch.zeros(4, dtype=torch.int64, device="cuda"))   # four empty bags
        assert torch.equal(y, torch.zeros(4, device="cuda"))
        y.sum().backward()
        torch.cuda.synchronize()
        assert torch.equal(t.get(), before), updater


def test_planted_ffm_trains_to_the_planted_log_loss(cuda):
    """Labels drawn from a planted FFM (F = 4 fields, k = 4, 200 Zipf ids, bags of 8 with fields 0..3 twice, linear
    weights ~ N(0, 0.5^2), factors ~ N(0, 0.3^2)): PSFieldAwareFactorizationMachine + sgd (lr 1, mean loss, 1500
    steps of 2048 bags, start uniform in +-0.1) reaches, on fresh data, a log-loss within 0.05 nats of the planted
    model's own (~0.5). An fp32 torch simulation of the same schedule on the CPU ends 0.024 above it: what remains
    is the noise of SGD at this step size and the fit of 3400 parameters to noisy labels. The untrained start is
    ~0.17 above it."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine, field_aware_factorization_machine_reference
    n, F, k, BAG, B = 200, 4, 4, 8, 2048
    D = F * k
    C = D + 1
    gen = torch.Generator(device="cuda").manual_seed(0)
    Wp = torch.cat([torch.randn(n, D, device="cuda", generator=gen) * 0.3,
                    torch.randn(n, 1, device="cuda", generator=gen) * 0.5], 1)
    # C = 17 has a row pitch of 20: a table over an explicit row map, pushed to by the fused sgd red.add
    W0 = (torch.rand(n, C, device="cuda", generator=gen) - 0.5) * 0.2
    rm, buf, _ = _sharded(W0, 1, 0)
    ffm = PSFieldAwareFactorizationMachine(_fake_table(rm, n, C, N.UPD_SGD), F, k, push_scale=1.0)
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    fields = (torch.arange(BAG, device="cuda") % F).repeat(1, 1)

    def batch(b):
        ids = _zipf_ids(n, b * BAG, gen).view(b, BAG)
        f = fields.expand(b, BAG)
        ys = field_aware_factorization_machine_reference(Wp, ids, f, num_fields=F, num_factors=k).float()
        return ids, f, (torch.rand(b, device="cuda", generator=gen) < torch.sigmoid(ys)).float(), ys

    def evaluate():
        ids, f, lab, ys = batch(65536)
        with torch.no_grad():
            return bce(ffm(ids, f), lab).item(), bce(ys, lab).item()

    start, floor = evaluate()
    for _ in range(1500):
        ids, f, lab, _ = batch(B)
        bce(ffm(ids, f), lab).backward()
    end, floor2 = evaluate()
    print(f"planted FFM: start {start:.4f} end {end:.4f} planted {floor:.4f} / {floor2:.4f}")
    assert start > floor + 0.12, (start, floor)
    assert end < floor2 + 0.05, (end, floor2)


def _ffm_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "ffm_fwd_kernel" in e.name)


def test_errors_raise_without_launching(cuda):
    """Every refusal of the layer and every return code of mvb_ffm_fwd raises before any launch. Two profiler
    sessions do the counting: the op first (seen as one kernel), then every error case in one session (none). A valid
    direct call is checked by what it writes: in a process that has run the rest of the GPU suite, a profiler session
    holding only a few launches can come back without their kernel records (the launches and their results are
    there), so a launch count is not asked of such a session."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSFieldAwareFactorizationMachine as FFM
    n, F, k = 1000, 3, 8
    C = F * k + 4
    W = torch.randn(n, C, device=cuda)
    rm, keep, _ = _sharded(W, 1, 0)
    t = _fake_table(rm, n, C, N.UPD_ADAGRAD)
    t.add_rows_async = lambda ids, vals, option=None: None
    ffm = FFM(t, F, k)
    ids = torch.arange(8, device=cuda)
    fields = torch.tensor([0, 1, 2, 0, 1, 2, 0, 1], device=cuda)
    offs = torch.tensor([0, 3], device=cuda)
    x = torch.rand(8, device=cuda)
    fi = fields.int()
    y = torch.empty(2, device=cuda)
    ldh = F * k + 4
    h = torch.empty(8, ldh, device=cuda)

    def args(**kw):
        a = N.Ffm()
        a.wmap, a.F, a.k = rm, F, k
        a.ids, a.fields, a.values, a.offsets = ids.data_ptr(), fi.data_ptr(), x.data_ptr(), offs.data_ptr()
        a.L, a.B, a.y, a.h, a.ldh = 8, 2, y.data_ptr(), h.data_ptr(), ldh
        for key, val in kw.items():
            if key == "shard0":
                a.wmap.shard_ptrs[0] = val
            elif key.startswith("map_"):
                setattr(a.wmap, key[4:], val)
            else:
                setattr(a, key, val)
        return a
    lib = N.cuda_lib()
    ffm(ids, fields, offs, x).sum().backward()                   # warm-up of the op
    assert _ffm_kernels(lambda: ffm(ids, fields, offs, x).sum().backward()) == 1       # the counter sees the op
    y.fill_(float("nan"))
    lib.mvb_ffm_fwd(args(), N.stream_ptr())                      # a valid direct call runs: it writes y
    with torch.no_grad():
        assert torch.equal(y, ffm(ids, fields, offs, x))
    layer_cases = [
        (ValueError, r"\[0, 1000\), got min 0 max 1000", (torch.tensor([0, 1, 2, 1000], device=cuda), fields[:4],
                                                          offs[:1], None)),
        (ValueError, r"fields must be in \[0, 3\), got min 1 max 3", (ids, fields + 1, offs, None)),
        (ValueError, r"fields must be in \[0, 3\), got min -1", (ids, fields - 1, offs, None)),
        (TypeError, "fields must be integers", (ids, fields.float(), offs, None)),
        (ValueError, "fields must have the shape of ids", (ids, fields[:7], offs, None)),
        (TypeError, "int32 or int64", (ids.float(), fields, offs, None)),
        (ValueError, "must start at 0", (ids, fields, offs + 1, None)),
        (ValueError, "non-decreasing", (ids, fields, torch.tensor([0, 5, 3], device=cuda), None)),
        (ValueError, "exceed the number of ids", (ids, fields, torch.tensor([0, 9], device=cuda), None)),
        (ValueError, "values must have the shape of ids", (ids, fields, offs, x[:7])),
        (TypeError, "floating point", (ids, fields, offs, torch.ones(8, dtype=torch.int64, device=cuda))),
        (ValueError, "get no gradient", (ids, fields, offs, x.clone().requires_grad_())),
    ]
    codes = [(N.BAD_ROW_MAP, dict(map_nservers=0)), (N.BAD_ROW_MAP, dict(map_nservers=9)),
             (N.BAD_ROW_MAP, dict(map_rows_per_server=0)),
             (-95, dict(k=0)), (-95, dict(k=6)), (-95, dict(k=-4)), (-95, dict(F=0)), (-95, dict(F=256, k=4)),
             (-95, dict(F=1, k=1024)),
             (-96, dict(map_num_col=24)), (-96, dict(map_num_col=26)), (-96, dict(shard0=W.data_ptr() + 4)),
             (-97, dict(B=-1)), (-97, dict(L=-1)),
             (-98, dict(offsets=None)), (-98, dict(y=None)), (-98, dict(ids=None)), (-98, dict(fields=None)),
             (-99, dict(ldh=26)), (-99, dict(ldh=24)), (-99, dict(h=h.data_ptr() + 4))]
    a0 = args(B=0, L=0)

    def every_error():
        for exc, msg, call_args in layer_cases:
            with pytest.raises(exc, match=msg):
                ffm(*call_args)
        for rc, kw in codes:
            with pytest.raises(N.NativeError, match=f"rc={rc}:"):
                lib.mvb_ffm_fwd(args(**kw), N.stream_ptr())
        lib.mvb_ffm_fwd(a0, N.stream_ptr())                      # B == 0 launches nothing
    assert _ffm_kernels(every_error) == 0
    # the layer's refusals of the table
    with pytest.raises(TypeError, match="MatrixTable"):
        FFM(W, F, k)
    with pytest.raises(TypeError, match="float32"):
        FFM(types.SimpleNamespace(**{**vars(t), "dtype": torch.float64}), F, k)
    with pytest.raises(ValueError, match="at least"):
        FFM(_fake_table(rm, n, F * k), F, k)
    with pytest.raises(ValueError, match="multiple of 4"):
        FFM(t, F, 6)
    rm6 = N.RowMap()
    rm6.num_row, rm6.num_col, rm6.nservers, rm6.rows_per_server = n, 30, 1, n
    rm6.shard_ptrs[0] = W.data_ptr()
    with pytest.raises(ValueError, match="row pitch"):
        FFM(_fake_table(rm6, n, 28), F, k)


def test_field_aware_factorization_machine_peer_shards_multi_gpu():
    """A table sharded over 2 GPUs (tests/mp_field_aware_factorization_machine_check.py under torchrun): the forward
    bitwise equal to a single-shard copy, async sgd pushes from every rank landing as W0 - lr * sum."""
    import os
    import subprocess
    import sys
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 1400
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_field_aware_factorization_machine_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == 2, tail
