"""The embedding-bag kernels (csrc/cuda/emb_bag.cuh, emb_bag.cu, emb_bag_coll.cu) against float64, at their register
class, chunk, segment and push-bound edges, with every byte of the table checked after each call.

Tables sit in a row pitch wider than their dim (4 to 7 padding columns), as shards of one buffer with gap rows before,
between and after them. Padding and gap cells hold a NaN with a payload (``SENTINEL``): a kernel that reads one makes a
dot product or a sum NaN, and one that writes it, even by adding zero, leaves the canonical NaN there instead. After
each call the whole buffer is read back: padding, gap rows and rows no lookup touched keep their bits exactly.

Two arms of data:

* exact: small-integer rows and dout, per-sample weights in {0.5, 1, 2}, and in the backward, bag lengths that are
  powers of two so that ``1 / len`` is exact. Every term is then a multiple of ``q`` (1, 1/2 with weights, 1 / the
  longest bag for a mean) and every sum of ``|terms|``, pushed row included, stays below ``2^24`` times its grain
  (asserted), so every fp32 partial sum is exact in any order: the forward, the
  pushed rows, the compact ``grads`` / ``uniq`` / unique count and ``dpsw`` equal the float64 result rounded to fp32,
  bit for bit. For a mean forward that is the exact sum divided in float64 and rounded (division rounds correctly,
  and float64 is wide enough for the double rounding to be innocuous). This arm sees a dropped, repeated or misranked
  piece however small it is.
* random: Gaussian data, checked against a bound derived from the documented summation order (``u = 2^-24``,
  ``gamma(n) = n u / (1 - n u)``):

  - backward: a row's gradient is an fp32 fma chain over each piece of its run (``n_r`` lookups in all), the pieces
    of a run that crosses chunks added in chunk order (``k_r`` pieces), and ``s = psw / len`` is rounded once. So
    ``|g - G| <= gamma(n_r + k_r + 1) M_r`` with ``M_r = sum |psw s_bag dout|`` over the run. The push adds
    ``fl(scale g)`` to the row in one fp32 add: ``|row' - (row + scale G)| <= |scale| gamma(n_r + k_r + 2) M_r +
    2 u |row + scale G|``; compact ``grads`` the same without the row.
  - forward: lane group ``g`` sums lookups ``g, g + NG, ...`` of the bag by an fp32 fma chain, the groups are combined
    by a butterfly of at most 5 adds and a mean divides once: ``|out - O| <= gamma(len + 6) sum |psw W| / len``.
  - ``dpsw``: per-lane fma chains over the row, 5 butterfly adds and one division:
    ``|dpsw - D| <= gamma(dim + 6) s_bag sum |dout W|``.

Chunk layouts are built on purpose: lookups sort by (id, position), so the per-id counts alone decide where each run
falls in sorted order. The layout tests (no GPU) check that every case really puts its runs where it says."""
import types

import pytest
import torch

CHUNK = 256                               # EMB_CHUNK: sorted lookups per backward warp
SENTINEL = 0x7FD1CE5D                     # a quiet NaN with a payload
U = 2.0 ** -24

# ------------------------------------------------------------------------------------------------ chunk layouts
# run lengths, in id order, and what the case claims about where its runs fall in sorted order
EDGES = [1, 255, 256, 257, 1, 3, 227, 600, 1000, 2100, 164, 1025, 1, 1022, 512] + [1] * 37


def _big(L, seed=7):
    """L lookups in 1024 or more chunks: one run over hundreds of chunks, the edge lengths, Zipf-like short runs."""
    head = [100_000, 1, 255, 256, 257, 2100]
    return head + _fill(L - sum(head), torch.Generator().manual_seed(seed))


def _fill(n, g, longest=60):
    """Run lengths of 1 .. longest - 1 that sum to n."""
    ends = torch.cumsum(torch.randint(1, longest, (n + 1,), generator=g), 0)
    ends = torch.cat([ends[ends < n], torch.tensor([n])]) if n else ends[:0]
    return torch.diff(ends, prepend=torch.tensor([0])).tolist()


CASES = {
    "edges": (EDGES, {"len1", "len255", "len256", "len257", "start_edge", "end_edge", "span2", "span4", "span5",
                      "span9", "middle", "head_whole_tail"}),
    "L1": ([1], {"len1", "chunks1"}),
    "L255": ([1, 200, 54], {"len1", "chunks1"}),
    "L256": ([3, 253], {"chunks1"}),
    "L257": ([2, 255], {"len255", "span2", "chunks2"}),
    "L262144": (_big(1024 * 256), {"len1", "len255", "len256", "len257", "span9", "middle", "chunks1024"}),
    "L262145": (_big(1024 * 256) + [1], {"len1", "len255", "len256", "len257", "span9", "middle", "chunks1025"}),
}


def _layout(counts, seed=0):
    """ids with counts[k] lookups of row 2 k + 1 (even rows are never looked up), positions shuffled: the stable sort
    puts run k at sorted positions [sum(counts[:k]), sum(counts[:k + 1]))."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.repeat_interleave(2 * torch.arange(len(counts)) + 1, torch.tensor(counts, dtype=torch.int64))
    return ids[torch.randperm(ids.numel(), generator=g)]


def _runs(ids):
    """(row, first sorted position, end) of every run of the stable sort of ids."""
    sid = torch.sort(ids.cpu(), stable=True).values
    rows, n = torch.unique_consecutive(sid, return_counts=True)
    end = torch.cumsum(n, 0)
    return rows, end - n, end


def _claims(ids):
    """What the sorted ids of one segment actually show."""
    rows, s, e = _runs(ids)
    L, n = ids.numel(), e - s
    span = (e - 1) // CHUNK - s // CHUNK + 1
    out = {f"len{k}" for k in (1, 255, 256, 257) if (n == k).any()}
    out |= {f"span{k}" for k in (2, 4, 5, 9) if (span == k).any()}
    out.add(f"chunks{(L + CHUNK - 1) // CHUNK}")
    if ((s % CHUNK == 0) & (s > 0)).any():
        out.add("start_edge")
    if ((e % CHUNK == 0) & (e < L)).any():
        out.add("end_edge")
    for c in range((L + CHUNK - 1) // CHUNK):
        c0, c1 = c * CHUNK, min((c + 1) * CHUNK, L)
        if ((s < c0) & (e > c1) & (c1 < L)).any():
            out.add("middle")                            # the chunk is the middle of one run
        head = ((s < c0) & (e > c0) & (e < c1)).any()     # a run continues into the chunk and ends in it
        whole = ((s >= c0) & (e <= c1) & (s > c0)).any()
        tail = ((s > c0) & (s < c1) & (e > c1)).any()     # a run starts in the chunk and goes on
        if head and whole and tail:
            out.add("head_whole_tail")
    return out


@pytest.mark.parametrize("case", sorted(CASES))
def test_layout_places_runs(case):
    counts, claims = CASES[case]
    ids = _layout(counts, seed=len(case))
    rows, s, e = _runs(ids)
    assert rows.tolist() == [2 * k + 1 for k in range(len(counts))]
    assert (e - s).tolist() == counts
    assert claims <= _claims(ids), claims - _claims(ids)


def _pow2_lengths(n, B, g, maxlen=64):
    """B bag lengths that sum to n, each 0 or a power of two <= maxlen, in random order: random powers of two while
    they fit, then the binary digits of what is left, then empty bags."""
    lens = 2 ** torch.randint(0, maxlen.bit_length(), (n,), generator=g)
    lens = lens[torch.cumsum(lens, 0) <= n].tolist()
    rest = n - sum(lens)
    lens += [1 << k for k in range(rest.bit_length()) if rest >> k & 1]
    assert len(lens) < B, (n, B)
    lens = torch.tensor(lens + [0] * (B - len(lens)), dtype=torch.int64)
    return lens[torch.randperm(B, generator=g)]


def _any_lengths(n, B, g):
    return torch.bincount(torch.randint(0, B, (n,), generator=g), minlength=B)


def test_pow2_lengths():
    g = torch.Generator().manual_seed(1)
    for n, B in ((1, 3), (255, 40), (7461, 1000), (262145, 16384)):
        lens = _pow2_lengths(n, B, g)
        nz = lens[lens > 0]
        assert lens.numel() == B and int(lens.sum()) == n and (lens == 0).any()
        assert ((nz & (nz - 1)) == 0).all() and int(nz.max()) <= 64


# ------------------------------------------------------------------------------------------------ GPU helpers
def gamma(n):
    return n * U / (1 - n * U)


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


class _Buf:
    """V x dim rows W in a row pitch of round4(dim) + 4 floats, as S shards of one buffer with `gap` SENTINEL rows
    before, between and after them; every cell that is not one of a row's dim columns holds SENTINEL."""

    def __init__(self, W, S=1, gap=3):
        from multiverso_b200 import _native as N
        V, dim = W.shape
        self.dim, self.pitch = dim, (dim + 3) // 4 * 4 + 4
        rps = max(V // S, 1)
        shard = torch.clamp(torch.arange(V) // rps, max=S - 1)
        self.pos = (torch.arange(V) + (shard + 1) * gap).to(W.device)
        self.buf = torch.full((V + (S + 1) * gap, self.pitch), SENTINEL, dtype=torch.int32,
                              device=W.device).view(torch.float32)
        self.buf[self.pos, :dim] = W
        self.init = self.buf.clone()
        self.rm = rm = N.RowMap()
        rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = V, self.pitch, S, rps
        for k in range(S):
            rm.shard_ptrs[k] = self.buf[k * rps + (k + 1) * gap].data_ptr()

    def rows(self):
        return self.buf[self.pos, :self.dim]

    def check(self, rows, what):
        """Rows [V, dim] expected in the table; every other cell keeps its bits."""
        exp = self.init.clone()
        exp[self.pos, :self.dim] = rows
        same = (self.buf == exp) | (self.buf.view(torch.int32) == exp.view(torch.int32))
        if not same.all():
            bad = (~same).nonzero()[:5].tolist()
            raise AssertionError(f"{what}: {int((~same).sum())} cells differ, first [buffer row, col] {bad}")


def _rows_of(lens):
    """The bag of every lookup."""
    return torch.repeat_interleave(torch.arange(lens.numel(), device=lens.device), lens)


def _fwd_ref(W64, ids, lens, psw, mean):
    """(float64 bags, sum of |terms| per element) of the forward."""
    bag = _rows_of(lens)
    t = W64[ids] * (psw.double()[:, None] if psw is not None else 1.0)
    out = torch.zeros(lens.numel(), W64.shape[1], dtype=torch.float64, device=W64.device).index_add_(0, bag, t)
    mag = torch.zeros_like(out).index_add_(0, bag, t.abs())
    if mean:
        d = lens.clamp_min(1).double()[:, None]
        out, mag = out / d, mag / d
    return out, mag


def _grad_ref(V, ids, s, drows):
    """(float64 gradient G, M = sum |terms|, n_r + k_r) of every row: s the scale of each lookup, drows its dout row."""
    t = s[:, None] * drows
    G = torch.zeros(V, drows.shape[1], dtype=torch.float64, device=drows.device).index_add_(0, ids, t)
    M = torch.zeros_like(G).index_add_(0, ids, t.abs())
    rows, a, e = _runs(ids)
    k = torch.zeros(V, dtype=torch.float64)
    k[rows] = ((e - a) + (e - 1) // CHUNK - a // CHUNK + 1).double()
    return G, M, k.to(drows.device)[:, None]


def _data(exact, shape, g, dev):
    if exact:
        return torch.randint(-8, 9, shape, generator=g).float().to(dev)
    return torch.randn(shape, generator=g).to(dev)


def _psw(exact, n, g, dev):
    if exact:
        return torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (n,), generator=g)].to(dev)
    return torch.randn(n, generator=g).to(dev)


def _expect(got, ref, err, what):
    """got (fp32) against the float64 ref: exactly its rounding when err is None, else within err."""
    if err is None:
        exp = ref.float()
        ok = got == exp
        if not ok.all():
            i = (~ok).nonzero()[0].tolist()
            raise AssertionError(f"{what}: {int((~ok).sum())} values differ, first at {i}: {got[tuple(i)].item()!r} "
                                 f"vs {exp[tuple(i)].item()!r}")
    else:
        d = (got.double() - ref).abs()
        ok = d <= err
        if not ok.all():
            raise AssertionError(f"{what}: {int((~ok).sum())} values out of bound, worst {(d / err).max().item():.3g}x")


def _assert_exact(G, M, W, psw, mean_lens):
    """The exact arm's premise: gradient sums and pushed rows (scale +-0.5) are exact in fp32."""
    q = (0.5 if psw is not None else 1.0) / (int(mean_lens.max()) if mean_lens is not None else 1)
    assert M.max().item() < 2 ** 24 * q and (W.abs().max() + 0.5 * M.max()).item() < 2 ** 23 * q, \
        "the exact arm's sums would round"


class _Capture(types.SimpleNamespace):
    """A table handle whose compact pushes are recorded instead of applied."""

    def add_rows_async(self, uniq, grads, option=None):
        self.pushed.append((uniq.clone(), grads.clone()))


# ------------------------------------------------------------------------------------------------ single table
DIMS = [1, 2, 3, 4, 20, 30, 32, 36, 128, 132, 256, 260, 384, 388, 512, 516, 1000, 2052]
MODES = [("sum", False), ("sum", True), ("mean", False)]


def _fwd_lengths(dim, g):
    """Bag lengths around the 32-lookup windows and the lane groups' in-flight groups of 4 NG, and empty bags."""
    nv = (dim + 3) // 4
    lg = 0
    while (1 << lg) < nv and lg < 5:
        lg += 1
    ng = 32 >> lg
    base = [0, 1, 31, 32, 33, 4 * ng - 1, 4 * ng, 4 * ng + 1, 0, 2, 63, 64, 65, 97, 0, 5]
    extra = torch.randint(0, 70, (48,), generator=g).tolist()
    return torch.tensor(base + extra)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", DIMS)
def test_forward(cuda, dim):
    from multiverso_b200.ops.embedding import _fwd_device
    g = torch.Generator().manual_seed(dim)
    V = 1500
    lens = _fwd_lengths(dim, g).to(cuda)
    L = int(lens.sum())
    offsets = torch.cumsum(lens, 0) - lens
    for exact in (True, False):
        W = _data(exact, (V, dim), g, cuda)
        tab = _Buf(W, S=3)
        ids = torch.randint(0, V, (L,), generator=g).to(cuda)
        for mode, weighted in MODES:
            psw = _psw(exact, L, g, cuda) if weighted else None
            out = _fwd_device(tab.rm, dim, ids, offsets, psw, mode)
            ref, mag = _fwd_ref(W.double(), ids, lens, psw, mode == "mean")
            _expect(out, ref, None if exact else gamma(lens.double()[:, None] + 6) * mag,
                    f"forward dim {dim} {mode} psw={weighted} exact={exact}")
            tab.check(W, "forward")


def _bwd_case(tab, W, dim, ids, lens, psw, mode, dout, exact, what, push_rows=0):
    """One backward over the table of _Buf tab through each epilogue, against float64: the pushed rows (sgd and
    default updaters: scale -0.5 and 0.5) and the compact grads / uniq (whose count is the count-only call's).
    push_rows: the bound the table handles carry (read when the test patches _push_rows to return it)."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import embedding
    V = W.shape[0]
    offsets = torch.cumsum(lens, 0) - lens
    bag = _rows_of(lens)
    s = psw.double() if psw is not None else torch.ones(ids.numel(), dtype=torch.float64, device=ids.device)
    if mode == "mean":
        s = s / lens[bag].double()
    G, M, k = _grad_ref(V, ids, s, dout.double()[bag])
    below = torch.arange(V, device=ids.device) < (push_rows if push_rows > 0 else V)
    looked = torch.zeros(V, dtype=torch.bool, device=ids.device)
    looked[ids] = True
    pushed = looked & below
    if exact:
        _assert_exact(G, M, W, psw, lens if mode == "mean" else None)
    for upd in (N.UPD_SGD, N.UPD_DEFAULT):
        scale = -0.5 if upd == N.UPD_SGD else 0.5
        exp = W.double() + scale * G * pushed[:, None]
        table = types.SimpleNamespace(updater=upd, is_sparse=False, num_col=tab.pitch, push_rows=push_rows)
        embedding._push_device(table, tab.rm, dim, ids, offsets, psw, mode, dout, 0.5, None)
        torch.cuda.synchronize()
        if exact:
            tab.check(exp.float(), f"{what} push scale {scale}")
        else:
            got = tab.rows()
            err = 0.5 * gamma(k + 2) * M + 2 * U * exp.abs()
            _expect(got[pushed], exp[pushed], err[pushed], f"{what} push scale {scale}")
            tab.check(torch.where(pushed[:, None], got, W), f"{what} push scale {scale}")
        tab.buf.copy_(tab.init)
    cap = _Capture(updater=N.UPD_ADAGRAD, is_sparse=False, num_col=tab.pitch, push_rows=push_rows, pushed=[])
    embedding._push_device(cap, tab.rm, dim, ids, offsets, psw, mode, dout, 0.5, None)
    torch.cuda.synchronize()
    tab.check(W, f"{what} compact")
    (uniq, grads), = cap.pushed
    want = pushed.nonzero().view(-1)
    assert torch.equal(uniq, want), f"{what}: compact uniq / unique count"
    assert grads.shape == (want.numel(), tab.pitch)
    assert (grads[:, dim:].view(torch.int32) == 0).all(), f"{what}: compact grads past dim"
    _expect(grads[:, :dim], 0.5 * G[want], None if exact else 0.5 * gamma(k[want] + 1) * M[want] + U * 0.5 *
            G[want].abs(), f"{what} compact grads")


def _dpsw_case(tab, W, dim, ids, lens, mode, dout, exact, what):
    from multiverso_b200.ops.embedding import _psw_grad_device
    offsets = torch.cumsum(lens, 0) - lens
    bag = _rows_of(lens)
    got = _psw_grad_device(tab.rm, dim, ids, offsets, mode, dout)
    t = dout.double()[bag] * W.double()[ids]
    ref, mag = t.sum(1), t.abs().sum(1)
    if mode == "mean":
        ref, mag = ref / lens[bag].double(), mag / lens[bag].double()
    _expect(got, ref, None if exact else gamma(dim + 6) * mag, f"{what} dpsw")
    tab.check(W, f"{what} dpsw")


def _single_backward(cuda, dim, case, seed, S=3):
    counts, _ = CASES[case]
    g = torch.Generator().manual_seed(seed)
    ids = _layout(counts, seed).to(cuda)
    L, V = ids.numel(), 2 * len(counts) + 3
    B = max(L // 8, 3)
    for exact in (True, False):
        W = _data(exact, (V, dim), g, cuda)
        tab = _Buf(W, S=S)
        lens = (_pow2_lengths(L, B, g) if exact else _any_lengths(L, B, g)).to(cuda)
        dout = _data(exact, (B, dim), g, cuda)
        for mode, weighted in MODES:
            psw = _psw(exact, L, g, cuda) if weighted else None
            what = f"{case} dim {dim} {mode} psw={weighted} exact={exact}"
            _bwd_case(tab, W, dim, ids, lens, psw, mode, dout, exact, what)
            _dpsw_case(tab, W, dim, ids, lens, mode, dout, exact, what)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", DIMS)
def test_backward_dims(cuda, dim):
    """Every register class and column slab over the chunk-edge layout: push, compact and dpsw."""
    _single_backward(cuda, dim, "edges", dim)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["L1", "L255", "L256", "L257", "L262144", "L262145"])
@pytest.mark.parametrize("dim", [3, 132])
def test_backward_lengths(cuda, case, dim):
    """Segments of 1, 255, 256 and 257 lookups, and of 1024 and 1025 chunks (the scan takes two chunks per thread)."""
    _single_backward(cuda, dim, case, dim + len(case), S=1 if case.startswith("L2621") else 2)


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [3, 132])
def test_backward_push_rows(cuda, monkeypatch, dim):
    """Rows at or above push_rows get no epilogue: they keep their bits, are not counted and shift no other rank.
    The bound falls inside a chunk, above a run that spans 9 chunks and below one that spans 5."""
    from multiverso_b200.ops import embedding
    monkeypatch.setattr(embedding, "_push_rows", lambda table: table.push_rows)
    g = torch.Generator().manual_seed(dim)
    ids = _layout(EDGES, 3).to(cuda)
    L, V = ids.numel(), 2 * len(EDGES) + 3
    bound = 2 * 10 + 1                    # runs 10 (row 21) and up are not pushed; run 9 spans 9 chunks
    B = L // 8
    W = _data(True, (V, dim), g, cuda)
    tab = _Buf(W, S=3)
    lens = _pow2_lengths(L, B, g).to(cuda)
    dout = _data(True, (B, dim), g, cuda)
    for mode, weighted in MODES:
        psw = _psw(True, L, g, cuda) if weighted else None
        _bwd_case(tab, W, dim, ids, lens, psw, mode, dout, True, f"push_rows dim {dim} {mode} psw={weighted}",
                  push_rows=bound)


# ------------------------------------------------------------------------------------------------ collection
# (dim, epilogue, features, lookups, leading run lengths, push bound as a run index or None). Lookups per table are
# 0, 1 or 255 mod 256, so every table's chunk numbering starts at an odd place; table 2 has none between two that
# have some; table 0's two features sit at dout columns 0 and 30 and table 1's at 60 (dims 30 and 3: the padded
# dout path); push and compact tables share the call, and every register class (dims up to 512) is present.
COLL = [
    (30, "sgd", ["a0", "a1"], 769, [300, 255], 1),
    (3, "default", ["b"], 255, [100], None),
    (1, "sgd", ["c"], 0, [], None),
    (36, "compact", ["d"], 512, [257], 1),
    (132, "default", ["e"], 1025, [600, 1], None),
    (260, "compact", ["f0", "f1"], 767, [400], 1),
    (388, "sgd", ["h"], 768, [256, 256], 1),
    (512, "compact", ["i"], 513, [300], None),
    (20, "default", ["j"], 511, [5], None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
def test_collection(cuda, monkeypatch, weighted, exact, bounded):
    """PSEmbeddingCollection over fake table handles: forward, every table's pushed rows or compact grads / uniq and
    dpsw against float64 over its features' bags stacked in feature order. bounded: four tables carry their own
    push_rows."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import EmbeddingBagConfig, PSEmbeddingCollection, embedding_collection
    monkeypatch.setattr(embedding_collection, "_push_rows", lambda table: table.push_rows)
    g = torch.Generator().manual_seed(4 * weighted + 2 * exact + bounded)
    B = 128
    upd = {"sgd": N.UPD_SGD, "default": N.UPD_DEFAULT, "compact": N.UPD_ADAGRAD}
    tabs, cfgs, feats = [], [], []                   # feats: (table, ids, lengths) in feature order
    for t, (dim, kind, names, n, head, run) in enumerate(COLL):
        counts = head + _fill(n - sum(head), g, 20)
        ids = _layout(counts, t)
        V = 2 * len(counts) + 3
        W = _data(exact, (V, dim), g, cuda)
        tab = _Buf(W, S=1 + t % 3)
        bound = 2 * run + 1 if bounded and run is not None else 0
        handle = _Capture(_rowmap=tab.rm, dtype=torch.float32, num_row=V, num_col=dim, updater=upd[kind],
                          is_sparse=False, rt=types.SimpleNamespace(device=cuda), push_rows=bound, pushed=[])
        mode = "mean" if t % 2 and not weighted else "sum"
        cfgs.append(EmbeddingBagConfig(handle, names, push_scale=0.5, mode=mode))
        cut = n // len(names)
        for k in range(len(names)):
            part = ids[k * cut:(k + 1) * cut if k + 1 < len(names) else n].to(cuda)
            lens = (_pow2_lengths if exact else _any_lengths)(part.numel(), B, g).to(cuda)
            feats.append((t, part, lens))
        tabs.append((tab, W, handle, mode, bound))
    ebc = PSEmbeddingCollection(cfgs)
    ids = torch.cat([f[1] for f in feats])
    lengths = torch.stack([f[2] for f in feats])
    psw = _psw(exact, ids.numel(), g, cuda).requires_grad_() if weighted else None
    dout = _data(exact, (B, ebc.out_dim), g, cuda)
    out = ebc(ids, lengths, psw)
    out.backward(dout)
    torch.cuda.synchronize()
    starts = [0] + torch.cumsum(lengths.sum(1), 0).tolist()
    for t, (tab, W, handle, mode, bound) in enumerate(tabs):
        dim, kind = COLL[t][0], COLL[t][1]
        what = f"table {t} (dim {dim}, {kind}, {mode}, psw={weighted}, exact={exact}, push_rows={bound})"
        V, mean = W.shape[0], mode == "mean"
        tids, s_all, drows = [], [], []
        for f, (tt, part, lens) in enumerate(feats):
            if tt != t:
                continue
            p = None if psw is None else psw.detach()[starts[f]:starts[f + 1]]
            col = ebc.cols[f]
            ref, mag = _fwd_ref(W.double(), part, lens, p, mean)
            _expect(out.detach()[:, col:col + dim], ref, None if exact else gamma(lens.double()[:, None] + 6) * mag,
                    f"{what} forward of {ebc.feature_names[f]}")
            bag = _rows_of(lens)
            d = dout.double()[:, col:col + dim][bag]
            s = p.double() if p is not None else torch.ones(part.numel(), dtype=torch.float64, device=cuda)
            if weighted:
                tt_ = d * W.double()[part]
                _expect(psw.grad[starts[f]:starts[f + 1]], tt_.sum(1), None if exact else
                        gamma(dim + 6) * tt_.abs().sum(1), f"{what} dpsw of {ebc.feature_names[f]}")
            tids.append(part)
            s_all.append(s / lens[bag].double() if mean else s)
            drows.append(d)
        tids = torch.cat(tids)
        if not tids.numel():
            assert not handle.pushed
            tab.check(W, what)
            continue
        G, M, k = _grad_ref(V, tids, torch.cat(s_all), torch.cat(drows))
        pushed = torch.zeros(V, dtype=torch.bool, device=cuda)
        pushed[tids] = True
        if bound:
            pushed[bound:] = False
        if exact:
            _assert_exact(G, M, W, psw, lengths.max() if mean else None)
        if kind == "compact":
            tab.check(W, what)
            (uniq, grads), = handle.pushed
            want = pushed.nonzero().view(-1)
            assert torch.equal(uniq, want), f"{what}: compact uniq / unique count"
            _expect(grads, 0.5 * G[want], None if exact else
                    0.5 * gamma(k[want] + 1) * M[want] + U * 0.5 * G[want].abs(), f"{what} compact grads")
            continue
        scale = -0.5 if kind == "sgd" else 0.5
        exp = W.double() + scale * G * pushed[:, None]
        if exact:
            tab.check(exp.float(), what)
        else:
            got = tab.rows()
            err = 0.5 * gamma(k + 2) * M + 2 * U * exp.abs()
            _expect(got[pushed], exp[pushed], err[pushed], f"{what} push")
            tab.check(torch.where(pushed[:, None], got, W), what)
