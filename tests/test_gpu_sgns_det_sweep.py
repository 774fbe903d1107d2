"""The deterministic skip-gram kernel (`mvb_sgns_train_det`) against the fp64 model of its wave schedule
(tests/sgns_det_model.py) over every shape it dispatches on.

Every case calls the kernel directly, takes its wave size from `mvb_sgns_win_inflight(dim, K, W)` and its slice
length S from the same rule as the host code, so no case depends on the SM count.  Each case checks:

  tables     the relative Frobenius error of each table's delta < 1e-4 (the bound of the other tests of this
             kernel: fp32 dots and products of order 2^-24 per pair, fast sigmoid, 2^-40 fixed-point sums);
  pairs      the pair count is exact;
  loss       within 1e-5 relative.  Each loss term is 8 softplus(-+f) from __expf and log1pf (a few ulp, u = 2^-24,
             against f's own error of about sqrt(dim) u |h||o|, far below); a sampled centre sums at most
             (1 + K) * 2W <= 8 (2W + 1) positive terms in fp32, which is off by at most (n - 1) u = 1.5e-5 if every
             rounding of every centre went the same way, and by about sqrt(n) u ~ 1e-6 in fact, since the errors of
             hundreds of centres are independent and of either sign; each centre's sum is then rounded to 2^-32
             (under 1e-9 of a centre's loss of 8 (2 + 2K) log 2 or so) and each wave's sum is rounded once to fp32
             and added to an fp32 total (2u per wave, 3-5 waves here);
  bits       rows no wave read, the padding columns [dim, ld) and 64 guard cells on each side of each table keep
             their bits: they hold a NaN with a payload, which a kernel that reads them spreads through a dot and
             one that rewrites them, even by adding zero, replaces by the canonical NaN.

The instances of `sgns_det_kernel<NJ, KO>` (NJ = ceil(dim / 32), KO = 6 for K <= 5 and 8 for K = 6, 7; NJ <= 10 runs
32 warps, NJ >= 11 16) and the instance case that runs each, as dim/K/W:

  NJ  | KO = 6            | KO = 8
  1   | 1/1/1, 32/2/3     | 1/6/2, 32/7/4
  2   | 33/3/5            | 33/6/6
  3   | 95/4/7            | 95/7/8
  4   | 128/5/9           | 128/6/10
  5   | 131/1/11          | 131/7/12
  6   | 190/2/13          | 190/6/14
  7   | 224/3/15          | 224/7/1
  8   | 250/4/2           | 250/6/3
  9   | 260/5/4           | 260/7/5
  10  | 319/1/6, 320/2/8  | 319/6/7, 320/7/9
  11  | 321/3/10          | 321/6/11
  12  | 384/4/12          | 384/7/13
  13  | 387/5/14          | 387/6/15
  14  | 445/1/1           | 445/7/2
  15  | 480/2/3           | 480/6/4
  16  | 512/3/5           | 512/7/6

Every K in 1..7 and every W in 1..15 appears at least twice; each instance case runs at least 3 waves.  Then: a
last wave of one slice of r = 1..5 and S - 1 centres, and blocks of 1 and 2 tokens; the 4-byte copy path with rows
of a multiple of 4 floats (ld % 4 != 0, or a base 4, 8 or 12 bytes past a 16-byte boundary), which must give the
bits of the 16-byte path; one repeated word, a one-word pool equal to every centre, breaks everywhere but one
position; compact row maps with padded rows and the pool size read from device memory, as the block protocol calls
the kernel; a block in 3 calls into one loss and pair count; and the configurations the kernel refuses."""
import json
import os
import struct
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sgns_det_model as sdm  # noqa: E402

pytestmark = pytest.mark.gpu

SENTINEL = 0x7FD1CE5D                     # a quiet NaN with a payload
GUARD = 64                                # guard cells before and after each table
TOL_TABLE, TOL_LOSS = 1e-4, 1e-5
ERRORS = {}                               # check -> largest error / bound seen (printed with -s)


def _lib():
    from multiverso_b200 import _native as N
    return N


def _wave(D, K, W):
    return _lib().cuda_lib().mvb_sgns_win_inflight(D, K, W)


def _smem(S, W, D, ko):
    """det_smem_bytes of csrc/cuda/sgns_win.cu."""
    dimp = (D + 3) // 4 * 4
    return ((S * ko + S + 2 * W) * dimp * 4 + S * (2 * W + 1) * ko * 8 + S * 8 + 4 * 8 + (S + 2 * W) * 12 +
            S * ko * 12 + S * 4 + S * W * 4 + 16)


def _slice(D, K, W):
    """Centres per CTA of the wave kernel, as mvb_sgns_train_det picks them."""
    props = torch.cuda.get_device_properties(0)
    sms, ko = props.multi_processor_count, 6 if K <= 5 else 8
    S = min(-(-_wave(D, K, W) // sms), 32)
    while S > 1 and _smem(S, W, D, ko) > props.shared_memory_per_block_optin:
        S -= 1
    return S


def _buffer(rows, D, LD, off, g):
    """A table of rows x LD floats starting `off` floats into a buffer of NaN sentinels: (buffer, table view)."""
    buf = torch.full((2 * GUARD + rows * LD + 4,), SENTINEL, dtype=torch.int32).view(torch.float32)
    t = buf[GUARD + off:GUARD + off + rows * LD].view(rows, LD)
    t[:, :D] = (torch.rand(rows, D, generator=g) - 0.5) * 0.4
    return buf, t


def _case(D, K, W, n_tok, *, rows=4096, LD=None, off=(0, 0), tokens=None, neg="pool", pool=None, pool_n=None,
          word_maps=None, V=None, scales=True, calls=None, seed=0, lr=2e-2):
    LD = D if LD is None else LD
    V = rows if V is None else V
    g = torch.Generator().manual_seed(1000 * D + 10 * K + W + seed)
    buf_in, w_in = _buffer(rows, D, LD, off[0], g)
    buf_out, w_out = _buffer(rows, D, LD, off[1], g)
    if tokens is None:                                   # a skewed corpus over 3/4 of the rows: hot and cold rows
        u = torch.rand(n_tok, generator=g, dtype=torch.float64)
        tokens = (u * u * (rows * 3 // 4)).to(torch.int32)
        tokens[41::97] = -1
    tokens = torch.as_tensor(tokens, dtype=torch.int32)
    assert len(tokens) == n_tok
    c = dict(V=V, D=D, LD=LD, W=W, K=K, n_tok=n_tok)
    if calls is not None:
        c["calls"] = calls
    case = dict(c=c, tokens=tokens, w_in=w_in, w_out=w_out, buf_in=buf_in, buf_out=buf_out, off=off,
                map=None, prob=None, alias=None, pool=None, lr=lr, seed=0x5EED + seed,
                s_in=0.5 + torch.rand(V, generator=g) if scales else None,
                s_out=0.5 + torch.rand(V, generator=g) if scales else None)
    if word_maps is not None:
        case["map_in"], case["map_out"] = (torch.as_tensor(m, dtype=torch.int32) for m in word_maps)
    if neg == "pool":
        case["pool"] = torch.randint(0, rows - 96, (4096,), generator=g, dtype=torch.int32) if pool is None \
            else torch.as_tensor(pool, dtype=torch.int32)
        if pool_n is not None:
            case["pool_n"] = pool_n
    else:
        case["prob"] = torch.rand(V, generator=g)
        case["alias"] = torch.randint(0, V, (V,), generator=g, dtype=torch.int32)
    return case


def _args(case, dev, s, e):
    N = _lib()
    c = case["c"]
    a = N.Sgns()
    toks = dev["tokens"][s:e]
    a.tokens, a.n_tokens = toks.data_ptr(), toks.numel()
    a.w_in = dev["buf_in"].data_ptr() + 4 * (GUARD + case["off"][0])
    a.w_out = dev["buf_out"].data_ptr() + 4 * (GUARD + case["off"][1])
    a.dim, a.ld, a.window, a.negative = c["D"], c["LD"], c["W"], c["K"]
    a.lr, a.seed, a.vocab = case["lr"], case["seed"] + s, c["V"]
    if case["pool"] is not None:
        a.neg_pool, a.neg_pool_size = dev["pool"].data_ptr(), dev["pool"].numel()
        if "pool_n" in case:                             # the size the kernel must read: not the host's
            a.neg_pool_size_ptr = dev["pool_n"].data_ptr()
    else:
        a.alias_prob, a.alias_idx = dev["prob"].data_ptr(), dev["alias"].data_ptr()
    a.map_in, a.map_out = N.ptr(dev.get("map_in")), N.ptr(dev.get("map_out"))
    if case["s_in"] is not None:
        a.scale_in, a.scale_out = dev["s_in"].data_ptr(), dev["s_out"].data_ptr()
    a.pair_count, a.loss_sum = dev["out"].data_ptr(), dev["out"].data_ptr() + 8
    return a


def _device(case):
    dev = {k: v.cuda() for k, v in case.items() if isinstance(v, torch.Tensor) and k not in ("w_in", "w_out")}
    if "pool_n" in case:
        dev["pool_n"] = torch.tensor([case["pool_n"]], dtype=torch.int32, device="cuda")
    dev["out"] = torch.zeros(2, dtype=torch.int64, device="cuda")
    return dev


def _run(case):
    """Trains the case on the GPU: dict(buf_in, buf_out on the host, pairs, loss, loss_bits)."""
    N = _lib()
    dev = _device(case)
    cuts = case["c"].get("calls", (0, case["c"]["n_tok"]))
    for s, e in zip(cuts[:-1], cuts[1:]):
        assert N.cuda_lib().mvb_sgns_train_det(_args(case, dev, s, e), N.stream_ptr()) == 0
    torch.cuda.synchronize()
    o = dev["out"].cpu()
    loss = o[1:].view(torch.float32)[0].item()
    return dict(buf_in=dev["buf_in"].cpu(), buf_out=dev["buf_out"].cpu(), pairs=int(o[0]), loss=loss,
                loss_bits=struct.unpack("<I", struct.pack("<f", loss))[0])


def _note(check, ratio):
    ERRORS[check] = max(ERRORS.get(check, 0.0), ratio)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _check(case, got, wave, trains=True):
    """The GPU result against the model: tables, pairs, loss, and every cell that must keep its bits."""
    c = case["c"]
    D, LD = c["D"], c["LD"]
    ref = sdm.model(case, wave)
    assert got["pairs"] == ref["pairs"], (got["pairs"], ref["pairs"])
    for t, buf, init_buf in (("in", got["buf_in"], case["buf_in"]), ("out", got["buf_out"], case["buf_out"])):
        off = GUARD + case["off"][0 if t == "in" else 1]
        rows = case["w_" + t].shape[0]
        end = off + rows * LD
        assert torch.equal(_bits(buf[:off]), _bits(init_buf[:off])), f"w_{t}: guard before the table written"
        assert torch.equal(_bits(buf[end:]), _bits(init_buf[end:])), f"w_{t}: guard after the table written"
        tab, init = buf[off:end].view(rows, LD), init_buf[off:end].view(rows, LD)
        assert torch.equal(_bits(tab[:, D:]), _bits(init[:, D:])), f"w_{t}: padding columns written"
        unread = torch.from_numpy(~ref["read_" + t])
        assert torch.equal(_bits(tab[unread]), _bits(init[unread])), f"w_{t}: a row no wave read was written"
        d_ref = ref["w_" + t] - init[:, :D].double()
        if not trains:
            assert torch.equal(_bits(tab), _bits(init)), f"w_{t}: written with no pair to train"
            continue
        d_got = tab[:, :D].double() - init[:, :D].double()
        err = float(torch.linalg.norm(d_got - d_ref) / torch.linalg.norm(d_ref))
        _note("table", err / TOL_TABLE)
        assert err < TOL_TABLE, (t, err)
    if not trains:
        assert got["pairs"] == 0 and got["loss"] == 0.0
        return
    lerr = abs(got["loss"] - ref["loss"]) / ref["loss"]
    _note("loss", lerr / TOL_LOSS)
    assert lerr < TOL_LOSS, (got["loss"], ref["loss"], lerr)


def _n_waves(wave, waves=3):
    """Token count of `waves` waves, the last a partial one."""
    return (waves - 1) * wave + wave // 3 + 5


# ---- every <NJ, KO> instance ----------------------------------------------------------------------------------
DIMS = [1, 32, 33, 95, 128, 131, 190, 224, 250, 260, 319, 320, 321, 384, 387, 445, 480, 512]
INSTANCES = []
for _j, _d in enumerate(DIMS):
    for _b, _k in enumerate((1 + _j % 5, 6 + _j % 2)):
        INSTANCES.append((_d, _k, 1 + (2 * _j + _b) % 15))
assert {((d + 31) // 32, 6 if k <= 5 else 8) for d, k, _ in INSTANCES} == \
    {(nj, ko) for nj in range(1, 17) for ko in (6, 8)}
assert all(sum(k == x for _, k, _ in INSTANCES) >= 2 for x in range(1, 8))
assert all(sum(w == x for _, _, w in INSTANCES) >= 2 for x in range(1, 16))


@pytest.mark.parametrize("D,K,W", INSTANCES, ids=[f"instance-d{d}-k{k}-w{w}-nj{(d + 31) // 32}-ko{6 if k <= 5 else 8}"
                                                  for d, k, w in INSTANCES])
def test_sgns_det_sweep_instance(mv_device, D, K, W):
    wave = _wave(D, K, W)
    n = _n_waves(wave)
    case = _case(D, K, W, n, neg="alias" if (D + K) % 2 else "pool")
    _check(case, _run(case), wave)


# ---- the last wave: one slice of r centres; blocks of 1 and 2 tokens -------------------------------------------
LAST = [(D, K, W, r) for D, K, W in ((32, 5, 5), (512, 7, 15)) for r in ("1", "2", "3", "4", "5", "S-1")]


@pytest.mark.parametrize("D,K,W,r", LAST, ids=[f"last-slice-d{d}-k{k}-w{w}-r{r}" for d, k, w, r in LAST])
def test_sgns_det_sweep_last_slice(mv_device, D, K, W, r):
    wave, S = _wave(D, K, W), _slice(D, K, W)
    rr = S - 1 if r == "S-1" else int(r)
    assert 1 <= rr < S
    case = _case(D, K, W, 2 * wave + rr)
    _check(case, _run(case), wave)


TINY = [(D, K, W, n) for D, K, W in ((32, 5, 5), (512, 7, 15)) for n in (1, 2)]


@pytest.mark.parametrize("D,K,W,n", TINY, ids=[f"tiny-d{d}-k{k}-w{w}-n{n}" for d, k, w, n in TINY])
def test_sgns_det_sweep_tiny_block(mv_device, D, K, W, n):
    """One token has no context: nothing changes.  Two tokens are each other's context: exactly two pairs."""
    case = _case(D, K, W, n, tokens=[5, 9][:n])
    got = _run(case)
    if n == 1:
        _check(case, got, _wave(D, K, W), trains=False)
    else:
        assert got["pairs"] == 2
        _check(case, got, _wave(D, K, W))


# ---- copy paths: the 4-byte copies give the bits of the 16-byte ones -------------------------------------------
COPY = [(128, 3, 4), (320, 6, 9)]
VARIANTS = [(1, (0, 0)), (2, (0, 0)), (3, (0, 0)), (0, (1, 1)), (0, (2, 2)), (0, (3, 3)), (0, (0, 2)), (0, (3, 0))]


@pytest.mark.parametrize("D,K,W", COPY, ids=[f"copy-d{d}-k{k}-w{w}" for d, k, w in COPY])
def test_sgns_det_sweep_copy_paths(mv_device, D, K, W):
    """Rows of a multiple of 4 floats at an ld that is not, or at a base 4, 8 or 12 bytes past a 16-byte boundary,
    are staged with 4-byte copies: same tables, loss and pair count, bit for bit, as the aligned 16-byte path."""
    wave = _wave(D, K, W)
    n = _n_waves(wave)
    base = _case(D, K, W, n)
    want = _run(base)
    _check(base, want, wave)
    for pad, off in VARIANTS:
        case = _case(D, K, W, n, LD=D + pad, off=off)
        assert torch.equal(case["tokens"], base["tokens"])
        got = _run(case)
        assert (got["pairs"], got["loss_bits"]) == (want["pairs"], want["loss_bits"]), (pad, off)
        for t in ("in", "out"):
            o_b, o_c = GUARD + base["off"][t == "out"], GUARD + off[t == "out"]
            rows = base["w_" + t].shape[0]
            tb = want["buf_" + t][o_b:o_b + rows * D].view(rows, D)
            tc = got["buf_" + t][o_c:o_c + rows * (D + pad)].view(rows, D + pad)[:, :D]
            assert torch.equal(_bits(tb), _bits(tc)), (t, pad, off)
            init = case["buf_" + t]
            assert torch.equal(_bits(got["buf_" + t][:o_c]), _bits(init[:o_c]))
            assert torch.equal(_bits(got["buf_" + t][o_c + rows * (D + pad):]), _bits(init[o_c + rows * (D + pad):]))
            pc = got["buf_" + t][o_c:o_c + rows * (D + pad)].view(rows, D + pad)[:, D:]
            assert torch.equal(_bits(pc), _bits(init[o_c:o_c + rows * (D + pad)].view(rows, D + pad)[:, D:]))


# ---- degenerate schedules ---------------------------------------------------------------------------------------
def test_sgns_det_sweep_one_word_corpus(mv_device):
    """Every reader of a wave shares one input row and one output row: every sum goes through the accumulator."""
    D, K, W = 64, 5, 5
    wave = _wave(D, K, W)
    n = _n_waves(wave)
    case = _case(D, K, W, n, tokens=np.full(n, 7), lr=2e-5)     # some 10^4 pairs a wave move the same two rows
    _check(case, _run(case), wave)


@pytest.mark.parametrize("K", [3, 7], ids=["one-word-pool-k3", "one-word-pool-k7"])
def test_sgns_det_sweep_one_word_pool(mv_device, K):
    """The pool is the one word of the corpus: every negative is the centre and skipped, only output row 0 is used."""
    D, W = 100, 6
    wave = _wave(D, K, W)
    n = _n_waves(wave)
    case = _case(D, K, W, n, tokens=np.full(n, 11), pool=[11], lr=2e-5)
    _check(case, _run(case), wave)


def test_sgns_det_sweep_breaks_all_but_one(mv_device):
    D, K, W = 96, 4, 7
    wave = _wave(D, K, W)
    n = _n_waves(wave)
    toks = np.full(n, -1)
    toks[wave + 3] = 17
    case = _case(D, K, W, n, tokens=toks)
    _check(case, _run(case), wave, trains=False)


def test_sgns_det_sweep_breaks_every_third(mv_device):
    """Sentences of two words: every centre has exactly one context."""
    D, K, W = 96, 4, 7
    wave = _wave(D, K, W)
    n = _n_waves(wave)
    toks = np.arange(n) % 3000
    toks[2::3] = -1
    case = _case(D, K, W, n, tokens=toks)
    got = _run(case)
    assert got["pairs"] == 2 * (n // 3) + (1 if n % 3 == 2 else 0) * 2
    _check(case, got, wave)


# ---- compact row maps and the pool size in device memory, as the block protocol calls the kernel ----------------
MAPS = [(37, 5, 5, 44), (100, 5, 5, 104), (300, 7, 10, 308)]


@pytest.mark.parametrize("D,K,W,LD", MAPS, ids=[f"maps-d{d}-k{k}-w{w}-ld{ld}" for d, k, w, ld in MAPS])
def test_sgns_det_sweep_maps_device_pool(mv_device, D, K, W, LD):
    """50k words, 2500 of them in the block, each mapped to its own row of a 2600-row cache per table; the pool
    holds 4096 words but the device says 1500, and the words past 1500 are never tokens."""
    V, used, rows = 50_000, 2500, 2600
    wave = _wave(D, K, W)
    n = _n_waves(wave)
    g = np.random.default_rng(D)
    words = g.choice(V, used + 1000, replace=False)
    block, extra = words[:used], words[used:]
    m_in, m_out = np.full(V, -1), np.full(V, -1)
    m_in[block] = g.permutation(rows)[:used]
    m_out[block] = g.permutation(rows)[:used]
    toks = block[(g.random(n) ** 2 * used).astype(np.int64)]
    toks[41::97] = -1
    pool = np.concatenate([block[g.integers(0, used, 1500)], extra[g.integers(0, 1000, 2596)]])
    case = _case(D, K, W, n, rows=rows, V=V, LD=LD, tokens=toks, pool=pool, pool_n=1500, word_maps=(m_in, m_out))
    _check(case, _run(case), wave)


# ---- one block in 3 calls into one loss and pair count ------------------------------------------------------------
@pytest.mark.parametrize("neg", ["pool", "alias"], ids=["3calls-pool", "3calls-alias"])
def test_sgns_det_sweep_three_calls(mv_device, neg):
    """Every call restarts positions at 0 (windows and loss sampling) and seeds with seed + start."""
    D, K, W = 100, 5, 5
    wave = _wave(D, K, W)
    n = 3 * wave + 500
    cuts = (0, wave + 123, 2 * wave + 7, n)
    case = _case(D, K, W, n, neg=neg, calls=cuts)
    _check(case, _run(case), wave)


# ---- refusals ----------------------------------------------------------------------------------------------------
REFUSALS = [("negative0", dict(negative=0), -20), ("negative8", dict(negative=8), -20), ("cbow", dict(cbow=1), -20),
            ("hs", dict(hs=1), -20), ("adagrad", dict(use_adagrad=1), -20), ("dim0", dict(dim=0), -21),
            ("dim513", dict(dim=513, ld=513), -21), ("window0", dict(window=0), -21),
            ("window16", dict(window=16), -21), ("nservers2", dict(nservers=2, rows_per_server=2048), -21),
            ("vocab0", dict(vocab=0), -21), ("tokens0", dict(n_tokens=0), 0)]


def _kernels(fn):
    """Names of the GPU kernels, memsets and copies fn ran, from torch.profiler; sorted."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted(e.name for e in prof.events() if e.device_type.name == "CUDA")


def _seen(fn, tries=3):
    """_kernels of fn, which launches something: a profiler session that recorded no GPU activity at all is taken
    again (the profiler now and then returns a session without its device events)."""
    for _ in range(tries):
        names = _kernels(fn)
        if names:
            return names
    raise AssertionError("the profiler saw no kernel of a call that launches some")


def test_sgns_det_sweep_refusals(mv_device):
    """Each refused configuration returns its code, launches nothing and leaves the tables alone.

    Launches are counted in a profiler session that runs the refused call and then a valid one: it must hold exactly
    the kernels of the valid call alone, which also shows that the session recorded the device's activity."""
    N = _lib()
    D, K, W = 64, 5, 5
    case = _case(D, K, W, 600, rows=1024)
    dev = _device(case)
    init_in, init_out = dev["buf_in"].clone(), dev["buf_out"].clone()

    def restore():
        dev["buf_in"].copy_(init_in)
        dev["buf_out"].copy_(init_out)
        dev["out"].zero_()

    def control():
        assert N.cuda_lib().mvb_sgns_train_det(_args(case, dev, 0, 600), N.stream_ptr()) == 0

    control()                                           # sizes the kernel's scratch: later calls clear nothing
    restore()
    want_names = _seen(control)
    restore()
    assert any("sgns_det_kernel" in x for x in want_names), want_names
    for name, fields, want in REFUSALS:
        a = _args(case, dev, 0, 600)
        for k, v in fields.items():
            setattr(a, k, v)

        def refused():
            if want == 0:
                assert N.cuda_lib().mvb_sgns_train_det(a, N.stream_ptr()) == 0
                return
            with pytest.raises(N.NativeError, match=f"rc={want}:"):
                N.cuda_lib().mvb_sgns_train_det(a, N.stream_ptr())

        refused()
        torch.cuda.synchronize()
        assert torch.equal(_bits(dev["buf_in"]), _bits(init_in)), name
        assert torch.equal(_bits(dev["buf_out"]), _bits(init_out)), name
        assert int(dev["out"][0]) == 0 and int(dev["out"][1]) == 0, name
        names = _seen(lambda: (refused(), control()))
        restore()
        assert names == want_names, (name, names, want_names)


def test_sgns_det_sweep_report():
    """Prints the largest error per check as a fraction of its bound over the cases run before it (pytest -s)."""
    print("\nsgns_det sweep, largest error / bound:", json.dumps({k: round(v, 4) for k, v in ERRORS.items()}))
