"""K6 (csrc/cuda/allreduce.cu) against the exact rank-order sum, with the W ranks of a call emulated on one GPU.

The kernels take nothing but pointers, so W ordinary device buffers stand for the peers' symmetric memory and W
zeroed pads for their signal pads; that runs the code of a multi-GPU call minus NVLink. The ranks of a case are
launched one after the other on the current stream. Before the first launch of a case its epoch is written into
every slot of the case's two channels on every pad, so each flag wait returns on its first load, and ``err_flag``
(set by a wait that gave up) and the grid counter must both be zero afterwards.

Schedules that are correct when ranks run in sequence:

* one-shot only reads ``bufs``, so the ranks run in any order, each into its own result;
* two-shot in place (``out == bufs[me]``): rank r reduces slice r and writes it into every buffer; slices are disjoint;
* two-shot with a separate ``out``: the finish kernel of rank ``me`` copies all of ``bufs[me]``, so ``me`` runs last,
  after every other rank ran in place;
* fused: the peers' data is put into their staging slots beforehand and rank ``me`` runs alone.

The model is exact, not a tolerance: ``((x0 + x1) + x2) + ...`` in the element type, wrapping for the integer types,
and for f32 / f64 the same left-to-right sum in that type on the CPU. Results are compared bit for bit, as whole
memory images: every buffer lies between guard regions filled with a sentinel byte, and the image a case must leave
(inputs, results, guards, the unused half of the fused staging) is compared in one piece. The f32 sum is also held
to W * 2^-24 * sum_r |x_r| of the fp64 sum, which keeps saying something should the order ever change on purpose.
"""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

from multiverso_b200 import _native as N

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GUARD = 512                       # bytes on each side of a buffer: 64 elements of the widest type
SENT = 0x5A
FUSED_BYTES = 1 << 20             # one half of the fused path's double-buffered staging
DTYPES = [torch.float32, torch.float64, torch.int32, torch.int64, torch.int8]
WORLDS = [1, 2, 3, 5, 8]
_ids = {"ids": lambda v: str(v).replace("torch.", "")}


def _es(dtype):
    return torch.empty(0, dtype=dtype).element_size()


def _vec(dtype):
    return 16 // _es(dtype)


def _bytes(x):
    return x.contiguous().view(torch.uint8) if x.numel() else x.new_empty(x.shape, dtype=torch.uint8)


@pytest.fixture
def lib():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return N.cuda_lib()


class _Rows:
    """``rows`` buffers of ``n`` elements in one allocation, each [guard | off bytes | n elements | guard] at a
    16-byte multiple, so ``ptr(r)`` is 16-byte aligned exactly when ``off`` is. Every byte is SENT until written."""

    def __init__(self, rows, n, dtype, off=0):
        self.rows, self.n, self.dtype, self.es = rows, n, dtype, _es(dtype)
        self.lo, self.nb = GUARD + off, n * self.es
        self.stride = -(-(self.lo + self.nb + GUARD) // 16) * 16
        self.raw = torch.full((rows, self.stride), SENT, dtype=torch.uint8, device="cuda")
        assert self.raw.data_ptr() % 16 == 0 and GUARD % 16 == 0

    def ptr(self, r):
        return self.raw.data_ptr() + r * self.stride + self.lo

    def reset(self):
        self.raw.fill_(SENT)

    def put(self, x, at=0, row=None):
        """Write x ([rows, k], or [k] into ``row``) at byte ``at`` of the data region."""
        b = _bytes(x).cuda()
        lo = self.lo + at
        if row is None:
            self.raw[:, lo:lo + b.shape[-1]] = b
        else:
            self.raw[row, lo:lo + b.shape[-1]] = b

    def image(self, x, at=0):
        """The bytes of the whole allocation when it holds x ([rows, k]) at byte ``at`` and nothing else."""
        img = torch.full_like(self.raw, SENT)
        b = _bytes(x).cuda()
        img[:, self.lo + at:self.lo + at + b.shape[-1]] = b
        return img

    def expect(self, x, what, at=0):
        exp = self.image(x, at)
        if torch.equal(self.raw, exp):
            return
        bad = (self.raw != exp).nonzero().cpu()
        r, b = bad[0].tolist()
        lo, k = self.lo + at, x.shape[-1]
        e = (b - lo) // self.es
        where = f"element {e} (vector {e // (16 // self.es)})" if 0 <= e < k else f"element {e}, outside the data"
        e_lo, e_hi = (int(bad[:, 1].min()) - lo) // self.es, (int(bad[:, 1].max()) - lo) // self.es
        pytest.fail(f"{what}: {len(bad)} bytes differ from the exact image, first in buffer {r} at {where}; "
                    f"buffers {sorted(set(bad[:, 0].tolist()))}, elements {e_lo}..{e_hi}, data is 0..{k - 1}")


class _Ranks:
    """Pads, flags and descriptors of W emulated ranks on channels ch (ready) and ch + 1 (done)."""

    def __init__(self, world, ch):
        self.world, self.ch, self.epoch = world, ch, 0
        self.pads = torch.zeros(max(world, 1), N.PAD_WORDS, dtype=torch.int64, device="cuda")
        ptrs = [self.pads[r].data_ptr() for r in range(min(world, N.MAX_RANKS))]
        self.pad_ptrs = (C.c_void_p * N.MAX_RANKS)(*ptrs)
        self.err = torch.zeros(1, dtype=torch.int32, device="cuda")
        self.counter = torch.zeros(1, dtype=torch.int32, device="cuda")

    def arm(self):
        """A new case: every flag any of its kernels will wait for is set before the first launch."""
        self.epoch += 1
        self.pads[:, self.ch * N.MAX_RANKS:(self.ch + 2) * N.MAX_RANKS] = self.epoch

    def desc(self, dtype, n, bufs, out, me, code=None):
        a = N.Allreduce()
        a.dtype = N.dtype_code(dtype) if code is None else code
        a.n = n
        for r in range(min(self.world, N.MAX_RANKS)):
            a.bufs[r] = bufs.ptr(r)
        a.out = out
        a.pads = C.cast(self.pad_ptrs, C.POINTER(C.c_void_p))
        a.me, a.world, a.ch, a.epoch = me, self.world, self.ch, self.epoch
        a.err_flag = self.err.data_ptr()
        a.done_counter = self.counter.data_ptr()
        a.timeout_s = 1.0
        return a

    def staged(self, fn, dtype, n, bufs, out, me):
        assert fn(self.desc(dtype, n, bufs, out, me), N.stream_ptr()) == 0

    def fused(self, lib, dtype, n, stage, src, out, me, slot):
        assert lib.mvb_allreduce_fused(self.desc(dtype, n, stage, out, me), src, slot, N.stream_ptr()) == 0

    def check(self, what):
        torch.cuda.synchronize()
        assert int(self.err.item()) == 0, f"{what}: a flag wait gave up, err_flag {int(self.err.item())}"
        assert int(self.counter.item()) == 0, f"{what}: the grid counter was not returned to zero"


def _data(dtype, world, n, seed):
    """[world, n] per-rank, per-element random data, every rank from its own seed. Floats spread over 13 binades
    so that another order of addition changes bits; integers over the full range so that sums wrap."""
    rows = []
    for r in range(world):
        g = torch.Generator().manual_seed(1_000_003 * seed + r)
        if dtype.is_floating_point:
            m = torch.randn(n, generator=g, dtype=torch.float64)
            e = torch.randint(-6, 7, (n,), generator=g)
            rows.append((m * torch.exp2(e.double())).to(dtype))
        elif dtype == torch.int64:
            hi = torch.randint(-2 ** 31, 2 ** 31, (n,), generator=g)
            rows.append((hi << 32) + torch.randint(0, 2 ** 32, (n,), generator=g))
        else:
            lim = 2 ** (8 * _es(dtype) - 1)
            rows.append(torch.randint(-lim, lim, (n,), generator=g).to(dtype))
    return torch.stack(rows)


def _model(x):
    """((x0 + x1) + x2) + ... in the element type; integer addition wraps."""
    s = x[0].clone()
    for r in range(1, x.shape[0]):
        s = s + x[r]
    assert s.dtype == x.dtype
    if x.dtype == torch.float32:
        x64 = x.double()
        bound = x.shape[0] * 2.0 ** -24 * x64.abs().sum(0)
        assert bool(((s.double() - x64.sum(0)).abs() <= bound).all())
    elif not x.dtype.is_floating_point and x.dtype != torch.int64:
        bits = 8 * _es(x.dtype)
        wide = x.to(torch.int64).sum(0)
        assert torch.equal(s.to(torch.int64), ((wide + 2 ** (bits - 1)) % 2 ** bits) - 2 ** (bits - 1))
        assert x.shape[0] == 1 or x.shape[1] < 64 or bool((wide != s).any()), "no element wraps"
    return s


def _all(s, world):
    return s.unsqueeze(0).expand(world, -1)


def _sizes(dtype, world):
    """Element counts around the vector width V, the two-shot slice ceil(n / V / W) (last slice short; trailing
    slices empty for fewer than W vectors, as (W - 1) V and 2 V at W = 8) and the n % V tail."""
    v = _vec(dtype)
    return sorted({0, 1, v - 1, v, v + 1, 2 * v, (world - 1) * v, world * v - 1, world * v, world * v + 1, 4099,
                   v * (world * 1000 + 1) + 3})


def _offsets(dtype):
    """Byte offsets of a result from a 16-byte boundary: none, one element, and 4 and 8 bytes for int8."""
    return [0, _es(dtype)] + ([4, 8] if dtype == torch.int8 else [])


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dtype", DTYPES, **_ids)
def test_oneshot(lib, dtype, world):
    rk = _Ranks(world, ch=1)
    for n in _sizes(dtype, world):
        x = _data(dtype, world, n, seed=n)
        exp = _model(x)
        for off in _offsets(dtype):
            what = f"one-shot n={n} out offset {off}"
            bufs, outs = _Rows(world, n, dtype), _Rows(world, n, dtype, off)
            bufs.put(x)
            rk.arm()
            for me in range(world):
                rk.staged(lib.mvb_allreduce_oneshot, dtype, n, bufs, outs.ptr(me), me)
            rk.check(what)
            outs.expect(_all(exp, world), what + ", results")
            bufs.expect(x, what + ", inputs")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dtype", DTYPES, **_ids)
def test_twoshot_in_place(lib, dtype, world):
    rk = _Ranks(world, ch=1)
    for n in _sizes(dtype, world):
        x = _data(dtype, world, n, seed=n + 1)
        exp = _model(x)
        for order in (range(world), reversed(range(world))):
            bufs = _Rows(world, n, dtype)
            bufs.put(x)
            rk.arm()
            for me in order:
                rk.staged(lib.mvb_allreduce_twoshot, dtype, n, bufs, bufs.ptr(me), me)
            rk.check(f"two-shot in place n={n}")
            bufs.expect(_all(exp, world), f"two-shot in place n={n}")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dtype", DTYPES, **_ids)
def test_twoshot_copy_out(lib, dtype, world):
    rk = _Ranks(world, ch=1)
    for n in _sizes(dtype, world):
        for off in _offsets(dtype):
            for me in range(world):
                what = f"two-shot n={n} rank {me} out offset {off}"
                x = _data(dtype, world, n, seed=17 * n + me)
                exp = _model(x)
                bufs, out = _Rows(world, n, dtype), _Rows(1, n, dtype, off)
                bufs.put(x)
                rk.arm()
                for r in [r for r in range(world) if r != me]:
                    rk.staged(lib.mvb_allreduce_twoshot, dtype, n, bufs, bufs.ptr(r), r)
                rk.staged(lib.mvb_allreduce_twoshot, dtype, n, bufs, out.ptr(0), me)
                rk.check(what)
                out.expect(_all(exp, 1), what + ", result")
                bufs.expect(_all(exp, world), what + ", buffers")


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("dtype", DTYPES, **_ids)
def test_fused(lib, dtype, world):
    rk = _Ranks(world, ch=3)
    stage = _Rows(world, 2 * FUSED_BYTES // _es(dtype), dtype)
    offs = _offsets(dtype)

    def case(n, me, slot, src_off, out_off, x, exp):
        what = f"fused n={n} rank {me} slot {slot} src offset {src_off}, " + (
            "out = src" if out_off is None else f"out offset {out_off}")
        stage.reset()
        for r in range(world):
            if r != me:
                stage.put(x[r], at=slot, row=r)
        src = _Rows(1, n, dtype, src_off)
        src.put(x[me:me + 1])
        out = src if out_off is None else _Rows(1, n, dtype, out_off)
        rk.arm()
        rk.fused(lib, dtype, n, stage, src.ptr(0), out.ptr(0), me, slot)
        rk.check(what)
        out.expect(_all(exp, 1), what + ", result")
        if out is not src:
            src.expect(x[me:me + 1], what + ", source")
        # rank me's slot now holds its data, the peers' slots are as given, the other half is untouched
        stage.expect(x, what + ", staging", at=slot)

    for n in _sizes(dtype, world):
        x = _data(dtype, world, n, seed=n + 2)
        exp = _model(x)
        for off in offs:
            for slot in (0, FUSED_BYTES):
                for me in range(world):
                    case(n, me, slot, off, None, x, exp)
        for src_off in offs:
            for out_off in offs:
                case(n, n % world, FUSED_BYTES * (n & 1), src_off, out_off, x, exp)


@pytest.mark.parametrize("world", [1, 2])
@pytest.mark.parametrize("dtype", [torch.float32, torch.int8], **_ids)
def test_grid_stride(lib, dtype, world):
    """Sizes beyond the grid caps (4 x SMs CTAs of 256 threads, 64 CTAs for the fused kernel), so that the loops
    go round more than once, with a partial last round and an n % V tail."""
    v, es = _vec(dtype), _es(dtype)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    lap = 4 * sms * 256 * v
    rk = _Ranks(world, ch=1)
    n = lap + 3 * 256 * v + v + 1
    x = _data(dtype, world, n, seed=5)
    exp = _model(x)
    for off in (0, es):
        bufs, outs = _Rows(world, n, dtype), _Rows(world, n, dtype, off)
        bufs.put(x)
        rk.arm()
        for me in range(world):
            rk.staged(lib.mvb_allreduce_oneshot, dtype, n, bufs, outs.ptr(me), me)
        rk.check(f"one-shot n={n}")
        outs.expect(_all(exp, world), f"one-shot n={n} out offset {off}")
        bufs.expect(x, f"one-shot n={n}, inputs")
    n = world * lap + 5 * 256 * v + v + 1
    x = _data(dtype, world, n, seed=6)
    exp = _model(x)
    bufs = _Rows(world, n, dtype)
    bufs.put(x)
    rk.arm()
    for me in range(world):
        rk.staged(lib.mvb_allreduce_twoshot, dtype, n, bufs, bufs.ptr(me), me)
    rk.check(f"two-shot in place n={n}")
    bufs.expect(_all(exp, world), f"two-shot in place n={n}")
    for me, off in ((0, es), (world - 1, 0)):
        bufs, out = _Rows(world, n, dtype), _Rows(1, n, dtype, off)
        bufs.put(x)
        rk.arm()
        for r in [r for r in range(world) if r != me]:
            rk.staged(lib.mvb_allreduce_twoshot, dtype, n, bufs, bufs.ptr(r), r)
        rk.staged(lib.mvb_allreduce_twoshot, dtype, n, bufs, out.ptr(0), me)
        rk.check(f"two-shot n={n} rank {me}")
        out.expect(_all(exp, 1), f"two-shot n={n} rank {me} out offset {off}")
        bufs.expect(_all(exp, world), f"two-shot n={n} rank {me}, buffers")
    # the fused kernel's largest message fills one half of the staging exactly
    rf = _Ranks(world, ch=3)
    n = FUSED_BYTES // es
    x = _data(dtype, world, n, seed=7)
    exp = _model(x)
    stage = _Rows(world, 2 * n, dtype)
    for me, slot, off in ((0, FUSED_BYTES, 0), (world - 1, 0, es), (0, 0, 0)):
        stage.reset()
        for r in range(world):
            if r != me:
                stage.put(x[r], at=slot, row=r)
        io = _Rows(1, n, dtype, off)
        io.put(x[me:me + 1])
        rf.arm()
        rf.fused(lib, dtype, n, stage, io.ptr(0), io.ptr(0), me, slot)
        rf.check(f"fused n={n}")
        io.expect(_all(exp, 1), f"fused n={n} rank {me} slot {slot} offset {off}")
        stage.expect(x, f"fused n={n} rank {me} slot {slot}, staging", at=slot)


def test_rejected_arguments(lib):
    """world outside 1..MVB_MAX_RANKS and a staging offset off a 16-byte boundary return -3, an unknown element
    type -1; none of them launches, so the result and the inputs keep their bytes."""
    n = 64
    x = _data(torch.float32, 2, n, seed=9)
    bufs, out = _Rows(2, n, torch.float32), _Rows(1, n, torch.float32)
    bufs.put(x)
    st = N.stream_ptr()
    for fn in (lib.mvb_allreduce_oneshot, lib.mvb_allreduce_twoshot):
        for world in (0, N.MAX_RANKS + 1):
            rk = _Ranks(2, ch=1)
            a = rk.desc(torch.float32, n, bufs, out.ptr(0), 0)
            a.world = world
            with pytest.raises(N.NativeError, match="rc=-3"):
                fn(a, st)
        rk = _Ranks(2, ch=1)
        with pytest.raises(N.NativeError, match="rc=-1"):
            fn(rk.desc(torch.float32, n, bufs, out.ptr(0), 0, code=5), st)
    rk = _Ranks(2, ch=3)
    src = _Rows(1, n, torch.float32)
    for world, slot, code, rc in ((0, 0, None, -3), (N.MAX_RANKS + 1, 0, None, -3), (2, 8, None, -3), (2, 0, 5, -1)):
        a = rk.desc(torch.float32, n, bufs, out.ptr(0), 0, code=code)
        a.world = world
        with pytest.raises(N.NativeError, match=f"rc={rc}"):
            lib.mvb_allreduce_fused(a, src.ptr(0), slot, st)
    rk.check("rejected calls")
    out.expect(torch.empty(1, 0), "rejected calls, result")
    src.expect(torch.empty(1, 0), "rejected calls, source")
    bufs.expect(x, "rejected calls, inputs")


def test_multi_gpu_aggregate():
    """``parallel.aggregate`` (thresholds, staging growth, symmetric tensors, epochs) over real peers:
    tests/mp_allreduce_check.py, one rank per GPU."""
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    n = min(n, N.MAX_RANKS)
    port = 29950 + (os.getpid() % 200)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "mp_allreduce_check.py")]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout, tail
