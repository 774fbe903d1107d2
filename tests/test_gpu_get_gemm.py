"""The TMA + wgmma GEMM of csrc/cuda/gemm_fused.cu (``get_gemm``, ``gemm_nt``) against fp64.

Two modes at every shape:

* exact: x and W are integers in [-8, 8], exact in TF32, and with K <= 4096 every partial sum is an integer below
  2^24, so the fp32 result is bitwise the fp64 product whatever the summation order or TF32 rounding. A dropped,
  duplicated or misplaced product changes it.
* rounding: randn activations, uniform weights, every element within (TF32 + K FP32) (|x| |W|^T)_ij of fp64 (TF32
  operands, then K fp32 additions in any order; the constants of test_gpu_sampled_softmax.py).

The output is written into a window of a sentinel buffer and nothing outside the window may change. Shapes cross
the 64-row consumer halves and the 128-row tiles, K crosses the 32-float k-block, the 6-stage ring (K = 192) and its
first phase wrap (K = 224), and two shapes have more items than SMs, so CTAs run the persistent loop. Shards are
faked on one GPU through an explicit row map: odd rows_per_server, a longer last shard, empty trailing shards and
garbage rows between them."""
import pytest
import torch

pytestmark = pytest.mark.gpu

TF32 = 4 * 2.0 ** -11
FP32 = 2.0 ** -24
SENTINEL = -1.2345e37
PAD = 1024                    # sentinel floats on each side of the output window
EDGES = (1, 63, 64, 65, 127, 128, 129, 257)


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _lib():
    from multiverso_b200 import _native as N
    return N, N.cuda_lib()


def _operands(M, Nr, K, exact, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    if exact:
        x = torch.randint(-8, 9, (M, K), device=dev, generator=g).float()
        w = torch.randint(-8, 9, (Nr, K), device=dev, generator=g).float()
    else:
        x = torch.randn(M, K, device=dev, generator=g)
        w = torch.rand(Nr, K, device=dev, generator=g) * 2 - 1
    return x, w


def _window(M, Nr, dev, shift=0):
    """An [M, Nr] output inside a sentinel buffer, starting ``shift`` floats past a 16-byte boundary."""
    buf = torch.full((2 * PAD + M * Nr + shift,), SENTINEL, device=dev)
    return buf, buf[PAD + shift:PAD + shift + M * Nr].view(M, Nr)


def _check(y, buf, x, w, exact, what, shift=0):
    """y against x w^T in fp64; with ``buf`` (the sentinel buffer of _window) also nothing outside the window."""
    torch.cuda.synchronize()
    M, Nr = y.shape
    K = x.shape[1]
    ref = x.double() @ w.double().T
    if exact:
        assert torch.equal(y.double(), ref), (what, (y.double() - ref).abs().max().item())
    else:
        tol = (TF32 + K * FP32) * (x.double().abs() @ w.double().abs().T)
        bad = (y.double() - ref).abs() > tol
        assert not bad.any(), (what, bad.nonzero()[:5].tolist())
    if buf is None:
        return
    lo, hi = buf[:PAD + shift], buf[PAD + shift + M * Nr:]
    assert bool((lo == SENTINEL).all()) and bool((hi == SENTINEL).all()), (what, "write outside the output window")


def _grid():
    return _lib()[1].mvb_get_gemm_last_config() % 1000


def _items(M, tiles_n):
    return tiles_n * ((M + 127) // 128)


@pytest.mark.parametrize("K", [4, 28, 32, 36, 192, 196, 224, 4096])
def test_gemm_nt_edges_exact_and_rounding(cuda, K):
    from multiverso_b200.ops.get_gemm import gemm_nt
    for M in EDGES:
        for Nr in EDGES:
            for exact in (True, False):
                x, w = _operands(M, Nr, K, exact, M * 1000 + Nr + K, cuda)
                buf, y = _window(M, Nr, cuda)
                assert gemm_nt(x, w, y) is y
                _check(y, buf, x, w, exact, (M, Nr, K, exact))


@pytest.mark.parametrize("M,Nr,K", [(1, 100003, 36), (4096, 1200, 224), (4096, 1200, 196)])
def test_persistent_loop_more_items_than_sms(cuda, M, Nr, K):
    """Each CTA takes several items: the accumulator reset, the ring stage and phase carried from one item to the
    next and the last empty-barrier arrive of each item are all on the path."""
    from multiverso_b200.ops.get_gemm import gemm_nt
    sms = torch.cuda.get_device_properties(cuda).multi_processor_count
    items = _items(M, (Nr + 127) // 128)
    assert items > sms and items % sms
    for exact in (True, False):
        x, w = _operands(M, Nr, K, exact, 11 + K, cuda)
        buf, y = _window(M, Nr, cuda)
        gemm_nt(x, w, y)
        assert _grid() == sms < items
        _check(y, buf, x, w, exact, (M, Nr, K, exact))


@pytest.mark.parametrize("M,Nrows,K", [(128, 64, 32), (256, 128, 64), (1000, 1000, 512), (77, 10, 784),
                                       (2048, 300, 300), (1300, 700, 1024)])
def test_get_gemm_matches_fp32_reference(mv_device, M, Nrows, K):
    """Through a MatrixTable: rounding mode on the table's own uniform weights, then exact mode on integer weights
    written into the shard, each into a sentinel window through ``out=``."""
    from multiverso_b200.ops import get_gemm, get_gemm_supported
    mv = mv_device
    assert get_gemm_supported()
    dev = torch.device("cuda", 0)
    t = mv.MatrixTable(Nrows, K, "float32", min_value=-1.0, max_value=1.0)
    for exact in (False, True):
        x, w = _operands(M, Nrows, K, exact, M + K, dev)
        if exact:
            t.shard.copy_(w.view(-1))
        else:
            w = t.get().view(Nrows, K).clone()
        buf, y = _window(M, Nrows, dev)
        assert get_gemm(t, x, out=y) is y
        _check(y, buf, x, w, exact, exact)
        y2 = get_gemm(t, x)
        torch.cuda.synchronize()
        assert torch.equal(y2, y)


def _rowmap(w, S, gap=29):
    """``w`` as S shards of pitch K at separate places of one buffer, NaN rows between and around them. The
    partition is the device table's: rows_per_server = num_row // S with the remainder on the last shard, or one
    row per server for the first num_row servers when num_row < S. An empty shard points at an aligned dummy row,
    as a device table's empty shard does."""
    N, _ = _lib()
    n, K = w.shape
    if n >= S:
        rps = n // S
        spans = [(s * rps, n if s == S - 1 else (s + 1) * rps) for s in range(S)]
    else:
        rps = 1
        spans = [(min(s, n), min(s + 1, n)) for s in range(S)]
    buf = torch.full((n + (S + 1) * gap, K), float("nan"), device=w.device)
    dummy = torch.full((1, K), float("nan"), device=w.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, K, S, rps
    for s, (lo, hi) in enumerate(spans):
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = w[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr() if hi > lo else dummy.data_ptr()
    return rm, (buf, dummy), spans


def _fused(rm, x, y, Nr):
    N, lib = _lib()
    g = N.GetGemm()
    g.x, g.y, g.w_cache = x.data_ptr(), y.data_ptr(), None
    g.M, g.N, g.K = x.shape[0], Nr, x.shape[1]
    g.wmap = rm
    g.local_server = 0
    lib.mvb_get_gemm_fused(g, N.stream_ptr())


# rows_per_server 501, 333, 129 (odd), 128 (tile-aligned shards, a 135-row last shard), and num_row < S
@pytest.mark.parametrize("S,Nr", [(2, 1003), (3, 1000), (8, 1037), (8, 8 * 128 + 7), (8, 5), (3, 2)])
@pytest.mark.parametrize("M", [1, 65, 300])
def test_sharded_row_map_on_one_gpu(cuda, S, Nr, M):
    """decode_tile and the per-shard tensor maps: odd rows_per_server puts odd shards at odd global columns (the
    scalar store path), the last shard is longer, and num_row < S leaves trailing shards empty."""
    K = 68
    for exact in (True, False):
        x, w = _operands(M, Nr, K, exact, S * 7 + Nr + M, cuda)
        rm, keep, spans = _rowmap(w, S)
        if Nr >= S:
            assert spans[-1][1] - spans[-1][0] > Nr // S          # the last shard takes the remainder
        buf, y = _window(M, Nr, cuda)
        _fused(rm, x, y, Nr)
        assert _grid() == min(_items(M, sum((hi - lo + 127) // 128 for lo, hi in spans)),
                              torch.cuda.get_device_properties(cuda).multi_processor_count)
        _check(y, buf, x, w, exact, (S, Nr, M, exact))


def test_nine_shards_return_an_error_without_a_launch(cuda):
    N, lib = _lib()
    x, w = _operands(4, 16, 8, True, 1, cuda)
    buf, y = _window(4, 16, cuda)
    _fused(_rowmap(w, 1)[0], x, y, 16)
    _check(y, buf, x, w, True, "one shard")
    assert _grid() == 1
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = 16, 8, N.MAX_RANKS + 1, 1
    for s in range(N.MAX_RANKS):
        rm.shard_ptrs[s] = w[s].data_ptr()
    buf2, y2 = _window(4, 16, cuda)
    with pytest.raises(N.NativeError, match="rc=-33"):
        _fused(rm, x, y2, 16)
    torch.cuda.synchronize()
    assert _grid() == 1 and bool((buf2 == SENTINEL).all())


def test_gemm_nt_call_patterns(cuda):
    """A row slice W[lo:hi] as the right operand (bench/full_softmax.py) and a row slice dout[B:] of a larger
    buffer as the output (the sampled-softmax backward)."""
    from multiverso_b200.ops.get_gemm import gemm_nt
    B, Sp, d, n = 37, 132, 96, 1000
    for exact in (True, False):
        x, W = _operands(B, n, d, exact, 5, cuda)
        lo, hi = 301, 301 + 259
        buf, y = _window(B, hi - lo, cuda)
        gemm_nt(x, W[lo:hi], y)
        _check(y, buf, x, W[lo:hi], exact, ("slice", exact))
        e_t, x_t = _operands(Sp, d, B + 3, exact, 6, cuda)
        dout = torch.full((B + Sp, d), SENTINEL, device=cuda)
        assert gemm_nt(e_t, x_t, dout[B:]).data_ptr() == dout[B].data_ptr()
        torch.cuda.synchronize()
        assert bool((dout[:B] == SENTINEL).all())
        _check(dout[B:], None, e_t, x_t, exact, ("dout", exact))


def test_gemm_nt_argument_contract(cuda):
    from multiverso_b200 import _native as N
    from multiverso_b200.ops.get_gemm import gemm_nt
    M, Nr, K = 20, 30, 64
    x, w = _operands(M, Nr, K, True, 2, cuda)
    for bad in (torch.empty(M, Nr + 1, device=cuda), torch.empty(M * Nr, device=cuda),
                torch.empty(M, Nr, dtype=torch.float64, device=cuda), torch.empty(M, Nr),
                torch.empty(Nr, M, device=cuda).t(), torch.empty(M, 2 * Nr, device=cuda)[:, ::2]):
        with pytest.raises(ValueError):
            gemm_nt(x, w, bad)
    with pytest.raises(ValueError):
        gemm_nt(x[:, :K - 2].contiguous(), w[:, :K - 2].contiguous(), torch.empty(M, Nr, device=cuda))
    with pytest.raises(ValueError):
        gemm_nt(x, w[:, :K - 4].contiguous(), torch.empty(M, Nr, device=cuda))
    # a base off 16 bytes cannot be described to TMA: the tensor-map encode refuses it
    xb = torch.zeros(M * K + 1, device=cuda)
    x_off = xb[1:].view(M, K)
    x_off.copy_(x)
    with pytest.raises(N.NativeError):
        gemm_nt(x_off, w, torch.empty(M, Nr, device=cuda))
    # an output one float off 8-byte alignment with an even row pitch: scalar stores, exact result
    for Ncol in (30, 256, 1200):
        x, w = _operands(M, Ncol, K, True, Ncol, cuda)
        buf, y = _window(M, Ncol, cuda, shift=1)
        assert y.data_ptr() % 8 == 4
        gemm_nt(x, w, y)
        _check(y, buf, x, w, True, ("shifted", Ncol), shift=1)


def test_get_gemm_argument_contract(mv_device):
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import get_gemm
    mv = mv_device
    dev = torch.device("cuda", 0)
    M, Nr, K = 33, 130, 64
    t = mv.MatrixTable(Nr, K, "float32")
    x, w = _operands(M, Nr, K, True, 3, dev)
    t.shard.copy_(w.view(-1))
    for bad in (torch.empty(M, Nr - 1, device=dev), torch.empty(M + 1, Nr, device=dev),
                torch.empty(M, Nr, dtype=torch.float16, device=dev), torch.empty(M, Nr),
                torch.empty(Nr, M, device=dev).t()):
        with pytest.raises(ValueError):
            get_gemm(t, x, out=bad)
    with pytest.raises(ValueError):
        get_gemm(mv.MatrixTable(8, 30, "float32"), torch.zeros(4, 30, device=dev))
    xb = torch.zeros(M * K + 2, device=dev)
    with pytest.raises(N.NativeError):
        get_gemm(t, xb[2:].view(M, K))
    buf, y = _window(M, Nr, dev, shift=1)
    assert get_gemm(t, x, out=y) is y
    _check(y, buf, x, w, True, "shifted", shift=1)
