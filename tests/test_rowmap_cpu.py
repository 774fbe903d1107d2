"""Every entry point of the kernel library that addresses a row-sharded table rejects a malformed map before any
CUDA call: nservers outside [1, MVB_MAX_RANKS] (the kernels hold MVB_MAX_RANKS shard pointers) or
rows_per_server < 1. Runs without a GPU: the arguments are well formed apart from the map, the pointers are dummies
that must never be dereferenced, and a CUDA call on a machine without a device would return a different code."""
import pytest

from multiverso_b200 import _native as N

DUMMY = 1 << 12          # 16-byte aligned, never dereferenced
BAD_MAPS = {"no_servers": (0, 4), "too_many_servers": (N.MAX_RANKS + 1, 4), "no_rows_per_server": (2, 0)}


def _map(rm, nservers, rps):
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = 16, 4, nservers, rps
    for s in range(N.MAX_RANKS):
        rm.shard_ptrs[s] = DUMMY


def _rows(lib, fn, S, rps):
    rm = N.RowMap()
    _map(rm, S, rps)
    if fn == "mvb_get_rows":
        return lib.mvb_get_rows(N.F32, rm, DUMMY, 1, DUMMY, 4, None)
    if fn == "mvb_add_rows_red":
        return lib.mvb_add_rows_red(N.F32, rm, DUMMY, 1, DUMMY, 4, 1.0, None)
    if fn == "mvb_add_rows_delta":
        return lib.mvb_add_rows_delta(rm, DUMMY, 1, DUMMY, DUMMY, 4, 1.0, None)
    if fn == "mvb_rows_pull":
        return lib.mvb_rows_pull(rm, 4, DUMMY, None, 1, DUMMY, DUMMY, 4, 1, None)
    return lib.mvb_rows_push_delta(rm, DUMMY, None, 1, DUMMY, DUMMY, 4, 1.0, 1, None)


def _rowbox(lib, fn, S, rps):
    b = N.RowBox()
    _map(b.map, S, rps)
    b.cap, b.slot_bytes = 16, lib.mvb_rowbox_slot_bytes(16, 4)
    opt = N.AddOpt()
    if fn == "mvb_rowbox_push_delta":
        return lib.mvb_rowbox_push_delta(b, DUMMY, None, 1, DUMMY, DUMMY, 4, 1.0, 1, opt, 1, None)
    if fn == "mvb_rowbox_push_vals":
        return lib.mvb_rowbox_push_vals(b, DUMMY, None, 1, DUMMY, 4, 1.0, 1, opt, 1, None)
    if fn == "mvb_rowbox_poll":
        return lib.mvb_rowbox_poll(b, -1, 0, None)
    return lib.mvb_rowbox_apply(b, N.UPD_DEFAULT, DUMMY, None, None, 0, 0, 0, 1, None)


def _keys(lib, fn, S, per):
    m = N.KeyMap()
    m.size, m.per_server, m.nservers, m.width = 16, per, S, 1
    for s in range(N.MAX_RANKS):
        m.shard_ptrs[s] = m.touched_ptrs[s] = DUMMY
    if fn == "mvb_keys_add":
        return lib.mvb_keys_add(m, DUMMY, DUMMY, 1, 1.0, None)
    if fn == "mvb_keys_get":
        return lib.mvb_keys_get(m, DUMMY, DUMMY, 1, None)
    return lib.mvb_keys_collect(m, DUMMY, DUMMY, DUMMY, 1, None)


def _gemm(lib, fn, S, rps):
    g = N.GetGemm()
    g.x, g.y, g.M, g.N, g.K = DUMMY, DUMMY, 4, 16, 4
    _map(g.wmap, S, rps)
    return lib.mvb_get_gemm_fused(g, None)


def _search(lib, fn, S, rps):
    a = N.TopkCos() if fn == "mvb_topk_cosine" else N.FullSoftmax()
    a.q, a.M, a.ldq, a.dim, a.n_rows, a.k = DUMMY, 1, 4, 4, 16, 1
    a.scores, a.ids, a.scratch, a.scratch_bytes = DUMMY, DUMMY, DUMMY, 1 << 30
    _map(a.wmap, S, rps)
    return getattr(lib, fn)(a, None)


def _emb_bag(lib, fn, S, rps):
    a = N.EmbBag()
    _map(a.wmap, S, rps)
    a.dim, a.ids, a.L, a.offsets, a.B = 4, DUMMY, 1, DUMMY, 1
    a.out, a.ldo, a.dout, a.ldd, a.perm, a.dpsw = DUMMY, 4, DUMMY, 4, DUMMY, DUMMY
    a.scratch, a.scratch_bytes = DUMMY, 1 << 30
    return getattr(lib, fn)(a, None)


def _sgns_direct(lib, fn, S, rps):
    """Direct mode (nservers > 1) of the window kernel: rows are addressed in the peers' shards."""
    h = N.Sgns()
    h.tokens, h.n_tokens, h.dim, h.ld, h.window, h.negative, h.lr, h.vocab = DUMMY, 64, 64, 64, 5, 5, 0.025, 16
    h.alias_prob = h.alias_idx = DUMMY
    h.nservers, h.rows_per_server = S, rps
    for s in range(N.MAX_RANKS):
        h.w_in_peers[s] = h.w_out_peers[s] = DUMMY
    return getattr(lib, fn)(h, None)


def _sgns_pool_size_ptr(lib, fn, case):
    """A device pool size (neg_pool_size_ptr) on an input that routes to the register or the generic kernel,
    which draw from neg_pool_size entries: refused with -23 before any CUDA call."""
    h = N.Sgns()
    h.tokens, h.n_tokens, h.dim, h.ld, h.window, h.negative, h.lr, h.vocab = DUMMY, 64, 64, 64, 5, 5, 0.025, 16
    h.w_in = h.w_out = DUMMY
    h.neg_pool, h.neg_pool_size, h.neg_pool_size_ptr = DUMMY, 16, DUMMY
    if case == "k8":
        h.negative = 8
    elif case == "k8_hogwild":
        h.negative, h.hogwild = 8, 1
    elif case == "cbow":
        h.cbow = 1
    elif case == "adagrad":
        h.use_adagrad, h.g2_in, h.g2_out = 1, DUMMY, DUMMY
    elif case == "hogwild_dim_37":
        h.dim = h.ld = 37
        h.hogwild = 1
    elif case == "hogwild_misaligned":
        h.w_in, h.hogwild = DUMMY + 4, 1
    return getattr(lib, fn)(h, None)


POOL_PTR_CASES = ["k8", "k8_hogwild", "cbow", "adagrad", "hogwild_dim_37", "hogwild_misaligned"]


@pytest.mark.parametrize("case", POOL_PTR_CASES)
def test_device_pool_size_is_refused_where_the_kernel_ignores_it(case):
    with pytest.raises(N.NativeError, match=r"^mvb_sgns_train failed rc=-23:"):
        _sgns_pool_size_ptr(N.cuda_lib(), "mvb_sgns_train", case)


# (entry point, caller, its map code)
ENTRIES = [(fn, _rows, N.BAD_ROW_MAP) for fn in
           ("mvb_get_rows", "mvb_add_rows_red", "mvb_add_rows_delta", "mvb_rows_pull", "mvb_rows_push_delta")]
ENTRIES += [(fn, _rowbox, N.BAD_ROW_MAP) for fn in
            ("mvb_rowbox_push_delta", "mvb_rowbox_push_vals", "mvb_rowbox_poll", "mvb_rowbox_apply")]
ENTRIES += [(fn, _keys, N.BAD_ROW_MAP) for fn in ("mvb_keys_add", "mvb_keys_get", "mvb_keys_collect")]
ENTRIES += [("mvb_get_gemm_fused", _gemm, -33), ("mvb_topk_cosine", _search, -41), ("mvb_full_softmax", _search, -41)]
ENTRIES += [(fn, _emb_bag, -50) for fn in
            ("mvb_embedding_bag_fwd", "mvb_embedding_bag_bwd", "mvb_embedding_bag_psw_grad")]
ENTRIES += [(fn, _sgns_direct, -21) for fn in ("mvb_sgns_train", "mvb_sgns_train_win")]


# nservers <= 1 is not a direct-mode call of the skip-gram kernels: it selects their local tables
CASES = [(fn, call, code, bad) for fn, call, code in ENTRIES for bad in sorted(BAD_MAPS)
         if not (call is _sgns_direct and BAD_MAPS[bad][0] <= 1)]


@pytest.mark.parametrize("fn,call,code,bad", CASES, ids=[f"{c[0]}-{c[3]}" for c in CASES])
def test_malformed_map_is_rejected_before_any_cuda_call(fn, call, code, bad):
    S, rps = BAD_MAPS[bad]
    with pytest.raises(N.NativeError, match=rf"^{fn} failed rc={code}:"):
        call(N.cuda_lib(), fn, S, rps)


def test_map_code_matches_the_header():
    header = (N._LIBDIR.parent.parent / "csrc" / "cuda" / "mvb200.h").read_text()
    assert f"enum {{ MVB_BAD_ROW_MAP = {N.BAD_ROW_MAP} }};" in header
