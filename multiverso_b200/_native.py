"""ctypes bindings of the two native libraries.

* :func:`cuda_lib` -> ``libmvb200.so`` (sm_90a kernels, ``csrc/cuda/mvb200.h``)
* :func:`host_lib` -> ``libmultiverso.so`` (C++ host runtime + C API, ``include/multiverso/c_api.h``)

The CUDA library is mandatory whenever a GPU is present: ops raise instead of silently
falling back to eager PyTorch, so a run that passes has really executed our kernels.
"""
from __future__ import annotations

import ctypes as C
import os
from pathlib import Path

import torch

MAX_RANKS = 8
PAD_CHANNELS = 64
PAD_WORDS = PAD_CHANNELS * MAX_RANKS
EPOCH_FIN = 1 << 62

F32, F64, I32, I64, I8 = 0, 1, 2, 3, 4
UPD_DEFAULT, UPD_SGD, UPD_MOMENTUM, UPD_ADAGRAD, UPD_DCASGD, UPD_DCASGDA = range(6)
UPD_ROWWISE_ADAGRAD = 7          # 6 is unassigned
UPD_ADAM = 8
UPD_FTRL = 9
UPDATER_NAMES = {
    "default": UPD_DEFAULT, "sgd": UPD_SGD, "momentum_sgd": UPD_MOMENTUM,
    "adagrad": UPD_ADAGRAD, "dcasgd": UPD_DCASGD, "dcasgda": UPD_DCASGDA,
    "rowwise_adagrad": UPD_ROWWISE_ADAGRAD, "adam": UPD_ADAM, "ftrl": UPD_FTRL,
}

_LIBDIR = Path(__file__).resolve().parent / "_lib"
_cuda = None
_host = None

vp = C.c_void_p
i64 = C.c_int64
VP8 = vp * MAX_RANKS
I64x8 = i64 * MAX_RANKS
I32x8 = C.c_int * MAX_RANKS


class AddOpt(C.Structure):
    """Reference AddOption layout: {worker_id, momentum, lr, rho, lambda} (20 bytes)."""
    _fields_ = [("worker_id", C.c_int), ("momentum", C.c_float), ("lr", C.c_float),
                ("rho", C.c_float), ("lam", C.c_float)]


AddOptx8 = AddOpt * MAX_RANKS


class DenseAdd(C.Structure):
    _fields_ = [
        ("dtype", C.c_int), ("updater", C.c_int), ("shard", vp), ("state0", vp), ("state1", vp),
        ("shard_len", i64), ("shard_off", i64), ("state_stride", i64), ("nworkers", C.c_int),
        ("worker_mask", C.c_uint32), ("delta_ptrs", VP8), ("delta_multicast", vp), ("opts", AddOptx8), ("replica_ptrs", VP8), ("replica_multicast", vp), ("scale", C.c_float),
        ("clip", C.c_float), ("pads", C.POINTER(vp)), ("me", C.c_int), ("world", C.c_int),
        ("ch_ready", C.c_int), ("ch_done", C.c_int), ("epoch", C.c_uint64), ("worker_rank", I32x8),
        ("is_worker", C.c_int), ("err_flag", vp), ("fin_flag", vp), ("done_counter", vp),
        ("timeout_s", C.c_double), ("opt_box", VP8), ("my_worker", C.c_int), ("num_col", i64),
    ]


class DenseGet(C.Structure):
    _fields_ = [
        ("dtype", C.c_int), ("out", vp), ("nservers", C.c_int), ("shard_ptrs", VP8),
        ("shard_offs", I64x8), ("shard_lens", I64x8), ("pads", C.POINTER(vp)), ("me", C.c_int),
        ("world", C.c_int), ("ch_done", C.c_int), ("epoch", C.c_uint64), ("server_rank", I32x8),
        ("err_flag", vp), ("timeout_s", C.c_double),
    ]


class RowMap(C.Structure):
    _fields_ = [("num_row", i64), ("num_col", i64), ("nservers", C.c_int),
                ("rows_per_server", i64), ("shard_ptrs", VP8)]


BAD_ROW_MAP = -70   # a row map without 1 <= nservers <= MAX_RANKS and rows_per_server >= 1


class KV(C.Structure):
    _fields_ = [("vtype", C.c_int), ("nservers", C.c_int), ("capacity", i64), ("keys", VP8),
                ("vals", VP8)]


HASH_INIT_CONST, HASH_INIT_UNIFORM = 0, 1
HASH_FULL, HASH_TIMEOUT, HASH_BAD_KEY = 1, 2, 3


class HashRows(C.Structure):
    _fields_ = [("nservers", C.c_int), ("slots", i64), ("keys", VP8), ("ready", VP8), ("count", VP8),
                ("map", RowMap), ("init", C.c_int), ("init_value", C.c_float), ("lo", C.c_float),
                ("hi", C.c_float), ("seed", C.c_uint64), ("last_seen", VP8), ("clock", vp), ("sketch", VP8),
                ("total", VP8), ("age", vp), ("width", i64), ("admit_after", C.c_int)]


class HashLookup(C.Structure):
    _fields_ = [("tables", vp), ("keys", vp), ("n", i64), ("seg_end", vp), ("seg_table", vp), ("G", C.c_int),
                ("insert", C.c_int), ("insert_ok", vp), ("rows", vp), ("status", vp), ("timeout_s", C.c_double),
                ("admit", C.c_int)]


class Allreduce(C.Structure):
    _fields_ = [("dtype", C.c_int), ("n", i64), ("bufs", VP8), ("out", vp),
                ("pads", C.POINTER(vp)), ("me", C.c_int), ("world", C.c_int), ("ch", C.c_int),
                ("epoch", C.c_uint64), ("err_flag", vp), ("done_counter", vp),
                ("timeout_s", C.c_double)]


class Sgns(C.Structure):
    _fields_ = [
        ("tokens", vp), ("n_tokens", i64), ("w_in", vp), ("w_out", vp), ("g2_in", vp),
        ("g2_out", vp), ("dim", C.c_int), ("ld", i64), ("window", C.c_int), ("negative", C.c_int),
        ("cbow", C.c_int), ("hs", C.c_int), ("use_adagrad", C.c_int), ("lr", C.c_float),
        ("alias_prob", vp), ("alias_idx", vp), ("vocab", C.c_int), ("neg_pool", vp),
        ("neg_pool_size", C.c_int), ("hs_points", vp), ("hs_codes", vp), ("hs_len", vp),
        ("hs_max_code", C.c_int), ("map_in", vp), ("map_out", vp), ("seed", C.c_uint64),
        ("loss_sum", vp), ("pair_count", vp), ("hogwild", C.c_int),
        ("scale_in", vp), ("scale_out", vp), ("neg_pool_size_ptr", vp),
        ("nservers", C.c_int), ("rows_per_server", i64), ("w_in_peers", VP8), ("w_out_peers", VP8),
    ]


class KeyMap(C.Structure):
    _fields_ = [("size", i64), ("per_server", i64), ("nservers", C.c_int), ("width", C.c_int),
                ("shard_ptrs", VP8), ("touched_ptrs", VP8)]


class RowBox(C.Structure):
    _fields_ = [
        ("map", RowMap), ("me", C.c_int), ("cap", i64), ("slot_bytes", i64), ("box", VP8), ("ack", VP8),
        ("seg", vp), ("done", vp), ("applied", vp), ("go", vp), ("err_flag", vp), ("timeout_s", C.c_double),
    ]


class WePrep(C.Structure):
    _fields_ = [
        ("tokens", vp), ("n_tokens", i64), ("vocab", C.c_int), ("negative", C.c_int),
        ("alias_prob", vp), ("alias_idx", vp), ("seed", C.c_uint64), ("bm_in", vp), ("bm_out", vp),
        ("chunk_sums", vp), ("map_in", vp), ("map_out", vp), ("ids_in", vp), ("ids_out", vp),
        ("neg_pool", vp), ("pool_cap", i64), ("counts", vp), ("cap_in", i64), ("cap_out", i64),
    ]


class LrSparse(C.Structure):
    _fields_ = [
        ("row_ptr", vp), ("keys", vp), ("vals", vp), ("labels", vp), ("sample_w", vp), ("n", i64),
        ("objective", C.c_int), ("w", vp), ("dim", i64), ("out", C.c_int), ("grad", vp),
        ("loss_sum", vp), ("correct", vp), ("pred", vp), ("err", vp), ("compute_grad", C.c_int),
    ]


class LrDense(C.Structure):
    _fields_ = [
        ("x", vp), ("labels", vp), ("n", i64), ("dim", i64), ("out", C.c_int),
        ("objective", C.c_int), ("w", vp), ("grad", vp), ("loss_sum", vp), ("correct", vp),
        ("pred", vp), ("err", vp), ("compute_grad", C.c_int),
    ]


class GetGemm(C.Structure):
    _fields_ = [("x", vp), ("y", vp), ("w_cache", vp), ("M", i64), ("N", i64), ("K", i64),
                ("wmap", RowMap), ("local_server", C.c_int)]


class TopkCos(C.Structure):
    _fields_ = [("q", vp), ("M", i64), ("ldq", i64), ("dim", i64), ("n_rows", i64), ("wmap", RowMap),
                ("k", C.c_int), ("scores", vp), ("ids", vp), ("scratch", vp), ("scratch_bytes", i64)]


class FullSoftmax(C.Structure):
    _fields_ = [("q", vp), ("M", i64), ("ldq", i64), ("dim", i64), ("n_rows", i64), ("wmap", RowMap),
                ("k", C.c_int), ("labels", vp), ("lse", vp), ("loss", vp), ("scores", vp), ("ids", vp),
                ("scratch", vp), ("scratch_bytes", i64)]


class FullSoftmaxBwd(C.Structure):
    _fields_ = [("q", vp), ("M", i64), ("ldq", i64), ("dim", i64), ("wmap", RowMap), ("labels", vp), ("lse", vp),
                ("g", vp), ("dq", vp), ("lddq", i64), ("dw", vp), ("lddw", i64), ("scale", C.c_float),
                ("scratch", vp), ("scratch_bytes", i64)]


EMB_PUSH, EMB_COMPACT = 0, 1


class EmbBag(C.Structure):
    _fields_ = [("wmap", RowMap), ("dim", i64), ("ids", vp), ("L", i64), ("offsets", vp), ("B", i64),
                ("psw", vp), ("mean", C.c_int), ("out", vp), ("ldo", i64), ("dout", vp), ("ldd", i64),
                ("perm", vp), ("epilogue", C.c_int), ("scale", C.c_float), ("grads", vp), ("ldg", i64),
                ("uniq", vp), ("n_unique", vp), ("dpsw", vp), ("scratch", vp), ("scratch_bytes", i64),
                ("push_rows", i64)]


EMB_NO_PUSH = 2


class EmbTable(C.Structure):
    _fields_ = [("wmap", RowMap), ("dim", i64), ("key_base", i64), ("mean", C.c_int), ("epilogue", C.c_int),
                ("scale", C.c_float), ("ldg", i64), ("push_rows", i64)]


class EmbFeature(C.Structure):
    _fields_ = [("table", C.c_int), ("col", i64)]


class EmbColl(C.Structure):
    _fields_ = [("tables", vp), ("features", vp), ("class_feats", vp), ("class_off", C.c_int * 5), ("T", C.c_int),
                ("F", C.c_int), ("B", i64), ("ids", vp), ("L", i64), ("offsets", vp), ("psw", vp), ("out", vp),
                ("ldo", i64), ("dout", vp), ("ldd", i64), ("keys", vp), ("skeys", vp), ("perm", vp), ("info", vp),
                ("grads", vp), ("uniq", vp), ("dpsw", vp), ("scratch", vp), ("scratch_bytes", i64)]


class SampledSoftmax(C.Structure):
    _fields_ = [("alias_prob", vp), ("alias_idx", vp), ("logq", vp), ("n", i64), ("seed", C.c_uint64),
                ("step", C.c_uint64), ("S", i64), ("S_pad", i64), ("log_s", C.c_float), ("cand", vp), ("logq_c", vp),
                ("x", vp), ("w_y", vp), ("B", i64), ("B_pad", i64), ("d", i64), ("labels", vp), ("logits", vp),
                ("loss", vp), ("lse", vp), ("t_true", vp), ("g", vp), ("e_t", vp), ("e_true", vp)]


HSM_MAX_DIM, HSM_MAX_PATH = 1024, 64


class Hsm(C.Structure):
    _fields_ = [("wmap", RowMap), ("dim", i64), ("hidden", vp), ("B", i64), ("ldh", i64), ("labels", vp),
                ("n_classes", i64), ("points", vp), ("codes", vp), ("lens", vp), ("ldp", i64), ("offsets", vp),
                ("loss", vp), ("ids", vp), ("g", vp), ("u", vp), ("ldu", i64)]


FM_MAX_DIM = 1024


class Fm(C.Structure):
    _fields_ = [("wmap", RowMap), ("dim", i64), ("ids", vp), ("L", i64), ("offsets", vp), ("B", i64),
                ("values", vp), ("y", vp), ("sp", vp), ("lds", i64), ("dy", vp), ("perm", vp), ("epilogue", C.c_int),
                ("scale", C.c_float), ("grads", vp), ("ldg", i64), ("uniq", vp), ("n_unique", vp), ("scratch", vp),
                ("scratch_bytes", i64), ("push_rows", i64)]


FFM_MAX_DIM = 1024


class Ffm(C.Structure):
    _fields_ = [("wmap", RowMap), ("F", i64), ("k", i64), ("ids", vp), ("fields", vp), ("values", vp),
                ("offsets", vp), ("L", i64), ("B", i64), ("max_len", i64), ("y", vp), ("h", vp), ("ldh", i64)]


class RandomWalk(C.Structure):
    _fields_ = [("indptr", vp), ("indices", vp), ("cum", vp), ("num_nodes", i64), ("starts", vp), ("n", i64),
                ("length", i64), ("pitch", i64), ("p", C.c_double), ("q", C.c_double), ("seed", C.c_uint64),
                ("first_walk", i64), ("out", vp), ("node_count", vp)]


class NativeError(RuntimeError):
    pass


class Ptr:
    """ctypes parameter type of a data pointer: a torch tensor (its ``data_ptr()``), an int address, or
    None for NULL. A ``c_void_p`` passes through unchanged, so callers that still wrap pointers by hand keep
    working. Anything else raises TypeError instead of reaching the kernel as a wrong value."""

    @classmethod
    def from_param(cls, obj):
        if isinstance(obj, torch.Tensor):
            return C.c_void_p(obj.data_ptr())
        if isinstance(obj, int) or obj is None:
            return C.c_void_p(obj)
        if isinstance(obj, C.c_void_p):
            return obj
        raise TypeError(f"expected a tensor, an int address, a c_void_p or None, got {type(obj).__name__}")


def _raise_on_error(rc, func, args):
    check(rc, func.__name__)
    return rc


def _status(*argtypes):
    """Returns 0 or an error code; an error raises NativeError with mvb_last_error()."""
    return C.c_int, argtypes, _raise_on_error


def _unchecked(restype, *argtypes):
    return restype, argtypes, None


# The entry points of csrc/cuda/mvb200.h that Python calls (tests/test_native_abi_cpu.py checks them
# against the header). Struct parameters take the struct itself, void* const* / void** a c_void_p array or
# instance, and the host int64_t arrays of the dense push a c_int64 array.
i32, u32, u64, f32, f64 = C.c_int, C.c_uint32, C.c_uint64, C.c_float, C.c_double
vpp, i64p = C.POINTER(vp), C.POINTER(i64)
_CUDA_FUNCS = {
    "mvb_last_error": _unchecked(C.c_char_p),
    "mvb_set_device": _status(i32),
    "mvb_symm_alloc": _status(i64, vpp),
    "mvb_ipc_get_handle": _status(Ptr, Ptr),
    "mvb_ipc_open_handle": _status(Ptr, vpp),
    # teardown: a failure must not stop the release of the remaining slabs
    "mvb_symm_free": _unchecked(i32, Ptr),
    "mvb_ipc_close_handle": _unchecked(i32, Ptr),
    "mvb_signal": _status(vpp, i32, i32, i32, u64, Ptr),
    "mvb_wait": _status(vpp, i32, i32, i32, u64, u32, Ptr, f64, Ptr),
    "mvb_barrier": _status(vpp, i32, i32, i32, u64, Ptr, f64, Ptr),
    "mvb_add_dense_fused": _status(C.POINTER(DenseAdd), Ptr),
    "mvb_updater_apply": _status(i32, i32, Ptr, Ptr, Ptr, Ptr, i64, C.POINTER(AddOpt), f32, Ptr),
    "mvb_get_dense": _status(C.POINTER(DenseGet), Ptr),
    "mvb_push_dense_red": _status(i32, Ptr, i32, vpp, i64p, i64p, f32, Ptr),
    "mvb_push_dense_stateful": _status(i32, i32, Ptr, i32, vpp, vpp, vpp, i64p, i64p, i64p, C.POINTER(AddOpt), i32,
                                       Ptr),
    "mvb_push_dense_rowwise": _status(i32, i32, Ptr, i32, vpp, vpp, i64p, i64p, i64p, i64, C.POINTER(AddOpt), i32,
                                      Ptr),
    "mvb_push_dense_adam": _status(i32, i32, Ptr, i32, vpp, vpp, vpp, i64p, i64p, i64p, i64, C.POINTER(AddOpt), i32,
                                   Ptr),
    "mvb_get_rows": _status(i32, C.POINTER(RowMap), Ptr, i64, Ptr, i64, Ptr),
    "mvb_add_rows_red": _status(i32, C.POINTER(RowMap), Ptr, i64, Ptr, i64, f32, Ptr),
    "mvb_add_rows_delta": _status(C.POINTER(RowMap), Ptr, i64, Ptr, Ptr, i64, f32, Ptr),
    "mvb_add_rows_owner": _status(i32, i32, Ptr, Ptr, Ptr, i64, i64, i64, i64, Ptr, i64, Ptr, i64, C.POINTER(AddOpt),
                                  Ptr),
    "mvb_row_nonzero_mask": _status(i32, Ptr, i64, i64, i64, Ptr, Ptr),
    "mvb_stale_mark": _status(Ptr, i64, i32, Ptr, i64, Ptr),
    "mvb_stale_take": _status(Ptr, i64, Ptr, i64, Ptr, Ptr),
    "mvb_kv_init": _status(Ptr, i64, Ptr),
    "mvb_kv_count": _status(Ptr, i64, Ptr, Ptr),
    "mvb_kv_rehash": _status(i32, Ptr, Ptr, i64, Ptr, Ptr, i64, Ptr, Ptr),
    "mvb_kv_add": _status(C.POINTER(KV), Ptr, Ptr, i64, Ptr, Ptr),
    "mvb_kv_get": _status(C.POINTER(KV), Ptr, Ptr, i64, Ptr),
    "mvb_kv_dump": _status(i32, Ptr, Ptr, i64, Ptr, Ptr, Ptr, Ptr),
    "mvb_hash_rows_init": _status(Ptr, Ptr, Ptr, i64, Ptr),
    "mvb_hash_rows_lookup": _status(C.POINTER(HashLookup), Ptr),
    "mvb_hash_rows_age": _status(C.POINTER(HashRows), Ptr),
    "mvb_hash_rows_count": _status(C.POINTER(HashRows), Ptr, Ptr),
    "mvb_hash_rows_dump": _status(C.POINTER(HashRows), i32, Ptr, Ptr, Ptr, Ptr),
    "mvb_hash_rows_mark": _status(C.POINTER(HashRows), Ptr, i64, Ptr),
    "mvb_hash_rows_evict": _status(C.POINTER(HashRows), i32, i64, Ptr, Ptr, i32, i64, i64, Ptr, Ptr, Ptr),
    "mvb_hash_rows_evict_ex": _status(C.POINTER(HashRows), i32, i64, Ptr, Ptr, i32, i64, i64, Ptr, Ptr, Ptr, Ptr,
                                      i64),
    "mvb_allreduce_oneshot": _status(C.POINTER(Allreduce), Ptr),
    "mvb_allreduce_twoshot": _status(C.POINTER(Allreduce), Ptr),
    "mvb_allreduce_fused": _status(C.POINTER(Allreduce), Ptr, i64, Ptr),
    "mvb_allreduce_nvls": _status(C.POINTER(Allreduce), Ptr, Ptr),
    "mvb_sgns_train": _status(C.POINTER(Sgns), Ptr),
    "mvb_sgns_train_win": _status(C.POINTER(Sgns), Ptr),
    "mvb_sgns_train_det": _status(C.POINTER(Sgns), Ptr),
    "mvb_sgns_last_launches": _unchecked(i32),
    "mvb_sgns_win_inflight": _unchecked(i32, i32, i32, i32),
    "mvb_keys_add": _status(C.POINTER(KeyMap), Ptr, Ptr, i64, f32, Ptr),
    "mvb_keys_get": _status(C.POINTER(KeyMap), Ptr, Ptr, i64, Ptr),
    "mvb_keys_collect": _status(C.POINTER(KeyMap), Ptr, Ptr, Ptr, i64, Ptr),
    "mvb_stale_on_add": _status(vpp, i32, Ptr, Ptr, Ptr, i32, Ptr),
    "mvb_stale_on_get": _status(vpp, i32, Ptr, Ptr, Ptr),
    "mvb_rowbox_slot_bytes": _unchecked(i64, i64, i64),
    "mvb_rowbox_slots": _unchecked(i32),
    "mvb_rowbox_push_delta": _status(C.POINTER(RowBox), Ptr, Ptr, i64, Ptr, Ptr, i64, f32, u64, C.POINTER(AddOpt), i32,
                                     Ptr),
    "mvb_rowbox_push_vals": _status(C.POINTER(RowBox), Ptr, Ptr, i64, Ptr, i64, f32, u64, C.POINTER(AddOpt), i32, Ptr),
    "mvb_rowbox_poll": _status(C.POINTER(RowBox), i32, i32, Ptr),
    "mvb_rowbox_apply": _status(C.POINTER(RowBox), i32, Ptr, Ptr, Ptr, i64, i64, i32, i32, Ptr),
    "mvb_we_prepare": _status(C.POINTER(WePrep), Ptr),
    "mvb_we_prepare_launches": _unchecked(i32, i32),
    "mvb_rows_pull": _status(C.POINTER(RowMap), i32, Ptr, Ptr, i64, Ptr, Ptr, i64, i32, Ptr),
    "mvb_rows_push_delta": _status(C.POINTER(RowMap), Ptr, Ptr, i64, Ptr, Ptr, i64, f32, i32, Ptr),
    "mvb_build_alias_table": _status(Ptr, i32, Ptr, Ptr),
    "mvb_lr_sparse_fwd_bwd": _status(C.POINTER(LrSparse), Ptr),
    "mvb_lr_dense_fwd_bwd": _status(C.POINTER(LrDense), Ptr),
    "mvb_lr_wide_epilogue": _status(Ptr, Ptr, i64, i32, i32, Ptr, i64, Ptr, Ptr, Ptr, Ptr),
    "mvb_transpose_pad_f32": _status(Ptr, i64, i64, i64, Ptr, i64, Ptr),
    "mvb_axpy_f32": _status(Ptr, Ptr, i64, f32, Ptr),
    "mvb_ftrl_weights": _status(Ptr, Ptr, Ptr, i64, f32, f32, f32, f32, Ptr),
    "mvb_ftrl_update": _status(Ptr, Ptr, Ptr, Ptr, i64, f32, Ptr),
    "mvb_ftrl_delta": _status(Ptr, Ptr, Ptr, Ptr, Ptr, i64, f32, Ptr),
    "mvb_regularize": _status(Ptr, Ptr, i64, i32, f32, Ptr),
    "mvb_get_gemm_fused": _status(C.POINTER(GetGemm), Ptr),
    "mvb_get_gemm_supported": _unchecked(i32),
    "mvb_get_gemm_last_config": _unchecked(i32),
    "mvb_topk_cos_scratch_bytes": _unchecked(i64, i64, i32, i64),
    "mvb_topk_cosine": _status(C.POINTER(TopkCos), Ptr),
    "mvb_full_softmax_scratch_bytes": _unchecked(i64, i64, i32, i64),
    "mvb_full_softmax": _status(C.POINTER(FullSoftmax), Ptr),
    "mvb_full_softmax_bwd_scratch_bytes": _unchecked(i64, i64, i64, i64, i32, i32),
    "mvb_full_softmax_bwd": _status(C.POINTER(FullSoftmaxBwd), Ptr),
    "mvb_embedding_bag_scratch_bytes": _unchecked(i64, i64, i64),
    "mvb_embedding_bag_fwd": _status(C.POINTER(EmbBag), Ptr),
    "mvb_embedding_bag_bwd": _status(C.POINTER(EmbBag), Ptr),
    "mvb_embedding_bag_psw_grad": _status(C.POINTER(EmbBag), Ptr),
    "mvb_emb_coll_scratch_bytes": _unchecked(i64, i64, i32, i64),
    "mvb_emb_coll_fwd": _status(C.POINTER(EmbColl), Ptr),
    "mvb_emb_coll_keys": _status(C.POINTER(EmbColl), Ptr),
    "mvb_emb_coll_count": _status(C.POINTER(EmbColl), Ptr),
    "mvb_emb_coll_bwd": _status(C.POINTER(EmbColl), Ptr),
    "mvb_emb_coll_psw_grad": _status(C.POINTER(EmbColl), Ptr),
    "mvb_ss_sample": _status(C.POINTER(SampledSoftmax), Ptr),
    "mvb_ss_fwd_epilogue": _status(C.POINTER(SampledSoftmax), Ptr),
    "mvb_ss_bwd_epilogue": _status(C.POINTER(SampledSoftmax), Ptr),
    "mvb_hsm_fwd": _status(C.POINTER(Hsm), Ptr),
    "mvb_fm_fwd": _status(C.POINTER(Fm), Ptr),
    "mvb_fm_bwd": _status(C.POINTER(Fm), Ptr),
    "mvb_ffm_fwd": _status(C.POINTER(Ffm), Ptr),
    "mvb_random_walk": _status(C.POINTER(RandomWalk), Ptr),
    "mvb_csr_cumsum": _status(Ptr, Ptr, i64, Ptr, Ptr),
}


def _ensure_built(name: str) -> Path:
    path = _LIBDIR / name
    if os.environ.get("MVB200_NO_BUILD") == "1" and path.exists():
        return path
    from . import _build
    try:
        if name == "libmvb200.so":
            _build.build_cuda()
        else:
            _build.build_host()
    except Exception:
        if not path.exists():
            raise
    return path


def cuda_lib():
    """Load (building if needed) the sm_90a kernel library."""
    global _cuda
    if _cuda is None:
        lib = C.CDLL(str(_ensure_built("libmvb200.so")), mode=C.RTLD_GLOBAL)
        for name, (restype, argtypes, errcheck) in _CUDA_FUNCS.items():
            f = getattr(lib, name)
            f.restype, f.argtypes = restype, argtypes
            if errcheck is not None:
                f.errcheck = errcheck
        _cuda = lib
    return _cuda


def host_lib():
    """Load (building if needed) the C++ host runtime."""
    global _host
    if _host is None:
        _host = C.CDLL(str(_ensure_built("libmultiverso.so")), mode=C.RTLD_GLOBAL)
    return _host


def check(rc: int, what: str = ""):
    """Raise NativeError for a non-zero status. The declared status functions already raise on their own;
    this serves code that checks a status by hand."""
    if rc != 0:
        msg = cuda_lib().mvb_last_error()
        raise NativeError(f"{what or 'mvb200 call'} failed rc={rc}: {msg.decode() if msg else ''}")


def ptr(t) -> int:
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return 0 if t is None else t.data_ptr()


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def dtype_code(torch_dtype) -> int:
    return {torch.float32: F32, torch.float64: F64, torch.int32: I32, torch.int64: I64,
            torch.int8: I8}[torch_dtype]
