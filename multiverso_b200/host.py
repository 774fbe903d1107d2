"""Host backend: the Python API served by the C++ runtime (libmultiverso.so) through its C API.

Used when no CUDA device is present (CPU plumbing mode, BASELINE config 1) and as the
semantic oracle of the device backend.  Reference analogue: the ctypes binding
binding/python/multiverso/{utils,api,tables}.py over include/multiverso/c_api.h -- here the
tables are typed (float32 / float64 / int32), 64-bit sized, accept AddOption, expose the
sparse Matrix options, the KV table, MV_Aggregate and checkpointing.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional

import numpy as np

from . import _native as N
from .tables.options import AddOption, GetOption, check_add_option
from .utils import FLAGS, Log

_DT = {"float32": (0, np.float32), "float": (0, np.float32), "float64": (1, np.float64),
       "double": (1, np.float64), "int32": (2, np.int32), "int": (2, np.int32)}
_KV_DT = {"float32": (0, np.float32), "float64": (1, np.float64), "int32": (2, np.int32),
          "int64": (3, np.int64)}

_started = False


def _lib():
    lib = N.host_lib()
    lib.MV_Version.restype = C.c_char_p
    return lib


def _dtype(d):
    key = str(d).replace("torch.", "")
    if key not in _DT:
        Log.fatal("host backend tables support float32/float64/int32, got %s", d)
    return _DT[key]


def _push_flags(lib) -> None:
    """MV_SetFlag for every flag the C++ registry knows."""
    for name, val in FLAGS.items():
        b = name.encode()
        if isinstance(val, bool):
            lib.MV_SetFlagBool(b, int(val))
        elif isinstance(val, int):
            lib.MV_SetFlagInt(b, int(val))
        elif isinstance(val, float):
            lib.MV_SetFlagDouble(b, C.c_double(val))
        else:
            lib.MV_SetFlagString(b, str(val).encode())


def init_backend(rt) -> None:
    """MV_Init of the C++ runtime; fills the Runtime's identity from the controller's answer."""
    global _started
    lib = _lib()
    _push_flags(lib)
    os.environ.setdefault("MV_RANK", os.environ.get("RANK", "0"))
    os.environ.setdefault("MV_SIZE", os.environ.get("WORLD_SIZE", "1"))
    lib.MV_Init(None, None)
    _started = True
    rt.rank, rt.size = lib.MV_Rank(), lib.MV_Size()
    nw, ns = lib.MV_NumWorkers(), lib.MV_NumServers()
    rt.worker_ranks = [lib.MV_WorkerIdToRank(i) for i in range(nw)]
    rt.server_ranks = [lib.MV_ServerIdToRank(i) for i in range(ns)]
    Log.rank = rt.rank if rt.size > 1 else None


def shutdown_backend(rt, finalize_net: bool = True) -> None:
    global _started
    if _started:
        _lib().MV_ShutDownEx(1 if finalize_net else 0)
        _started = False


def barrier() -> None:
    _lib().MV_Barrier()


def aggregate(data):
    """MV_Aggregate on host memory (numpy array or CPU tensor), in place."""
    import torch
    lib = _lib()
    arr = data.numpy() if torch.is_tensor(data) else data
    arr = np.ascontiguousarray(arr)
    fn = {np.dtype(np.float32): lib.MV_AggregateFloat, np.dtype(np.float64): lib.MV_AggregateDouble,
          np.dtype(np.int32): lib.MV_AggregateInt, np.dtype(np.int8): lib.MV_AggregateChar}.get(arr.dtype)
    if fn is None:
        Log.fatal("aggregate: unsupported dtype %s", arr.dtype)
    fn(arr.ctypes.data_as(C.c_void_p), C.c_int64(arr.size))
    if torch.is_tensor(data):
        if arr.ctypes.data != data.data_ptr():
            data.copy_(torch.from_numpy(arr))
    elif arr is not data:
        np.copyto(data, arr)
    return data


def net_bind(rank: int, endpoint: str) -> None:
    if _lib().MV_NetBindC(rank, endpoint.encode()) != 0:
        Log.fatal("MV_NetBind(%d, %s) failed", rank, endpoint)


def net_connect(ranks: List[int], endpoints: List[str]) -> None:
    n = len(ranks)
    r = (C.c_int * n)(*ranks)
    e = (C.c_char_p * n)(*[x.encode() for x in endpoints])
    _lib().MV_NetConnectC(r, e, n)


def net_finalize() -> None:
    _lib().MV_NetFinalizeC()


def _opt_bytes(option: Optional[AddOption], npdt=None):
    """The 20-byte AddOption of an Add; a float table checks it against the servers' updater (-updater_type)."""
    opt = option or AddOption()
    if npdt is not None and np.issubdtype(npdt, np.floating):
        check_add_option(str(FLAGS.get("updater_type")), opt)
    return opt.pack()


def _as_np(data, npdt) -> np.ndarray:
    try:
        import torch
        if torch.is_tensor(data):
            data = data.detach().cpu().numpy()
    except ImportError:
        pass
    return np.ascontiguousarray(np.asarray(data, dtype=npdt))


class _HostTable:
    def __init__(self):
        self.handle = C.c_void_p()

    @property
    def table_id(self) -> int:
        return _lib().MV_TableId(self.handle) if self.handle.value else -1

    def wait(self, handle=None) -> None:
        """Async handles of this backend are already complete (the C API waits for Gets; async Adds are
        applied by the servers in order), kept so that scripts written for the device backend run here."""
        return None

    def finish_train(self) -> None:
        """Server_Finish_Train is sent by MV_ShutDown on this backend."""
        return None

    def store(self, uri: str) -> bool:
        return _lib().MV_SaveTableC(self.table_id, str(uri).encode()) == 0

    def load(self, uri: str) -> bool:
        return _lib().MV_LoadTableC(self.table_id, str(uri).encode()) == 0


class HostArrayTable(_HostTable):
    """ArrayTable<T> on the C++ runtime."""

    def __init__(self, size: int, dtype="float32", init_value=None):
        super().__init__()
        self.size = int(size)
        self.code, self.npdt = _dtype(dtype)
        _lib().MV_NewArrayTable64(C.c_int64(self.size), self.code, C.byref(self.handle))
        if init_value is not None:
            # master-init protocol of the reference binding (tables.py:51-57): every worker
            # issues a sync add; the master adds the initial value, the others add zeros
            from .runtime import Runtime
            init = np.zeros(self.size, self.npdt)
            if Runtime.get().worker_id() == 0:
                init += np.asarray(init_value, dtype=self.npdt).reshape(-1)
            self.add(init)
            barrier()

    def get(self, out=None):
        buf = np.empty(self.size, self.npdt) if out is None else out
        _lib().MV_GetArrayTable64(self.handle, self.code, buf.ctypes.data_as(C.c_void_p), C.c_int64(self.size))
        return buf

    def add(self, data, option: Optional[AddOption] = None, sync: bool = True) -> None:
        arr = _as_np(data, self.npdt).reshape(-1)
        assert arr.size == self.size
        _lib().MV_AddArrayTable64(self.handle, self.code, arr.ctypes.data_as(C.c_void_p),
                                  C.c_int64(self.size), _opt_bytes(option, self.npdt), 0 if sync else 1)

    def add_async(self, data, option: Optional[AddOption] = None):
        self.add(data, option, sync=False)
        return 0

    def get_async(self, out=None):
        """(handle, buffer) like the device backend; the buffer is already filled."""
        return 0, self.get(out)


class HostMatrixTable(_HostTable):
    """MatrixTable<T> / Matrix<T> (is_sparse) on the C++ runtime."""

    def __init__(self, num_row, num_col, dtype="float32", init_value=None, min_value=None,
                 max_value=None, is_sparse=False, is_pipeline=False):
        super().__init__()
        self.num_row, self.num_col = int(num_row), int(num_col)
        self.size = self.num_row * self.num_col
        self.code, self.npdt = _dtype(dtype)
        rnd = min_value is not None and max_value is not None
        _lib().MV_NewMatrixTable64(C.c_int64(self.num_row), C.c_int64(self.num_col), self.code,
                                   int(bool(is_sparse)), int(bool(is_pipeline)), int(rnd),
                                   C.c_double(min_value or 0.0), C.c_double(max_value or 0.0),
                                   C.byref(self.handle))
        self.is_sparse = bool(is_sparse)
        if init_value is not None:
            from .runtime import Runtime
            init = np.zeros(self.size, self.npdt)
            if Runtime.get().worker_id() == 0:
                init += np.broadcast_to(np.asarray(init_value, dtype=self.npdt), (self.num_row, self.num_col)).reshape(-1) \
                    if np.ndim(init_value) == 0 else np.asarray(init_value, dtype=self.npdt).reshape(-1)
            self.add(init)
            barrier()

    def get(self, out=None, option: Optional[GetOption] = None):
        buf = np.zeros((self.num_row, self.num_col), self.npdt) if out is None else out
        wid = option.worker_id if option else (-1 if not self.is_sparse else GetOption().worker_id)
        _lib().MV_GetMatrixTable64(self.handle, self.code, buf.ctypes.data_as(C.c_void_p),
                                   C.c_int64(self.size), None, C.c_int64(0), wid)
        return buf

    def get_rows(self, row_ids, out=None):
        ids = np.ascontiguousarray(np.asarray(row_ids, dtype=np.int64))
        buf = np.empty((ids.size, self.num_col), self.npdt) if out is None else out
        _lib().MV_GetMatrixTable64(self.handle, self.code, buf.ctypes.data_as(C.c_void_p),
                                   C.c_int64(ids.size * self.num_col), ids.ctypes.data_as(C.c_void_p),
                                   C.c_int64(ids.size), -1)
        return buf

    def get_row(self, row_id: int):
        return self.get_rows([row_id])[0]

    def add(self, data, option: Optional[AddOption] = None, sync: bool = True) -> None:
        arr = _as_np(data, self.npdt).reshape(-1)
        assert arr.size == self.size
        _lib().MV_AddMatrixTable64(self.handle, self.code, arr.ctypes.data_as(C.c_void_p),
                                   C.c_int64(self.size), None, C.c_int64(0), _opt_bytes(option, self.npdt),
                                   0 if sync else 1)

    def add_rows(self, row_ids, values, option: Optional[AddOption] = None, sync: bool = True) -> None:
        ids = np.ascontiguousarray(np.asarray(row_ids, dtype=np.int64))
        arr = _as_np(values, self.npdt).reshape(-1)
        assert arr.size == ids.size * self.num_col
        _lib().MV_AddMatrixTable64(self.handle, self.code, arr.ctypes.data_as(C.c_void_p),
                                   C.c_int64(arr.size), ids.ctypes.data_as(C.c_void_p),
                                   C.c_int64(ids.size), _opt_bytes(option, self.npdt), 0 if sync else 1)

    def add_row(self, row_id: int, values, option: Optional[AddOption] = None) -> None:
        self.add_rows([row_id], values, option)

    # the *_async spellings of the device backend (same return shapes)
    def add_async(self, data, option: Optional[AddOption] = None):
        self.add(data, option, sync=False)
        return 0

    def add_rows_async(self, row_ids, values, option: Optional[AddOption] = None):
        self.add_rows(row_ids, values, option, sync=False)
        return 0

    def get_async(self, out=None, option: Optional[GetOption] = None):
        return 0, self.get(out, option)

    def get_rows_async(self, row_ids, out=None):
        return 0, self.get_rows(row_ids, out)

    def get_stale(self, option: Optional[GetOption] = None):
        """Delta pull of a sparse table: (row_ids, rows) that changed since this worker's previous
        pull (explicit empty result when nothing changed).  The servers return only the stale rows and
        the C API scatters them into the caller's buffer, so the table keeps that buffer between pulls
        and reports the rows whose values moved."""
        cache = getattr(self, "_pull_cache", None)
        if not self.is_sparse or cache is None:
            # first pull (every row is stale) or a dense table: everything
            self._pull_cache = self.get(option=option)
            return np.arange(self.num_row, dtype=np.int64), self._pull_cache.copy()
        prev = cache.copy()
        self.get(out=cache, option=option)          # the servers overwrite only the stale rows
        changed = np.flatnonzero((cache != prev).any(axis=1)).astype(np.int64)
        return changed, cache[changed]


class HostKVTable(_HostTable):
    """KVTable<int64, V> on the C++ runtime; ``raw()`` is the worker-side cache."""

    def __init__(self, key_dtype="int64", val_dtype="float32"):
        super().__init__()
        key = str(val_dtype).replace("torch.", "")
        self.code, self.npdt = _KV_DT[key]
        _lib().MV_NewKVTable(self.code, C.byref(self.handle))
        self._cache = {}

    def raw(self):
        return self._cache

    def add(self, keys, vals) -> None:
        k = np.ascontiguousarray(np.atleast_1d(np.asarray(keys, dtype=np.int64)))
        v = np.ascontiguousarray(np.atleast_1d(np.asarray(vals, dtype=self.npdt)))
        assert k.size == v.size
        _lib().MV_KVAdd(self.handle, self.code, k.ctypes.data_as(C.c_void_p), v.ctypes.data_as(C.c_void_p),
                        C.c_int64(k.size))

    def get(self, keys):
        scalar = np.ndim(keys) == 0
        k = np.ascontiguousarray(np.atleast_1d(np.asarray(keys, dtype=np.int64)))
        out = np.empty(k.size, self.npdt)
        _lib().MV_KVGet(self.handle, self.code, k.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                        C.c_int64(k.size))
        for kk, vv in zip(k.tolist(), out.tolist()):
            self._cache[kk] = vv
        return out[0].item() if scalar else out
