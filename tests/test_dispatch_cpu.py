"""The kernel library's argument codes, checked without a GPU: -2 for an unknown updater, -1 for an element type an
entry point does not serve, -3 for a server count outside [1, MVB_MAX_RANKS] where an entry point copies one
pointer per server into a fixed array of MVB_MAX_RANKS, -4 for a KV capacity that is not a power of two >= 1 (the
probe chains wrap with capacity - 1 as a mask), and -8 for a key-table width outside [1, 16]. Every other argument is
well formed, the pointers are dummies that must never be dereferenced, and a CUDA call on a machine without a device
would return a different code.

The calls run in a child process that sees no CUDA device (CUDA_VISIBLE_DEVICES=""), also where a GPU is present: an
argument check that stopped working then returns a CUDA error instead of launching a kernel on a dummy pointer."""
import ctypes as C
import json
import os
import re
import subprocess
import sys
from pathlib import Path

if __name__ == "__main__":
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

import pytest

from multiverso_b200 import _native as N

DUMMY = 1 << 12          # 16-byte aligned, never dereferenced
BAD_UPDATER = 6
BAD_DTYPE = 99


def _host_arrays(S):
    vp = (C.c_void_p * N.MAX_RANKS)(*([DUMMY] * N.MAX_RANKS))
    i64 = (C.c_int64 * N.MAX_RANKS)(*([4] * N.MAX_RANKS))
    return vp, i64


def _add_dense_fused(lib, dtype, upd):
    a = N.DenseAdd()
    a.dtype, a.updater, a.shard, a.shard_len, a.nworkers, a.worker_mask, a.world = dtype, upd, DUMMY, 4, 1, 1, 1
    a.delta_ptrs[0] = DUMMY
    return lib.mvb_add_dense_fused(a, None)


def _updater_apply(lib, dtype, upd):
    return lib.mvb_updater_apply(dtype, upd, DUMMY, DUMMY, DUMMY, DUMMY, 4, N.AddOpt(), 1.0, None)


def _push_stateful(lib, dtype, upd, S=1):
    vp, i64 = _host_arrays(S)
    return lib.mvb_push_dense_stateful(dtype, upd, DUMMY, S, vp, vp, vp, i64, i64, i64, N.AddOpt(), 0, None)


def _add_rows_owner(lib, dtype, upd):
    return lib.mvb_add_rows_owner(dtype, upd, DUMMY, DUMMY, DUMMY, 0, 4, 4, 16, DUMMY, 1, DUMMY, 4, N.AddOpt(), None)


def _rowbox_apply(lib, dtype, upd):
    b = N.RowBox()
    b.map.num_row, b.map.num_col, b.map.nservers, b.map.rows_per_server = 16, 4, 1, 16
    b.map.shard_ptrs[0] = b.box[0] = b.ack[0] = DUMMY
    b.cap, b.slot_bytes = 16, lib.mvb_rowbox_slot_bytes(16, 4)
    return lib.mvb_rowbox_apply(b, upd, DUMMY, DUMMY, DUMMY, 16, 0, 0, 1, None)


def _get_dense(lib, dtype):
    g = N.DenseGet()
    g.dtype, g.out, g.nservers, g.world = dtype, DUMMY, 1, 1
    g.shard_ptrs[0], g.shard_lens[0] = DUMMY, 4
    return lib.mvb_get_dense(g, None)


def _push_red(lib, dtype, S=1):
    vp, i64 = _host_arrays(S)
    return lib.mvb_push_dense_red(dtype, DUMMY, S, vp, i64, i64, 1.0, None)


def _rowmap():
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = 16, 4, 1, 16
    rm.shard_ptrs[0] = DUMMY
    return rm


def _get_rows(lib, dtype):
    return lib.mvb_get_rows(dtype, _rowmap(), DUMMY, 1, DUMMY, 4, None)


def _add_rows_red(lib, dtype):
    return lib.mvb_add_rows_red(dtype, _rowmap(), DUMMY, 1, DUMMY, 4, 1.0, None)


def _row_nonzero(lib, dtype):
    return lib.mvb_row_nonzero_mask(dtype, DUMMY, 4, 4, 4, DUMMY, None)


def _kv(dtype, S=1, cap=16):
    kv = N.KV()
    kv.vtype, kv.nservers, kv.capacity = dtype, S, cap
    for s in range(N.MAX_RANKS):
        kv.keys[s] = kv.vals[s] = DUMMY
    return kv


def _kv_add(lib, dtype, S=1):
    return lib.mvb_kv_add(_kv(dtype, S), DUMMY, DUMMY, 1, DUMMY, None)


def _kv_get(lib, dtype, S=1):
    return lib.mvb_kv_get(_kv(dtype, S), DUMMY, DUMMY, 1, None)


def _kv_capacity(fn, cap):
    def call(lib):
        if fn == "mvb_kv_rehash":
            return lib.mvb_kv_rehash(N.F32, DUMMY, DUMMY, 16, DUMMY, DUMMY, cap, DUMMY, None)
        return getattr(lib, fn)(_kv(N.F32, 1, cap), DUMMY, DUMMY, *((1, DUMMY) if fn == "mvb_kv_add" else (1,)), None)
    return call


def _keys_width(fn, width):
    def call(lib):
        m = N.KeyMap()
        m.size, m.per_server, m.nservers, m.width = 16, 16, 1, width
        m.shard_ptrs[0] = m.touched_ptrs[0] = DUMMY
        if fn == "mvb_keys_add":
            return lib.mvb_keys_add(m, DUMMY, DUMMY, 1, 1.0, None)
        if fn == "mvb_keys_get":
            return lib.mvb_keys_get(m, DUMMY, DUMMY, 1, None)
        return lib.mvb_keys_collect(m, DUMMY, DUMMY, DUMMY, 1, None)
    return call


def _kv_dump(lib, dtype):
    return lib.mvb_kv_dump(dtype, DUMMY, DUMMY, 16, DUMMY, DUMMY, DUMMY, None)


def _kv_rehash(lib, dtype):
    return lib.mvb_kv_rehash(dtype, DUMMY, DUMMY, 16, DUMMY, DUMMY, 32, DUMMY, None)


def _allreduce(fn):
    def call(lib, dtype):
        h = N.Allreduce()
        h.dtype, h.n, h.out, h.world = dtype, 4, DUMMY, 1
        h.bufs[0] = DUMMY
        if fn == "mvb_allreduce_fused":
            return lib.mvb_allreduce_fused(h, DUMMY, 0, None)
        return getattr(lib, fn)(h, None)
    return call


UPDATER_ENTRIES = {"mvb_add_dense_fused": _add_dense_fused, "mvb_updater_apply": _updater_apply,
                   "mvb_push_dense_stateful": _push_stateful, "mvb_add_rows_owner": _add_rows_owner,
                   "mvb_rowbox_apply": _rowbox_apply}
DTYPE_ENTRIES = {"mvb_add_dense_fused": lambda lib, dt: _add_dense_fused(lib, dt, N.UPD_DEFAULT),
                 "mvb_updater_apply": lambda lib, dt: _updater_apply(lib, dt, N.UPD_DEFAULT),
                 "mvb_push_dense_stateful": lambda lib, dt: _push_stateful(lib, dt, N.UPD_ADAGRAD),
                 "mvb_add_rows_owner": lambda lib, dt: _add_rows_owner(lib, dt, N.UPD_DEFAULT),
                 "mvb_get_dense": _get_dense, "mvb_push_dense_red": _push_red, "mvb_get_rows": _get_rows,
                 "mvb_add_rows_red": _add_rows_red, "mvb_row_nonzero_mask": _row_nonzero, "mvb_kv_add": _kv_add,
                 "mvb_kv_get": _kv_get, "mvb_kv_dump": _kv_dump, "mvb_kv_rehash": _kv_rehash,
                 **{fn: _allreduce(fn) for fn in ("mvb_allreduce_oneshot", "mvb_allreduce_twoshot",
                                                  "mvb_allreduce_fused")}}
SERVER_ENTRIES = {"mvb_push_dense_red": lambda lib, S: _push_red(lib, N.F32, S),
                  "mvb_push_dense_stateful": lambda lib, S: _push_stateful(lib, N.F32, N.UPD_ADAGRAD, S),
                  "mvb_kv_add": lambda lib, S: _kv_add(lib, N.F32, S),
                  "mvb_kv_get": lambda lib, S: _kv_get(lib, N.F32, S)}



def _cases():
    """case id -> (call, args) of every check below"""
    c = {}
    for fn, call in UPDATER_ENTRIES.items():
        for dt, name in ((N.F32, "f32"), (N.F64, "f64")):
            c[f"updater/{fn}/{name}"] = (call, (dt, BAD_UPDATER))
    for fn, call in DTYPE_ENTRIES.items():
        c[f"dtype/{fn}/{BAD_DTYPE}"] = (call, (BAD_DTYPE,))
    for dt in (N.I32, N.I64, N.I8):
        c[f"dtype/mvb_push_dense_stateful/{dt}"] = (DTYPE_ENTRIES["mvb_push_dense_stateful"], (dt,))
    for dt in (N.I64, N.I8):
        c[f"dtype/mvb_updater_apply/{dt}"] = (DTYPE_ENTRIES["mvb_updater_apply"], (dt,))
    for upd in (N.UPD_DEFAULT, N.UPD_SGD):
        c[f"stateless/mvb_push_dense_stateful/{upd}"] = (_push_stateful, (N.F32, upd))
    for fn, call in SERVER_ENTRIES.items():
        for S in (0, N.MAX_RANKS + 1):
            c[f"servers/{fn}/{S}"] = (call, (S,))
    for fn in ("mvb_kv_add", "mvb_kv_get", "mvb_kv_rehash"):
        for cap in (0, -16, 3, 48):
            c[f"capacity/{fn}/{cap}"] = (_kv_capacity(fn, cap), ())
    for fn in ("mvb_keys_add", "mvb_keys_get", "mvb_keys_collect"):
        for width in (0, -1, 17):
            c[f"width/{fn}/{width}"] = (_keys_width(fn, width), ())
    return c


def _codes():
    """The status of every case, or the message of any other exception."""
    lib, out = N.cuda_lib(), {}
    for cid, (call, args) in _cases().items():
        try:
            out[cid] = call(lib, *args)
        except N.NativeError as e:
            m = re.search(r"failed rc=(-?\d+):", str(e))
            out[cid] = int(m.group(1)) if m else str(e)
    return out


@pytest.fixture(scope="module")
def codes():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [str(Path(__file__).resolve())]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _ids(prefix):
    return sorted(k for k in _cases() if k.startswith(prefix))


@pytest.mark.parametrize("case", _ids("updater/"))
def test_unknown_updater_is_rejected(codes, case):
    assert codes[case] == -2


@pytest.mark.parametrize("case", _ids("dtype/"))
def test_unknown_element_type_is_rejected(codes, case):
    """-1 for an unknown code, and for a type outside an entry point's set: the one-sided stateful push serves f32
    and f64 only, and no updater entry point serves int64 or int8."""
    assert codes[case] == -1


@pytest.mark.parametrize("case", _ids("stateless/"))
def test_stateful_push_rejects_stateless_updaters(codes, case):
    assert codes[case] == -2


@pytest.mark.parametrize("case", _ids("servers/"))
def test_server_count_is_checked(codes, case):
    assert codes[case] == -3


@pytest.mark.parametrize("case", _ids("capacity/"))
def test_kv_capacity_is_checked(codes, case):
    assert codes[case] == -4


@pytest.mark.parametrize("case", _ids("width/"))
def test_key_table_width_is_checked(codes, case):
    assert codes[case] == -8


if __name__ == "__main__":
    print(json.dumps(_codes()))
