"""The rowwise_adagrad updater against an fp64 model, and its argument checks, without a GPU.

``RowwiseModel`` holds a table of rows of ``C`` elements and one accumulator per (worker, row) in fp64 and applies
worker ``w``'s delta row ``g`` to row ``r`` as the server does (include/multiverso/updater/rowwise_adagrad_updater.h,
``Updater<MVB_UPD_ROWWISE_ADAGRAD>`` in csrc/cuda/mvb_common.cuh):

    gn_j = g_j / lr ;  h[w, r] += (1/C) sum_j gn_j^2 ;  d_j -= rho / sqrt(h[w, r] + 1e-6) * gn_j

with ``lr`` and ``rho`` rounded to fp32 (they travel as ``MvbAddOpt`` / ``AddOption`` fp32 fields) and 1e-6 a
constant of the element type. A repeated row of a row Add is stepped once per occurrence in list order; ids outside
the table are ignored.

Error bound. ``u`` is the unit roundoff of the element type (2^-24, 2^-53). The square sum is the one term that
grows with the row: ``C`` terms ``fl(fl(g_j / lr)^2)`` (each within ``3 u`` relative) are added by the host in a
chain of ``C`` additions and by the device in lane partials of at most ``ceil(C / 32)`` terms followed by the five
levels of the xor tree, so both are within ``(C + 3) u`` relative of the exact sum (the terms are non-negative,
so relative errors of partial sums never exceed that of the whole). Dividing by ``C`` and adding it to ``h`` adds
``2 u``; ``h`` is a sum of non-negative increments, so after ``n`` steps it is within ``(C + 3 + 2 n) u`` of the
model, relative. The factor ``rho * rsqrt(h + eps)`` takes half of ``h``'s relative error plus at most ``4 u``
(``rsqrtf`` is within 2 ulp; the host's ``sqrt`` and division round twice), and the step ``f * gn`` adds ``2 u``,
so a step is within ``(C / 2 + n + 8) u`` of its model value, relative. ``d - step`` rounds once more, within
``u (|d| + |step|)``. A step does not depend on ``d``, so the error of ``d`` after ``n`` steps is the sum of the
step errors, below ``(C + 2 n + 10) u (|ref| + M)`` with ``M`` the start value's magnitude plus the sum of the
step magnitudes (``RowwiseModel.mag``). The tests allow ``8 (n + C + 2) u`` times that scale, for values and for
every accumulator (scale: its own model value); the model's own fp64 rounding is far inside that for fp32 and of
the same order as the device's for fp64, which the factor 8 covers.
"""
import ctypes as C
import json
import os
import re
import subprocess
import sys
from pathlib import Path

if __name__ == "__main__":
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    sys.path.insert(0, str(Path(__file__).resolve().parent))

import numpy as np
import pytest
import torch

from test_table_numerics import _assert_close, _delta, _opt, _UNIT

EPS = 1e-6


def _f32(x):
    return float(np.float32(x))


class RowwiseModel:
    """A table of ``num_col``-element rows and one accumulator per (worker, row), in fp64."""

    def __init__(self, start, num_col, dtype, workers=1):
        self.npdt = np.dtype(dtype)
        self.data = np.asarray(start, dtype=np.float64).reshape(-1, num_col).copy()
        self.num_row, self.num_col = self.data.shape
        self.h = np.zeros((workers, self.num_row))
        self.hn = np.zeros((workers, self.num_row), dtype=np.int64)   # steps taken by each accumulator
        self.mag = np.abs(self.data)                                   # |start| + sum of |steps|, per element
        self.nupd = np.zeros(self.data.shape, dtype=np.int64)
        self.eps = float(self.npdt.type(EPS))

    def _step(self, r, g, opt):
        """Worker ``opt.worker_id`` steps rows ``r`` (an index or a slice) with delta rows ``g``."""
        lr, rho, w = _f32(opt.learning_rate), _f32(opt.rho), opt.worker_id
        gn = np.asarray(g, dtype=np.float64).reshape(self.data[r].shape) / lr
        h = self.h[w, r] + (gn * gn).mean(axis=-1)
        f = rho / np.sqrt(h + self.eps)
        step = np.asarray(f)[..., None] * gn if gn.ndim == 2 else f * gn
        self.h[w, r] = h
        self.hn[w, r] += 1
        self.data[r] -= step
        self.mag[r] += np.abs(step)
        self.nupd[r] += 1

    def add(self, delta, opt):
        self._step(slice(None), np.asarray(delta, dtype=np.float64).reshape(self.data.shape), opt)

    def add_rows(self, ids, vals, opt):
        vals = np.asarray(vals, dtype=np.float64).reshape(len(ids), self.num_col)
        for i, r in enumerate(np.asarray(ids).tolist()):
            if 0 <= r < self.num_row:
                self._step(r, vals[i], opt)

    def bound_n(self):
        """The update count of the module docstring's bound: n + C + 2."""
        return self.nupd + self.num_col + 2

    def check_values(self, got, dtype, what, rows=None):
        sel = slice(None) if rows is None else rows
        got = np.asarray(got, dtype=np.float64).reshape(self.data.shape)
        _assert_close(got[sel], self.data[sel], (np.abs(self.data) + self.mag)[sel], self.bound_n()[sel], dtype,
                      f"{what} values")

    def check_state(self, got, w, dtype, what):
        """Worker ``w``'s accumulators (``num_row`` values) against the model."""
        got = np.asarray(got, dtype=np.float64).reshape(-1)[:self.num_row]
        _assert_close(got, self.h[w], self.h[w], self.hn[w] + self.num_col + 2, dtype,
                      f"{what} state[worker {w}]")


def test_model_is_adagrad_at_one_column():
    """At C = 1 the model is AdaGrad's rule, element by element."""
    from test_table_numerics import ServerModel
    import multiverso_b200 as mv
    rng = np.random.default_rng(3)
    start = rng.uniform(-1, 1, 40)
    a, b = ServerModel(start, 1, "adagrad", "float64"), RowwiseModel(start, 1, "float64")
    for k in range(4):
        d = _delta(rng, (40,), "float64")
        a.add(d, _opt(mv, k))
        b.add(d, _opt(mv, k))
    np.testing.assert_allclose(b.data, a.data, rtol=1e-13, atol=0)
    np.testing.assert_allclose(b.h[0], a.state[0][0].reshape(-1), rtol=1e-13, atol=0)


# ----------------------------------------------------------------------------------- host runtime
@pytest.fixture
def host_backend():
    """The host runtime (libmultiverso.so) at world size 1 with ``-updater_type=rowwise_adagrad``."""
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.FLAGS.set("updater_type", "rowwise_adagrad")
    mv.init()
    yield mv
    mv.shutdown(finalize_net=False)
    mv.FLAGS.reset()


def _repeated_ids(rng, num_row, reps):
    """A shuffled id list: row 0 ``reps`` times, the last row twice, and a few unique rows in between."""
    hot = [0, num_row - 1] if num_row > 1 else [0]
    others = np.setdiff1d(np.arange(num_row), hot)
    uniq = rng.choice(others, min(len(others), 6), replace=False) if len(others) else np.zeros(0, np.int64)
    ids = np.concatenate([np.repeat(hot, [reps, 2][:len(hot)]), uniq])
    return rng.permutation(ids).astype(np.int64)


def _host_steps(mv, t, model, rng, rows, cols, dtype, steps=6):
    for k in range(steps):
        opt = _opt(mv, k)
        if k % 2 == 0:
            d = _delta(rng, (rows, cols), dtype)
            t.add(d, opt)
            model.add(d, opt)
        else:
            ids = _repeated_ids(rng, rows, 5 + k)
            v = _delta(rng, (ids.size, cols), dtype)
            t.add_rows(ids, v, opt)
            model.add_rows(ids, v, opt)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("cols", [1, 5, 37])
def test_host_matrix_table_matches_model(host_backend, cols, dtype):
    """Whole-table Adds interleaved with row Adds that repeat rows, the AddOption changing at every step."""
    mv = host_backend
    rng = np.random.default_rng(cols)
    rows = 23
    t = mv.MatrixTable(rows, cols, dtype, min_value=-1.0, max_value=1.0)
    model = RowwiseModel(t.get(), cols, dtype)
    _host_steps(mv, t, model, rng, rows, cols, dtype)
    model.check_values(t.get(), dtype, f"host MatrixTable C={cols} {dtype}")


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_host_array_table_matches_model(host_backend, dtype):
    """An ArrayTable has rows of one element: its updater is AdaGrad, one accumulator per element."""
    mv = host_backend
    rng = np.random.default_rng(8)
    n = 11
    a = mv.ArrayTable(n, dtype, init_value=0.75)
    model = RowwiseModel(np.zeros(n), 1, dtype)
    model.add(np.full(n, 0.75), mv.AddOption(worker_id=0))
    for k in range(5):
        d = _delta(rng, (n,), dtype)
        a.add(d, _opt(mv, k))
        model.add(d, _opt(mv, k))
    model.check_values(a.get(), dtype, f"host ArrayTable {dtype}")


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_host_store_load_roundtrip(host_backend, tmp_path, dtype):
    """save_table writes the shard and then one accumulator per (worker, row), which match the model; a table
    loaded from it continues bitwise like the table that wrote it."""
    mv = host_backend
    rng = np.random.default_rng(12)
    rows, cols = 17, 6
    t = mv.MatrixTable(rows, cols, dtype, min_value=-1.0, max_value=1.0)
    model = RowwiseModel(t.get(), cols, dtype)
    _host_steps(mv, t, model, rng, rows, cols, dtype, steps=4)
    uri = str(tmp_path / "ck")
    assert mv.save_table(t, uri)
    raw = Path(f"{uri}.shard0").read_bytes()
    esz = np.dtype(dtype).itemsize
    assert len(raw) == (rows * cols + mv.num_workers() * rows) * esz
    model.check_state(np.frombuffer(raw[rows * cols * esz:], dtype=dtype), 0, dtype, "host checkpoint")
    t2 = mv.MatrixTable(rows, cols, dtype)
    assert mv.load_table(t2, uri)
    assert np.array_equal(t2.get(), t.get())
    d = _delta(rng, (rows, cols), dtype)
    ids = np.array([3, 3, 16], dtype=np.int64)
    v = _delta(rng, (3, cols), dtype)
    for tab in (t, t2):
        tab.add(d, _opt(mv, 4))
        tab.add_rows(ids, v, _opt(mv, 5))
    assert np.array_equal(t2.get(), t.get())


# ----------------------------------------------------------------------------------- argument codes
DUMMY = 1 << 12          # 16-byte aligned, never dereferenced


def _fused(lib, dtype, num_col, shard_len=8, state_stride=8):
    from multiverso_b200 import _native as N
    a = N.DenseAdd()
    a.dtype, a.updater, a.shard, a.state0 = dtype, N.UPD_ROWWISE_ADAGRAD, DUMMY, DUMMY
    a.shard_len, a.state_stride, a.num_col = shard_len, state_stride, num_col
    a.nworkers, a.worker_mask, a.world = 1, 1, 1
    a.delta_ptrs[0] = DUMMY
    return lib.mvb_add_dense_fused(a, None)


def _push_rowwise(lib, dtype, upd, S=1, num_col=2, lens=8, stride=4):
    from multiverso_b200 import _native as N
    vp = (C.c_void_p * N.MAX_RANKS)(*([DUMMY] * N.MAX_RANKS))
    offs = (C.c_int64 * N.MAX_RANKS)(*([0] * N.MAX_RANKS))
    ln = (C.c_int64 * N.MAX_RANKS)(*([lens] * N.MAX_RANKS))
    st = (C.c_int64 * N.MAX_RANKS)(*([stride] * N.MAX_RANKS))
    return lib.mvb_push_dense_rowwise(dtype, upd, DUMMY, S, vp, vp, offs, ln, st, num_col, N.AddOpt(), 0, None)


def _cases():
    from multiverso_b200 import _native as N
    R = N.UPD_ROWWISE_ADAGRAD
    vp = (C.c_void_p * N.MAX_RANKS)(*([DUMMY] * N.MAX_RANKS))
    i64 = (C.c_int64 * N.MAX_RANKS)(*([4] * N.MAX_RANKS))
    c = {}
    for dt, name in ((N.F32, "f32"), (N.F64, "f64")):
        c[f"norows/mvb_updater_apply/{name}"] = (
            lambda lib, dt=dt: lib.mvb_updater_apply(dt, R, DUMMY, DUMMY, DUMMY, DUMMY, 4, N.AddOpt(), 1.0, None), -2)
        c[f"norows/mvb_push_dense_stateful/{name}"] = (
            lambda lib, dt=dt: lib.mvb_push_dense_stateful(dt, R, DUMMY, 1, vp, vp, vp, i64, i64, i64, N.AddOpt(), 0,
                                                           None), -2)
        # num_col < 1, a shard that is not whole rows, a state stride below the row count
        for tag, kw in (("num_col0", dict(num_col=0)), ("num_col-1", dict(num_col=-1)),
                        ("partial_row", dict(num_col=3)), ("short_stride", dict(num_col=2, state_stride=3))):
            c[f"geometry/mvb_add_dense_fused/{name}/{tag}"] = (lambda lib, dt=dt, kw=kw: _fused(lib, dt, **kw),
                                                               N.BAD_ROW_MAP)
            pkw = {"num_col": kw["num_col"]}
            if "state_stride" in kw:
                pkw["stride"] = kw["state_stride"]
            c[f"geometry/mvb_push_dense_rowwise/{name}/{tag}"] = (
                lambda lib, dt=dt, pkw=pkw: _push_rowwise(lib, dt, R, **pkw), N.BAD_ROW_MAP)
        # valid geometry passes the checks and reaches the launch, which fails without a device
        c[f"launch/mvb_add_dense_fused/{name}"] = (lambda lib, dt=dt: _fused(lib, dt, 2, state_stride=4), "cuda")
        c[f"launch/mvb_push_dense_rowwise/{name}"] = (lambda lib, dt=dt: _push_rowwise(lib, dt, R), "cuda")
        for upd in (N.UPD_DEFAULT, N.UPD_SGD, N.UPD_MOMENTUM, N.UPD_ADAGRAD, N.UPD_DCASGD, N.UPD_DCASGDA, 6):
            c[f"updater/mvb_push_dense_rowwise/{name}/{upd}"] = (
                lambda lib, dt=dt, upd=upd: _push_rowwise(lib, dt, upd), -2)
    for dt in (N.I32, N.I64, N.I8, 99):
        c[f"dtype/mvb_push_dense_rowwise/{dt}"] = (lambda lib, dt=dt: _push_rowwise(lib, dt, R), -1)
    for S in (0, N.MAX_RANKS + 1):
        c[f"servers/mvb_push_dense_rowwise/{S}"] = (lambda lib, S=S: _push_rowwise(lib, N.F32, R, S=S), -3)
    return c


def _codes():
    from multiverso_b200 import _native as N
    lib, out = N.cuda_lib(), {}
    for cid, (call, _) in _cases().items():
        try:
            out[cid] = call(lib)
        except N.NativeError as e:
            m = re.search(r"failed rc=(-?\d+):", str(e))
            out[cid] = int(m.group(1)) if m else str(e)
    return out


@pytest.fixture(scope="module")
def codes():
    """The codes, from a child process that sees no CUDA device: a check that stopped working returns a CUDA error
    instead of launching a kernel on the dummy pointers."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [str(Path(__file__).resolve())]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("case", sorted(_cases()))
def test_argument_codes(codes, case):
    want = _cases()[case][1]
    if want == "cuda":
        assert isinstance(codes[case], int) and codes[case] > 0, codes[case]
    else:
        assert codes[case] == want, codes[case]


def test_updater_code_matches_header():
    from multiverso_b200 import _native as N
    hdr = (Path(__file__).resolve().parents[1] / "csrc" / "cuda" / "mvb200.h").read_text()
    assert re.search(r"MVB_UPD_ROWWISE_ADAGRAD\s*=\s*7\b", hdr)
    assert N.UPD_ROWWISE_ADAGRAD == 7 and N.UPDATER_NAMES["rowwise_adagrad"] == 7
    assert 6 not in N.UPDATER_NAMES.values()


if __name__ == "__main__":
    print(json.dumps(_codes()))
