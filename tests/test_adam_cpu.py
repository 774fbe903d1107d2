"""The adam updater against an fp64 model, and its option and argument checks, without a GPU.

``AdamModel`` holds a table of rows of ``C`` elements, the moments ``m`` and ``v`` of every element and the step
count ``t`` of every row, in fp64, and steps a row with a delta row ``g`` as the server does
(include/multiverso/updater/adam_updater.h, ``Updater<MVB_UPD_ADAM>`` in csrc/cuda/mvb_common.cuh):

    t += 1 ;  gn = g / lr ;  m = b1 m + (1 - b1) gn ;  v = b2 v + (1 - b2) gn^2 ;
    d -= rho / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)

``b1`` (``momentum``), ``lr`` and ``rho`` are rounded to fp32 (they travel as fp32 fields), ``1 - b1`` is formed in
fp32, and ``b2 = 0.999``, ``1 - b2`` and ``eps = 1e-8`` are constants of the element type, as in the kernels and the
host updater. The state is shared by every worker, so a worker's delta is one more step of the row whoever sends it.
A repeated row of a row Add is one step per occurrence, in list order; ids outside the table are ignored.

Error bound. ``u`` is the unit roundoff of the element type. Every rounded operation is within ``u`` of its result.
* ``m`` is a convex recurrence: with ``mm = b1 mm + (1 - b1) |gn|`` (its magnitude, ``AdamModel.mm``), a step adds
  at most ``3 u mm`` (the quotient ``g / lr``, two products, one sum) and shrinks the earlier error by ``b1``, so
  after ``n`` steps ``|m - m_model| <= 3 n u mm``. ``v`` has non-negative terms: within ``4 n u v`` relative.
* The denominator ``sqrt(v) / c2 + eps`` (``c2`` the fp64 bias factor rounded once) is within ``(2 n + 4) u``
  relative, the factor ``a = rho / (1 - b1^t)`` within ``u``, and the quotient and product round twice. So step
  ``n`` of an element is within ``(3 n + 7) u a (mm + |m|) / den`` of the model's (``|m| <= mm``).
* The bias factors are formed in fp64 from ``pow``, which is within 2 fp64 ulp: ``1 - b^t`` then carries
  ``2^-51 b^t / (1 - b^t)`` relative, large at small ``t`` for ``b`` near 1 and negligible for fp32 tables. The
  step takes that error of ``1 - b1^t`` and half of that of ``1 - b2^t``.
* A step does not depend on ``d``, and ``d - step`` rounds once more (``u |d|``).
``AdamModel.err`` adds these per element over the steps; values must lie within ``4 err`` of the model (the factor
covers the model's own fp64 rounding, of the same order as the device's for fp64 tables). ``m`` is held to
``8 (n + 1) u mm``, ``v`` to ``8 (n + 1) u v`` and ``t`` exactly.
"""
import ctypes as C
import json
import os
import re
import subprocess
import sys
from pathlib import Path
from types import SimpleNamespace

if __name__ == "__main__":
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    sys.path.insert(0, str(Path(__file__).resolve().parent))

import numpy as np
import pytest
import torch

from test_table_numerics import _delta, _UNIT

B2, EPS, MAX_STEP = 0.999, 1e-8, 2 ** 24
# (beta1, learning_rate, rho) of consecutive Adds: beta1 0.9 (torch's default), 0 (RMSProp with bias correction),
# 0.5 and 0.99 (the largest bias factor at small t)
OPTS = [(0.9, 0.05, 0.01), (0.0, 0.02, 0.02), (0.5, 0.1, 0.005), (0.99, 0.03, 0.01), (0.9, 0.07, 0.001)]


def _f32(x):
    return float(np.float32(x))


def _o(b1, lr, rho):
    """An AddOption-like record, for the model alone."""
    return SimpleNamespace(momentum=b1, learning_rate=lr, rho=rho, worker_id=0)


def aopt(mv, k, worker_id=0):
    b1, lr, rho = OPTS[k % len(OPTS)]
    return mv.AddOption(worker_id=worker_id, momentum=b1, learning_rate=lr, rho=rho)


class AdamModel:
    """A table of ``num_col``-element rows with Adam's m, v per element and t per row, in fp64."""

    def __init__(self, start, num_col, dtype):
        self.npdt = np.dtype(dtype)
        self.u = _UNIT[self.npdt]
        self.data = np.asarray(start, dtype=np.float64).reshape(-1, num_col).copy()
        self.num_row, self.num_col = self.data.shape
        self.m = np.zeros(self.data.shape)
        self.v = np.zeros(self.data.shape)
        self.t = np.zeros(self.num_row, dtype=np.int64)
        self.mm = np.zeros(self.data.shape)                 # magnitude of m
        self.nupd = np.zeros(self.data.shape, dtype=np.int64)
        self.err = np.zeros(self.data.shape)                # the bound of the module docstring
        c = self.npdt.type
        self.b2, self.c2, self.eps = float(c(B2)), float(c(1.0 - B2)), float(c(EPS))

    def _step(self, r, g, opt):
        """One step of rows ``r`` (an index or a slice) with delta rows ``g``."""
        b1, lr, rho = _f32(opt.momentum), _f32(opt.learning_rate), _f32(opt.rho)
        c1 = float(np.float32(1.0) - np.float32(b1))
        gn = np.asarray(g, dtype=np.float64).reshape(self.data[r].shape) / lr
        t = np.minimum(self.t[r] + 1, MAX_STEP)
        self.t[r] = t
        t = np.asarray(t, dtype=np.float64)
        p1, p2 = b1 ** t, B2 ** t
        a = rho / (1.0 - p1)
        bc2 = np.sqrt(1.0 - p2)
        eb = 2.0 ** -51 * (p1 / (1.0 - p1) + 0.5 * p2 / (1.0 - p2))
        if gn.ndim == 2:
            a, bc2, eb = a[:, None], bc2[:, None], eb[:, None]
        m = b1 * self.m[r] + c1 * gn
        v = self.b2 * self.v[r] + self.c2 * gn * gn
        mm = b1 * self.mm[r] + c1 * np.abs(gn)
        den = np.sqrt(v) / bc2 + self.eps
        step = a * m / den
        n = self.nupd[r] + 1
        self.m[r], self.v[r], self.mm[r], self.nupd[r] = m, v, mm, n
        self.data[r] -= step
        self.err[r] += (3 * n + 7) * self.u * a * (mm + np.abs(m)) / den + np.abs(step) * eb \
            + self.u * np.abs(self.data[r])

    def add(self, delta, opt):
        self._step(slice(None), np.asarray(delta, dtype=np.float64).reshape(self.data.shape), opt)

    def add_rows(self, ids, vals, opt):
        vals = np.asarray(vals, dtype=np.float64).reshape(len(ids), self.num_col)
        for i, r in enumerate(np.asarray(ids).tolist()):
            if 0 <= r < self.num_row:
                self._step(r, vals[i], opt)

    def check_values(self, got, what, rows=None):
        sel = slice(None) if rows is None else rows
        got = np.asarray(got, dtype=np.float64).reshape(self.data.shape)[sel]
        _within(got, self.data[sel], 4.0 * self.err[sel], f"{what} values")

    def check_state(self, m, v, t, what, rows=None):
        """m and v (``num_row x num_col`` elements) and t (``num_row``) against the model."""
        sel = slice(None) if rows is None else rows
        n = (self.nupd + 1)[sel]
        m = np.asarray(m, dtype=np.float64).reshape(-1)[:self.data.size].reshape(self.data.shape)[sel]
        v = np.asarray(v, dtype=np.float64).reshape(-1)[:self.data.size].reshape(self.data.shape)[sel]
        _within(m, self.m[sel], 8.0 * n * self.u * self.mm[sel], f"{what} m")
        _within(v, self.v[sel], 8.0 * n * self.u * self.v[sel], f"{what} v")
        t = np.asarray(t, dtype=np.float64).reshape(-1)[:self.num_row][sel]
        assert np.array_equal(t, self.t[sel].astype(np.float64)), f"{what} t: {t} != {self.t[sel]}"


def _within(got, ref, bound, what):
    bad = ~(np.abs(got - ref) <= bound)
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, np.abs(got - ref) - bound, -np.inf)), ref.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound; worst at {i}: "
                             f"got {got[i]!r} model {ref[i]!r} bound {bound[i]:.3g}")


# ----------------------------------------------------------------------------------- the model itself
def _torch_adam_run(start, grads, lr, b1, dtype):
    """torch.optim.Adam(lr, betas=(b1, 0.999), eps=1e-8) on a parameter stepped with ``grads`` in turn."""
    p = torch.nn.Parameter(torch.tensor(start, dtype=dtype))
    opt = torch.optim.Adam([p], lr=lr, betas=(b1, B2), eps=EPS, foreach=False)
    for g in grads:
        p.grad = torch.tensor(g, dtype=dtype)
        opt.step()
    return p.detach().numpy().astype(np.float64), opt.state[p]


@pytest.mark.parametrize("b1", [0.9, 0.5, 0.0])
def test_model_is_torch_adam(b1):
    """A single worker's sequence of whole-table steps, pushed as delta = lr * grad, is torch.optim.Adam with
    lr = rho (fp64 throughout: 1e-12 relative)."""
    rng = np.random.default_rng(4)
    start = rng.uniform(-1, 1, (6, 5))
    grads = [rng.normal(0, 10.0 ** rng.uniform(-3, 1), start.shape) for _ in range(30)]
    b1 = _f32(b1)
    lr, rho = _f32(0.125), _f32(0.01)
    model = AdamModel(start, 5, "float64")
    for g in grads:
        model.add(g * lr, _o(b1, lr, rho))
    ref, st = _torch_adam_run(start, grads, rho, b1, torch.float64)
    np.testing.assert_allclose(model.data, ref, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(model.m, st["exp_avg"].numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(model.v, st["exp_avg_sq"].numpy(), rtol=1e-12, atol=1e-20)
    assert (model.t == 30).all() and float(st["step"]) == 30


def test_late_row_gets_a_bias_corrected_first_step():
    """The step count is per row: a row first stepped after 1000 steps of another row moves by about rho (Adam's
    first step), not by about 3 rho as a table-wide count would give at beta1 0.9."""
    O = _o(_f32(0.9), _f32(0.1), _f32(0.01))
    model = AdamModel(np.zeros((2, 4)), 4, "float32")
    for _ in range(1000):
        model.add_rows([0], np.full((1, 4), 0.01), O)
    model.add_rows([1], np.full((1, 4), 0.01), O)
    assert model.t.tolist() == [1000, 1]
    np.testing.assert_allclose(model.data[1], -O.rho, rtol=1e-6)


def test_step_count_stops_at_two_to_the_24():
    O = _o(_f32(0.9), _f32(0.1), _f32(0.01))
    model = AdamModel(np.zeros((1, 1)), 1, "float32")
    model.t[:] = MAX_STEP - 1
    model.add([[0.01]], O)
    model.add([[0.01]], O)
    assert model.t[0] == MAX_STEP


# ----------------------------------------------------------------------------------- host runtime
@pytest.fixture
def host_backend():
    """The host runtime (libmultiverso.so) at world size 1 with ``-updater_type=adam``."""
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.FLAGS.set("updater_type", "adam")
    mv.init()
    yield mv
    mv.shutdown(finalize_net=False)
    mv.FLAGS.reset()
    # the C++ flag registry outlives the runtime: later tests of this process start with the default updater
    from multiverso_b200 import host
    host._lib().MV_SetFlagString(b"updater_type", b"default")


def _repeated_ids(rng, num_row, reps):
    """A shuffled id list: row 0 ``reps`` times, the last row twice, and a few unique rows in between."""
    hot = [0, num_row - 1] if num_row > 1 else [0]
    others = np.setdiff1d(np.arange(num_row), hot)
    uniq = rng.choice(others, min(len(others), 6), replace=False) if len(others) else np.zeros(0, np.int64)
    ids = np.concatenate([np.repeat(hot, [reps, 2][:len(hot)]), uniq])
    return rng.permutation(ids).astype(np.int64)


def _host_steps(mv, t, model, rng, rows, cols, dtype, steps=6):
    for k in range(steps):
        opt = aopt(mv, k)
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
    model = AdamModel(t.get(), cols, dtype)
    _host_steps(mv, t, model, rng, rows, cols, dtype)
    model.check_values(t.get(), f"host MatrixTable C={cols} {dtype}")


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_host_array_table_matches_model(host_backend, dtype):
    """An ArrayTable has rows of one element, so every element has its own step count. The master-init Add of
    ``init_value`` is the first step."""
    mv = host_backend
    rng = np.random.default_rng(8)
    n = 11
    a = mv.ArrayTable(n, dtype, init_value=0.75)
    model = AdamModel(np.zeros(n), 1, dtype)
    model.add(np.full(n, 0.75), mv.AddOption(worker_id=0))
    for k in range(5):
        d = _delta(rng, (n,), dtype)
        a.add(d, aopt(mv, k))
        model.add(d, aopt(mv, k))
    model.check_values(a.get(), f"host ArrayTable {dtype}")


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_host_store_load_roundtrip(host_backend, tmp_path, dtype):
    """save_table writes the shard, then m, v and t, which match the model; a table loaded from it continues
    bitwise like the table that wrote it."""
    mv = host_backend
    rng = np.random.default_rng(12)
    rows, cols = 17, 6
    t = mv.MatrixTable(rows, cols, dtype, min_value=-1.0, max_value=1.0)
    model = AdamModel(t.get(), cols, dtype)
    _host_steps(mv, t, model, rng, rows, cols, dtype, steps=4)
    uri = str(tmp_path / "ck")
    assert mv.save_table(t, uri)
    raw = np.frombuffer(Path(f"{uri}.shard0").read_bytes(), dtype=dtype)
    n = rows * cols
    assert raw.size == 3 * n + rows
    model.check_state(raw[n:2 * n], raw[2 * n:3 * n], raw[3 * n:], "host checkpoint")
    t2 = mv.MatrixTable(rows, cols, dtype)
    assert mv.load_table(t2, uri)
    assert np.array_equal(t2.get(), t.get())
    d = _delta(rng, (rows, cols), dtype)
    ids = np.array([3, 3, 16], dtype=np.int64)
    v = _delta(rng, (3, cols), dtype)
    for tab in (t, t2):
        tab.add(d, aopt(mv, 4))
        tab.add_rows(ids, v, aopt(mv, 0))
    assert np.array_equal(t2.get(), t.get())


def test_host_matches_torch_adam(host_backend):
    """A single-worker sequence on the host runtime against CPU torch.optim.Adam (fp64 tables, 1e-10 relative)."""
    mv = host_backend
    rng = np.random.default_rng(21)
    rows, cols = 9, 4
    t = mv.MatrixTable(rows, cols, "float64", min_value=-1.0, max_value=1.0)
    start = t.get().reshape(rows, cols).copy()
    lr, rho, b1 = 0.125, 0.01, 0.9
    grads = [rng.normal(0, 1, (rows, cols)) for _ in range(20)]
    for g in grads:
        t.add(g * lr, mv.AddOption(worker_id=0, momentum=b1, learning_rate=lr, rho=rho))
    ref, _ = _torch_adam_run(start, grads, _f32(rho), _f32(b1), torch.float64)
    np.testing.assert_allclose(t.get().reshape(rows, cols), ref, rtol=1e-10, atol=1e-12)


# ----------------------------------------------------------------------------------- option checks
BAD_OPTS = {"beta1=1": (1.0, 0.1, 0.01), "beta1<0": (-0.1, 0.1, 0.01), "beta1 rounds to 1": (0.99999999, 0.1, 0.01),
            "lr=0": (0.9, 0.0, 0.01), "lr<0": (0.9, -0.1, 0.01), "rho<0": (0.9, 0.1, -0.01),
            "nan": (float("nan"), 0.1, 0.01)}


@pytest.mark.parametrize("case", sorted(BAD_OPTS))
def test_option_check(case):
    from multiverso_b200.tables.options import AddOption, check_add_option
    b1, lr, rho = BAD_OPTS[case]
    with pytest.raises(ValueError, match="adam needs"):
        check_add_option("adam", AddOption(worker_id=0, momentum=b1, learning_rate=lr, rho=rho))
    check_add_option("adagrad", AddOption(worker_id=0, momentum=b1, learning_rate=lr, rho=rho))
    check_add_option("adam", AddOption(worker_id=0, momentum=0.9, learning_rate=0.1, rho=0.0))


def test_host_option_check_raises(host_backend):
    """The host backend raises ValueError before the request leaves Python; the table is unchanged."""
    mv = host_backend
    t = mv.MatrixTable(3, 4, "float32", min_value=-1.0, max_value=1.0)
    a = mv.ArrayTable(5, "float32")
    before = t.get().copy()
    bad = mv.AddOption(worker_id=0, momentum=1.0, learning_rate=0.1, rho=0.01)
    with pytest.raises(ValueError):
        t.add(np.ones((3, 4), np.float32), bad)
    with pytest.raises(ValueError):
        t.add_rows(np.array([1]), np.ones((1, 4), np.float32), bad)
    with pytest.raises(ValueError):
        a.add(np.ones(5, np.float32), mv.AddOption(worker_id=0, momentum=0.9, learning_rate=0.0, rho=0.01))
    assert np.array_equal(t.get(), before)


_CHECK_CHILD = r"""
import sys
sys.path.insert(0, sys.argv[1])
import ctypes as C
import numpy as np
import multiverso_b200 as mv
from multiverso_b200 import host
mv.FLAGS.set("updater_type", "adam")
mv.init()
a = mv.ArrayTable(4, "float32")
data = np.ones(4, np.float32)
opt = mv.AddOption(worker_id=0, momentum=float(sys.argv[2]), learning_rate=float(sys.argv[3]), rho=float(sys.argv[4]))
host._lib().MV_AddArrayTable64(a.handle, a.code, data.ctypes.data_as(C.c_void_p), C.c_int64(4), opt.pack(), 0)
print("APPLIED", flush=True)
"""


@pytest.mark.parametrize("case", ["beta1=1", "lr=0", "rho<0", "ok"])
def test_host_runtime_check(case):
    """The host runtime's own CHECK, reached through the C API without the Python check: a bad option stops the
    process with 'Check failed', a good one is applied."""
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    b1, lr, rho = BAD_OPTS.get(case, (0.9, 0.1, 0.01))
    root = str(Path(__file__).resolve().parents[1])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHECK_CHILD, root, str(b1), str(lr),
                                                                           str(rho)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    out = r.stdout + r.stderr
    if case == "ok":
        assert r.returncode == 0 and "APPLIED" in out, out[-2000:]
    else:
        assert r.returncode != 0 and "APPLIED" not in out and "Check failed" in out, out[-2000:]


# ----------------------------------------------------------------------------------- argument codes
DUMMY = 1 << 12          # 16-byte aligned, never dereferenced


def _fused(lib, dtype, num_col, shard_len=8, state_stride=8):
    from multiverso_b200 import _native as N
    a = N.DenseAdd()
    a.dtype, a.updater, a.shard, a.state0, a.state1 = dtype, N.UPD_ADAM, DUMMY, DUMMY, DUMMY
    a.shard_len, a.state_stride, a.num_col = shard_len, state_stride, num_col
    a.nworkers, a.worker_mask, a.world = 1, 1, 1
    a.delta_ptrs[0] = DUMMY
    return lib.mvb_add_dense_fused(a, None)


def _push_adam(lib, dtype, upd, S=1, num_col=2, lens=8, stride=8):
    from multiverso_b200 import _native as N
    vp = (C.c_void_p * N.MAX_RANKS)(*([DUMMY] * N.MAX_RANKS))
    offs = (C.c_int64 * N.MAX_RANKS)(*([0] * N.MAX_RANKS))
    ln = (C.c_int64 * N.MAX_RANKS)(*([lens] * N.MAX_RANKS))
    st = (C.c_int64 * N.MAX_RANKS)(*([stride] * N.MAX_RANKS))
    return lib.mvb_push_dense_adam(dtype, upd, DUMMY, S, vp, vp, vp, offs, ln, st, num_col, N.AddOpt(), 0, None)


def _rows_owner(lib, dtype, state_stride):
    from multiverso_b200 import _native as N
    return lib.mvb_add_rows_owner(dtype, N.UPD_ADAM, DUMMY, DUMMY, DUMMY, 0, 4, 4, state_stride, DUMMY, 1, DUMMY, 4,
                                  N.AddOpt(), None)


def _evict_ex(lib, state2_row):
    from multiverso_b200 import _native as N
    h = N.HashRows()
    h.nservers, h.slots = 1, 4
    h.map.num_row, h.map.num_col, h.map.nservers, h.map.rows_per_server = 5, 4, 1, 5
    work = (C.c_int64 * 8)()
    return lib.mvb_hash_rows_evict_ex(h, 0, -2 ** 63, DUMMY, DUMMY, 1, 16, 4, DUMMY, C.addressof(work), None, DUMMY,
                                      state2_row)


def _cases():
    from multiverso_b200 import _native as N
    A = N.UPD_ADAM
    vp = (C.c_void_p * N.MAX_RANKS)(*([DUMMY] * N.MAX_RANKS))
    i64 = (C.c_int64 * N.MAX_RANKS)(*([4] * N.MAX_RANKS))
    c = {}
    for dt, name in ((N.F32, "f32"), (N.F64, "f64")):
        c[f"norows/mvb_updater_apply/{name}"] = (
            lambda lib, dt=dt: lib.mvb_updater_apply(dt, A, DUMMY, DUMMY, DUMMY, DUMMY, 4, N.AddOpt(), 1.0, None), -2)
        c[f"norows/mvb_push_dense_stateful/{name}"] = (
            lambda lib, dt=dt: lib.mvb_push_dense_stateful(dt, A, DUMMY, 1, vp, vp, vp, i64, i64, i64, N.AddOpt(), 0,
                                                           None), -2)
        c[f"norows/mvb_push_dense_rowwise/{name}"] = (
            lambda lib, dt=dt: lib.mvb_push_dense_rowwise(dt, A, DUMMY, 1, vp, vp, i64, i64, i64, 2, N.AddOpt(), 0,
                                                          None), -2)
        # num_col < 1, a shard that is not whole rows, a state stride below the shard's elements
        for tag, kw in (("num_col0", dict(num_col=0)), ("num_col-1", dict(num_col=-1)),
                        ("partial_row", dict(num_col=3)), ("short_stride", dict(num_col=2, state_stride=7))):
            c[f"geometry/mvb_add_dense_fused/{name}/{tag}"] = (lambda lib, dt=dt, kw=kw: _fused(lib, dt, **kw),
                                                               N.BAD_ROW_MAP)
            pkw = {"num_col": kw["num_col"]}
            if "state_stride" in kw:
                pkw["stride"] = kw["state_stride"]
            c[f"geometry/mvb_push_dense_adam/{name}/{tag}"] = (
                lambda lib, dt=dt, pkw=pkw: _push_adam(lib, dt, A, **pkw), N.BAD_ROW_MAP)
        c[f"geometry/mvb_add_rows_owner/{name}"] = (lambda lib, dt=dt: _rows_owner(lib, dt, 15), N.BAD_ROW_MAP)
        # valid geometry passes the checks and reaches the launch, which fails without a device
        c[f"launch/mvb_add_dense_fused/{name}"] = (lambda lib, dt=dt: _fused(lib, dt, 2), "cuda")
        c[f"launch/mvb_push_dense_adam/{name}"] = (lambda lib, dt=dt: _push_adam(lib, dt, A), "cuda")
        c[f"launch/mvb_add_rows_owner/{name}"] = (lambda lib, dt=dt: _rows_owner(lib, dt, 16), "cuda")
        for upd in (N.UPD_DEFAULT, N.UPD_SGD, N.UPD_MOMENTUM, N.UPD_ADAGRAD, N.UPD_DCASGD, N.UPD_DCASGDA,
                    N.UPD_ROWWISE_ADAGRAD, 6):
            c[f"updater/mvb_push_dense_adam/{name}/{upd}"] = (lambda lib, dt=dt, upd=upd: _push_adam(lib, dt, upd), -2)
    for dt in (N.I32, N.I64, N.I8, 99):
        c[f"dtype/mvb_push_dense_adam/{dt}"] = (lambda lib, dt=dt: _push_adam(lib, dt, A), -1)
    for S in (0, N.MAX_RANKS + 1):
        c[f"servers/mvb_push_dense_adam/{S}"] = (lambda lib, S=S: _push_adam(lib, N.F32, A, S=S), -3)
    for r in (0, -1):
        c[f"state2_row/mvb_hash_rows_evict_ex/{r}"] = (lambda lib, r=r: _evict_ex(lib, r), -6)
    c["launch/mvb_hash_rows_evict_ex"] = (lambda lib: _evict_ex(lib, 1), "cuda")
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
    assert re.search(r"MVB_UPD_ADAM\s*=\s*8\b", hdr)
    assert N.UPD_ADAM == 8 and N.UPDATER_NAMES["adam"] == 8
    assert 6 not in N.UPDATER_NAMES.values()


if __name__ == "__main__":
    print(json.dumps(_codes()))
