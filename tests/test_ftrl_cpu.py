"""The ftrl updater against an fp64 model, and its option and argument checks, without a GPU.

``FtrlModel`` holds a table of rows of ``C`` elements and FTRL-Proximal's ``z`` and ``n`` of every element, in fp64,
and steps an element with a delta ``delta`` as the server does (include/multiverso/updater/ftrl_updater.h,
``Updater<MVB_UPD_FTRL>`` in csrc/cuda/mvb_common.cuh), with ``alpha = rho``, ``l1 = lambda_``, ``l2 = momentum`` and
``beta = 1``, in this operation order:

    g = delta / lr ;  if g == 0: nothing changes
    sigma = g^2 / (alpha (sqrt(n + g^2) + sqrt(n))) ;  z += g - sigma d ;  n += g^2 ;
    d = |z| <= l1 ? 0 : (sign(z) l1 - z) / ((beta + sqrt(n)) / alpha + l2)

The options are rounded to fp32 (they travel as fp32 fields). The state is shared by every worker, so a worker's
delta is one more step of the element whoever sends it. A repeated row of a row Add is one step per occurrence, in
list order; ids outside the table are ignored.

Error bound. ``u`` is the unit roundoff of the element type; every rounded operation is within ``u`` of its result.
For one step of an element, with ``ez``, ``en`` and ``ed`` the bounds on the device's z, n and d before the step:
* ``g`` is within ``u |g|``. ``n`` is a sum of non-negative terms: each step adds ``g^2`` with at most 4 roundings
  (the quotient, the square, the sum), so ``en' = en + 4 u n'``.
* ``sigma`` takes 7 roundings (square, two square roots, sum, product, quotient, and those of g) and, through the
  denominator, half of n's relative error: it is within ``(10 u + en / n) sigma``.
* ``z' = z + g - sigma d`` takes the errors of z, g, sigma and d, the last scaled by ``sigma``, and rounds at most
  three times: ``ez' = ez + u |g| + sigma ed + (10 u + en / n) |sigma d| + 3 u (|z| + |g| + |sigma d|)``.
* The closed form ``d(z, n)`` is continuous at ``|z| = l1``, where both branches are 0, and its slope in z is
  ``L = alpha / (beta + sqrt(n) + alpha l2) <= alpha`` on either side. So a z that is ``ez'`` away moves d by at most
  ``L ez'`` wherever the two values fall relative to the threshold: one may be exactly 0 and the other not. Its
  slope in n gives ``|d| en' / (2 n')``, and the formula rounds at most 8 times (``8 u |d|``).
* The one-sided push adds the device's step to the old value, ``d_old + (d' - d_old)``, which rounds twice:
  ``2 u (|d_old| + |d'|)``. The model adds it to every step, so one bound serves every path.
So ``ed' = L ez' + (8 u + en' / (2 n')) |d'| + 2 u (|d| + |d'|)``. A step does not read the old d except through
``sigma d``. Values, z and n must lie within 4 times their bounds (the factor covers the model's own fp64 rounding,
of the same order as the device's for fp64 tables). An element that was never stepped must keep its bits.
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

BETA = 1.0
# (learning_rate, rho = alpha, lambda_ = l1, momentum = l2) of consecutive Adds: l1 from 0 (no sparsity) to 1, l2
# from 0 to 1
OPTS = [(0.05, 0.1, 0.2, 0.0), (0.02, 0.05, 0.5, 0.1), (0.1, 0.2, 0.1, 1.0), (0.03, 0.1, 1.0, 0.0),
        (0.07, 0.3, 0.0, 0.5)]


def _f32(x):
    return float(np.float32(x))


def _o(lr, alpha, l1, l2):
    """An AddOption-like record, for the model alone."""
    return SimpleNamespace(learning_rate=lr, rho=alpha, lambda_=l1, momentum=l2, worker_id=0)


def fopt(mv, k, worker_id=0):
    lr, alpha, l1, l2 = OPTS[k % len(OPTS)]
    return mv.AddOption(worker_id=worker_id, momentum=l2, learning_rate=lr, rho=alpha, lambda_=l1)


def ftrl_weight(z, n, alpha, l1, l2):
    """The closed-form weight of (z, n), elementwise, beta = 1."""
    sgn = np.where(z < 0, -1.0, 1.0)
    with np.errstate(invalid="ignore", divide="ignore"):
        w = (sgn * l1 - z) / ((BETA + np.sqrt(n)) / alpha + l2)
    return np.where(sgn * z > l1, w, 0.0)


class FtrlModel:
    """A table of ``num_col``-element rows with FTRL's z and n per element, in fp64, and the bounds of the module
    docstring."""

    def __init__(self, start, num_col, dtype):
        self.npdt = np.dtype(dtype)
        self.u = _UNIT[self.npdt]
        self.data = np.asarray(start, dtype=np.float64).reshape(-1, num_col).copy()
        self.start = self.data.copy()
        self.num_row, self.num_col = self.data.shape
        shape = self.data.shape
        self.z, self.n = np.zeros(shape), np.zeros(shape)
        self.ez, self.en, self.ed = np.zeros(shape), np.zeros(shape), np.zeros(shape)
        self.nupd = np.zeros(shape, dtype=np.int64)

    def _step(self, r, delta, opt):
        """One step of rows ``r`` (an index or a slice) with delta rows ``delta``."""
        lr, alpha = _f32(opt.learning_rate), _f32(opt.rho)
        l1, l2 = _f32(opt.lambda_), _f32(opt.momentum)
        u = self.u
        d, z, n = self.data[r], self.z[r], self.n[r]
        ed, ez, en = self.ed[r], self.ez[r], self.en[r]
        g = np.asarray(delta, dtype=np.float64).reshape(d.shape) / lr
        act = g != 0
        g2 = g * g
        den = alpha * (np.sqrt(n + g2) + np.sqrt(n))
        sigma = np.where(den > 0, g2 / np.where(den > 0, den, 1.0), np.abs(g) / alpha)
        z1 = z + (g - sigma * d)
        n1 = n + g2
        d1 = ftrl_weight(z1, n1, alpha, l1, l2)
        rel_n = np.where(n > 0, en / np.where(n > 0, n, 1.0), 0.0)
        sd = np.abs(sigma * d)
        ez1 = ez + u * np.abs(g) + sigma * ed + (10 * u + rel_n) * sd + 3 * u * (np.abs(z) + np.abs(g) + sd)
        en1 = en + 4 * u * n1
        L = alpha / (BETA + np.sqrt(n1) + alpha * l2)
        rel_n1 = np.where(n1 > 0, en1 / np.where(n1 > 0, n1, 1.0), 0.0)
        ed1 = L * ez1 + (8 * u + 0.5 * rel_n1) * np.abs(d1) + 2 * u * (np.abs(d) + np.abs(d1))
        for arr, new in ((self.data, d1), (self.z, z1), (self.n, n1), (self.ez, ez1), (self.en, en1), (self.ed, ed1)):
            arr[r] = np.where(act, new, arr[r])
        self.nupd[r] += act

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
        _within(got, self.data[sel], 4.0 * self.ed[sel], f"{what} values")
        # an element never stepped keeps its starting value bit for bit
        idle = self.nupd[sel] == 0
        assert np.array_equal(got[idle], self.start[sel][idle]), f"{what}: an element that was never stepped moved"

    def check_state(self, z, n, what, rows=None):
        """z and n (``num_row x num_col`` elements) against the model."""
        sel = slice(None) if rows is None else rows
        z = np.asarray(z, dtype=np.float64).reshape(-1)[:self.data.size].reshape(self.data.shape)[sel]
        n = np.asarray(n, dtype=np.float64).reshape(-1)[:self.data.size].reshape(self.data.shape)[sel]
        _within(z, self.z[sel], 4.0 * self.ez[sel], f"{what} z")
        _within(n, self.n[sel], 4.0 * self.en[sel], f"{what} n")


def _within(got, ref, bound, what):
    bad = ~(np.abs(got - ref) <= bound)
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, np.abs(got - ref) - bound, -np.inf)), ref.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound; worst at {i}: "
                             f"got {got[i]!r} model {ref[i]!r} bound {bound[i]:.3g}")


def _sparse_delta(rng, shape, dtype, zero=0.2):
    """``_delta`` with a fraction ``zero`` of exact zeros: those elements must not be stepped."""
    d = _delta(rng, shape, dtype)
    d[rng.random(d.shape) < zero] = 0
    return d


# ----------------------------------------------------------------------------------- the model itself
def _mcmahan_algorithm_1(grads, alpha, beta, l1, l2):
    """McMahan et al. 2013, Algorithm 1 (per-coordinate FTRL-Proximal with L1 and L2), transcribed per coordinate:
    each round computes w_i from z_i, n_i for the coordinates in play (here: those with a non-zero gradient), then
    updates z_i and n_i with the round's gradient. Returns w, z, n after the last round, the weights being those the
    state implies (what the next round would predict with)."""
    dim = len(grads[0])
    z, n = [0.0] * dim, [0.0] * dim

    def weight(i):
        if abs(z[i]) <= l1:
            return 0.0
        sgn = 1.0 if z[i] > 0 else -1.0
        return -(z[i] - sgn * l1) / ((beta + n[i] ** 0.5) / alpha + l2)

    for g in grads:
        for i in range(dim):
            if g[i] == 0:
                continue
            w_i = weight(i)
            sigma = ((n[i] + g[i] * g[i]) ** 0.5 - n[i] ** 0.5) / alpha
            z[i] += g[i] - sigma * w_i
            n[i] += g[i] * g[i]
    return np.array([weight(i) for i in range(dim)]), np.array(z), np.array(n)


@pytest.mark.parametrize("l1,l2", [(0.0, 0.0), (0.5, 0.0), (0.5, 1.0), (3.0, 0.1)])
def test_model_is_mcmahan_algorithm_1(l1, l2):
    """From a zero table (whose weights are the closed form of z = n = 0), a single worker's sequence of whole-table
    Adds, pushed as delta = lr * grad, is Algorithm 1 with beta = 1 (fp64 throughout: 1e-12 relative). A fifth of the
    gradients are 0 and take no step, as coordinates absent from a round of Algorithm 1."""
    rng = np.random.default_rng(4)
    dim, steps = 40, 30
    scale = 10.0 ** rng.uniform(-3, 1, dim)         # per coordinate: the small ones stay inside l1
    grads = [rng.normal(0, scale) * (rng.random(dim) > 0.2) for _ in range(steps)]
    lr, alpha = _f32(0.125), _f32(0.1)
    l1, l2 = _f32(l1), _f32(l2)
    model = FtrlModel(np.zeros(dim), 1, "float64")
    for g in grads:
        model.add((g * lr).reshape(dim, 1), _o(lr, alpha, l1, l2))
    w, z, n = _mcmahan_algorithm_1([g.tolist() for g in grads], alpha, BETA, l1, l2)
    np.testing.assert_allclose(model.z.ravel(), z, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(model.n.ravel(), n, rtol=1e-12, atol=0)
    np.testing.assert_allclose(model.data.ravel(), w, rtol=1e-12, atol=1e-14)
    if l1 > 0:
        assert (model.data == 0).any() and (model.data != 0).any()


def test_zero_gradient_keeps_the_element():
    """An element whose delta is 0 keeps its value, z and n, even where the closed form of its state is 0."""
    O = _o(_f32(0.1), _f32(0.1), _f32(0.5), 0.0)
    model = FtrlModel([[0.3, -0.7, 0.2]], 3, "float32")
    model.add([[0.0, 0.01, 0.0]], O)
    assert model.data[0, 0] == 0.3 and model.data[0, 2] == 0.2 and model.z[0, 0] == 0 and model.n[0, 2] == 0
    assert model.nupd.tolist() == [[0, 1, 0]]


def test_initial_value_enters_through_sigma():
    """With z = n = 0 every table would start at the closed form 0; the initial value still matters, through
    sigma * d on the first step: z = g - (|g| / alpha) d0."""
    O = _o(_f32(0.1), _f32(0.5), 0.0, 0.0)
    a, b = FtrlModel([[0.0]], 1, "float64"), FtrlModel([[1.0]], 1, "float64")
    a.add([[0.01]], O)
    b.add([[0.01]], O)
    g = 0.01 / O.learning_rate
    assert a.z[0, 0] == pytest.approx(g) and b.z[0, 0] == pytest.approx(g - g / O.rho * 1.0)
    assert a.data[0, 0] != b.data[0, 0]


def test_sigma_is_the_reference_difference():
    """sigma = g^2 / (alpha (sqrt(n + g^2) + sqrt(n))) equals (sqrt(n + g^2) - sqrt(n)) / alpha, and keeps its
    relative accuracy where the difference cancels (g^2 << n)."""
    n = np.array([0.0, 1.0, 1e6, 1e12])
    g = np.array([0.5, 0.5, 1e-3, 1e-3])
    alpha = 0.1
    exact = g * g / (alpha * (np.sqrt(n + g * g) + np.sqrt(n)))
    diff = (np.sqrt(n + g * g) - np.sqrt(n)) / alpha
    np.testing.assert_allclose(exact[:2], diff[:2], rtol=1e-15)
    f32 = np.float32
    s32 = f32(g[2]) * f32(g[2]) / (f32(alpha) * (np.sqrt(f32(n[2]) + f32(g[2]) * f32(g[2])) + np.sqrt(f32(n[2]))))
    d32 = (np.sqrt(f32(n[2]) + f32(g[2]) * f32(g[2])) - np.sqrt(f32(n[2]))) / f32(alpha)
    assert abs(s32 / exact[2] - 1) < 1e-6 and abs(d32 / exact[2] - 1) > 1e-2


# ----------------------------------------------------------------------------------- host runtime
@pytest.fixture
def host_backend():
    """The host runtime (libmultiverso.so) at world size 1 with ``-updater_type=ftrl``."""
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    import multiverso_b200 as mv
    mv.FLAGS.reset()
    mv.FLAGS.set("updater_type", "ftrl")
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
        opt = fopt(mv, k)
        if k % 2 == 0:
            d = _sparse_delta(rng, (rows, cols), dtype)
            t.add(d, opt)
            model.add(d, opt)
        else:
            ids = _repeated_ids(rng, rows, 5 + k)
            v = _sparse_delta(rng, (ids.size, cols), dtype)
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
    model = FtrlModel(t.get(), cols, dtype)
    _host_steps(mv, t, model, rng, rows, cols, dtype)
    model.check_values(t.get(), f"host MatrixTable C={cols} {dtype}")
    assert model.nupd.max() >= 5 and (model.data == 0).any()


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_host_array_table_matches_model(host_backend, dtype):
    """An ArrayTable through the host runtime: the master-init Add of ``init_value`` is the first step."""
    mv = host_backend
    rng = np.random.default_rng(8)
    n = 11
    a = mv.ArrayTable(n, dtype, init_value=0.75)
    model = FtrlModel(np.zeros(n), 1, dtype)
    model.add(np.full(n, 0.75), mv.AddOption(worker_id=0))
    for k in range(5):
        d = _sparse_delta(rng, (n,), dtype)
        a.add(d, fopt(mv, k))
        model.add(d, fopt(mv, k))
    model.check_values(a.get(), f"host ArrayTable {dtype}")


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_host_store_load_roundtrip(host_backend, tmp_path, dtype):
    """save_table writes the shard, then z, then n, which match the model; a table loaded from it continues
    bitwise like the table that wrote it."""
    mv = host_backend
    rng = np.random.default_rng(12)
    rows, cols = 17, 6
    t = mv.MatrixTable(rows, cols, dtype, min_value=-1.0, max_value=1.0)
    model = FtrlModel(t.get(), cols, dtype)
    _host_steps(mv, t, model, rng, rows, cols, dtype, steps=4)
    uri = str(tmp_path / "ck")
    assert mv.save_table(t, uri)
    raw = np.frombuffer(Path(f"{uri}.shard0").read_bytes(), dtype=dtype)
    n = rows * cols
    assert raw.size == 3 * n
    model.check_state(raw[n:2 * n], raw[2 * n:], "host checkpoint")
    t2 = mv.MatrixTable(rows, cols, dtype)
    assert mv.load_table(t2, uri)
    assert np.array_equal(t2.get(), t.get())
    d = _sparse_delta(rng, (rows, cols), dtype)
    ids = np.array([3, 3, 16], dtype=np.int64)
    v = _delta(rng, (3, cols), dtype)
    for tab in (t, t2):
        tab.add(d, fopt(mv, 4))
        tab.add_rows(ids, v, fopt(mv, 0))
    assert np.array_equal(t2.get(), t.get())


def test_host_zero_gradient_keeps_the_element(host_backend):
    """A whole-table Add with zeros leaves those elements bitwise at their random initial values."""
    mv = host_backend
    t = mv.MatrixTable(4, 8, "float32", min_value=-1.0, max_value=1.0)
    before = t.get().copy()
    d = np.zeros((4, 8), np.float32)
    d[1, 2] = 0.01
    t.add(d, fopt(mv, 0))
    after = t.get()
    changed = np.argwhere(after.reshape(4, 8) != before.reshape(4, 8)).tolist()
    assert changed in ([], [[1, 2]])
    mask = np.ones((4, 8), bool)
    mask[1, 2] = False
    assert np.array_equal(after.reshape(4, 8)[mask], before.reshape(4, 8)[mask])


# ----------------------------------------------------------------------------------- option checks
# (learning_rate, rho, lambda_, momentum)
BAD_OPTS = {"lr=0": (0.0, 0.1, 0.1, 0.0), "lr<0": (-0.1, 0.1, 0.1, 0.0), "rho=0": (0.1, 0.0, 0.1, 0.0),
            "rho<0": (0.1, -0.1, 0.1, 0.0), "lambda<0": (0.1, 0.1, -0.1, 0.0), "momentum<0": (0.1, 0.1, 0.1, -0.5),
            "nan": (0.1, float("nan"), 0.1, 0.0), "inf": (0.1, 0.1, float("inf"), 0.0),
            "beyond fp32": (0.1, 0.1, 0.1, 1e39), "lr rounds to 0": (1e-46, 0.1, 0.1, 0.0)}


@pytest.mark.parametrize("case", sorted(BAD_OPTS))
def test_option_check(case):
    from multiverso_b200.tables.options import AddOption, check_add_option
    lr, rho, l1, l2 = BAD_OPTS[case]
    bad = AddOption(worker_id=0, momentum=l2, learning_rate=lr, rho=rho, lambda_=l1)
    with pytest.raises(ValueError, match="ftrl needs"):
        check_add_option("ftrl", bad)
    check_add_option("momentum_sgd", bad)
    check_add_option("ftrl", AddOption(worker_id=0, momentum=0.0, learning_rate=0.1, rho=0.1, lambda_=0.0))


def test_host_option_check_raises(host_backend):
    """The host backend raises ValueError before the request leaves Python; the table is unchanged."""
    mv = host_backend
    t = mv.MatrixTable(3, 4, "float32", min_value=-1.0, max_value=1.0)
    a = mv.ArrayTable(5, "float32")
    before = t.get().copy()
    bad = mv.AddOption(worker_id=0, momentum=0.0, learning_rate=0.1, rho=0.0, lambda_=0.1)
    with pytest.raises(ValueError):
        t.add(np.ones((3, 4), np.float32), bad)
    with pytest.raises(ValueError):
        t.add_rows(np.array([1]), np.ones((1, 4), np.float32), bad)
    with pytest.raises(ValueError):
        a.add(np.ones(5, np.float32), mv.AddOption(worker_id=0, learning_rate=0.1, rho=0.1, lambda_=-1.0))
    assert np.array_equal(t.get(), before)


_CHECK_CHILD = r"""
import sys
sys.path.insert(0, sys.argv[1])
import ctypes as C
import numpy as np
import multiverso_b200 as mv
from multiverso_b200 import host
mv.FLAGS.set("updater_type", "ftrl")
mv.init()
a = mv.ArrayTable(4, "float32")
data = np.ones(4, np.float32)
lr, rho, l1, l2 = (float(x) for x in sys.argv[2:6])
opt = mv.AddOption(worker_id=0, momentum=l2, learning_rate=lr, rho=rho, lambda_=l1)
host._lib().MV_AddArrayTable64(a.handle, a.code, data.ctypes.data_as(C.c_void_p), C.c_int64(4), opt.pack(), 0)
print("APPLIED", flush=True)
"""


@pytest.mark.parametrize("case", ["lr=0", "rho=0", "lambda<0", "momentum<0", "nan", "ok"])
def test_host_runtime_check(case):
    """The host runtime's own CHECK, reached through the C API without the Python check: a bad option stops the
    process with 'Check failed', a good one is applied."""
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    vals = BAD_OPTS.get(case, (0.1, 0.1, 0.1, 0.0))
    root = str(Path(__file__).resolve().parents[1])
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", _CHECK_CHILD, root] + \
        [str(v) for v in vals]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    out = r.stdout + r.stderr
    if case == "ok":
        assert r.returncode == 0 and "APPLIED" in out, out[-2000:]
    else:
        assert r.returncode != 0 and "APPLIED" not in out and "Check failed" in out, out[-2000:]


# ----------------------------------------------------------------------------------- argument codes
DUMMY = 1 << 12          # 16-byte aligned, never dereferenced


def _cases():
    """ftrl is element-wise: the element-wise entry points launch for it (which fails without a device), the
    row-state pushes refuse it."""
    from multiverso_b200 import _native as N
    F = N.UPD_FTRL
    vp = (C.c_void_p * N.MAX_RANKS)(*([DUMMY] * N.MAX_RANKS))
    i64 = (C.c_int64 * N.MAX_RANKS)(*([4] * N.MAX_RANKS))
    c = {}
    for dt, name in ((N.F32, "f32"), (N.F64, "f64")):
        c[f"launch/mvb_updater_apply/{name}"] = (
            lambda lib, dt=dt: lib.mvb_updater_apply(dt, F, DUMMY, DUMMY, DUMMY, DUMMY, 4, N.AddOpt(), 1.0, None),
            "cuda")
        c[f"launch/mvb_push_dense_stateful/{name}"] = (
            lambda lib, dt=dt: lib.mvb_push_dense_stateful(dt, F, DUMMY, 1, vp, vp, vp, i64, i64, i64, N.AddOpt(), 0,
                                                           None), "cuda")
        c[f"launch/mvb_add_rows_owner/{name}"] = (
            lambda lib, dt=dt: lib.mvb_add_rows_owner(dt, F, DUMMY, DUMMY, DUMMY, 0, 4, 4, 16, DUMMY, 1, DUMMY, 4,
                                                      N.AddOpt(), None), "cuda")
        c[f"norows/mvb_push_dense_rowwise/{name}"] = (
            lambda lib, dt=dt: lib.mvb_push_dense_rowwise(dt, F, DUMMY, 1, vp, vp, i64, i64, i64, 2, N.AddOpt(), 0,
                                                          None), -2)
        c[f"norows/mvb_push_dense_adam/{name}"] = (
            lambda lib, dt=dt: lib.mvb_push_dense_adam(dt, F, DUMMY, 1, vp, vp, vp, i64, i64, i64, 2, N.AddOpt(), 0,
                                                       None), -2)
    for dt in (N.I64, N.I8, 99):
        c[f"dtype/mvb_push_dense_stateful/{dt}"] = (
            lambda lib, dt=dt: lib.mvb_push_dense_stateful(dt, F, DUMMY, 1, vp, vp, vp, i64, i64, i64, N.AddOpt(), 0,
                                                           None), -1)
    c["unknown/mvb_updater_apply/10"] = (
        lambda lib: lib.mvb_updater_apply(N.F32, 10, DUMMY, DUMMY, DUMMY, DUMMY, 4, N.AddOpt(), 1.0, None), -2)
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
    assert re.search(r"MVB_UPD_FTRL\s*=\s*9\b", hdr)
    assert N.UPD_FTRL == 9 and N.UPDATER_NAMES["ftrl"] == 9
    assert 6 not in N.UPDATER_NAMES.values()


if __name__ == "__main__":
    print(json.dumps(_codes()))
