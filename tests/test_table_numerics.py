"""Table Adds, Gets and row ops against an fp64 model of the parameter server.

``ServerModel`` holds one table and its updater state in fp64 and applies Adds the way the server does
(include/multiverso/updater/*.h, the updater functors of csrc/cuda/mvb_common.cuh):

* the AddOption fields travel as fp32 (``<iffff>`` / ``MvbAddOpt``), so momentum, learning rate, rho and
  lambda are rounded to fp32, and ``1 - momentum`` is computed in fp32 (exact for the momenta used here,
  0 and [0.5, 1], so the host updaters, which form it in the element type, agree);
* AdaGrad adds 1e-6 and DC-ASGD-A 1e-7 to the square sums, as constants of the element type;
* momentum keeps one shared state slab; AdaGrad, DC-ASGD and DC-ASGD-A keep one slab per worker, and
  DC-ASGD-A two (shadow copy, mean square);
* a row Add applies its entries in list order, so a repeated row is updated once per occurrence; ids
  outside ``[0, num_row)`` are ignored (the device contract; the host runtime CHECKs them).

Error bound.  One updater step rounds a handful of operations, each within one unit roundoff ``u``
(2^-24 for fp32, 2^-53 for fp64) of its result; ``rsqrtf`` is within 2 ulp and FMA contraction only
removes roundings.  Every rounded intermediate of a step is bounded by the sum of the magnitudes of the
step's terms, so the error a step adds is below ``8 u (|d| + sum |terms|)``.  Errors of earlier steps are
carried forward by factors of at most one (the DC-ASGD factor ``1 - lr lambda g^2`` stays in [0, 1] for
the deltas used here) and a state error enters a later step the same way.  After ``n`` updates of an
element the difference to the model is therefore below ``8 n u (|ref| + M)`` where ``M`` is |start value|
plus the sum of the magnitudes of every term applied to that element (``ServerModel.mag``); each state
element has the analogous scale (``ServerModel.state_scale``).  Integer tables are exact.

The CPU test ties the model to the host runtime (libmultiverso.so at world size 1), the semantic oracle
of the device backend; the GPU tests hold the device kernels to the model at world size 1.
"""
import io

import numpy as np
import pytest
import torch

UPDATERS = ["default", "sgd", "momentum_sgd", "adagrad", "dcasgd", "dcasgda"]
STATEFUL = ["momentum_sgd", "adagrad", "dcasgd", "dcasgda"]
_STATES = {"default": (0, False), "sgd": (0, False), "momentum_sgd": (1, False), "adagrad": (1, True),
           "dcasgd": (1, True), "dcasgda": (2, True)}
_UNIT = {np.dtype(np.float32): 2.0 ** -24, np.dtype(np.float64): 2.0 ** -53}
# (momentum, learning_rate, rho, lambda) of five consecutive Adds
_OPTS = [(0.0, 0.05, 0.1, 0.2), (0.5, 0.02, 0.05, 0.5), (0.99, 0.1, 0.2, 0.1), (0.5, 0.03, 0.1, 1.0),
         (0.0, 0.07, 0.3, 0.3)]


def _f32(x):
    return float(np.float32(x))


class ServerModel:
    """One table (``num_row x num_col``, element type ``dtype``) and its updater state, in fp64."""

    def __init__(self, start, num_col, updater, dtype, workers=1):
        self.npdt = np.dtype(dtype)
        self.is_int = self.npdt.kind == "i"
        self.updater = "default" if self.is_int else updater
        self.data = np.asarray(start, dtype=np.float64).reshape(-1, num_col).copy()
        self.num_row, self.num_col = self.data.shape
        nst, per_worker = _STATES[self.updater]
        self.state = [np.zeros((workers if per_worker else 1,) + self.data.shape) for _ in range(nst)]
        self.smag = [np.zeros_like(s) for s in self.state]
        self.per_worker = per_worker
        self.mag = np.abs(self.data)                     # |start| + sum of |terms| applied, per element
        self.nupd = np.zeros(self.data.shape, dtype=np.int64)
        self.stale = set()                               # rows a sparse table marks as changed
        eps = {"adagrad": 1e-6, "dcasgda": 1e-7}.get(self.updater, 0.0)
        self.eps = float(self.npdt.type(eps)) if not self.is_int else 0.0

    def _apply(self, r, g, opt):
        """One update of rows ``r`` (an index or a slice) with delta rows ``g``."""
        m, lr, rho, lam = _f32(opt.momentum), _f32(opt.learning_rate), _f32(opt.rho), _f32(opt.lambda_)
        one_m = float(np.float32(1.0) - np.float32(m))
        w = opt.worker_id if self.per_worker else 0
        g = np.asarray(g, dtype=np.float64)
        d = self.data[r]
        u = self.updater
        if u == "default":
            new, terms = d + g, np.abs(g)
        elif u == "sgd":
            new, terms = d - g, np.abs(g)
        elif u == "momentum_sgd":
            s = self.state[0][0, r]
            s_new = m * s + one_m * g
            self.smag[0][0, r] = m * self.smag[0][0, r] + one_m * np.abs(g)
            self.state[0][0, r] = s_new
            new, terms = d - s_new, np.abs(m * s) + np.abs(one_m * g)
        elif u == "adagrad":
            gn = g / lr
            h = self.state[0][w, r] + gn * gn
            step = rho / np.sqrt(h + self.eps) * gn
            self.state[0][w, r] = h
            self.smag[0][w, r] = h
            new, terms = d - step, np.abs(step)
        elif u == "dcasgd":
            gn = g / lr
            comp = lr * lam * gn * gn * (d - self.state[0][w, r])
            new, terms = d - (lr * gn + comp), np.abs(lr * gn) + np.abs(comp)
        else:  # dcasgda
            gn = g / lr
            ms = m * self.state[1][w, r] + one_m * gn * gn
            comp = lr * lam / np.sqrt(ms + self.eps) * gn * gn * (d - self.state[0][w, r])
            self.state[1][w, r] = ms
            self.smag[1][w, r] = ms
            new, terms = d - (lr * gn + comp), np.abs(lr * gn) + np.abs(comp)
        self.data[r] = new
        self.mag[r] += terms
        self.nupd[r] += 1
        if u in ("dcasgd", "dcasgda"):
            self.state[0][w, r] = new
            self.smag[0][w, r] = np.abs(new) + self.mag[r]

    def add(self, delta, opt):
        delta = np.asarray(delta, dtype=np.float64).reshape(self.data.shape)
        self._apply(slice(None), delta, opt)
        self.stale.update(np.flatnonzero((delta != 0).any(axis=1)).tolist())

    def add_rows(self, ids, vals, opt):
        vals = np.asarray(vals, dtype=np.float64).reshape(len(ids), self.num_col)
        for i, r in enumerate(np.asarray(ids).tolist()):
            if 0 <= r < self.num_row:
                self._apply(r, vals[i], opt)
                self.stale.add(r)

    def take_stale(self):
        rows = sorted(self.stale)
        self.stale.clear()
        return rows

    def state_scale(self, i, w=0):
        return self.smag[i][w]


def _opt(mv, k):
    m, lr, rho, lam = _OPTS[k % len(_OPTS)]
    return mv.AddOption(worker_id=0, momentum=m, learning_rate=lr, rho=rho, lambda_=lam)


def _delta(rng, shape, dtype):
    """Deltas of both signs over three decades (|delta| in [1e-4, 0.1]): the small ones make the square
    sums comparable to the AdaGrad / DC-ASGD-A epsilons, so a wrong epsilon moves the result."""
    n = int(np.prod(shape))
    if np.dtype(dtype).kind == "i":
        return rng.integers(-1000, 1000, n).astype(dtype).reshape(shape)
    mag = 0.1 * 10.0 ** rng.uniform(-3.0, 0.0, n)
    return (rng.choice([-1.0, 1.0], n) * mag).astype(dtype).reshape(shape)


def _assert_close(got, ref, scale, nupd, dtype, what):
    got = np.asarray(got, dtype=np.float64).reshape(ref.shape)
    if np.dtype(dtype).kind == "i":
        assert np.array_equal(got, ref), f"{what}: integer table differs"
        return
    bound = 8.0 * np.maximum(nupd, 1) * _UNIT[np.dtype(dtype)] * scale
    bad = np.abs(got - ref) > bound
    if bad.any():
        i = np.unravel_index(np.argmax(np.abs(got - ref) - bound), ref.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound; worst at {i}: "
                             f"got {got[i]!r} model {ref[i]!r} bound {bound[i]:.3g}")


def _check_model(t, model, dtype, what, rows=None):
    """Values and updater state of device table ``t`` against ``model`` (rows: restrict to these rows)."""
    sel = slice(None) if rows is None else rows
    got = t.get().cpu().numpy().reshape(model.data.shape)
    _assert_close(got[sel], model.data[sel], (np.abs(model.data) + model.mag)[sel], model.nupd[sel], dtype,
                  f"{what} values")
    for i in range(len(model.state)):
        for w in range(model.state[i].shape[0]):
            st = _device_state(t, i, w).reshape(model.data.shape)
            _assert_close(st[sel], model.state[i][w][sel], model.state_scale(i, w)[sel], model.nupd[sel], dtype,
                          f"{what} state{i}[worker {w}]")


def _device_state(t, i, w=0):
    """Worker ``w``'s slice of state slab ``i`` of a device table (the whole slab for momentum)."""
    off = w * t.state_stride if t.state_per_worker else 0
    return t.state[i][off:off + t.my_len].cpu().numpy()


# ----------------------------------------------------------------------------------- CPU tier: host runtime
@pytest.fixture
def host_backend():
    """The host runtime (libmultiverso.so) at world size 1; call the fixture with the updater type."""
    if torch.cuda.is_available():
        pytest.skip("host-backend test (runs where there is no GPU)")
    import multiverso_b200 as mv
    started = []

    def start(updater):
        mv.FLAGS.reset()
        mv.FLAGS.set("updater_type", updater)
        mv.init()
        started.append(True)
        return mv

    yield start
    if started:
        mv.shutdown(finalize_net=False)
    mv.FLAGS.reset()


def _repeated_ids(rng, num_row, hot, reps, n_unique, out_of_range=()):
    """A shuffled id list: each hot row ``reps[j]`` times, interleaved with unique other rows."""
    others = np.setdiff1d(np.arange(num_row), hot)
    ids = np.concatenate([np.repeat(hot, reps), rng.choice(others, n_unique, replace=False),
                          np.asarray(out_of_range, dtype=np.int64)])
    return rng.permutation(ids).astype(np.int64)


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", UPDATERS)
def test_host_runtime_matches_model(host_backend, updater, dtype):
    """The host runtime against the model: whole-table Adds interleaved with row Adds that repeat rows,
    on a randomly initialised MatrixTable (so DC-ASGD's compensation term starts non-zero) and on an
    ArrayTable whose ``init_value`` goes through the updater as the master-init Add."""
    mv = host_backend(updater)
    rng = np.random.default_rng(11)
    rows, cols = 37, 5
    t = mv.MatrixTable(rows, cols, dtype, min_value=-1.0, max_value=1.0)
    start = t.get()
    assert np.abs(start).min() > 0
    model = ServerModel(start, cols, updater, dtype)
    for k in range(5):
        opt = _opt(mv, k)
        if k % 2 == 0:
            d = _delta(rng, (rows, cols), dtype)
            t.add(d, opt)
            model.add(d, opt)
        else:
            ids = _repeated_ids(rng, rows, [2, 30], [9, 4], 12)
            v = _delta(rng, (ids.size, cols), dtype)
            t.add_rows(ids, v, opt)
            model.add_rows(ids, v, opt)
    _assert_close(t.get(), model.data, np.abs(model.data) + model.mag, model.nupd, dtype, "host MatrixTable")

    n = 11
    a = mv.ArrayTable(n, dtype, init_value=0.75)
    am = ServerModel(np.zeros(n), 1, updater, dtype)
    am.add(np.full(n, 0.75), mv.AddOption(worker_id=0))
    for k in range(5):
        d = _delta(rng, (n,), dtype)
        a.add(d, _opt(mv, k))
        am.add(d, _opt(mv, k))
    _assert_close(a.get(), am.data.reshape(-1), (np.abs(am.data) + am.mag).reshape(-1), am.nupd.reshape(-1), dtype,
                  "host ArrayTable")


# ----------------------------------------------------------------------------------- GPU tier: device tables
_SHAPES = [("array", 1), ("array", 3), ("array", 4), ("array", 5), ("array", 4099), ("array", (1 << 20) + 3),
           ("matrix", (1, 1)), ("matrix", (7, 3)), ("matrix", (1000, 300)), ("matrix", (513, 1025))]


def _make_table(mv, kind, shape, dtype, updater, **kw):
    """A device table with non-zero starting values, and the model seeded from its ``get()``."""
    if kind == "array":
        t = mv.ArrayTable(shape, dtype, updater=updater,
                          init_value=(7 if np.dtype(dtype).kind == "i" else 0.75))
        cols = 1
    else:
        rows, cols = shape
        if np.dtype(dtype).kind == "i":
            t = mv.MatrixTable(rows, cols, dtype, updater=updater, init_value=7, **kw)
        else:
            t = mv.MatrixTable(rows, cols, dtype, updater=updater, min_value=-1.0, max_value=1.0, **kw)
    start = t.get().cpu().numpy()
    assert np.abs(start.astype(np.float64)).min() > 0
    return t, ServerModel(start, cols, updater, dtype)


def _on_device(x, offset=0):
    """``x`` on the GPU; ``offset`` > 0 returns it as a view ``offset`` elements into a larger buffer, so
    that it is not 16-byte aligned and the kernels take their element-wise paths."""
    x = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    if offset == 0:
        return x
    buf = torch.zeros(x.numel() + offset + 1, dtype=x.dtype, device="cuda")
    v = buf[offset:offset + x.numel()].view(x.shape)
    v.copy_(x)
    return v


def _whole_table_steps(mv, t, model, kind, shape, dtype, offset):
    rng = np.random.default_rng(5)
    full = (shape,) if kind == "array" else shape
    for k in range(5):
        d = _delta(rng, full, dtype)
        t.add(_on_device(d, offset), _opt(mv, k))
        model.add(d, _opt(mv, k))


@pytest.mark.gpu
@pytest.mark.parametrize("kind,shape", _SHAPES)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", UPDATERS)
def test_whole_table_add(mv_device, updater, dtype, kind, shape):
    """Five whole-table Adds, the AddOption changing at every step, through the fused Add kernel's 16-byte
    path and its scalar tail (sizes that are not a multiple of the vector width); values and state against
    the model within the bound of the module docstring."""
    mv = mv_device
    t, model = _make_table(mv, kind, shape, dtype, updater)
    _whole_table_steps(mv, t, model, kind, shape, dtype, offset=0)
    _check_model(t, model, dtype, f"{updater} {dtype} {kind}{shape}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind,shape", [("array", 5), ("array", 4099), ("matrix", (7, 3)), ("matrix", (513, 1025))])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", UPDATERS)
def test_whole_table_add_scalar_path(mv_device, updater, dtype, kind, shape):
    """The delta is a view one element into a larger buffer: the fused Add takes its element-wise kernel
    (VEC = 1) and must meet the same bound as the vector path."""
    mv = mv_device
    t, model = _make_table(mv, kind, shape, dtype, updater)
    _whole_table_steps(mv, t, model, kind, shape, dtype, offset=1)
    _check_model(t, model, dtype, f"{updater} {dtype} {kind}{shape} scalar")


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("kind,shape", [("array", 1), ("array", 5), ("array", 4099), ("array", (1 << 20) + 3),
                                        ("matrix", (7, 3)), ("matrix", (513, 1025))])
def test_whole_table_add_int32_exact(mv_device, kind, shape, offset):
    mv = mv_device
    t, model = _make_table(mv, kind, shape, "int32", "default")
    _whole_table_steps(mv, t, model, kind, shape, "int32", offset)
    assert np.array_equal(t.get().cpu().numpy().reshape(model.data.shape), model.data)


def _row_case(rng, rows, repeated):
    if repeated:
        # hot rows repeated up to 50 times, shuffled among unique rows
        return _repeated_ids(rng, rows, [3, 17, 150], [50, 20, 7], 40)
    return rng.choice(rows, 60, replace=False).astype(np.int64)


@pytest.mark.gpu
@pytest.mark.parametrize("ids_kind", ["unique", "repeated"])
@pytest.mark.parametrize("cols", [1, 3, 4, 5, 300, 1025])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", STATEFUL)
def test_row_add_stateful(mv_device, updater, dtype, cols, ids_kind):
    """Stateful row Adds applied by the owner kernel: every occurrence of a repeated row is applied, in list
    order; an empty list changes nothing; ids -1 and num_row are ignored; rows never named stay bitwise
    unchanged in the shard and in the state."""
    mv = mv_device
    rows = 200
    rng = np.random.default_rng(cols)
    t, model = _make_table(mv, "matrix", (rows, cols), dtype, updater)
    start = model.data.copy()
    named = set()
    for k in range(3):
        ids = _row_case(rng, rows, ids_kind == "repeated")
        if k == 1:
            ids = rng.permutation(np.concatenate([ids, [-1, rows]])).astype(np.int64)
        v = _delta(rng, (ids.size, cols), dtype)
        t.add_rows(torch.from_numpy(ids).cuda(), _on_device(v), _opt(mv, k))
        model.add_rows(ids, v, _opt(mv, k))
        named.update(r for r in ids.tolist() if 0 <= r < rows)
    t.add_rows(torch.empty(0, dtype=torch.int64, device="cuda"),
               torch.empty(0, cols, dtype=getattr(torch, dtype), device="cuda"), _opt(mv, 3))
    what = f"{updater} {dtype} cols={cols} {ids_kind}"
    _check_model(t, model, dtype, what)
    untouched = np.setdiff1d(np.arange(rows), sorted(named))
    got = t.get().cpu().numpy().reshape(rows, cols)
    assert np.array_equal(got[untouched], start[untouched]), f"{what}: a row never named changed"
    for i in range(len(model.state)):
        st = _device_state(t, i).reshape(rows, cols)
        assert not st[untouched].any(), f"{what}: state{i} of a row never named changed"


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("cols", [1, 4, 5, 1025])
@pytest.mark.parametrize("dtype,updater", [("float32", "default"), ("float32", "sgd"), ("float64", "default"),
                                           ("float64", "sgd"), ("int32", "default")])
def test_row_add_stateless_repeated(mv_device, dtype, updater, cols, offset):
    """default / sgd row Adds (atomic adds into the owner) with repeated and out-of-range ids; ``offset``
    puts the values one element into a larger buffer so the element-wise ``red.add`` path runs. The
    atomics apply the occurrences in any order: exact for int32, within the bound for floats."""
    mv = mv_device
    rows = 200
    rng = np.random.default_rng(100 + cols)
    t, model = _make_table(mv, "matrix", (rows, cols), dtype, updater)
    for k in range(2):
        ids = _repeated_ids(rng, rows, [3, 17, 150], [50, 20, 7], 40, out_of_range=[-1, rows])
        v = _delta(rng, (ids.size, cols), dtype)
        t.add_rows(torch.from_numpy(ids).cuda(), _on_device(v, offset), _opt(mv, k))
        model.add_rows(ids, v, _opt(mv, k))
    _check_model(t, model, dtype, f"{updater} {dtype} cols={cols} offset={offset}")


_SENTINEL = {"float32": -123.5, "float64": -123.5, "int32": -12345}


@pytest.mark.gpu
@pytest.mark.parametrize("cols", [1, 4, 5, 300])
@pytest.mark.parametrize("dtype", ["float32", "float64", "int32"])
def test_get_rows_layouts(mv_device, dtype, cols):
    """get_rows with repeated and out-of-range ids into (a) a fresh tensor, (b) a column slice of a wider
    buffer (ld > num_col), (c) a view at an element offset, (d) a column slice starting at column 1.
    In-range rows equal the table's rows; out-of-range rows and every element outside ``out`` keep the
    sentinel."""
    mv = mv_device
    rows = 50
    tdt = getattr(torch, dtype)
    t = mv.MatrixTable(rows, cols, dtype)
    rng = np.random.default_rng(cols)
    t.add(torch.from_numpy(_delta(rng, (rows, cols), dtype)).cuda())
    full = t.get().view(rows, cols)
    ids = torch.tensor([5, 5, 0, 49, -1, 50, 5, 12, 0], device="cuda")
    ok = (ids >= 0) & (ids < rows)
    k = ids.numel()
    sent = _SENTINEL[dtype]

    got = t.get_rows(ids)
    assert torch.equal(got[ok], full[ids[ok]])

    for lead, extra in ((0, 3), (1, 2)):
        wide = torch.full((k, cols + lead + extra), sent, dtype=tdt, device="cuda")
        out = wide[:, lead:lead + cols]
        t.get_rows(ids, out=out)
        assert torch.equal(out[ok], full[ids[ok]])
        assert bool((out[~ok] == sent).all()), "out-of-range rows were written"
        assert bool((wide[:, :lead] == sent).all()) and bool((wide[:, lead + cols:] == sent).all())

    flat = torch.full((k * cols + 2,), sent, dtype=tdt, device="cuda")
    out = flat[1:1 + k * cols].view(k, cols)
    t.get_rows(ids, out=out)
    assert torch.equal(out[ok], full[ids[ok]])
    assert bool((out[~ok] == sent).all()) and float(flat[0]) == sent and float(flat[-1]) == sent


@pytest.mark.gpu
@pytest.mark.parametrize("kind,shape", [("array", 5), ("array", 4099), ("array", (1 << 20) + 3), ("matrix", (7, 3))])
@pytest.mark.parametrize("dtype", ["float32", "float64", "int32"])
def test_get_into_unaligned_view(mv_device, dtype, kind, shape):
    """Whole-table ``get(out=...)`` into a view one element into a larger buffer (not 16-byte aligned)."""
    mv = mv_device
    t, model = _make_table(mv, kind, shape, dtype, "default")
    n = model.data.size
    sent = _SENTINEL[dtype]
    flat = torch.full((n + 2,), sent, dtype=getattr(torch, dtype), device="cuda")
    out = t.get(out=flat[1:n + 1])
    assert np.array_equal(out.cpu().numpy().astype(np.float64), model.data.reshape(-1))
    assert float(flat[0]) == sent and float(flat[-1]) == sent


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", STATEFUL)
def test_sparse_table_stale_rows(mv_device, updater, dtype):
    """A sparse MatrixTable with a stateful updater: after mixed row Adds (repeated and out-of-range ids) and
    whole-table Adds (all-zero rows are not marked), ``get_stale()`` returns exactly the rows the model
    marked, with the model's values."""
    mv = mv_device
    rows, cols = 64, 6
    rng = np.random.default_rng(2)
    t, model = _make_table(mv, "matrix", (rows, cols), dtype, updater, is_sparse=True)
    ids0, _ = t.get_stale()
    assert ids0.numel() == rows
    model.take_stale()

    def delta_rows(which):
        d = np.zeros((rows, cols), dtype=dtype)
        d[which] = _delta(rng, (len(which), cols), dtype)
        return d

    def check(what):
        sid, srows = t.get_stale()
        exp = model.take_stale()
        assert sid.cpu().tolist() == exp, f"{what}: stale rows {sid.cpu().tolist()} != {exp}"
        if exp:
            _assert_close(srows.cpu().numpy(), model.data[exp], (np.abs(model.data) + model.mag)[exp],
                          model.nupd[exp], dtype, what)

    ids = _repeated_ids(rng, rows, [9, 40], [12, 5], 6, out_of_range=[-1])
    v = _delta(rng, (ids.size, cols), dtype)
    t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(v).cuda(), _opt(mv, 0))
    model.add_rows(ids, v, _opt(mv, 0))
    d = delta_rows([7, 20, 40])
    t.add(torch.from_numpy(d).cuda(), _opt(mv, 1))
    model.add(d, _opt(mv, 1))
    ids = np.array([20, 3, 20, 63], dtype=np.int64)
    v = _delta(rng, (ids.size, cols), dtype)
    t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(v).cuda(), _opt(mv, 2))
    model.add_rows(ids, v, _opt(mv, 2))
    check("after row and whole-table Adds")
    d = delta_rows([33])
    t.add(torch.from_numpy(d).cuda(), _opt(mv, 3))
    model.add(d, _opt(mv, 3))
    check("after a one-row whole-table Add")
    check("with nothing new")
    _check_model(t, model, dtype, f"sparse {updater} {dtype}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", ["dcasgd", "dcasgda"])
def test_checkpoint_roundtrip_dcasgd(mv_device, tmp_path, updater, dtype):
    """save_table / load_table carry DC-ASGD's per-worker shadow (and DC-ASGD-A's mean square): the loaded
    table is bitwise equal in values and state, and the next Add gives the same result on both."""
    mv = mv_device
    rows, cols = 33, 7
    rng = np.random.default_rng(4)
    t, model = _make_table(mv, "matrix", (rows, cols), dtype, updater)
    for k in range(2):
        d = _delta(rng, (rows, cols), dtype)
        t.add(torch.from_numpy(d).cuda(), _opt(mv, k))
        model.add(d, _opt(mv, k))
    ids = np.array([4, 4, 30], dtype=np.int64)
    v = _delta(rng, (3, cols), dtype)
    t.add_rows(torch.from_numpy(ids).cuda(), torch.from_numpy(v).cuda(), _opt(mv, 2))
    model.add_rows(ids, v, _opt(mv, 2))
    assert mv.save_table(t, str(tmp_path / "ck"))
    t2 = mv.MatrixTable(rows, cols, dtype, updater=updater)
    assert mv.load_table(t2, str(tmp_path / "ck"))
    assert torch.equal(t2.get(), t.get())
    for a, b in zip(t.state, t2.state):
        assert torch.equal(a, b)
    d = torch.from_numpy(_delta(rng, (rows, cols), dtype)).cuda()
    t.add(d, _opt(mv, 3))
    t2.add(d, _opt(mv, 3))
    model.add(d.cpu().numpy(), _opt(mv, 3))
    assert torch.equal(t2.get(), t.get())
    _check_model(t2, model, dtype, f"{updater} {dtype} after load")


@pytest.mark.gpu
def test_int64_tables_rejected(mv_device):
    """No kernel serves int64 dense tables: creating one is an error that names the supported types."""
    from multiverso_b200.utils import FatalError
    mv = mv_device
    with pytest.raises(FatalError, match="float32/float64/int32"):
        mv.ArrayTable(8, "int64")
    with pytest.raises(FatalError, match="float32/float64/int32"):
        mv.MatrixTable(4, 4, "int64")


# ------------------------------------------------------------------ GPU tier: updater kernels called directly
_KSENT = -123.5           # sentinel of every buffer region a kernel must not write


def _kopt(k, worker_id):
    """The k-th AddOption of ``_OPTS`` for ``worker_id``, and its C struct."""
    from multiverso_b200.tables.options import AddOption
    from multiverso_b200.tables.device import _opt_struct
    m, lr, rho, lam = _OPTS[k % len(_OPTS)]
    o = AddOption(worker_id=worker_id, momentum=m, learning_rate=lr, rho=rho, lambda_=lam)
    return o, _opt_struct(o)


def _start_values(rng, n, dtype):
    return (rng.choice([-1.0, 1.0], n) * rng.uniform(0.25, 1.0, n)).astype(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("dtype", ["float32", "float64", "int32"])
@pytest.mark.parametrize("updater", STATEFUL)
def test_updater_apply(mv_device, updater, dtype, scale):
    """The stand-alone updater (``mvb_updater_apply``) over more elements than its grid covers at once: five
    steps, the AddOption changing at every step, the delta scaled by ``scale``; values and the state slabs
    (one shared slab each, whatever the updater) against the model. An int32 table always takes the plain
    add, ignores ``scale`` and touches no state."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    n = 300_001
    rng = np.random.default_rng(21)
    is_int = dtype == "int32"
    start = rng.integers(-1000, 1000, n).astype(dtype) if is_int else _start_values(rng, n, dtype)
    data = torch.from_numpy(start).cuda()
    nst = 0 if is_int else _STATES[updater][0]
    states = [torch.zeros(n, dtype=getattr(torch, dtype), device="cuda") for _ in range(nst)]
    model = ServerModel(start, 1, updater, dtype)
    for k in range(5):
        opt, copt = _kopt(k, 0)
        d = _delta(rng, (n,), dtype)
        lib.mvb_updater_apply(N.dtype_code(data.dtype), N.UPDATER_NAMES[updater], data, torch.from_numpy(d).cuda(),
                              states[0] if nst >= 1 else None, states[1] if nst >= 2 else None, n, copt, scale, st)
        model.add(d if is_int else d * scale, opt)
    torch.cuda.synchronize()
    what = f"updater_apply {updater} {dtype} scale={scale}"
    _assert_close(data.cpu().numpy(), model.data.reshape(-1), (np.abs(model.data) + model.mag).reshape(-1),
                  model.nupd.reshape(-1), dtype, f"{what} values")
    for i in range(nst):
        _assert_close(states[i].cpu().numpy(), model.state[i][0].reshape(-1), model.state_scale(i).reshape(-1),
                      model.nupd.reshape(-1), dtype, f"{what} state{i}")


@pytest.mark.gpu
@pytest.mark.parametrize("worker_id", [0, 2])
@pytest.mark.parametrize("nservers", [1, 3])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", STATEFUL)
def test_push_dense_stateful(mv_device, updater, dtype, nservers, worker_id):
    """The one-sided stateful push (``mvb_push_dense_stateful``) of worker ``worker_id`` into ``nservers``
    servers, emulated as slices of one device buffer laid out out of order with sentinel gaps; each server's
    state is a slab of three workers (one shared slab for momentum) at a padded stride. Three pushes; values
    and the worker's state slab against the model, every other word of the buffers bitwise unchanged."""
    from multiverso_b200 import _native as N
    import ctypes as C
    lib, st = N.cuda_lib(), N.stream_ptr()
    n, gap, W = 10007, 16, 3
    lens = [n] if nservers == 1 else [3000, 3000, n - 6000]
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
    order = list(range(nservers))[::-1]                       # the last server first in the buffers
    nst, per_worker = _STATES[updater]
    nslab = W if per_worker else 1
    strides = [(ln + 3) // 4 * 4 + 8 for ln in lens]          # padding between a server's worker slabs
    tdt = getattr(torch, dtype)
    data_at, state_at, pos, spos = {}, {}, gap, gap
    for s in order:
        data_at[s], state_at[s] = pos, spos
        pos += lens[s] + gap
        spos += strides[s] * nslab + gap
    rng = np.random.default_rng(nservers * 10 + worker_id)
    start = _start_values(rng, n, dtype)
    data = torch.full((pos,), _KSENT, dtype=tdt, device="cuda")
    states = [torch.full((spos,), _KSENT, dtype=tdt, device="cuda") for _ in range(nst)]
    slab = worker_id if per_worker else 0
    for s in range(nservers):
        data[data_at[s]:data_at[s] + lens[s]] = torch.from_numpy(start[offs[s]:offs[s] + lens[s]]).cuda()
        for t in states:
            o = state_at[s] + slab * strides[s]
            t[o:o + lens[s]] = 0
    data0, states0 = data.clone(), [t.clone() for t in states]
    esz = data.element_size()
    sp = (C.c_void_p * nservers)(*[data.data_ptr() + data_at[s] * esz for s in range(nservers)])
    s0 = (C.c_void_p * nservers)(*[(states[0].data_ptr() + state_at[s] * esz) if nst >= 1 else 0
                                   for s in range(nservers)])
    s1 = (C.c_void_p * nservers)(*[(states[1].data_ptr() + state_at[s] * esz) if nst >= 2 else 0
                                   for s in range(nservers)])
    so, sl = (C.c_int64 * nservers)(*offs), (C.c_int64 * nservers)(*lens)
    ss = (C.c_int64 * nservers)(*strides)
    model = ServerModel(start, 1, updater, dtype, workers=W)
    for k in range(3):
        opt, copt = _kopt(k, worker_id)
        d = _delta(rng, (n,), dtype)
        lib.mvb_push_dense_stateful(N.dtype_code(tdt), N.UPDATER_NAMES[updater], torch.from_numpy(d).cuda(), nservers,
                                    sp, s0, s1, so, sl, ss, copt, 1, st)
        model.add(d, opt)
    torch.cuda.synchronize()
    what = f"push_dense_stateful {updater} {dtype} S={nservers} worker {worker_id}"
    got = torch.cat([data[data_at[s]:data_at[s] + lens[s]] for s in range(nservers)]).cpu().numpy()
    _assert_close(got, model.data.reshape(-1), (np.abs(model.data) + model.mag).reshape(-1),
                  model.nupd.reshape(-1), dtype, f"{what} values")
    written = torch.zeros(pos, dtype=torch.bool, device="cuda")
    for s in range(nservers):
        written[data_at[s]:data_at[s] + lens[s]] = True
    assert torch.equal(data[~written], data0[~written]), f"{what}: data written outside the shards"
    mw = worker_id if per_worker else 0
    for i, t in enumerate(states):
        got = torch.cat([t[state_at[s] + slab * strides[s]:][:lens[s]] for s in range(nservers)]).cpu().numpy()
        _assert_close(got, model.state[i][mw].reshape(-1), model.state_scale(i, mw).reshape(-1),
                      model.nupd.reshape(-1), dtype, f"{what} state{i}")
        mine = torch.zeros(spos, dtype=torch.bool, device="cuda")
        for s in range(nservers):
            mine[state_at[s] + slab * strides[s]:][:lens[s]] = True
        assert torch.equal(t[~mine], states0[i][~mine]), f"{what}: state{i} written outside worker's slab"


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("updater", STATEFUL)
def test_fused_add_three_workers(mv_device, updater, dtype):
    """The fused whole-table Add (``mvb_add_dense_fused``, no signal pads) with three workers' deltas on one
    device: the owner applies worker 0, 1, 2 in that order, each with its own AddOption and, for the per-worker
    updaters, its own state slab. 4099 elements: the 16-byte path and the scalar tail. Values and every
    worker's state against the model; the padding between the state slabs stays untouched."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    n, W = 4099, 3
    nst, per_worker = _STATES[updater]
    stride = (n + 3) // 4 * 4 + 8
    tdt = getattr(torch, dtype)
    rng = np.random.default_rng(31)
    start = _start_values(rng, n, dtype)
    shard = torch.from_numpy(start).cuda()
    states = [torch.full((stride * (W if per_worker else 1),), _KSENT, dtype=tdt, device="cuda")
              for _ in range(nst)]
    for t in states:
        t.view(-1, stride)[:, :n] = 0
    model = ServerModel(start, 1, updater, dtype, workers=W)
    a = N.DenseAdd()
    a.dtype, a.updater = N.dtype_code(tdt), N.UPDATER_NAMES[updater]
    a.shard = shard.data_ptr()
    a.state0 = states[0].data_ptr() if nst >= 1 else None
    a.state1 = states[1].data_ptr() if nst >= 2 else None
    a.shard_len, a.shard_off, a.state_stride = n, 0, stride
    a.nworkers, a.worker_mask, a.world = W, (1 << W) - 1, 1
    a.scale, a.clip, a.my_worker = 0.5, 0.0, 0
    for k in range(2):
        deltas = [torch.from_numpy(_delta(rng, (n,), dtype)).cuda() for _ in range(W)]
        for w in range(W):
            opt, a.opts[w] = _kopt(k * W + w, w)
            a.delta_ptrs[w] = deltas[w].data_ptr()
            model.add(deltas[w].cpu().numpy() * 0.5, opt)
        lib.mvb_add_dense_fused(a, st)
        torch.cuda.synchronize()
    what = f"fused Add {updater} {dtype} W={W}"
    _assert_close(shard.cpu().numpy(), model.data.reshape(-1), (np.abs(model.data) + model.mag).reshape(-1),
                  model.nupd.reshape(-1), dtype, f"{what} values")
    for i, t in enumerate(states):
        slabs = t.view(-1, stride)
        for w in range(slabs.shape[0]):
            _assert_close(slabs[w, :n].cpu().numpy(), model.state[i][w].reshape(-1),
                          model.state_scale(i, w).reshape(-1), model.nupd.reshape(-1), dtype,
                          f"{what} state{i}[worker {w}]")
        assert bool((slabs[:, n:] == _KSENT).all()), f"{what}: state{i} padding written"


@pytest.mark.gpu
@pytest.mark.parametrize("updater", STATEFUL)
def test_row_mailbox_apply(mv_device, updater):
    """Row Adds through the row mailbox of a one-process fp32 MatrixTable (``push_vals`` then
    ``drain(wait=True)``, ``mvb_rowbox_apply`` on the owner), held to the model. With one rank the push waits
    only for acks of its own earlier drains and the drain only for the push's doorbell; one push per drain, and
    the push has completed (device synchronise) before the drain polls, so nothing waits on work not yet run.
    Rows never named stay bitwise unchanged in the shard and in the state."""
    from multiverso_b200.runtime import Runtime
    mv = mv_device
    rows, cols = 300, 68
    rng = np.random.default_rng(41)
    t, model = _make_table(mv, "matrix", (rows, cols), "float32", updater)
    start = model.data.copy()
    mb = t.enable_row_mailbox()
    named = set()
    for k in range(4):
        ids = np.sort(rng.choice(rows, 90, replace=False)).astype(np.int32)
        v = _delta(rng, (ids.size, cols), "float32")
        opt, _ = _kopt(k, 0)
        mb.push_vals(torch.from_numpy(ids).cuda(), torch.from_numpy(v).cuda(), opt)
        torch.cuda.synchronize()
        mb.drain(wait=True)
        mb.drain_stream.synchronize()
        model.add_rows(ids.astype(np.int64), v, opt)
        named.update(ids.tolist())
    Runtime.get().check_watchdog()
    what = f"row mailbox {updater}"
    _check_model(t, model, "float32", what)
    untouched = np.setdiff1d(np.arange(rows), sorted(named))
    assert np.array_equal(t.get().cpu().numpy().reshape(rows, cols)[untouched], start[untouched])
    for i in range(len(model.state)):
        assert not _device_state(t, i).reshape(rows, cols)[untouched].any(), f"{what}: state{i} of an unnamed row"
