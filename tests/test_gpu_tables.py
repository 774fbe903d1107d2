"""GPU numerics: every table kernel against a plain PyTorch fp32/fp64 reference.
Scenarios mirror Test/unittests/test_array.cpp, test_kv.cpp, Test/test_matrix_table.cpp."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref_update(name, data, delta, st, opt):
    m, lr, rho, lam = opt["momentum"], opt["lr"], opt["rho"], opt["lam"]
    if name == "default":
        data += delta
    elif name == "sgd":
        data -= delta
    elif name == "momentum_sgd":
        st[0].mul_(m).add_((1 - m) * delta)
        data -= st[0]
    elif name == "adagrad":
        g = delta / lr
        st[0] += g * g
        data -= rho / torch.sqrt(st[0] + 1e-6) * g
    elif name == "dcasgd":
        g = delta / lr
        data -= lr * (g + lam * g * g * (data - st[0]))
        st[0].copy_(data)
    elif name == "dcasgda":
        g = delta / lr
        st[1].mul_(m).add_((1 - m) * g * g)
        data -= lr * (g + lam / torch.sqrt(st[1] + 1e-7) * g * g * (data - st[0]))
        st[0].copy_(data)


@pytest.mark.parametrize("updater", ["default", "sgd", "momentum_sgd", "adagrad", "dcasgd", "dcasgda"])
@pytest.mark.parametrize("size", [1, 1000, 4099, 1 << 20])
def test_array_add_get_matches_reference(mv_device, updater, size):
    mv = mv_device
    t = mv.ArrayTable(size, "float32", updater=updater)
    torch.manual_seed(0)
    ref = torch.zeros(size, dtype=torch.float64)
    st = [torch.zeros(size, dtype=torch.float64), torch.zeros(size, dtype=torch.float64)]
    opt = mv.AddOption(momentum=0.9, learning_rate=0.05, rho=0.1, lambda_=0.2)
    o = dict(momentum=0.9, lr=0.05, rho=0.1, lam=0.2)
    for it in range(3):
        delta = torch.randn(size, device="cuda") * 0.1
        t.add(delta, opt)
        _ref_update(updater, ref, delta.double().cpu(), st, o)
    got = t.get().cpu().double()
    assert torch.allclose(got, ref, rtol=2e-4, atol=2e-5), (got - ref).abs().max()


def test_array_integer_scenario_exact(mv_device):
    """test_array.cpp:26-44: Add(delta) -> Get == delta; AddAsync+GetAsync+Wait == 2*delta."""
    mv = mv_device
    n = 100000
    t = mv.ArrayTable(n, "float32")
    delta = torch.arange(n, dtype=torch.float32, device="cuda")
    t.add(delta)
    assert torch.equal(t.get(), delta)
    h = t.add_async(delta)
    t.wait(h)
    h2, out = t.get_async()
    t.wait(h2)
    assert torch.equal(out, 2 * delta)
    ti = mv.ArrayTable(1001, "int32")
    di = torch.arange(1001, dtype=torch.int32, device="cuda")
    ti.add(di)
    ti.add(di)
    assert torch.equal(ti.get(), 2 * di)
    td = mv.ArrayTable(513, "float64", updater="sgd")
    dd = torch.randn(513, dtype=torch.float64, device="cuda")
    td.add(dd)
    assert torch.allclose(td.get(), -dd)


def test_matrix_rows_exact_integer_scenario(mv_device):
    """Test/test_matrix_table.cpp:9-99 at world size 1: whole-table and row-set Add/Get with
    the exact integer expectation (i*cols+j+1)*count (doubled for rows 0,1,3,7)."""
    mv = mv_device
    rows, cols = 11, 10
    t = mv.MatrixTable(rows, cols, "float32")
    base = (torch.arange(rows * cols, dtype=torch.float32, device="cuda") + 1).view(rows, cols)
    ids = torch.tensor([0, 1, 3, 7], device="cuda")
    for count in range(1, 4):
        t.add(base)
        t.add_rows(ids, base[ids])
        got = t.get().view(rows, cols)
        exp = base * count
        exp[ids] *= 2
        assert torch.equal(got, exp)
        assert torch.equal(t.get_rows(ids), exp[ids])
        assert torch.equal(t.get_row(5), exp[5])


@pytest.mark.parametrize("cols", [1, 7, 300, 512])
def test_matrix_get_add_rows_random(mv_device, cols):
    mv = mv_device
    rows = 5000
    t = mv.MatrixTable(rows, cols, "float32", min_value=-1.0, max_value=1.0)
    full = t.get().view(rows, cols).clone()
    g = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.randperm(rows, device="cuda", generator=g)[:777]
    assert torch.equal(t.get_rows(ids), full[ids])
    vals = torch.randn(777, cols, device="cuda")
    t.add_rows(ids, vals)
    full[ids] += vals
    assert torch.allclose(t.get().view(rows, cols), full, atol=1e-6)


def test_matrix_stateful_rows_and_sparse_stale(mv_device):
    mv = mv_device
    rows, cols = 64, 16
    t = mv.MatrixTable(rows, cols, "float32", updater="momentum_sgd", is_sparse=True)
    ids0, r0 = t.get_stale()
    assert ids0.numel() == rows           # everything stale before the first pull
    ids1, _ = t.get_stale()
    assert ids1.numel() == 0              # explicit empty result (Q12)
    ids = torch.tensor([3, 9, 40], device="cuda")
    vals = torch.ones(3, cols, device="cuda")
    opt = mv.AddOption(momentum=0.5)
    t.add_rows(ids, vals, opt)
    sid, srows = t.get_stale()
    assert sid.tolist() == [3, 9, 40]
    assert torch.allclose(srows, torch.full((3, cols), -0.5, device="cuda"))
    d = torch.zeros(rows, cols, device="cuda")
    d[5] = 2.0
    t.add(d, opt)                          # zero rows are skipped when marking
    sid, _ = t.get_stale()
    assert sid.tolist() == [5]


def test_kv_table(mv_device):
    """test_kv.cpp:25-39: Get 0 -> 0, Add 3 -> 3, Add -4 -> -1."""
    mv = mv_device
    kv = mv.KVTable("int64", "float32")
    assert kv.get(0) == 0
    kv.add(0, 3.0)
    assert kv.get(0) == 3.0
    kv.add(0, -4.0)
    assert kv.get(0) == -1.0
    keys = torch.arange(-500, 500, device="cuda") * 7919 + 1
    kv.add(keys, torch.ones(1000, device="cuda"))
    kv.add(keys, torch.ones(1000, device="cuda"))
    assert torch.equal(kv.get(keys), torch.full((1000,), 2.0, device="cuda"))
    assert kv.raw()[0] == -1.0
    kvi = mv.KVTable("int64", "int64")
    kvi.add(4, 10**12)
    kvi.add(4, 5)
    assert kvi.get(4) == 10**12 + 5


def test_kv_table_grows(mv_device):
    """The reference's server map is unbounded (kv_table.h:86-106): start with 1024 slots, insert 50 000 distinct
    keys in batches with repeated hits, every value must survive the re-hashes."""
    import multiverso_b200 as mv
    kv = mv.KVTable("int64", "float32", capacity=1024)
    g = torch.Generator().manual_seed(0)
    keys = torch.randperm(10_000_000, generator=g)[:50_000] - 5_000_000          # negative keys too
    for lo in range(0, 50_000, 700):
        k = keys[lo:lo + 700].cuda()
        kv.add(k, torch.ones(k.numel(), device="cuda"))
        kv.add(k[:100], torch.full((min(100, k.numel()),), 2.0, device="cuda"))
    torch.cuda.synchronize()
    assert kv.growths >= 5 and kv.capacity >= 2 * 50_000
    got = kv.get(keys.cuda())
    exp = torch.ones(50_000)
    for lo in range(0, 50_000, 700):
        exp[lo:lo + 100] += 2.0
    assert torch.equal(got.cpu(), exp)
    assert float(kv.get(123456789)) == 0.0                                        # missing key -> default value
    assert kv.live_keys() == 50_000


def test_app_defined_tables_sparse_and_ftrl(mv_device):
    """The reference's application tables (sparse_table.h, ftrl_sparse_table.h) on the device extension point:
    server subtracts, whole-table Get returns only the keys ever written, FTRL carries {z, n} pairs."""
    import multiverso_b200 as mv
    from multiverso_b200.tables.custom import SparseTableOption, FTRLDeviceTable
    n = 1_000_003
    t = mv.create_table(SparseTableOption(n))
    g = torch.Generator().manual_seed(0)
    keys = torch.randperm(n, generator=g)[:5000]
    vals = torch.randn(5000, generator=g)
    t.add(keys, vals)
    t.add(keys[:100], torch.ones(100))
    exp = -vals.clone(); exp[:100] -= 1.0
    assert torch.allclose(t.get(keys).cpu(), exp, atol=1e-6)
    assert float(t.get([n - 1 if (n - 1) not in keys.tolist() else 7]).abs().sum()) >= 0.0
    k_all, v_all = t.get()
    order = torch.argsort(keys)
    assert torch.equal(k_all.cpu(), keys[order]) and torch.allclose(v_all.cpu(), exp[order], atol=1e-6)
    f = FTRLDeviceTable(4099)
    fk = torch.arange(0, 4099, 7)
    f.add(fk, torch.stack([torch.full((fk.numel(),), 0.5), torch.full((fk.numel(),), 2.0)], 1))
    got = f.get(fk).cpu()
    assert torch.allclose(got[:, 0], torch.full((fk.numel(),), -0.5)) and torch.allclose(got[:, 1], torch.full((fk.numel(),), -2.0))
    ka, va = f.get()
    assert ka.numel() == fk.numel() and va.shape == (fk.numel(), 2)


def test_custom_device_table_extension_point(mv_device, tmp_path):
    """A user-defined table on the extension point: subclass CustomDeviceTable, express the ops on the peer-mapped
    shard tensors, get table id / partition / checkpoint plumbing from the base."""
    import multiverso_b200 as mv
    from multiverso_b200.tables.custom import CustomDeviceTable

    class MaxTable(CustomDeviceTable):                     # Add keeps the element-wise maximum
        def __init__(self, size):
            super().__init__(size, 4)

        def add(self, keys, vals):
            keys = torch.as_tensor(keys, device="cuda"); vals = torch.as_tensor(vals, dtype=torch.float32, device="cuda")
            for s in range(self.S):
                m = (keys >= self.lo[s]) & (keys < self.hi[s])
                if bool(m.any()):
                    shard = self.peer_tensor(s)
                    idx = keys[m] - self.lo[s]
                    shard[idx] = torch.maximum(shard[idx], vals[m])

        def get(self, keys):
            keys = torch.as_tensor(keys, device="cuda")
            out = torch.empty(keys.numel(), device="cuda")
            for s in range(self.S):
                m = (keys >= self.lo[s]) & (keys < self.hi[s])
                if bool(m.any()):
                    out[m] = self.peer_tensor(s)[keys[m] - self.lo[s]]
            return out

    t = MaxTable(1000)
    t.add([1, 5, 999], [3.0, -1.0, 7.0])
    t.add([1, 5], [2.0, 4.0])
    assert t.get([1, 5, 999, 0]).tolist() == [3.0, 4.0, 7.0, 0.0]
    assert mv.save_table(t, str(tmp_path / "max"))
    t.add([1], [100.0])
    assert mv.load_table(t, str(tmp_path / "max"))
    assert t.get([1]).tolist() == [3.0]


def test_aggregate_single_rank(mv_device):
    x = torch.ones(10, device="cuda")
    mv_device.aggregate(x)
    assert torch.equal(x, torch.ones(10, device="cuda"))


def test_checkpoint_roundtrip(mv_device, tmp_path):
    import io
    mv = mv_device
    t = mv.ArrayTable(1000, "float32", updater="momentum_sgd")
    t.add(torch.randn(1000, device="cuda"), mv.AddOption(momentum=0.9))
    buf = io.BytesIO()
    t.store(buf)
    want = t.get().clone()
    t2 = mv.ArrayTable(1000, "float32", updater="momentum_sgd")
    buf.seek(0)
    t2.load(buf)
    assert torch.equal(t2.get(), want)
    assert torch.equal(t2.state[0], t.state[0])


@pytest.mark.gpu
def test_watchdog_reports_dead_peer(mv_device):
    """Fault injection (SURVEY 5.3): a device-side wait on a flag that nobody will ever write must end
    with a diagnostic naming the channel / peer after -barrier_timeout_s, not hang the GPU."""
    import time
    from multiverso_b200 import _native as N
    from multiverso_b200.runtime import Runtime
    from multiverso_b200.utils.log import FatalError, Log
    rt = Runtime.get()
    ch = rt.new_channels(1)
    kill, Log.kill_fatal = Log.kill_fatal, False
    try:
        t0 = time.time()
        N.cuda_lib().mvb_wait(rt.pads_array(), rt.rank, rt.size, ch, 7, 1, rt.err_flag, 0.05, N.stream_ptr())
        torch.cuda.synchronize()
        assert time.time() - t0 < 10.0                     # gave up after the budget, did not spin forever
        with pytest.raises(FatalError, match="watchdog"):
            rt.check_watchdog()
        rt.check_watchdog()                                # the flag is cleared: the runtime stays usable
        t = mv_device.ArrayTable(1000, "float32")
        t.add(torch.ones(1000, device="cuda"))
        assert bool((t.get() == 1).all())
    finally:
        Log.kill_fatal = kill
