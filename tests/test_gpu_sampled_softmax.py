"""PSSampledSoftmax on the GPU (csrc/cuda/sampled_softmax.cu): device draws equal to the host replay, loss, dL/dhidden
and the table after one sgd step against fp64 within a TF32 bound derived from the operands, bitwise equality over
1 / 3 / 8 shards and across runs, stateful updaters, host synchronisations and errors raised without a launch."""
import os
import subprocess
import sys
import types
import warnings

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# The GEMM feeds raw fp32 to TF32 wgmma, which keeps 10 explicit mantissa bits of each operand: 2^-11 relative
# with round-to-nearest, up to twice that when the hardware drops the low bits. A product of two operands is then
# within 4 * 2^-11 of the exact one, and a dot product within 4 * 2^-11 * |x| |w| (Cauchy-Schwarz).
TF32 = 4 * 2.0 ** -11
FP32 = 2.0 ** -24


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _sharded(W, S, gap=37):
    """W as S shards at separate places of one buffer with garbage rows between them (reference rows_per_server
    rule, the last shard takes the remainder), and a function reading the table back."""
    from multiverso_b200 import _native as N
    n, pitch = W.shape
    rps = n // S
    buf = torch.full((n + S * gap, pitch), 1e3, device=W.device)
    rm = N.RowMap()
    rm.num_row, rm.num_col, rm.nservers, rm.rows_per_server = n, pitch, S, rps
    spans = []
    for s in range(S):
        lo, hi = s * rps, (n if s == S - 1 else (s + 1) * rps)
        at = lo + (s + 1) * gap
        buf[at:at + hi - lo] = W[lo:hi]
        rm.shard_ptrs[s] = buf[at].data_ptr()
        spans.append((at, hi - lo))
    return rm, buf, lambda: torch.cat([buf[a:a + k] for a, k in spans])


def _fake_table(rm, num_row, num_col, updater=None):
    """A MatrixTable handle over an explicit row map: what the op reads of a device table."""
    from multiverso_b200 import _native as N
    return types.SimpleNamespace(_rowmap=rm, dtype=torch.float32, num_row=num_row, num_col=num_col,
                                 updater=N.UPD_SGD if updater is None else updater, is_sparse=False,
                                 rt=types.SimpleNamespace(device=torch.device("cuda", 0)))


def _logq64(ssm):
    """log(S q) in fp64 from the sampler's definition."""
    n = ssm.num_classes
    k = np.arange(n, dtype=np.float64)
    q = np.log((k + 2) / (k + 1)) / np.log(n + 1)
    return torch.from_numpy(np.log(ssm.num_sampled * q)).cuda()


def _reference(x, W, y, cand, logsq, mean=True):
    """fp64 loss, dL/dx (of loss.mean(), or loss.sum()) and dL/dW, with the bounds of the device result derived from
    TF32."""
    B, d = x.shape
    x64 = x.double().requires_grad_()
    W64 = W.double().requires_grad_()
    t = (x64 * W64[y]).sum(1) - logsq[y]
    s = (x64 @ W64[cand].t() - logsq[cand][None, :]).masked_fill(cand[None, :] == y[:, None], float("-inf"))
    z = torch.cat([t[:, None], s], 1)
    lse = torch.logsumexp(z, 1)
    loss = lse - t
    (loss.mean() if mean else loss.sum()).backward()
    with torch.no_grad():
        xn = x64.norm(dim=1)
        wmax = W64[torch.cat([y, cand])].norm(dim=1).max()
        # error of one logit: TF32 products plus fp32 accumulation over d terms, plus the fp32 log(S q)
        delta = (TF32 + d * FP32) * xn * wmax + 4 * FP32 * (1 + logsq.abs().max() + lse.abs())
        p = torch.softmax(z, 1)[:, 1:]                            # sampled-column probabilities
        g = 1.0 / B if mean else 1.0
        tol_loss = 2 * delta
        # dX_b = sum_j E_bj w_j + e_true w_y: E off by g p (2 delta), the E W_S product by TF32, e_true by g 2 delta
        tol_dx = g * wmax * (4 * delta + TF32) + 8 * FP32 * x64.grad.abs().max()
        # row r: label uses (e_true error times |x_b|) plus candidate uses (sum_b E error and TF32 times |x_b|)
        rows = torch.zeros(W.shape[0], dtype=torch.float64, device=x.device)
        rows.index_add_(0, y, g * 2 * delta * xn)
        rows.index_add_(0, cand, (g * p * (2 * delta + TF32)[:, None] * xn[:, None]).sum(0))
        # fp32 sums: the E^T X product over B terms and the coalescing over at most B + S uses, each within
        # (terms) * 2^-24 of the sum of the magnitudes of its terms
        mag = torch.zeros_like(rows)
        mag.index_add_(0, y, g * (1 - torch.softmax(z, 1)[:, 0]) * xn)
        mag.index_add_(0, cand, (g * p * xn[:, None]).sum(0))
        rows += (B + cand.numel()) * FP32 * mag
    return loss.detach(), x64.grad, W64.grad, tol_loss, tol_dx, rows


@pytest.mark.parametrize("sampler", ["log_uniform", "counts"])
def test_device_draws_equal_host_replay(cuda, sampler):
    from multiverso_b200.ops import PSSampledSoftmax
    from multiverso_b200.ops.sampled_softmax import draw_reference
    n = 200003
    rm, keep, _ = _sharded(torch.zeros(n, 4, device=cuda), 1, 0)
    counts = torch.randint(0, 50, (n,)) if sampler == "counts" else None
    kw = {"counts": counts} if counts is not None else {"sampler": "log_uniform"}
    ssm = PSSampledSoftmax(_fake_table(rm, n, 4), num_sampled=100003, seed=2**40 + 3, **kw)
    for step in (0, 1, 12345):
        dev = ssm.draw(step)
        assert dev.is_cuda and dev.dtype == torch.int64
        assert np.array_equal(dev.cpu().numpy(), draw_reference(ssm._prob, ssm._alias, ssm.seed, step, 100003))
    if counts is not None:
        assert (counts[ssm.draw(0).cpu()] > 0).all()


@pytest.mark.parametrize("d", [4, 32, 100, 128, 300, 512, 1024])
def test_matches_fp64(cuda, d):
    """Loss, dL/dhidden and the table after one sgd step against fp64, within the TF32 bound of every value."""
    from multiverso_b200.ops import PSSampledSoftmax
    g = torch.Generator(device=cuda).manual_seed(d)
    n, B, S, lr = 5003, 301, 1001, 0.5
    W = torch.randn(n, d, device=cuda, generator=g) / d ** 0.5
    rm, keep, back = _sharded(W, 1, 0)
    ssm = PSSampledSoftmax(_fake_table(rm, n, d), num_sampled=S, sampler="log_uniform", push_scale=lr, seed=d)
    x = (torch.randn(B, d, device=cuda, generator=g) * 2).requires_grad_()
    y = torch.randint(0, n, (B,), device=cuda, generator=g)
    y[:20] = ssm.draw(0)[:20]                                      # accidental hits
    loss = ssm(x, y)
    loss.mean().backward()
    torch.cuda.synchronize()
    ref, dx, dW, tol_loss, tol_dx, tol_rows = _reference(x.detach(), W, y, ssm.draw(0), _logq64(ssm))
    assert ((loss.double() - ref).abs() <= tol_loss).all(), ((loss.double() - ref).abs() / tol_loss).max().item()
    err_dx = (x.grad.double() - dx).abs().max(1).values
    assert (err_dx <= tol_dx).all(), (err_dx / tol_dx).max().item()
    exp = W.double() - lr * dW
    err_w = (back().double() - exp).abs().max(1).values
    bound = lr * tol_rows + 4 * FP32 * exp.abs().max()
    assert (err_w <= bound).all(), (err_w / bound).max().item()
    touched = torch.zeros(n, dtype=torch.bool, device=cuda)
    touched[torch.cat([y, ssm.draw(0)])] = True
    assert torch.equal(back()[~touched], W[~touched])


def _step(W, S, x, y, n_shards, lr=0.25):
    from multiverso_b200.ops import PSSampledSoftmax
    rm, keep, back = _sharded(W, n_shards, 0 if n_shards == 1 else 37)
    ssm = PSSampledSoftmax(_fake_table(rm, W.shape[0], W.shape[1]), num_sampled=S, sampler="log_uniform",
                           push_scale=lr, seed=4)
    xx = x.clone().requires_grad_()
    loss = ssm(xx, y)
    loss.mean().backward()
    torch.cuda.synchronize()
    return loss.detach(), xx.grad, back()


def test_bitwise_over_shards_and_runs(cuda):
    g = torch.Generator(device=cuda).manual_seed(9)
    n, d, B, S = 20011, 128, 1024, 2048
    W = torch.randn(n, d, device=cuda, generator=g) * 0.1
    x = torch.randn(B, d, device=cuda, generator=g)
    y = (torch.rand(B, device=cuda, generator=g) ** 3 * n).long()   # a Zipf-like head of repeated labels
    ref = _step(W, S, x, y, 1)
    for shards in (1, 3, 8):
        got = _step(W, S, x, y, shards)
        for a, b in zip(ref, got):
            assert torch.equal(a, b), shards


@pytest.mark.parametrize("updater", ["momentum_sgd", "adagrad"])
def test_stateful_one_step_per_row(mv_device, updater):
    """A stateful table takes exactly one updater step per unique row with the gradient summed over the row's label
    and candidate uses. The same call over a recording table yields the compact push: one row per touched id, each
    within the TF32 bound of the fp64 gradient. The table after the real call is bitwise equal to an identical table
    given that one explicit add_rows_async; for momentum (linear in the gradient) it also matches fp64."""
    from multiverso_b200 import _native as N
    from multiverso_b200.ops import PSSampledSoftmax
    from multiverso_b200.tables.options import AddOption
    mv = mv_device
    n, d, B, S, scale = 3000, 32, 256, 512, 0.1
    t = mv.MatrixTable(n, d, "float32", updater=updater, min_value=-0.5, max_value=0.5, seed=11)
    twin = mv.MatrixTable(n, d, "float32", updater=updater, min_value=-0.5, max_value=0.5, seed=11)
    W0 = t.get().view(n, d).clone()
    assert torch.equal(twin.get().view(n, d), W0)
    opt = AddOption(momentum=0.9, learning_rate=0.5, rho=0.2)
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, d, device="cuda", generator=g)
    y = torch.randint(0, 50, (B,), device="cuda", generator=g)      # labels that are also frequent candidates
    # the compact push of the call, recorded instead of applied
    rm, keep, _ = _sharded(W0, 1, 0)
    pushes = []
    rec = _fake_table(rm, n, d, N.UPDATER_NAMES[updater])
    rec.add_rows_async = lambda ids, vals, option=None: pushes.append((ids.clone(), vals.clone(), option))
    PSSampledSoftmax(rec, num_sampled=S, sampler="log_uniform", push_scale=scale, option=opt, seed=1)(x, y) \
        .mean().backward()
    ssm = PSSampledSoftmax(t, num_sampled=S, sampler="log_uniform", push_scale=scale, option=opt, seed=1)
    ssm(x, y).mean().backward()
    torch.cuda.synchronize()
    cand = ssm.draw(0)
    touched = torch.unique(torch.cat([y, cand]))
    assert len(pushes) == 1
    uniq, grads, option = pushes[0]
    assert torch.equal(uniq, touched) and option is opt                 # one row per touched id, once
    _, _, dW, _, _, tol_rows = _reference(x, W0, y, cand, _logq64(ssm))
    err = (grads.double() - scale * dW[touched]).abs().max(1).values
    assert (err <= scale * tol_rows[touched]).all(), (err / (scale * tol_rows[touched])).max().item()
    twin.wait(twin.add_rows_async(uniq, grads, opt))
    torch.cuda.synchronize()
    got = t.get().view(n, d)
    assert torch.equal(got, twin.get().view(n, d))
    assert ((got - W0).abs().max(1).values[touched] > 0).float().mean() > 0.9
    if updater == "momentum_sgd":
        exp = W0.double().clone()
        exp[touched] -= (1.0 - 0.9) * scale * dW[touched]
        bound = (1.0 - 0.9) * scale * tol_rows[touched] + 4 * FP32 * exp[touched].abs().max(1).values
        err = (got.double() - exp)[touched].abs().max(1).values
        assert (err <= bound).all(), (err / bound).max().item()


def test_empty_batch_pushes_nothing(mv_device):
    """B = 0 right after a full call (whose buffers the allocator hands back): an empty loss, and the backward pushes
    nothing into an sgd or a momentum table."""
    from multiverso_b200.ops import PSSampledSoftmax
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(8)
    for updater in ("sgd", "momentum_sgd"):
        t = mv.MatrixTable(2000, 64, "float32", updater=updater, min_value=-0.5, max_value=0.5)
        ssm = PSSampledSoftmax(t, num_sampled=1000, sampler="log_uniform", push_scale=0.1)
        ssm(torch.randn(300, 64, device="cuda", generator=g), torch.randint(0, 2000, (300,), device="cuda")).sum()\
            .backward()
        torch.cuda.synchronize()
        before = t.get().clone()
        x = torch.zeros(0, 64, device="cuda", requires_grad=True)
        loss = ssm(x, torch.zeros(0, dtype=torch.int64, device="cuda"))
        assert loss.shape == (0,)
        loss.sum().backward()
        torch.cuda.synchronize()
        assert torch.equal(t.get(), before), updater
        assert x.grad.shape == (0, 64)


def test_second_backward_raises(cuda):
    """The backward turns the saved logits into E: a second backward through a retained graph raises instead of
    computing from E and pushing again."""
    from multiverso_b200.ops import PSSampledSoftmax
    rm, keep, back = _sharded(torch.randn(500, 32, device=cuda), 1, 0)
    ssm = PSSampledSoftmax(_fake_table(rm, 500, 32), num_sampled=64, sampler="log_uniform", push_scale=0.1)
    x = torch.randn(16, 32, device=cuda, requires_grad=True)
    loss = ssm(x, torch.arange(16, device=cuda))
    loss.sum().backward(retain_graph=True)
    torch.cuda.synchronize()
    after, dx = back().clone(), x.grad.clone()
    with pytest.raises(RuntimeError, match="backward ran twice"):
        loss.sum().backward()
    torch.cuda.synchronize()
    assert torch.equal(back(), after) and torch.equal(x.grad, dx)


def _syncs(fn):
    """Synchronising torch calls made by fn (torch's sync debug mode in 'warn')."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("called a synchronizing CUDA operation" in str(x.message) for x in w)


def test_host_syncs(mv_device):
    """1 per forward (the label checks), 0 per sgd backward, 1 per backward with a compact (adagrad) push."""
    from multiverso_b200.ops import PSSampledSoftmax
    mv = mv_device
    g = torch.Generator(device="cuda").manual_seed(6)
    x = torch.randn(512, 64, device="cuda", generator=g, requires_grad=True)
    y = torch.randint(0, 4000, (512,), device="cuda", generator=g)
    for updater, want in (("sgd", 0), ("adagrad", 1)):
        t = mv.MatrixTable(4000, 64, "float32", updater=updater)
        ssm = PSSampledSoftmax(t, num_sampled=1000, sampler="log_uniform", push_scale=0.1)
        ssm(x, y).mean().backward()                                   # warm-up
        out = []
        assert _syncs(lambda: out.append(ssm(x, y))) == 1
        assert _syncs(lambda: out[0].mean().backward()) == want, updater


def _ss_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if "ss_" in e.name and "kernel" in e.name or "gemm" in e.name)


def test_errors_raise_without_launching(cuda):
    from multiverso_b200.ops import PSSampledSoftmax
    n, d = 1000, 32
    rm, keep, _ = _sharded(torch.randn(n, d, device=cuda), 1, 0)
    counts = torch.ones(n)
    counts[5] = 0
    ssm = PSSampledSoftmax(_fake_table(rm, n, d), num_sampled=64, counts=counts)
    x = torch.randn(8, d, device=cuda)
    ok = torch.arange(8, device=cuda) + 10
    assert _ss_kernels(lambda: ssm(x, ok)) >= 3                      # the counter does see the op's kernels
    cases = [
        (ValueError, r"\[0, 1000\)", x, torch.tensor([0, 1, 2, 3, 4, 6, 7, 1000], device=cuda)),
        (ValueError, "count zero", x, torch.tensor([0, 1, 2, 3, 4, 5, 7, 8], device=cuda)),
        (ValueError, "hidden has 16 columns", torch.randn(8, 16, device=cuda), ok),
        (ValueError, "one label per row", x, ok[:7]),
        (TypeError, "2-D float32", x.half(), ok),
    ]
    steps = ssm.steps
    for exc, msg, h, y in cases:
        def call():
            with pytest.raises(exc, match=msg):
                ssm(h, y)
        assert _ss_kernels(call) == 0, msg
    assert ssm.steps == steps


@pytest.mark.parametrize("nproc", [2, 4])
def test_sampled_softmax_peer_shards_multi_gpu(nproc):
    """A table sharded over 2 / 4 GPUs (tests/mp_sampled_softmax_check.py under torchrun): identical draws on every
    rank, forward bitwise equal to a single-shard copy, async sgd pushes from every rank landing as W0 - lr * sum."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < nproc:
        pytest.skip(f"needs >= {nproc} GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    port = 29500 + (os.getpid() % 150) + 800 + nproc
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "tests", "mp_sampled_softmax_check.py")]
    r = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=900)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    assert "FAIL" not in r.stdout and r.stdout.count("PASS") == nproc, tail
