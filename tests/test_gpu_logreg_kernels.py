"""K8 numerics against plain PyTorch references: the sparse / dense CUDA-core kernels, FTRL, regularisers
(csrc/cuda/logreg.cu) and the wide dense path whose two products run on the hand-written wgmma kernel
(no library GEMM), each compared with fp32/fp64 torch on the same inputs.

The bounds below follow the operations each kernel does, with u = 2^-24 the fp32 unit roundoff and an ulp at most
2^-23 of the value:

* logit z_ic: the CUDA-core kernels sum m fp32 fmaf terms per lane and then over the warp (5 more levels), so
  |dz| <= (m + 6) u A_ic with A = |x| |W|^T; the wgmma GEMM gives (TF32 + m FP32) A_ic (test_gpu_get_gemm.py).
* __expf(t) is within 2 + floor(1.173 |t|) ulp, taken as (3 + 1.2 |t|) 2^-23 relative; __logf(p) is within 2^-21.41
  absolute on [0.5, 2] and 3 ulp elsewhere, taken as 2^-21 + 3 2^-23 |log p|.
* sigmoid p = 1 / (1 + exp(-z)): |dp| <= p ((1 - p)(dz + E(z)) + 2u). softmax p_c = exp(t_c) / sum exp(t_k) with
  t = z - max: |dp_c| <= p_c (E(t_c) + dt_c + sum_k p_k (E(t_k) + dt_k) + (out + 7) u), dt_c <= dz_c + max dz + u |t_c|.
  linear p = z: |dp| <= dz.
* err = (p - y) w / n: |derr| <= (|dp| + 4u |p - y|) w / n. The per-sample loss is propagated through p and __logf
  the same way, and the loss sum, added in fp32 in any order, gets (count + 2) u sum |l|.
* grad = E^T X, added with fp32 fma and red.add in any order over c contributions: |dg| <= |dE|^T |X|
  + (c + 2) u |E|^T |X|; through the GEMM, (TF32 + n_pad FP32)(|E| + |dE|)^T |X| instead of the second term.
* correct: the argmax (or threshold) of the fp64 reference decides a sample only where its top-two margin exceeds
  twice the logit bound (or its distance to the threshold exceeds the bound of p). The kernel's count must lie
  between the sure hits and the sure hits plus the undecided samples, which is exact when none is undecided.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ULP = 2.0 ** -23
TF32 = 4 * 2.0 ** -11
FP32 = 2.0 ** -24


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _exp_rel(t):
    return (3 + 1.2 * t.abs()) * ULP


def _log_abs(p):
    return 2.0 ** -21 + 3 * ULP * p.log().abs()


def _epilogue64(Z, dz, labels, objective, wgt):
    """fp64 reference of finish_sample / lr_wide_epilogue_kernel on logits Z (|z_fp32 - Z| <= dz) and per-sample
    weights ``wgt``: p, err, loss sum, the bounds of each and the [lo, hi] range of the correct count."""
    n, out = Z.shape
    y = labels.double()
    w = wgt.double().view(n, 1)
    lab = labels.long().view(n, 1).clamp(0, out - 1)
    if out == 1:
        T = y.view(n, 1)
    else:
        T = torch.zeros_like(Z).scatter_(1, lab, 1.0)
    if objective == 2 and out > 1:
        t = Z - Z.max(1, keepdim=True).values
        P = torch.softmax(Z, 1)
        dt = dz + dz.max(1, keepdim=True).values + U * t.abs()
        e = _exp_rel(t) + dt
        dP = P * (e + (P * e).sum(1, keepdim=True) + (out + 7) * U)
        py = P.gather(1, lab)
        L = -py.log()
        dL = dP.gather(1, lab) / py + _log_abs(py) + U * L
    elif objective >= 1:
        P = torch.sigmoid(Z)
        dP = P * ((1 - P) * (dz + _exp_rel(Z)) + 2 * U)
        Q = 1 - P
        L = -(T * P.log() + (1 - T) * Q.log())
        dL = T * (dP / P + _log_abs(P)) + (1 - T) * ((dP + U * Q) / Q + _log_abs(Q)) + 3 * U * L
    else:
        P, dP = Z, dz
        L = 0.5 * (P - T) ** 2
        dL = (P - T).abs() * dz + dz ** 2 + 4 * U * L
    L, dL = L * w, dL * w.abs() + U * (L * w).abs()
    err = (P - T) * w / n
    derr = (dP + 4 * U * (P - T).abs()) * w.abs() / n
    loss, dloss = L.sum().item(), dL.sum().item() + (L.numel() + 2) * U * L.abs().sum().item()
    if out > 1:
        top = Z.topk(2, 1).values
        sure = top[:, 0] - top[:, 1] > 2 * dz.max(1).values
        hit = Z.argmax(1) == labels.long()
    elif objective >= 1:
        sure = (P[:, 0] - 0.5).abs() > dP[:, 0]
        hit = (P[:, 0] > 0.5) == (y > 0.5)
    else:
        sure = ((P[:, 0] - y).abs() - 0.5).abs() > dP[:, 0] + U
        hit = (P[:, 0] - y).abs() < 0.5
    lo = int((hit & sure).sum())
    return dict(P=P, dP=dP, err=err, derr=derr, loss=loss, dloss=dloss, correct=(lo, lo + int((~sure).sum())))


def _within(got, ref, tol, what):
    bad = (got.double() - ref).abs() > tol
    assert not bad.any(), (what, bad.nonzero()[:4].tolist(), (got.double() - ref).abs().max().item())


def _check_outputs(r, pred, err, loss, correct, what):
    n, out = r["P"].shape
    if pred is not None:
        _within(pred.view(n, out), r["P"], r["dP"], (what, "pred"))
    if err is not None:
        _within(err.view(n, out), r["err"], r["derr"], (what, "err"))
    assert abs(loss.item() - r["loss"]) <= r["dloss"], (what, "loss", loss.item(), r["loss"], r["dloss"])
    lo, hi = r["correct"]
    assert lo <= int(correct.item()) <= hi, (what, "correct", int(correct.item()), lo, hi)


def _ref_dense(x, labels, w, objective, out):
    n, dim = x.shape
    logits = x.double() @ w.double().view(out, dim).t()
    if out == 1:
        tgt = labels.view(n, 1).double()
    else:
        tgt = torch.zeros_like(logits); tgt.scatter_(1, labels.view(n, 1).long(), 1.0)
    if objective == 2 and out > 1:
        p = torch.softmax(logits, 1)
        loss = -torch.log(p.gather(1, labels.view(n, 1).long())).sum()
    elif objective >= 1:
        p = torch.sigmoid(logits)
        loss = -(tgt * torch.log(p) + (1 - tgt) * torch.log(1 - p)).sum()
    else:
        p = logits
        loss = 0.5 * ((p - tgt) ** 2).sum()
    grad = (p - tgt).t() @ x.double() / n
    if out > 1:
        correct = (p.argmax(1) == labels.long()).sum()
    elif objective >= 1:
        correct = ((p.view(-1) > 0.5) == (labels > 0.5)).sum()
    else:
        correct = ((p.view(-1) - labels.double()).abs() < 0.5).sum()
    return loss.item(), int(correct), p.float(), grad.float()


@pytest.mark.parametrize("n,dim,out,objective", [(256, 40, 5, 2), (100, 785, 10, 2), (64, 33, 1, 1), (50, 20, 1, 0)])
def test_dense_cuda_core_kernel(mv_device, n, dim, out, objective):
    from multiverso_b200 import _native as N
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, dim, device="cuda", generator=g)
    w = torch.randn(out * dim, device="cuda", generator=g) * 0.1
    labels = (torch.randint(0, out, (n,), device="cuda", generator=g) if out > 1
              else torch.randint(0, 2, (n,), device="cuda", generator=g)).float()
    grad = torch.zeros(out * dim, device="cuda"); loss = torch.zeros(1, device="cuda")
    correct = torch.zeros(1, dtype=torch.int32, device="cuda")
    pred = torch.zeros(n * out, device="cuda"); err = torch.zeros(n * out, device="cuda")
    a = N.LrDense()
    a.x, a.labels, a.n, a.dim, a.out, a.objective = x.data_ptr(), labels.data_ptr(), n, dim, out, objective
    a.w, a.grad, a.loss_sum, a.correct = w.data_ptr(), grad.data_ptr(), loss.data_ptr(), correct.data_ptr()
    a.pred, a.err, a.compute_grad = pred.data_ptr(), err.data_ptr(), 1
    N.cuda_lib().mvb_lr_dense_fwd_bwd(a, N.stream_ptr())
    torch.cuda.synchronize()
    rl, rc, rp, rg = _ref_dense(x, labels, w, objective, out)
    assert abs(loss.item() - rl) / max(abs(rl), 1e-6) < 1e-3
    assert int(correct.item()) == rc
    assert torch.allclose(pred.view(n, out), rp, atol=2e-4)
    assert torch.allclose(grad.view(out, dim), rg, atol=2e-4)


def _wide_model(dim, out, objective, n):
    from multiverso_b200.models.logreg import LogRegConfig, LogRegModel
    cfg = LogRegConfig(input_size=dim - 1, output_size=out, sparse=False, use_ps=False,
                       objective_type={2: "softmax", 1: "sigmoid", 0: "default"}[objective], minibatch_size=n)
    m = LogRegModel(cfg)
    assert m.dim == dim and m.objective == objective
    return m


def _wide_step_checked(m, x, labels, g0, train=True):
    """One forward_backward_dense on the wide path from grad = g0, checked against fp64: the logits within the
    GEMM bound, the epilogue's outputs within _epilogue64's bounds, and grad = g0 + E^T X within the GEMM bound of
    the error matrix times X (TF32 operands, n_pad fp32 terms) plus the rounding of the axpy."""
    n, dim = x.shape
    out = m.out
    pred = torch.full((n * out,), float("nan"), device=x.device)
    m.loss.zero_(); m.correct.zero_(); m.grad.copy_(g0)
    m.forward_backward_dense(x, labels, train=train, pred=pred)
    torch.cuda.synchronize()
    W, X = m.w.double().view(out, dim), x.double()
    Z = X @ W.T
    dz = (TF32 + dim * FP32) * (X.abs() @ W.abs().T)
    r = _epilogue64(Z, dz, labels, m.objective, torch.ones(n, device=x.device))
    _check_outputs(r, pred, None, m.loss, m.correct, ("wide", n, out, m.objective))
    if not train:
        assert torch.equal(m.grad, g0)
        return
    n_pad = (n + 3) // 4 * 4
    G = r["err"].T @ X
    dG = r["derr"].T @ X.abs() + (TF32 + n_pad * FP32) * ((r["err"].abs() + r["derr"]).T @ X.abs())
    ref = g0.double().view(out, dim) + G
    _within(m.grad.view(out, dim), ref, dG + U * (ref.abs() + dG), ("wide grad", n, out, m.objective))


@pytest.mark.parametrize("n,dim,out,objective", [(512, 256, 128, 2), (301, 64, 70, 2), (257, 128, 96, 1), (1000, 512, 1000, 2)])
def test_dense_wide_path_on_tcgen05(mv_device, n, dim, out, objective):
    """> 64 classes: LogRegModel.forward_backward_dense through gemm_fused.cu + the epilogue kernel (TF32
    products, fp32 accumulation): predictions / loss / correct / gradient within the bounds of the module
    docstring around the fp64 reference."""
    m = _wide_model(dim, out, objective, n)
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(n, dim, device="cuda", generator=g)
    m.w.copy_(torch.randn(out * dim, device="cuda", generator=g) * 0.05)
    labels = torch.randint(0, out, (n,), device="cuda", generator=g).float()
    _wide_step_checked(m, x, labels, torch.zeros(out * dim, device="cuda"))


@pytest.mark.parametrize("out", [65, 129, 1000])
@pytest.mark.parametrize("objective", [0, 1, 2])
def test_dense_wide_path_edges(mv_device, objective, out):
    """n_pad padding (n = 1, 3, 5, 129), labels at class 0 and out - 1, the gradient accumulated onto a nonzero
    grad, and train=False leaving grad bitwise alone."""
    dim = 36
    m = _wide_model(dim, out, objective, 129)
    g = torch.Generator(device="cuda").manual_seed(out + objective)
    m.w.copy_(torch.randn(out * dim, device="cuda", generator=g) * 0.1)
    for n in (1, 3, 5, 129):
        x = torch.randn(n, dim, device="cuda", generator=g)
        labels = torch.randint(0, out, (n,), device="cuda", generator=g).float()
        labels[-1] = out - 1
        if n > 1:
            labels[0] = 0
        g0 = torch.randn(out * dim, device="cuda", generator=g)
        _wide_step_checked(m, x, labels, g0, train=True)
        _wide_step_checked(m, x, labels, g0, train=False)


@pytest.mark.parametrize("objective", [0, 1])
def test_wide_epilogue_single_output(cuda, objective):
    """The out == 1 branch of lr_wide_epilogue_kernel (the model reaches it only at n dim >= 2^26): err_t's pad
    columns are zero, the rest within the bounds of the exact fp32 logits."""
    from multiverso_b200 import _native as N
    g = torch.Generator(device=cuda).manual_seed(9)
    for n in (1, 5, 70):
        n_pad = (n + 3) // 4 * 4 + 4
        logits = torch.randn(n, device=cuda, generator=g) * 3
        labels = torch.randint(0, 2, (n,), device=cuda, generator=g).float()
        err_t = torch.full((n_pad,), float("nan"), device=cuda)
        pred = torch.full((n,), float("nan"), device=cuda)
        loss = torch.zeros(1, device=cuda); correct = torch.zeros(1, dtype=torch.int32, device=cuda)
        N.cuda_lib().mvb_lr_wide_epilogue(logits, labels, n, 1, objective, err_t, n_pad, pred, loss, correct,
                                          N.stream_ptr())
        torch.cuda.synchronize()
        assert torch.equal(err_t[n:], torch.zeros(n_pad - n, device=cuda))
        r = _epilogue64(logits.double().view(n, 1), torch.zeros(n, 1, dtype=torch.float64, device=cuda), labels,
                        objective, torch.ones(n, device=cuda))
        _check_outputs(r, pred, err_t[:n], loss, correct, ("out=1", n, objective))


def test_sparse_kernel_matches_reference(mv_device):
    from multiverso_b200 import _native as N
    g = torch.Generator(device="cuda").manual_seed(3)
    n, dim, nnz_per = 300, 5000, 12
    keys = torch.randint(0, dim, (n * nnz_per,), device="cuda", generator=g)
    vals = torch.rand(n * nnz_per, device="cuda", generator=g)
    row_ptr = torch.arange(0, n * nnz_per + 1, nnz_per, device="cuda")
    w = torch.randn(dim, device="cuda", generator=g) * 0.3
    labels = torch.randint(0, 2, (n,), device="cuda", generator=g).float()
    grad = torch.zeros(dim, device="cuda"); loss = torch.zeros(1, device="cuda")
    correct = torch.zeros(1, dtype=torch.int32, device="cuda"); err = torch.zeros(n, device="cuda")
    pred = torch.zeros(n, device="cuda")
    a = N.LrSparse()
    a.row_ptr, a.keys, a.vals, a.labels, a.n = row_ptr.data_ptr(), keys.data_ptr(), vals.data_ptr(), labels.data_ptr(), n
    a.objective, a.w, a.dim, a.out = 1, w.data_ptr(), dim, 1
    a.grad, a.loss_sum, a.correct, a.pred, a.err, a.compute_grad = (grad.data_ptr(), loss.data_ptr(), correct.data_ptr(),
                                                                      pred.data_ptr(), err.data_ptr(), 1)
    N.cuda_lib().mvb_lr_sparse_fwd_bwd(a, N.stream_ptr())
    torch.cuda.synchronize()
    X = torch.zeros(n, dim, dtype=torch.float64, device="cuda")
    X.index_put_((torch.arange(n, device="cuda").repeat_interleave(nnz_per), keys), vals.double(), accumulate=True)
    z = X @ w.double()
    p = torch.sigmoid(z)
    rl = -(labels.double() * torch.log(p) + (1 - labels.double()) * torch.log(1 - p)).sum().item()
    rg = ((p - labels.double())[:, None] * X).sum(0) / n
    assert abs(loss.item() - rl) / rl < 1e-3
    assert torch.allclose(pred, p.float(), atol=1e-4)
    assert torch.allclose(grad, rg.float(), atol=1e-4)


def test_ftrl_and_regularisers(mv_device):
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    g = torch.Generator(device="cuda").manual_seed(5)
    L = 10007
    z = torch.randn(L, device="cuda", generator=g); nn = torch.rand(L, device="cuda", generator=g) * 4
    w = torch.zeros(L, device="cuda")
    alpha, beta, l1, l2 = 0.1, 1.0, 0.5, 0.2
    lib.mvb_ftrl_weights(z, nn, w, L, alpha, beta, l1, l2, st)
    ref = torch.where(z.abs() <= l1, torch.zeros_like(z),
                      -(z - torch.sign(z) * l1) / ((beta + nn.sqrt()) / alpha + l2))
    torch.cuda.synchronize()
    assert torch.allclose(w, ref, atol=1e-6)
    grad = torch.randn(L, device="cuda", generator=g)
    for typ, fn in ((1, lambda w_: torch.sign(w_) * 0.01), (2, lambda w_: w_ * 0.01)):
        gg = grad.clone()
        lib.mvb_regularize(gg, w, L, typ, 0.01, st)
        torch.cuda.synchronize()
        assert torch.allclose(gg, grad + fn(w), atol=1e-7)


def _sparse_case(dev, n, dim, out, use_vals, use_sw, seed):
    """CSR minibatch with empty rows (the second and the last), keys < 0 or >= dim in the first row and scattered
    elsewhere, duplicate keys, optional values and per-sample weights; and its fp64 dense form."""
    g = torch.Generator(device=dev).manual_seed(seed)
    cnt = torch.randint(0, 40, (n,), device=dev, generator=g)
    cnt[0] = 20
    if n >= 5:
        cnt[1] = 0
        cnt[-1] = 0
    row_ptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    row_ptr[1:] = cnt.cumsum(0)
    nnz = int(row_ptr[-1])
    keys = torch.randint(-4, dim + 4, (nnz,), device=dev, generator=g)
    keys[:4] = torch.tensor([-1, dim, dim + 1000, -(1 << 40)], device=dev)
    vals = torch.rand(nnz, device=dev, generator=g) + 0.25 if use_vals else None
    w = torch.randn(out * dim, device=dev, generator=g) * 0.3
    labels = torch.randint(0, max(out, 2), (n,), device=dev, generator=g).float()
    sw = torch.rand(n, device=dev, generator=g) * 1.5 + 0.25 if use_sw else None
    rows = torch.arange(n, device=dev).repeat_interleave(cnt)
    ok = (keys >= 0) & (keys < dim)
    v = vals.double() if use_vals else torch.ones(nnz, dtype=torch.float64, device=dev)
    X = torch.zeros(n, dim, dtype=torch.float64, device=dev)
    X.index_put_((rows[ok], keys[ok]), v[ok], accumulate=True)
    one = torch.ones_like(v[ok])
    per_row = torch.zeros(n, dtype=torch.float64, device=dev).index_add_(0, rows[ok], one)
    per_col = torch.zeros(dim, dtype=torch.float64, device=dev).index_add_(0, keys[ok], one)
    return dict(row_ptr=row_ptr, keys=keys, vals=vals, w=w, labels=labels, sw=sw, X=X, per_row=per_row,
                per_col=per_col)


def _sparse_run(c, n, dim, out, objective, grad, compute_grad=1):
    from multiverso_b200 import _native as N
    dev = grad.device
    bufs = dict(loss=torch.zeros(1, device=dev), correct=torch.zeros(1, dtype=torch.int32, device=dev),
                pred=torch.full((n * out,), float("nan"), device=dev),
                err=torch.full((n * out,), float("nan"), device=dev))
    a = N.LrSparse()
    a.row_ptr, a.keys, a.vals, a.labels = c["row_ptr"].data_ptr(), c["keys"].data_ptr(), N.ptr(c["vals"]), \
        c["labels"].data_ptr()
    a.sample_w, a.n, a.objective, a.w, a.dim, a.out = N.ptr(c["sw"]), n, objective, c["w"].data_ptr(), dim, out
    a.grad, a.loss_sum, a.correct = grad.data_ptr(), bufs["loss"].data_ptr(), bufs["correct"].data_ptr()
    a.pred, a.err, a.compute_grad = bufs["pred"].data_ptr(), bufs["err"].data_ptr(), compute_grad
    N.cuda_lib().mvb_lr_sparse_fwd_bwd(a, N.stream_ptr())
    torch.cuda.synchronize()
    return bufs


def _sparse_ref(c, n, dim, out, objective):
    X, W = c["X"], c["w"].double().view(out, dim)
    Z = X @ W.T
    dz = (c["per_row"][:, None] + 6) * U * (X @ W.abs().T)
    wgt = c["sw"] if c["sw"] is not None else torch.ones(n, device=X.device)
    return _epilogue64(Z, dz, c["labels"], objective, wgt)


@pytest.mark.parametrize("out", [1, 2, 17, 64])
@pytest.mark.parametrize("objective", [0, 1, 2])
def test_sparse_kernel_classes_weights_and_keys(cuda, objective, out):
    """lr_sparse_fwd_kernel: loss, correct, pred, err and grad against fp64 with and without sample weights and
    values, keys outside [0, dim) contributing nothing, empty rows, n = 1, 5, 1000."""
    dim = 1500
    for n in (1, 5, 1000):
        for use_vals in (True, False):
            for use_sw in (True, False):
                what = (n, use_vals, use_sw)
                c = _sparse_case(cuda, n, dim, out, use_vals, use_sw, seed=n * 4 + 2 * use_vals + use_sw + out)
                grad = torch.zeros(out * dim, device=cuda)
                b = _sparse_run(c, n, dim, out, objective, grad)
                r = _sparse_ref(c, n, dim, out, objective)
                _check_outputs(r, b["pred"], b["err"], b["loss"], b["correct"], what)
                X = c["X"]
                G = r["err"].T @ X
                dG = r["derr"].T @ X + (c["per_col"][None, :] + 2) * U * (r["err"].abs().T @ X)
                _within(grad.view(out, dim), G, dG, (what, "grad"))


def test_sparse_kernel_without_gradient_leaves_grad_alone(cuda):
    n, dim, out = 300, 700, 17
    c = _sparse_case(cuda, n, dim, out, True, True, seed=4)
    grad = torch.randn(out * dim, device=cuda)
    keep = grad.clone()
    b = _sparse_run(c, n, dim, out, 2, grad, compute_grad=0)
    assert torch.equal(grad, keep)
    _check_outputs(_sparse_ref(c, n, dim, out, 2), b["pred"], b["err"], b["loss"], b["correct"], "no grad")


def _dense_run(x, labels, w, out, objective, grad, compute_grad=1):
    from multiverso_b200 import _native as N
    n, dim = x.shape
    dev = x.device
    bufs = dict(loss=torch.zeros(1, device=dev), correct=torch.zeros(1, dtype=torch.int32, device=dev),
                pred=torch.full((n * out,), float("nan"), device=dev),
                err=torch.full((n * out,), float("nan"), device=dev))
    a = N.LrDense()
    a.x, a.labels, a.n, a.dim, a.out, a.objective = x.data_ptr(), labels.data_ptr(), n, dim, out, objective
    a.w, a.grad, a.loss_sum, a.correct = w.data_ptr(), grad.data_ptr(), bufs["loss"].data_ptr(), \
        bufs["correct"].data_ptr()
    a.pred, a.err, a.compute_grad = bufs["pred"].data_ptr(), bufs["err"].data_ptr(), compute_grad
    N.cuda_lib().mvb_lr_dense_fwd_bwd(a, N.stream_ptr())
    torch.cuda.synchronize()
    return bufs


@pytest.mark.parametrize("out", [15, 16, 17, 33, 64])
@pytest.mark.parametrize("objective", [0, 1, 2])
def test_dense_cuda_core_class_passes_and_slabs(cuda, objective, out):
    """lr_dense_fwd_kernel + lr_dense_grad_kernel: one to four 16-class passes of the gradient, n across the
    128-sample slabs, dim across the warp width; the gradient accumulates onto a nonzero grad."""
    g = torch.Generator(device=cuda).manual_seed(out * 3 + objective)
    for n in (1, 127, 128, 129, 300):
        for dim in (1, 31, 33):
            x = torch.randn(n, dim, device=cuda, generator=g)
            w = torch.randn(out * dim, device=cuda, generator=g) * 0.3
            labels = torch.randint(0, out, (n,), device=cuda, generator=g).float()
            g0 = torch.randn(out * dim, device=cuda, generator=g)
            grad = g0.clone()
            b = _dense_run(x, labels, w, out, objective, grad)
            X, W = x.double(), w.double().view(out, dim)
            r = _epilogue64(X @ W.T, (dim + 6) * U * (X.abs() @ W.abs().T), labels, objective,
                            torch.ones(n, device=cuda))
            _check_outputs(r, b["pred"], b["err"], b["loss"], b["correct"], (n, dim))
            ref = g0.double().view(out, dim) + r["err"].T @ X
            dG = r["derr"].T @ X.abs() + (n + n // 128 + 2) * U * (r["err"].abs().T @ X.abs()) + U * ref.abs()
            _within(grad.view(out, dim), ref, dG, (n, dim, "grad"))


def test_more_than_64_classes_is_an_error_on_both_abis(cuda):
    from multiverso_b200 import _native as N
    n, dim, out = 8, 16, 65
    x = torch.randn(n, dim, device=cuda)
    labels = torch.zeros(n, device=cuda)
    w = torch.randn(out * dim, device=cuda)
    grad = torch.zeros(out * dim, device=cuda)
    with pytest.raises(N.NativeError, match="rc=-8"):
        _dense_run(x, labels, w, out, 2, grad)
    c = _sparse_case(cuda, n, dim, out, True, False, seed=1)
    with pytest.raises(N.NativeError, match="rc=-8"):
        _sparse_run(c, n, dim, out, 2, grad)
    torch.cuda.synchronize()
    assert not grad.any()


@pytest.mark.parametrize("objective", [0, 1, 2])
def test_planted_ties_pick_the_lowest_class(mv_device, objective):
    """W = 0 makes every logit exactly 0, in TF32 too: the CUDA-core kernels, the wide epilogue and
    dense_gemm_step all take class 0, so correct counts the label-0 samples; the softmax loss is n log(out)."""
    from multiverso_b200.models.logreg import dense_gemm_step
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(objective)
    n, dim = 300, 36
    for out in (17, 64, 65, 300):
        x = torch.randn(n, dim, device=dev, generator=g)
        labels = torch.randint(0, 3, (n,), device=dev, generator=g).float()
        zeros = int((labels == 0).sum())
        r = _epilogue64(torch.zeros(n, out, dtype=torch.float64, device=dev),
                        torch.zeros(n, out, dtype=torch.float64, device=dev), labels, objective,
                        torch.ones(n, device=dev))
        if objective == 2:
            assert abs(r["loss"] - n * math.log(out)) < 1e-9 * n * math.log(out)
        results = {}
        if out <= 64:
            b = _dense_run(x, labels, torch.zeros(out * dim, device=dev), out, objective,
                           torch.zeros(out * dim, device=dev))
            results["dense"] = (b["loss"], b["correct"])
            c = _sparse_case(dev, n, dim, out, True, False, seed=out)
            c["labels"] = labels
            c["w"].zero_()
            b = _sparse_run(c, n, dim, out, objective, torch.zeros(out * dim, device=dev))
            results["sparse"] = (b["loss"], b["correct"])
        else:
            m = _wide_model(dim, out, objective, n)
            m.forward_backward_dense(x, labels, train=False)
            results["wide"] = (m.loss, m.correct)
        loss, correct, _ = dense_gemm_step(x, labels, torch.zeros(out * dim, device=dev), None, objective, out)
        results["dense_gemm_step"] = (loss.view(1), correct.view(1))
        torch.cuda.synchronize()
        for k, (lo, co) in results.items():
            assert int(co.item()) == zeros, (k, out)
            assert abs(lo.item() - r["loss"]) <= r["dloss"], (k, out, lo.item(), r["loss"])


@pytest.mark.parametrize("rows,cols,ld_in,ld_out", [(45, 70, 75, 100), (33, 1, 4, 36), (1, 40, 41, 4),
                                                     (129, 65, 67, 132)])
def test_transpose_pad(cuda, rows, cols, ld_in, ld_out):
    """out[c][r] = in[r][c] bitwise, and the pad columns r in [rows, ld_out) are zero."""
    from multiverso_b200 import _native as N
    src = torch.randn(rows, ld_in, device=cuda)
    out = torch.full((cols, ld_out), float("nan"), device=cuda)
    N.cuda_lib().mvb_transpose_pad_f32(src, rows, cols, ld_in, out, ld_out, N.stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(out[:, :rows], src[:, :cols].T)
    assert torch.equal(out[:, rows:], torch.zeros(cols, ld_out - rows, device=cuda))


def _ftrl_sigma64(n, g, alpha):
    return ((n + g * g).sqrt() - n.sqrt()) / alpha


def _ftrl_sigma_tol(n, g, alpha):
    """fp32 n + g g, two sqrtf, their difference and the division by alpha."""
    s = (n + g * g).sqrt()
    return (2 * U * s + U * n.sqrt()) / alpha + 3 * U * _ftrl_sigma64(n, g, alpha).abs() + U * s / alpha


def test_ftrl_update_and_delta_against_fp64(cuda):
    """mvb_ftrl_update (local FTRL) and mvb_ftrl_delta (the negated (dz, dn) pushed to a subtracting server) from the
    same fp32 state, chained over a few steps through mvb_ftrl_weights; g = 0 leaves z and n bitwise alone and
    n = 0 entries take sigma = |g| / alpha."""
    from multiverso_b200 import _native as N
    lib, st = N.cuda_lib(), N.stream_ptr()
    gen = torch.Generator(device=cuda).manual_seed(13)
    L = 20011
    alpha, beta, l1, l2 = 0.1, 1.0, 0.5, 0.2
    z = torch.randn(L, device=cuda, generator=gen) * 3
    nacc = torch.rand(L, device=cuda, generator=gen) * 4
    nacc[::7] = 0
    w = torch.empty(L, device=cuda)
    for step in range(4):
        lib.mvb_ftrl_weights(z, nacc, w, L, alpha, beta, l1, l2, st)
        torch.cuda.synchronize()
        z64, n64 = z.double(), nacc.double()
        den = (beta + n64.sqrt()) / alpha + l2
        w64 = torch.where(z64.abs() <= l1, torch.zeros_like(z64), -(z64 - z64.sign() * l1) / den)
        # seven roundings, and alpha = 0.1 and l2 = 0.2 are fp32 constants in the kernel
        _within(w, w64, 8 * U * w64.abs(), ("weights", step))
        g = torch.randn(L, device=cuda, generator=gen)
        g[::5] = 0
        w64, g64 = w.double(), g.double()
        sig, dsig = _ftrl_sigma64(n64, g64, alpha), _ftrl_sigma_tol(n64, g64, alpha)
        dz, dn = torch.empty(L, device=cuda), torch.empty(L, device=cuda)
        lib.mvb_ftrl_delta(nacc, w, g, dz, dn, L, alpha, st)
        z0, n0 = z.clone(), nacc.clone()
        lib.mvb_ftrl_update(z, nacc, w, g, L, alpha, st)
        torch.cuda.synchronize()
        step_z = g64 - sig * w64
        tol_z = w64.abs() * dsig + 2 * U * (g64.abs() + (sig * w64).abs())
        _within(dz, -step_z, tol_z, ("delta z", step))
        _within(dn, -g64 * g64, U * g64 * g64, ("delta n", step))
        moved = g != 0
        assert torch.equal(z[~moved], z0[~moved]) and torch.equal(nacc[~moved], n0[~moved])
        _within(z[moved], z64[moved] + step_z[moved], tol_z[moved] + U * (z64 + step_z).abs()[moved], ("z", step))
        _within(nacc[moved], (n64 + g64 * g64)[moved], 2 * U * (n64 + g64 * g64)[moved], ("n", step))
