"""K8 numerics against plain PyTorch references: the sparse / dense CUDA-core kernels, FTRL, regularisers
(csrc/cuda/logreg.cu) and the wide dense path whose two products run on the hand-written wgmma kernel
(no library GEMM), each compared with fp32/fp64 torch on the same inputs."""
import pytest
import torch

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize("n,dim,out,objective", [(512, 256, 128, 2), (301, 64, 70, 2), (257, 128, 96, 1), (1000, 512, 1000, 2)])
def test_dense_wide_path_on_tcgen05(mv_device, n, dim, out, objective):
    """> 64 classes: LogRegModel.forward_backward_dense through gemm_fused.cu + the epilogue kernel (TF32
    products, fp32 accumulation): predictions / loss / gradient within TF32 accuracy of the fp64 reference."""
    from multiverso_b200.models.logreg import LogRegConfig, LogRegModel
    cfg = LogRegConfig(input_size=dim - 1, output_size=out, sparse=False, use_ps=False,
                       objective_type={2: "softmax", 1: "sigmoid", 0: "default"}[objective], minibatch_size=n)
    m = LogRegModel(cfg)
    assert m.dim == dim
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(n, dim, device="cuda", generator=g)
    m.w.copy_(torch.randn(out * dim, device="cuda", generator=g) * 0.05)
    labels = torch.randint(0, out, (n,), device="cuda", generator=g).float()
    pred = torch.zeros(n * out, device="cuda")
    m.loss.zero_(); m.correct.zero_(); m.grad.zero_()
    m.forward_backward_dense(x, labels, train=True, pred=pred)
    torch.cuda.synchronize()
    rl, rc, rp, rg = _ref_dense(x, labels, m.w, objective, out)
    assert abs(m.loss.item() - rl) / abs(rl) < 2e-3
    assert abs(int(m.correct.item()) - rc) <= max(2, n // 100)          # TF32 can flip near-ties of the argmax
    assert (pred.view(n, out) - rp).abs().max().item() < 5e-3
    assert (m.grad.view(out, dim) - rg).abs().max().item() < 5e-3 * max(1.0, rg.abs().max().item() * 50)


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
