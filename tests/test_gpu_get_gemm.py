"""wgmma / TMA fused Get+GEMM against a plain PyTorch fp32 reference (TF32 operands:
10-bit mantissa, so the tolerance is relative to |x||w| sqrt(K))."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,Nrows,K", [(128, 64, 32), (256, 128, 64), (1000, 1000, 512), (77, 10, 784), (2048, 300, 300), (1300, 700, 1024)])
def test_get_gemm_matches_fp32_reference(mv_device, M, Nrows, K):
    from multiverso_b200.ops import get_gemm, get_gemm_supported
    mv = mv_device
    assert get_gemm_supported()
    t = mv.MatrixTable(Nrows, K, "float32", min_value=-1.0, max_value=1.0)
    W = t.get().view(Nrows, K).clone()
    torch.manual_seed(1)
    x = torch.randn(M, K, device="cuda")
    y = get_gemm(t, x)
    torch.cuda.synchronize()
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = x.double() @ W.double().T
    torch.backends.cuda.matmul.allow_tf32 = prev
    err = (y.double() - ref).abs().max().item()
    scale = (x.abs().max() * W.abs().max()).item() * K ** 0.5
    assert err < 4e-3 * scale, (err, scale)
