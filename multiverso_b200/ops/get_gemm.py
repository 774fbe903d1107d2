"""Fused Get + GEMM (K2-fused): ``y = x @ W^T`` where W is a row-sharded MatrixTable.

The pulled row block is never materialised: a persistent, warp-specialised kernel streams each
W tile from its owner (local or peer HBM over NVLink) with TMA into shared memory and multiplies
it with Hopper warp-group MMAs (wgmma, TF32 operands, fp32 accumulation in registers) against
the local activations.
Reference analogue: MatrixWorkerTable::Get followed by the application's first GEMM
(e.g. LogReg Objective::Predict, Applications/LogisticRegression/src/objective/objective.cpp:113-120).
"""
from __future__ import annotations

import torch

from .. import _native as N
from .topk import _rowmap_of


def get_gemm_supported() -> bool:
    """True when the fused wgmma kernel can run here (sm_90a device present)."""
    if not torch.cuda.is_available():
        return False
    return bool(N.cuda_lib().mvb_get_gemm_supported())


def _check_out(what: str, out: torch.Tensor, M: int, Nrows: int, device: torch.device) -> None:
    """The kernel writes M x Nrows floats at row pitch Nrows from out's first element: anything else in `out`
    would be written out of bounds or into the wrong elements."""
    if (out.dtype != torch.float32 or out.device != device or tuple(out.shape) != (M, Nrows)
            or not out.is_contiguous()):
        raise ValueError(f"{what}: out must be a contiguous float32 [{M}, {Nrows}] tensor on {device}, got "
                         f"{out.dtype} {tuple(out.shape)} stride {out.stride()} on {out.device}")


def get_gemm(table, x: torch.Tensor, out: torch.Tensor = None) -> torch.Tensor:
    """``x``: [M, K] fp32 CUDA, ``table``: MatrixDeviceTable with num_col == K. Returns [M, num_row], written
    into ``out`` when given (a contiguous fp32 [M, num_row] tensor on x's device, else ValueError).
    On the host backend (no GPU) the same call is a plain Get followed by a matmul."""
    from ..runtime import Runtime
    if Runtime.get().backend == "host":
        w = torch.as_tensor(table.get()).view(table.num_row, table.num_col).to(torch.float32)
        y = torch.as_tensor(x, dtype=torch.float32) @ w.t()
        if out is not None:
            out.copy_(y)
            return out
        return y
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.is_contiguous()
    M, K = x.shape
    assert K == table.num_col and table.dtype == torch.float32
    if K % 4 != 0:
        raise ValueError("get_gemm needs K % 4 == 0 (16-byte row pitch for TMA)")
    Nrows = table.num_row
    if out is None:
        out = torch.empty(M, Nrows, dtype=torch.float32, device=x.device)
    _check_out("get_gemm", out, M, Nrows, x.device)
    g = N.GetGemm()
    g.x, g.y, g.w_cache = x.data_ptr(), out.data_ptr(), None
    g.M, g.N, g.K = M, Nrows, K
    g.wmap = _rowmap_of(table, "get_gemm")[0]
    g.local_server = table.sid if table.S > 1 else 0
    N.cuda_lib().mvb_get_gemm_fused(g, N.stream_ptr())
    return out


def gemm_nt(x: torch.Tensor, w: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[M, N] = x[M, K] @ w[N, K]^T on the hand-written wgmma kernel (gemm_fused.cu: TMA-fed
    wgmma, TF32 operands, fp32 accumulation in registers) -- `w` is presented as a one-server
    row map, so the same kernel that streams table shards multiplies two local matrices.  K % 4 == 0."""
    for name, t in (("x", x), ("w", w)):
        if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.is_contiguous()):
            raise ValueError(f"gemm_nt: {name} must be a contiguous 2-D float32 CUDA tensor")
    M, K = x.shape
    Nr = w.shape[0]
    if w.shape[1] != K or w.device != x.device:
        raise ValueError(f"gemm_nt: w {tuple(w.shape)} on {w.device} does not match x {tuple(x.shape)} on {x.device}")
    if K % 4 != 0:
        raise ValueError("gemm_nt needs K % 4 == 0 (16-byte row pitch for TMA)")
    _check_out("gemm_nt", out, M, Nr, x.device)
    g = N.GetGemm()
    g.x, g.y, g.w_cache = x.data_ptr(), out.data_ptr(), None
    g.M, g.N, g.K = M, Nr, K
    g.wmap = _rowmap_of(w, "gemm_nt")[0]
    g.local_server = 0
    N.cuda_lib().mvb_get_gemm_fused(g, N.stream_ptr())
    return out
