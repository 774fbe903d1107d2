"""Full-softmax evaluation and inner-product top-k over a MatrixTable whose rows are the classes of an output layer.

``full_softmax(table, hidden, labels=None, k=0, rows=None)`` returns, for every row ``x_b`` of ``hidden`` [B, d], with
``z_bn = x_b . w_n`` over the first ``d`` columns of the rows ``n`` in ``[0, rows)``:

* ``lse`` [B] fp32, ``log sum_n exp(z_bn)``;
* ``loss`` [B] fp32, ``lse_b - z_{b, y_b}`` (the exact cross-entropy; ``None`` without labels);
* ``scores`` / ``ids`` [B, k] fp32 / int64, the k rows with the largest logit, sorted by score descending with ties
  to the smaller id (``None`` when ``k == 0``); missing slots (fewer than ``k`` rows) hold id -1 and score -inf.

``topk_dot(table, queries, k)`` is the top-k alone: maximum-inner-product search, ranked by ``q . w``. Unlike
``topk_cosine`` the row norms count, which is the ranking of an output layer (its norms carry the class prior) and
of two-tower retrieval. There is no log-Q correction, no accidental-hit mask and no bias term: fold a bias into a
column of the table and append a constant 1 to ``hidden``.

On the device it is one pass over the table (``csrc/cuda/topk_cos.cu``, the fused search of ``topk_cosine`` with the
dot product as the score): W tiles stream from their owners' shards by TMA into tf32 wgmma, and the epilogue keeps a
running log-sum-exp per query and, for ``k > 0``, k + 8 candidates whose dot products are then recomputed in fp64.
The ``[B, N]`` logits are never written, so B = 8192 over a 1M-row table needs no 32 GB buffer. A loss-only call
(``k == 0``) runs no top-k bookkeeping. Reads follow ``get_rows`` / ``topk_cosine``: the caller orders a call after
the Adds it wants to see (barrier / ``flush``). Evaluation only: the outputs do not require grad and nothing is
pushed.

Numerics: logits are tf32 products with fp32 accumulation (the convention of the sampled-softmax training path), so

    |lse - lse_fp64| <= 2^-10 * ||x_b|| * max_n ||w_n|| + 1e-5 * (1 + |lse_fp64|).

``lse`` is folded in the kernel's tile and range order: it is bitwise the same on every call with the same inputs,
but across shardings of the table and batch sizes it agrees only within that bound. The label logit is recomputed in
fp64, so ``loss`` is not clamped: when the label dominates it can come out slightly below zero. Top-k scores are the
fp64 dot products rounded to fp32, and top-k ids are the exact fp64 top-k except where rows lie within the tf32 error
of the k-th score; both are bitwise independent of the sharding and of the query chunking.

Without a GPU (CPU tensors, host-backend tables) the same call is :func:`full_softmax_reference`, chunked fp64.
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Tuple

import torch

from .. import _native as N
from .topk import TOPK_MAX, _Q_CHUNK, _rowmap_of, check_queries, merge_topk, padded_queries

_INT = (torch.int32, torch.int64)


class FullSoftmaxResult(NamedTuple):
    lse: torch.Tensor                   # [B] fp32
    loss: Optional[torch.Tensor]        # [B] fp32, with labels
    scores: Optional[torch.Tensor]      # [B, k] fp32, k > 0
    ids: Optional[torch.Tensor]         # [B, k] int64, k > 0


def _check_k(k, lo: int, what: str) -> int:
    k = int(k)
    if not lo <= k <= TOPK_MAX:
        raise ValueError(f"{what}: k must be in [{lo}, {TOPK_MAX}], got {k}")
    return k


def _check_rows(rows, num_row: int, what: str) -> int:
    n = num_row if rows is None else int(rows)
    if not 1 <= n <= num_row:
        raise ValueError(f"{what}: rows={n} outside [1, {num_row}]")
    return n


def _check_labels(labels, B: int, n: int, device, what: str) -> Optional[torch.Tensor]:
    """int64 labels on ``device``, checked to lie in [0, n) with one host read (None stays None)."""
    if labels is None:
        return None
    y = torch.as_tensor(labels)
    if y.dtype not in _INT:
        raise TypeError(f"{what}: labels must be int32 or int64, got {y.dtype}")
    if y.dim() != 1 or y.shape[0] != B:
        raise ValueError(f"{what}: labels must be 1-D with one label per row of hidden ({B}), got {tuple(y.shape)}")
    y = y.to(device=device, dtype=torch.int64).contiguous()
    if y.numel():
        lo, hi = torch.stack(list(torch.aminmax(y))).tolist()
        if lo < 0 or hi >= n:
            raise ValueError(f"{what}: labels must be in [0, {n}), got min {lo} max {hi}")
    return y


def _check_hidden(h, width: int, name: str, what: str) -> torch.Tensor:
    h = torch.as_tensor(h)
    if h.dtype != torch.float32 or h.dim() != 2:
        raise TypeError(f"{what}: {name} must be a 2-D float32 tensor, got {h.dtype} {tuple(h.shape)}")
    if not 1 <= h.shape[1] <= width:
        raise ValueError(f"{what}: {name} have {h.shape[1]} columns, the table rows {width}")
    return h


def _reference(w: torch.Tensor, x: torch.Tensor, y: Optional[torch.Tensor], k: int, n: int, want_lse: bool,
               row_chunk: int) -> FullSoftmaxResult:
    B, d = x.shape
    x64 = x.detach().to(torch.float64)
    lse = torch.full((B,), float("-inf"), dtype=torch.float64) if want_lse else None
    best_s = torch.full((B, k), float("-inf"), dtype=torch.float32)
    best_i = torch.full((B, k), -1, dtype=torch.int64)
    for lo in range(0, n if B else 0, row_chunk):        # an empty batch reads nothing
        hi = min(n, lo + row_chunk)
        z = x64 @ w[lo:hi, :d].to(torch.float64).t()
        if want_lse:
            lse = torch.logaddexp(lse, torch.logsumexp(z, 1))
        if k:
            best_s, best_i = merge_topk(best_s, best_i, z.to(torch.float32), lo, k)
    loss = None
    if y is not None:
        loss = (lse - (x64 * w[y, :d].to(torch.float64)).sum(1)).to(torch.float32)
    return FullSoftmaxResult(lse.to(torch.float32) if want_lse else None, loss,
                             best_s if k else None, best_i if k else None)


def full_softmax_reference(weights, hidden, labels=None, k: int = 0, rows: Optional[int] = None,
                           row_chunk: int = 65536) -> FullSoftmaxResult:
    """Host implementation in fp64 (top-k scores rounded to fp32 and ranked as on the device). ``weights``:
    [N, >= d] (columns beyond ``hidden``'s width are ignored), ``hidden``: [B, d] fp32."""
    what = "full_softmax"
    k = _check_k(k, 0, what)
    w = torch.as_tensor(weights)
    if w.dim() != 2:
        raise ValueError(f"{what}: the table must be 2-D, got {tuple(w.shape)}")
    x = _check_hidden(hidden, w.shape[1], "hidden", what).cpu()
    n = _check_rows(rows, w.shape[0], what)
    y = _check_labels(labels, x.shape[0], n, "cpu", what)
    return _reference(w.cpu(), x, y, k, n, True, row_chunk)


def _device(rm: N.RowMap, width: int, hidden: torch.Tensor, y: Optional[torch.Tensor], k: int, n: int,
            want_lse: bool) -> FullSoftmaxResult:
    """Kernel path over an explicit row map (``width``: usable columns of a row); arguments already checked."""
    B, d = hidden.shape
    dev = hidden.device
    f32 = dict(dtype=torch.float32, device=dev)
    lse = torch.empty(B, **f32) if want_lse else None
    loss = torch.empty(B, **f32) if y is not None else None
    scores = torch.empty(B, k, **f32) if k else None
    ids = torch.empty(B, k, dtype=torch.int64, device=dev) if k else None
    if B == 0:
        return FullSoftmaxResult(lse, loss, scores, ids)
    q = padded_queries(hidden.detach())
    lib = N.cuda_lib()
    # the scratch need is not monotone in the query count: size it for the full chunks and the last one
    nbytes = max(lib.mvb_full_softmax_scratch_bytes(c, k, n) for c in {min(B, _Q_CHUNK), B % _Q_CHUNK or _Q_CHUNK})
    scratch = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=dev)
    a = N.FullSoftmax()
    a.ldq, a.dim, a.n_rows, a.wmap, a.k = q.shape[1], d, n, rm, k
    a.scratch, a.scratch_bytes = scratch.data_ptr(), scratch.numel()

    def at(t, i):
        return None if t is None else t[i].data_ptr()
    for lo in range(0, B, _Q_CHUNK):
        a.q, a.M = q[lo].data_ptr(), min(B, lo + _Q_CHUNK) - lo
        a.labels, a.lse, a.loss, a.scores, a.ids = at(y, lo), at(lse, lo), at(loss, lo), at(scores, lo), at(ids, lo)
        lib.mvb_full_softmax(a, N.stream_ptr())
    return FullSoftmaxResult(lse, loss, scores, ids)


def _call(table, hidden, labels, k: int, rows, want_lse: bool, name: str, what: str) -> FullSoftmaxResult:
    if isinstance(table, torch.Tensor) and not table.is_cuda or \
            not isinstance(table, torch.Tensor) and not hasattr(table, "_rowmap"):
        # a CPU tensor or a host-backend table: the host implementation over its Get
        w = table if isinstance(table, torch.Tensor) else \
            torch.as_tensor(table.get()).view(table.num_row, table.num_col)
        if w.dtype != torch.float32 or w.dim() != 2:
            raise TypeError(f"{what}: a table tensor must be 2-D float32, got {w.dtype} {tuple(w.shape)}")
        x = _check_hidden(hidden, w.shape[1], name, what)
        n = _check_rows(rows, w.shape[0], what)
        y = _check_labels(labels, x.shape[0], n, "cpu", what)
        r = _reference(w, x.cpu(), y, k, n, want_lse, 65536)
        return FullSoftmaxResult(*(None if t is None else t.to(x.device) for t in r))
    rm, num_row, width = _rowmap_of(table, what)
    x = torch.as_tensor(hidden)
    check_queries(rm, width, x, name, what)
    n = _check_rows(rows, num_row, what)
    y = _check_labels(labels, x.shape[0], n, x.device, what)
    return _device(rm, width, x, y, k, n, want_lse)


def full_softmax(table, hidden, labels=None, k: int = 0, rows: Optional[int] = None) -> FullSoftmaxResult:
    """Exact log-partition, cross-entropy and top-k classes of ``hidden`` [B, d] fp32 over the table's rows
    ``[0, rows)`` (see the module docstring). ``table``: MatrixDeviceTable, 2-D fp32 CUDA tensor (a column slice of
    a wider pitch is fine), host-backend table or CPU tensor; ``labels``: [B] int32 / int64 in ``[0, rows)``;
    ``k`` in ``[0, TOPK_MAX]``; ``rows`` in ``[1, num_row]``. Returns ``FullSoftmaxResult(lse, loss, scores,
    ids)``."""
    k = _check_k(k, 0, "full_softmax")
    return _call(table, hidden, labels, k, rows, True, "hidden", "full_softmax")


def topk_dot(table, queries, k: int, rows: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """Maximum-inner-product search: the ``k`` rows (``k`` in ``[1, TOPK_MAX]``) with the largest ``q . w`` for each
    query of ``queries`` [M, d] fp32, with the conventions of :func:`full_softmax`. Returns (scores [M, k] fp32,
    ids [M, k] int64)."""
    k = _check_k(k, 1, "topk_dot")
    r = _call(table, queries, None, k, rows, False, "queries", "topk_dot")
    return r.scores, r.ids
