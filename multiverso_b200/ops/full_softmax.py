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


# ------------------------------------------------------------------------------------------------ training
_WHAT = "PSFullSoftmax"


def _lse64(w: torch.Tensor, x64: torch.Tensor, row_chunk: int) -> torch.Tensor:
    lse = torch.full((x64.shape[0],), float("-inf"), dtype=torch.float64)
    for lo in range(0, w.shape[0] if x64.shape[0] else 0, row_chunk):
        z = x64 @ w[lo:lo + row_chunk, :x64.shape[1]].to(torch.float64).t()
        lse = torch.logaddexp(lse, torch.logsumexp(z, 1))
    return lse


def full_softmax_grad_reference(weights, hidden, labels, g, row_chunk: int = 65536):
    """The exact full-softmax cross-entropy and its gradients in fp64, chunked over the rows of ``weights``
    [N, d] so that no [B, N] buffer is formed: returns ``(loss, dX, dW)`` for ``hidden`` [B, d], ``labels`` [B]
    and upstream gradient ``g`` [B], with ``dX = g (P W - W_y)`` and ``dW = (g (P - Y))^T X``."""
    w = torch.as_tensor(weights).cpu()
    x64 = torch.as_tensor(hidden).detach().cpu().to(torch.float64)
    y = torch.as_tensor(labels).cpu().to(torch.int64)
    g64 = torch.as_tensor(g).detach().cpu().to(torch.float64)
    B, d = x64.shape
    lse = _lse64(w, x64, row_chunk)
    loss = lse - (x64 * w[y, :d].to(torch.float64)).sum(1)
    dx = torch.zeros(B, d, dtype=torch.float64)
    dw = torch.zeros(w.shape[0], d, dtype=torch.float64)
    for lo in range(0, w.shape[0] if B else 0, row_chunk):
        wc = w[lo:lo + row_chunk, :d].to(torch.float64)
        p = torch.exp(x64 @ wc.t() - lse[:, None]) * g64[:, None]
        dx += p @ wc
        dw[lo:lo + wc.shape[0]] = p.t() @ x64
    dx -= g64[:, None] * w[y, :d].to(torch.float64)
    dw.index_add_(0, y, -g64[:, None] * x64)
    return loss, dx, dw


class PSFullSoftmax(torch.nn.Module):
    """Output layer trained with the exact softmax over every row of a MatrixTable::

        fsm = mv.ops.PSFullSoftmax(table, push_scale=lr, option=None)
        loss = fsm(hidden, labels)        # [B] exact cross-entropy, hidden [B, num_col] fp32
        loss.mean().backward()            # dL/dhidden to autograd; one dense Add of push_scale * dL/dW
        r = fsm.evaluate(hidden, labels, k=10)   # = full_softmax(table, hidden, labels, k)

    The forward is :func:`full_softmax` (lse and loss, one host read for the label check) and saves hidden, the
    labels and lse. With ``G_bn = g_b (p_bn - [y_b = n])``, ``p_bn = exp(z_bn - lse_b)`` and ``g_b`` the upstream
    gradient of ``loss_b``, the backward computes ``dL/dhidden = G W`` (only when hidden requires grad) and
    ``dL/dW = G^T hidden`` for every row, written times ``push_scale`` into the table's ``staging()`` buffer and
    pushed as one dense ``add_async(staged=True)`` through the table's updater (``push_scale=None``: neither the
    dW pass nor the Add runs). On the device both products run in ``csrc/cuda/full_softmax_bwd.cu``, which
    recomputes the tf32 logits tile by tile and never writes the [B, N] logits or their gradient; the backward
    makes no host read.

    Every backward issues exactly one Add, also for an empty batch (a zero gradient): a dense Add is collective
    under BSP with several workers. With momentum or adam every row takes a step, as with any dense Add.

    The backward reads the table again: an Add that lands between a call's forward and its backward changes the
    recomputed logits. In one process, or under BSP, that happens only if the caller adds; in async mode it is
    ordinary staleness.

    Numerics on the device: with ``T = 2^-10`` (tf32 truncation of each operand), ``|x_b|`` and ``|w_n|`` the
    largest row norms, every logit is within ``e_z = 2 T |x| |w| + 1e-6`` of fp64, so ``|p - p_fp64| <= p (2 e_z +
    e_lse)`` with ``e_lse = |lse - lse_fp64|`` (the forward's bound); G then enters a second tf32 product. With
    ``f_b = 1.1 (2 e_z + e_lse + 2 T)`` (1.1 covers exp(e) - 1 <= 1.1 e for small e) and ``U = 2^-24`` for the
    fp32 accumulation of the products over the N classes (dX) and the B queries (dW), per element,

        |dX_bj - dX_fp64| <= |g_b| ((f_b + N U) sum_n p_bn |w_nj| + (2 T + N U) |w_{y_b, j}|) + 1e-6
        |dW_nj - dW_fp64| <= |scale| (sum_b |g_b| ((f_b + B U) p_bn + (2 T + B U) [y_b = n]) |x_bj| + 1e-6)

    and ``sum_n p_bn |w_nj| <= max_n |w_nj|``. The bound is checked against fp64 up to N = 1,000,003. dW is bitwise the same for every sharding of the table and every run;
    dX is bitwise repeatable and within its bound across shardings.

    Refused before anything runs: HashMatrixTable, ``is_sparse`` tables (their staged Adds do not mark rows
    stale), non-fp32 tables, a row pitch that is not a multiple of 4, hidden whose width is not ``num_col`` and
    CPU hidden with a device table. On the host backend the same formula runs in fp64, chunked over rows
    (:func:`full_softmax_grad_reference`), and the gradient goes out as one ``table.add``.
    """

    def __init__(self, table, push_scale: Optional[float] = 1.0, option=None):
        super().__init__()
        from ..tables.device import HashMatrixTable
        from .embedding import _device_of, _dtype_of
        if isinstance(table, torch.Tensor):
            raise TypeError(f"{_WHAT}: the weight must be a MatrixTable (a tensor has no updater to push to)")
        if isinstance(table, HashMatrixTable):
            raise TypeError(f"{_WHAT}: a HashMatrixTable has no dense Add over all rows; use a MatrixTable")
        if getattr(table, "is_sparse", False):
            raise ValueError(f"{_WHAT}: is_sparse tables are not supported (a staged Add does not mark rows stale)")
        if _dtype_of(table) != torch.float32:
            raise TypeError(f"{_WHAT}: the table must be float32, got {_dtype_of(table)}")
        self.table, self.push_scale, self.option = table, push_scale, option
        self.num_classes, self.in_features = int(table.num_row), int(table.num_col)
        self._device = _device_of(table)
        if self._device is not None:
            self._rm = _rowmap_of(table, _WHAT)[0]
            if self._rm.num_col % 4 != 0:
                raise ValueError(f"{_WHAT}: the table's row pitch ({self._rm.num_col} floats) must be a multiple of "
                                 "4 (16-byte TMA rows)")
        # hidden may not require grad: the anchor makes autograd run the backward, and so the push
        self.anchor = torch.nn.Parameter(torch.zeros(0))

    def _check(self, hidden, labels):
        h = hidden
        if not isinstance(h, torch.Tensor) or h.dim() != 2 or h.dtype != torch.float32:
            raise TypeError(f"{_WHAT}: hidden must be a 2-D float32 tensor, got "
                            f"{getattr(h, 'dtype', type(h).__name__)} {tuple(getattr(h, 'shape', ()))}")
        if h.shape[1] != self.in_features:
            raise ValueError(f"{_WHAT}: hidden has {h.shape[1]} columns, the table rows {self.in_features}")
        if self._device is not None and not h.is_cuda:
            raise ValueError(f"{_WHAT}: the table is on the GPU, hidden must be too")
        return _check_labels(labels, h.shape[0], self.num_classes, self._device or "cpu", _WHAT)

    def forward(self, hidden: torch.Tensor, labels) -> torch.Tensor:
        y = self._check(hidden, labels)
        if self._device is None:
            return _FullSoftmaxHostFn.apply(self.anchor, hidden, y, self)
        return _FullSoftmaxFn.apply(self.anchor, hidden, y, self)

    def evaluate(self, hidden: torch.Tensor, labels, k: int = 0) -> FullSoftmaxResult:
        """:func:`full_softmax` over the table: ``lse``, ``loss`` and for ``k > 0`` the top-k classes. Nothing is
        pushed."""
        h = torch.as_tensor(hidden)
        if self._device is not None and not h.is_cuda:
            raise ValueError(f"{_WHAT}: the table is on the GPU, hidden must be too")
        return full_softmax(self.table, h, labels, k)

    def extra_repr(self) -> str:
        return (f"{self.in_features}, {self.num_classes}, push_scale={self.push_scale}, "
                f"weight=MatrixTable#{getattr(self.table, 'table_id', '?')}")


def full_softmax_bwd(rm: N.RowMap, q: torch.Tensor, d: int, y: torch.Tensor, lse: torch.Tensor, g: torch.Tensor,
                     dq: Optional[torch.Tensor], dw: Optional[torch.Tensor], scale: float) -> None:
    """One ``mvb_full_softmax_bwd`` call: ``q`` [B, ldq] fp32 (ldq % 4 == 0), ``dq`` [B, >= d] and / or ``dw``
    [num_row, >= d] written (see ``csrc/cuda/mvb200.h``); arguments already checked."""
    lib = N.cuda_lib()
    B = q.shape[0]
    nbytes = lib.mvb_full_softmax_bwd_scratch_bytes(B, d, rm.num_row, dq is not None, dw is not None)
    scratch = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=q.device)
    a = N.FullSoftmaxBwd()
    a.q, a.M, a.ldq, a.dim, a.wmap = q.data_ptr(), B, q.shape[1], d, rm
    a.labels, a.lse, a.g = y.data_ptr(), lse.data_ptr(), g.data_ptr()
    if dq is not None:
        a.dq, a.lddq = dq.data_ptr(), dq.stride(0)
    if dw is not None:
        a.dw, a.lddw, a.scale = dw.data_ptr(), dw.stride(0), float(scale)
    a.scratch, a.scratch_bytes = scratch.data_ptr(), scratch.numel()
    lib.mvb_full_softmax_bwd(a, N.stream_ptr())


class _FullSoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, hidden, y, fsm):
        x = hidden.detach()
        r = _device(fsm._rm, fsm.in_features, x, y, 0, fsm.num_classes, True)
        ctx.fsm = fsm
        ctx.save_for_backward(padded_queries(x) if x.shape[0] else x.contiguous(), y, r.lse)
        return r.loss

    @staticmethod
    def backward(ctx, grad):
        q, y, lse = ctx.saved_tensors
        fsm = ctx.fsm
        B, d = q.shape[0], fsm.in_features
        want_dx = ctx.needs_input_grad[1]
        dq = torch.empty(B, d, dtype=torch.float32, device=q.device) if want_dx else None
        dw = None
        if fsm.push_scale is not None:
            dw = fsm.table.staging().view(fsm.num_classes, fsm.table.num_col)
        if dq is not None or dw is not None:
            g = grad.to(torch.float32).contiguous()
            full_softmax_bwd(fsm._rm, q, d, y, lse, g, dq, dw, 0.0 if dw is None else fsm.push_scale)
        if dw is not None:
            fsm.table.add_async(None, fsm.option, staged=True)
        return torch.zeros_like(fsm.anchor), dq, None, None


class _FullSoftmaxHostFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, hidden, y, fsm):
        w = torch.as_tensor(fsm.table.get()).view(fsm.num_classes, fsm.in_features)
        x64 = hidden.detach().cpu().to(torch.float64)
        loss = _lse64(w, x64, 65536) - (x64 * w[y].to(torch.float64)).sum(1)
        ctx.fsm = fsm
        ctx.save_for_backward(hidden.detach(), y)
        return loss.to(torch.float32).to(hidden.device)

    @staticmethod
    def backward(ctx, grad):
        x, y = ctx.saved_tensors
        fsm = ctx.fsm
        want_dx = ctx.needs_input_grad[1]
        dx = None
        if want_dx or fsm.push_scale is not None:
            w = torch.as_tensor(fsm.table.get()).view(fsm.num_classes, fsm.in_features)
            _, dx64, dw64 = full_softmax_grad_reference(w, x, y, grad)
            dx = dx64.to(torch.float32).to(x.device) if want_dx else None
            if fsm.push_scale is not None:
                fsm.table.add((dw64 * float(fsm.push_scale)).to(torch.float32).reshape(-1).numpy(), fsm.option)
        return torch.zeros_like(fsm.anchor), dx, None, None
