"""Hierarchical softmax over a MatrixTable: an exactly normalised output layer at O(log N) work per example.

The classes are the leaves of the Huffman tree of their counts, and row ``p`` of the table holds inner node ``p``::

    hsm = mv.ops.PSHierarchicalSoftmax(table, counts, push_scale=lr)
    loss = hsm(hidden, labels)       # [B] per-example loss; hidden [B, num_col] float32, labels [B] int32 / int64
    loss.mean().backward()           # dL/dhidden goes to autograd, the inner-node gradient to the table's updater

The tree is the one word2vec's hierarchical softmax uses: ``MVA_HuffmanBuild`` over
``HuffmanTables.int_frequencies(counts)`` (N >= 2 classes, inner nodes 0..N-2, the root N-2), so the V-row output
table of a word2vec model trained with ``hs`` reads as this layer's table. With label y's path ``p_1..p_L`` (root
first) and branch codes ``c_1..c_L``:

* ``z_i = hidden . w_{p_i}``, ``s_i = 1 - 2 c_i``;
* ``loss = sum_i softplus(-s_i z_i)``, so ``exp(-loss)`` summed over all N labels is 1;
* ``dloss / dz_i = g_i = sigmoid(z_i) - (1 - c_i)`` (word2vec's error ``1 - c - sigmoid(z)`` with the sign of a loss).

The inner-node gradient of a call, ``sum over (b, i) with p_i = n of dloss_b g_bi hidden_b``, is coalesced over the
batch, multiplied by ``push_scale`` and pushed once per unique node (``None``: no push): ``default`` / ``sgd``
tables that are not ``is_sparse`` get a ``red.add`` into the owners' rows, other tables the compact rows through
``add_rows_async``, so every stateful updater takes exactly one step per touched node. Reads follow ``get_rows``'
rule: the caller orders a call after the Adds it wants to see (barrier / ``flush``). Under ``torch.no_grad()`` the
forward is the exact evaluation: the per-example negative log-likelihood (perplexity ``exp(loss.mean())``), with
nothing else computed or kept.

On the device a call reads the labels' path lengths and range in one host read, then ``mvb_hsm_fwd``
(``csrc/cuda/hier_softmax.cu``) runs one warp per example: the path rows come straight from the owners' shards, and
the kernel writes the loss, the path node and ``g`` of every step and ``u_b = sum_i g_bi w_{p_i}``. The backward
is ``dL/dhidden = dloss u`` and the embedding-bag push of ``ids`` with per-sample weights ``g`` over bags of
``dloss hidden``; it does not synchronise with the host for the fused push and reads the unique-node count once for
a compact one. Widths above 1024 floats are refused. On the host backend the same formula runs in torch fp32 over
``get_rows`` of the unique path nodes, and the node gradient goes out in one coalesced ``add_rows``.

Accuracy of the device result against exact arithmetic, with ``u = 2^-24``, for step i of example b with
``a_bi = sum_k |h_bk w_{p_i} k|``:

* ``z``: an fp32 dot of d terms in any fixed order, ``|dz_bi| <= d u a_bi``;
* ``loss``: softplus is 1-Lipschitz, and expf / log1pf / the additions are each within a few ulp, so
  ``|dloss_b| <= sum_i (|dz_bi| + 4 u (1 + softplus_bi)) + L u loss_b``;
* ``g``: sigmoid' <= 1/4 and ``|g| <= 1``, so ``|dg_bi| <= |dz_bi| / 4 + 4 u``;
* ``dL/dhidden = dloss_b u_b``: an fma chain of L terms, ``|d| <= |dloss_b| (sum_i |dg_bi| |w_i| + (L + 1) u
  sum_i |g_bi w_i|)`` per column;
* node n's gradient: the embedding-bag sum of its m uses ``dloss_b g_bi h_b`` (each rounded once in ``dloss h``),
  ``|d| <= sum |dloss_b| |dg_bi| |h_b| + (m + 2) u sum |dloss_b g_bi h_b|`` per column.

``tests/test_gpu_hierarchical_softmax.py`` checks every value against fp64 within these bounds.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .. import _native as N
from ..tables.device import HashMatrixTable
from ..tables.options import AddOption
from ..utils import monitor
from .embedding import _INT, _device_of, _dtype_of, _host_rows, _push_device
from .topk import _rowmap_of

_WHAT = "PSHierarchicalSoftmax"


def huffman_tree(counts) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(points [N, depth] int32, codes [N, depth] int8, lens [N] int32) of the Huffman tree over the class counts:
    label y's path is ``points[y, :lens[y]]``, root first, with branch codes ``codes[y, :lens[y]]``. Raises
    ValueError for fewer than 2 classes, counts that are not finite and non-negative, or a code longer than
    ``HuffmanTables.MAX_CODE``."""
    from ..models.wordembedding import HuffmanTables
    c = np.asarray(torch.as_tensor(counts).detach().cpu().to(torch.float64).numpy())
    if c.ndim != 1:
        raise ValueError(f"{_WHAT}: counts must be 1-D, got shape {c.shape}")
    if c.size < 2:
        raise ValueError(f"{_WHAT}: a tree needs at least 2 classes, got {c.size}")
    if not np.isfinite(c).all() or (c < 0).any():
        raise ValueError(f"{_WHAT}: counts must be finite and non-negative")
    P, Cd, lens, longest = HuffmanTables.encode(c)
    if longest < 0:
        raise ValueError(f"{_WHAT}: the Huffman code of these counts is longer than {HuffmanTables.MAX_CODE} "
                         "(counts that grow like a Fibonacci sequence make a chain)")
    return (torch.from_numpy(np.ascontiguousarray(P[:, :longest])),
            torch.from_numpy(np.ascontiguousarray(Cd[:, :longest])), torch.from_numpy(lens))


def _steps(points, codes, lens, y):
    """The flattened path steps of labels y: (example of each step, node ids int64, codes, offsets [B])."""
    ln = lens[y].to(torch.int64)
    offsets = torch.cumsum(ln, 0) - ln
    bag = torch.repeat_interleave(torch.arange(y.numel(), device=y.device), ln)
    pos = torch.arange(bag.numel(), device=y.device) - offsets[bag]
    return bag, points[y[bag], pos].to(torch.int64), codes[y[bag], pos], offsets


def _path_loss(x, rows, bag, codes, B):
    """sum over each example's steps of softplus(-s z), z = x[bag] . rows (rows: one per step)."""
    z = (x[bag] * rows).sum(1)
    s = 1 - 2 * codes.to(z.dtype)
    return torch.zeros(B, dtype=z.dtype, device=z.device).index_add(0, bag, F.softplus(-s * z))


def hierarchical_softmax_reference(weights, hidden, labels, counts) -> torch.Tensor:
    """Host implementation in fp64: the loss [B] of ``hidden`` [B, d] against ``labels`` over the Huffman tree of
    ``counts``, with inner node p in row p of ``weights`` [>= N - 1, d]. Differentiable in weights and hidden."""
    points, codes, lens = huffman_tree(counts)
    w = torch.as_tensor(weights).cpu().to(torch.float64)
    x = torch.as_tensor(hidden).cpu().to(torch.float64)
    y = torch.as_tensor(labels).cpu().to(torch.int64)
    bag, ids, cds, _ = _steps(points, codes, lens, y)
    return _path_loss(x, w[ids], bag, cds, y.numel())


class PSHierarchicalSoftmax(torch.nn.Module):
    """Hierarchical-softmax output layer whose inner nodes are the rows of a MatrixTable (see the module
    docstring). ``counts``: the N class counts the Huffman tree is built from (the table needs >= N - 1 rows);
    ``push_scale``: the node gradient is multiplied by it before the push (``None``: no push); ``option``: the
    AddOption of the push."""

    def __init__(self, table, counts, push_scale: Optional[float] = 1.0, option: Optional[AddOption] = None):
        super().__init__()
        if isinstance(table, torch.Tensor):
            raise TypeError(f"{_WHAT}: the weight must be a MatrixTable (a tensor has no updater to push to)")
        if isinstance(table, HashMatrixTable):
            raise TypeError(f"{_WHAT}: inner nodes are dense row ids 0..N-2; a HashMatrixTable is keyed by ids")
        if _dtype_of(table) != torch.float32:
            raise TypeError(f"{_WHAT}: the table must be float32, got {_dtype_of(table)}")
        n, d = int(table.num_row), int(table.num_col)
        if d % 4 != 0:
            raise ValueError(f"{_WHAT}: the table's row width ({d} floats) must be a multiple of 4 (16-byte row "
                             "loads)")
        points, codes, lens = huffman_tree(counts)
        self.num_classes, self.in_features = int(lens.numel()), d
        if n < self.num_classes - 1:
            raise ValueError(f"{_WHAT}: {self.num_classes} classes need {self.num_classes - 1} inner-node rows, "
                             f"the table has {n}")
        self.table, self.push_scale, self.option = table, push_scale, option
        self.depth = int(points.shape[1])
        self._device = _device_of(table)
        if self._device is not None:
            self._rm = _rowmap_of(table, _WHAT)[0]
            if self._rm.num_col % 4 != 0:
                raise ValueError(f"{_WHAT}: the table's row pitch ({self._rm.num_col} floats) must be a multiple "
                                 "of 4")
            if d > N.HSM_MAX_DIM:
                raise ValueError(f"{_WHAT}: the device kernel reads rows of at most {N.HSM_MAX_DIM} floats, the "
                                 f"table has {d}")
            points, codes, lens = (t.to(self._device) for t in (points, codes, lens))
        self.points, self.codes, self.lens = points, codes, lens
        # labels never require grad and hidden may not: the anchor makes autograd run the backward, and so the push
        self.anchor = torch.nn.Parameter(torch.zeros(0))

    # ------------------------------------------------------------------------------------------------ checks
    def _check(self, hidden, labels):
        """(labels int64 on the table's device, their path lengths, the total path length L): one host read."""
        if not isinstance(hidden, torch.Tensor) or hidden.dim() != 2 or hidden.dtype != torch.float32:
            raise TypeError(f"{_WHAT}: hidden must be a 2-D float32 tensor, got "
                            f"{getattr(hidden, 'dtype', type(hidden).__name__)} {tuple(getattr(hidden, 'shape', ()))}")
        if hidden.shape[1] != self.in_features:
            raise ValueError(f"{_WHAT}: hidden has {hidden.shape[1]} columns, the table rows {self.in_features}")
        labels = torch.as_tensor(labels)
        if labels.dtype not in _INT:
            raise TypeError(f"{_WHAT}: labels must be int32 or int64, got {labels.dtype}")
        if labels.dim() != 1 or labels.shape[0] != hidden.shape[0]:
            raise ValueError(f"{_WHAT}: labels must be 1-D with one label per row of hidden ({hidden.shape[0]}), "
                             f"got {tuple(labels.shape)}")
        dev = self._device
        if dev is not None and not hidden.is_cuda:
            raise ValueError(f"{_WHAT}: the table is on the GPU, hidden must be too")
        y = labels.to(device=dev if dev is not None else "cpu", dtype=torch.int64).contiguous()
        ln = self.lens[y.clamp(0, self.num_classes - 1)].to(torch.int64)    # never indexes out of range
        L = 0
        if y.numel():
            lo, hi = torch.aminmax(y)
            lo, hi, L = torch.stack([lo, hi, ln.sum()]).tolist()
            if lo < 0 or hi >= self.num_classes:
                raise ValueError(f"{_WHAT}: labels must be in [0, {self.num_classes}), got min {lo} max {hi}")
        return y, ln, L

    # ------------------------------------------------------------------------------------------------ forward
    def forward(self, hidden: torch.Tensor, labels) -> torch.Tensor:
        y, ln, L = self._check(hidden, labels)
        if y.numel() == 0:
            # an empty batch: an empty loss, nothing read or pushed (the anchor keeps backward() valid)
            return hidden.sum(1) + self.anchor.sum().to(hidden.device)
        if self._device is None:
            return self._forward_host(hidden, y)
        if not torch.is_grad_enabled():
            return self._launch(hidden.detach(), y, ln, L, grad=False)[0]
        return _HsmFn.apply(self.anchor, hidden, y, ln, L, self)

    def _launch(self, x, y, ln, L, grad: bool):
        """mvb_hsm_fwd: loss, and with ``grad`` the step node ids, offsets, g and u."""
        x = x.contiguous()
        if x.data_ptr() % 16:
            x = x.clone()
        B, d = x.shape
        dev = self._device
        a = N.Hsm()
        a.wmap, a.dim, a.hidden, a.B, a.ldh = self._rm, d, x.data_ptr(), B, d
        a.labels, a.n_classes = y.data_ptr(), self.num_classes
        a.points, a.codes, a.lens, a.ldp = self.points.data_ptr(), self.codes.data_ptr(), self.lens.data_ptr(), \
            self.depth
        loss = torch.empty(B, dtype=torch.float32, device=dev)
        a.loss = loss.data_ptr()
        offsets = ids = g = u = None
        if grad:
            offsets = torch.cumsum(ln, 0) - ln
            ids = torch.empty(L, dtype=torch.int64, device=dev)
            g = torch.empty(L, dtype=torch.float32, device=dev)
            u = torch.empty(B, d, dtype=torch.float32, device=dev)
            a.offsets, a.ids, a.g, a.u, a.ldu = offsets.data_ptr(), ids.data_ptr(), g.data_ptr(), u.data_ptr(), d
        with monitor("WORKER_TABLE_HIERARCHICAL_SOFTMAX", cuda=True, nbytes=L * d * 4):
            N.cuda_lib().mvb_hsm_fwd(a, N.stream_ptr())
        return loss, x, ids, offsets, g, u

    def _forward_host(self, hidden: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
        bag, ids, cds, _ = _steps(self.points, self.codes, self.lens, y)
        uniq, inv = torch.unique(ids, return_inverse=True)
        rows = _host_rows(self.table, uniq).to(torch.float32)
        if not torch.is_grad_enabled():
            return _path_loss(hidden.detach().cpu(), rows[inv], bag, cds, y.numel()).to(hidden.device)
        rows.requires_grad_()
        loss = _path_loss(hidden.cpu(), rows[inv], bag, cds, y.numel())
        table, scale, option = self.table, self.push_scale, self.option

        def push(grad):
            if scale is not None:
                table.add_rows(uniq.numpy(), (grad * float(scale)).numpy(), option)
        rows.register_hook(push)
        return loss.to(hidden.device)

    def extra_repr(self) -> str:
        return (f"{self.in_features}, {self.num_classes}, depth={self.depth}, "
                f"weight=MatrixTable#{getattr(self.table, 'table_id', '?')}")


class _HsmFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, hidden, y, ln, L, hsm):
        loss, x, ids, offsets, g, u = hsm._launch(hidden.detach(), y, ln, L, grad=True)
        ctx.hsm = hsm
        ctx.save_for_backward(x, ids, offsets, g, u)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        x, ids, offsets, g, u = ctx.saved_tensors
        hsm = ctx.hsm
        dloss = dloss.to(torch.float32).contiguous()
        dx = dloss[:, None] * u if ctx.needs_input_grad[1] else None
        if hsm.push_scale is not None:
            _push_device(hsm.table, hsm._rm, hsm.in_features, ids, offsets, g, "sum", dloss[:, None] * x,
                         float(hsm.push_scale), hsm.option)
        return torch.zeros_like(hsm.anchor), dx, None, None, None, None
