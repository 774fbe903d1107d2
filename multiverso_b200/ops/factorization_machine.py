"""Factorization machine over a MatrixTable: the second-order model of sparse CTR features (Rendle 2010), with its
factors and linear weights in the parameter server.

Row ``r`` of a table of width ``C`` (2 <= C <= 1024) holds the ``k = C - 1`` factors ``v_r = W[r, 0:k]`` and the
linear weight ``w_r = W[r, k]``; the factors start at column 0, so their loads stay 16-byte aligned::

    fm = mv.ops.PSFactorizationMachine(table, push_scale=lr)       # table: MatrixTable(num_row, k + 1, "float32")
    y = fm(ids, offsets, values)      # [B] float32; bags in torch's embedding_bag layout, values: the shape of ids
    loss = F.binary_cross_entropy_with_logits(y + bias, labels)    # a global bias is the caller's Parameter
    loss.backward()                   # the row gradient goes to the table's updater, once per touched row

Bag ``b`` holds the lookups ``j`` with ids ``i_j`` and values ``x_j`` (``values=None``: every x is 1), as
``embedding_bag`` takes them: 1-D ``ids`` with ``offsets`` or a 2-D ``[B, n]`` tensor. Then

* ``S_b = sum_j x_j W[i_j, :]`` (C columns: ``s_b = S_b[:k]``, ``lin_b = S_b[k]``),
* ``q_b = sum_j x_j^2 |v_{i_j}|^2``,
* ``y_b = lin_b + (|s_b|^2 - q_b) / 2 = sum_j x_j w_{i_j} + sum_{j < l} x_j x_l <v_{i_j}, v_{i_l}>``.

An empty bag gives 0. Repeated ids in one bag interact as distinct positions (the pair term of an id with itself
is counted): to get the FM of a feature vector, merge its duplicate ids (adding their values) first.

With ``g_b = dL/dy_b``, the gradient of row ``r`` coalesced over the batch is
``G_r = sum_{j: i_j = r} g_b x_j (S'_b - x_j v'_r)``, where ``S'_b`` is ``S_b`` with column k set to 1 and ``v'_r``
is ``v_r`` with 0 in column k. It is multiplied by ``push_scale`` and pushed once per unique row (``None``: no
push): ``default`` / ``sgd`` tables that are not ``is_sparse`` get a ``red.add`` into the owners' rows without a
host synchronisation, any other table the compact rows through one ``add_rows_async`` after one read of the
unique-row count, so every stateful updater takes exactly one step per touched row. ``values`` get no gradient; a
``values`` tensor that requires grad is refused. Reads follow ``get_rows``' rule: the caller orders a call after
the Adds it wants to see (barrier / ``flush``). Under ``torch.no_grad()`` the forward computes ``y`` only and keeps
nothing.

On the device, the forward checks the ids and offsets in one host read, then ``mvb_fm_fwd``
(``csrc/cuda/fm.cu``) runs one warp per bag: rows come straight from the owners' shards and are summed in
registers exactly as ``embedding_bag`` sums them (so ``S_b`` is bitwise ``embedding_bag(table, ids, offsets,
per_sample_weights=values)``), together with each lane's share of ``q``; the kernel writes ``y`` and, for the
backward, ``S'`` (``[B, round4(C)]``). Nothing of size lookups x C is written, and ``y`` is bitwise reproducible
and the same for every sharding. ``mvb_fm_bwd`` is the embedding-bag backward with the weight ``g_b x_j`` over the
dout row ``S'_b``, each run piece corrected by ``-c v'_r`` with ``c = sum g_b x_j^2``.

Over a :class:`~multiverso_b200.tables.device.HashMatrixTable` the ids are keys, as in ``PSEmbedding``: training
mode inserts missing keys, eval mode reads them as the zero row (and a backward after such a forward raises), and
keys not yet admitted under ``admit_after`` read the zero row, add 0 to ``y`` and are never pushed. A hash table's
width is a multiple of 4, so its factor count is 3, 7, 15, 31, 63, ... On the host backend the same maths runs in
torch fp32 over ``get_rows`` of the unique ids, and the gradient goes out in one coalesced ``add_rows``.

Accuracy of the device results against exact arithmetic, to first order in ``u = 2^-24``, for bag b of n lookups
with ``A_bc = sum_j |x_j W[i_j, c]|``, ``P_b = sum_{c < k} A_bc^2``, ``ss_b = |s_b|^2``:

* ``S``: an fma chain of at most n terms per lane group, then a butterfly of at most 5 levels:
  ``|dS_bc| <= (n + 5) u A_bc``;
* ``|s|^2``: at most 18 roundings on any term from a rounded S: ``|d ss_b| <= 2 (n + 5) u P_b + 18 u ss_b``;
* ``q``: a sum of non-negative terms, none rounded more than ``2 n + 14`` times: ``|dq_b| <= (2 n + 14) u q_b``;
* ``y``: ``|dy_b| <= u ((n + 5) (A_bk + P_b) + 9 ss_b + (n + 7) q_b + |ss_b - q_b| / 2 + |y_b|)``.
  The pair term is a difference ``(ss - q) / 2`` that cancels: for a bag of one lookup it is exactly 0 in exact
  arithmetic, and on the device it is rounding noise of order ``u (ss + q)``, not 0;
* ``G_r`` over the m lookups of row r (the weights ``g_b x_j`` and ``g_b x_j^2`` rounded once each, the pieces of
  a run summed in chunk order, one correction per piece): ``|dG_rc| <= u sum_j |g_b x_j| (n_b + 5) A_bc +
  (2 m + 4) u (sum_j |g_b x_j S'_bc| + |v'_rc| sum_j |g_b| x_j^2)``. ``S' - x v'`` cancels in the same way: a row
  looked up once in a bag of one lookup has a factor gradient of exactly 0, and gets rounding noise of order
  ``u |g x^2 v|``;
* the fused push adds ``scale * G_r`` with ``red.add``: one more rounding, ``u |W_rc + scale G_rc|``, and
  ``u |scale G_rc|`` for the product when ``|scale| != 1``.

``tests/test_gpu_factorization_machine.py`` checks ``y`` and ``G`` against fp64 within these bounds.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _native as N
from ..tables.device import HashMatrixTable
from ..tables.options import AddOption
from ..utils import monitor
from .embedding import _bag_index, _bags, _check_values, _device_of, _dtype_of, _host_rows, _prepare, _push_rows
from .topk import _rowmap_of

_WHAT = "PSFactorizationMachine"


def _fm_y(rows: torch.Tensor, x: torch.Tensor, bag: torch.Tensor, B: int) -> torch.Tensor:
    """y [B] from the row of every lookup ``rows`` [L, C], the values x [L] and the bag of every lookup."""
    k = rows.shape[1] - 1
    S = torch.zeros(B, k + 1, dtype=rows.dtype, device=rows.device).index_add(0, bag, x[:, None] * rows)
    q = torch.zeros(B, dtype=rows.dtype, device=rows.device).index_add(0, bag, x * x * (rows[:, :k] ** 2).sum(1))
    return S[:, k] + 0.5 * ((S[:, :k] ** 2).sum(1) - q)


def factorization_machine_reference(weights, ids, offsets=None, values=None) -> torch.Tensor:
    """Host implementation in fp64: y [B] of the bags over ``weights`` [num_row, C] (factors in columns 0..C-2, the
    linear weight in column C-1). Differentiable in ``weights``."""
    w = torch.as_tensor(weights)
    if w.dim() != 2 or w.shape[1] < 2:
        raise ValueError(f"factorization_machine_reference: weights must be [num_row, C >= 2], got {tuple(w.shape)}")
    ids, offsets, x = _bags(ids, offsets, values, "sum")
    _check_values(ids, offsets, w.shape[0])
    ids, offsets = ids.to(w.device), offsets.to(w.device)
    x = torch.ones(ids.numel(), dtype=torch.float64, device=w.device) if x is None else \
        x.to(device=w.device, dtype=torch.float64)
    bag, _ = _bag_index(offsets, ids.numel())
    return _fm_y(w.to(torch.float64)[ids], x, bag, offsets.numel())


class PSFactorizationMachine(torch.nn.Module):
    """Factorization-machine layer whose factors and linear weights are the rows of a MatrixTable (see the module
    docstring). ``push_scale``: the row gradient is multiplied by it before the push (``None``: no push);
    ``option``: the AddOption of the push."""

    def __init__(self, table, push_scale: Optional[float] = 1.0, option: Optional[AddOption] = None):
        super().__init__()
        if isinstance(table, torch.Tensor):
            raise TypeError(f"{_WHAT}: the weight must be a MatrixTable (a tensor has no updater to push to)")
        if _dtype_of(table) != torch.float32:
            raise TypeError(f"{_WHAT}: the table must be float32, got {_dtype_of(table)}")
        C = int(table.num_col)
        if not 2 <= C <= N.FM_MAX_DIM:
            raise ValueError(f"{_WHAT}: the table's width C = k + 1 must be in [2, {N.FM_MAX_DIM}], got {C}")
        self.table, self.push_scale, self.option = table, push_scale, option
        self.num_col, self.num_factors = C, C - 1
        self._device = _device_of(table)
        if self._device is not None:
            self._rm = _rowmap_of(table, _WHAT)[0]
            if self._rm.num_col % 4 != 0:
                raise ValueError(f"{_WHAT}: the table's row pitch ({self._rm.num_col} floats) must be a multiple "
                                 "of 4 (16-byte row loads)")
        # ids never require grad: without an input that does, autograd would skip the backward and so the push
        self.anchor = torch.nn.Parameter(torch.zeros(0))

    def forward(self, ids, offsets=None, values=None) -> torch.Tensor:
        if values is not None:
            values = torch.as_tensor(values)
            if not values.is_floating_point():
                raise TypeError(f"{_WHAT}: values must be floating point, got {values.dtype}")
            if values.requires_grad:
                raise ValueError(f"{_WHAT}: values get no gradient; pass values.detach()")
            shape = torch.as_tensor(ids).shape
            if values.shape != shape:
                raise ValueError(f"{_WHAT}: values must have the shape of ids {tuple(shape)}, got "
                                 f"{tuple(values.shape)}")
        # over a HashMatrixTable the ids are keys: training inserts the missing ones, eval reads them as zeros
        frozen = isinstance(self.table, HashMatrixTable) and not self.training
        ids, offsets, x = _prepare(self.table, ids, offsets, values, "sum", insert=self.training)
        if self._device is None:
            return self._forward_host(ids, offsets, x)
        x = None if x is None else x.to(device=self._device, dtype=torch.float32).contiguous()
        if not torch.is_grad_enabled():
            return self._launch(ids, offsets, x, grad=False)[0]
        return _FmFn.apply(self.anchor, ids, offsets, x, frozen, self)

    # ------------------------------------------------------------------------------------------------ device
    def _args(self, ids, offsets, x) -> N.Fm:
        a = N.Fm()
        a.wmap, a.dim = self._rm, self.num_col
        a.ids, a.L = ids.data_ptr(), ids.numel()
        a.offsets, a.B = offsets.data_ptr(), offsets.numel()
        a.values = N.ptr(x)
        return a

    def _launch(self, ids, offsets, x, grad: bool):
        """mvb_fm_fwd: y [B], and with ``grad`` S' [B, round4(C)]."""
        B, C = offsets.numel(), self.num_col
        a = self._args(ids, offsets, x)
        y = torch.empty(B, dtype=torch.float32, device=self._device)
        a.y = y.data_ptr()
        sp = None
        if grad:
            lds = (C + 3) // 4 * 4
            sp = torch.empty(B, lds, dtype=torch.float32, device=self._device)
            a.sp, a.lds = sp.data_ptr(), lds
        with monitor("WORKER_TABLE_FACTORIZATION_MACHINE", cuda=True, nbytes=ids.numel() * C * 4):
            N.cuda_lib().mvb_fm_fwd(a, N.stream_ptr())
        return y, sp

    def _push(self, ids, offsets, x, sp, dy) -> None:
        """mvb_fm_bwd: the coalesced row gradient times push_scale, fused red.add or compact + add_rows_async."""
        L, C, table = ids.numel(), self.num_col, self.table
        if L == 0:
            return
        lib = N.cuda_lib()
        sid, perm = torch.sort(ids, stable=True)               # (id, position) order
        nbytes = lib.mvb_embedding_bag_scratch_bytes(L, C)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=ids.device)
        a = self._args(sid, offsets, x)
        a.sp, a.lds, a.dy, a.perm = sp.data_ptr(), sp.shape[1], dy.data_ptr(), perm.data_ptr()
        a.scratch, a.scratch_bytes = scratch.data_ptr(), nbytes
        a.push_rows = _push_rows(table)
        st = N.stream_ptr()
        scale = float(self.push_scale)
        fused = table.updater in (N.UPD_DEFAULT, N.UPD_SGD) and not table.is_sparse
        with monitor("WORKER_TABLE_FACTORIZATION_MACHINE_GRAD", cuda=True, nbytes=L * C * 4):
            if fused:
                a.epilogue = N.EMB_PUSH
                a.scale = (-1.0 if table.updater == N.UPD_SGD else 1.0) * scale
                lib.mvb_fm_bwd(a, st)
                return
            a.epilogue, a.scale = N.EMB_COMPACT, scale
            n_unique = torch.empty(1, dtype=torch.int64, device=ids.device)
            a.n_unique = n_unique.data_ptr()
            lib.mvb_fm_bwd(a, st)          # count only
            U = int(n_unique.item())
            ldg = sp.shape[1]
            grads = torch.empty(U, ldg, dtype=torch.float32, device=ids.device)
            uniq = torch.empty(U, dtype=torch.int64, device=ids.device)
            a.grads, a.ldg, a.uniq = grads.data_ptr(), ldg, uniq.data_ptr()
            lib.mvb_fm_bwd(a, st)
        table.add_rows_async(uniq, grads if ldg == C else grads[:, :C], self.option)

    # ------------------------------------------------------------------------------------------------ host
    def _forward_host(self, ids, offsets, x) -> torch.Tensor:
        ids, offsets = ids.cpu(), offsets.cpu()
        L, B = ids.numel(), offsets.numel()
        bag, _ = _bag_index(offsets, L)
        uniq, inv = torch.unique(ids, return_inverse=True)
        rows = _host_rows(self.table, uniq).to(torch.float32)
        x = torch.ones(L) if x is None else x.detach().cpu().to(torch.float32)
        if not torch.is_grad_enabled():
            return _fm_y(rows[inv], x, bag, B)
        rows.requires_grad_()
        table, scale, option = self.table, self.push_scale, self.option

        def push(grad):
            if scale is not None and uniq.numel():
                table.add_rows(uniq.numpy(), (grad * float(scale)).numpy(), option)
        rows.register_hook(push)
        return _fm_y(rows[inv], x, bag, B)

    def extra_repr(self) -> str:
        return f"factors={self.num_factors}, weight=MatrixTable#{getattr(self.table, 'table_id', '?')}"


class _FmFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, ids, offsets, x, frozen, fm):
        y, sp = fm._launch(ids, offsets, x, grad=True)
        ctx.fm, ctx.frozen = fm, frozen
        ctx.save_for_backward(ids, offsets, x, sp)
        return y

    @staticmethod
    def backward(ctx, dy):
        fm = ctx.fm
        if fm.push_scale is not None:
            if ctx.frozen:
                raise RuntimeError(f"{_WHAT}: backward after a forward that inserted no keys (eval mode): missing "
                                   "keys share the zero row, which must not be pushed to; run the forward in training "
                                   "mode")
            ids, offsets, x, sp = ctx.saved_tensors
            fm._push(ids, offsets, x, sp, dy.to(torch.float32).contiguous())
        return torch.zeros_like(fm.anchor), None, None, None, None, None
