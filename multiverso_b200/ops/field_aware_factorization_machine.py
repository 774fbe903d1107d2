"""Field-aware factorization machine over a MatrixTable: the FFM of sparse CTR features (Juan et al., RecSys 2016;
libffm), with its factors and linear weights in the parameter server.

Take F fields of k factors each (k >= 4, k % 4 == 0, so every field segment starts on a 16-byte boundary) and
D = F k. Row ``r`` of the table holds the F factor vectors ``V_r[f] = W[r, f k : (f + 1) k]`` and the linear weight
``w_r = W[r, D]``. The table's width must be at least D + 1; columns past D are not part of the model and are never
read (a HashMatrixTable, whose width is a multiple of 4, takes width D + 4)::

    ffm = mv.ops.PSFieldAwareFactorizationMachine(table, num_fields=F, num_factors=k, push_scale=lr)
    y = ffm(ids, fields, offsets, values)   # [B] float32; bags in embedding_bag's layout; fields, values: ids' shape
    loss = F.binary_cross_entropy_with_logits(y + bias, labels)    # a global bias is the caller's Parameter
    loss.backward()                         # the row gradient goes to the table's updater, once per touched row

Bag ``b`` holds the lookups ``j`` with ids ``i_j``, fields ``f_j`` in [0, F) and values ``x_j`` (``values=None``:
every x is 1), as ``embedding_bag`` takes them: 1-D ``ids`` with ``offsets`` or a 2-D ``[B, n]`` tensor (one-hot
Criteo rows: ``fields`` is the column index). Then

    y_b = sum_j x_j w_{i_j} + sum_{j < l} x_j x_l <V_{i_j}[f_l], V_{i_l}[f_j]>.

An empty bag gives 0. Repeated ids and repeated fields in a bag are distinct positions (multi-hot fields just work);
a position never interacts with itself. With F = 1 this is ``PSFactorizationMachine`` with C = k + 1.

The gradient of y_b with respect to the row values at position j is one row ``H_j`` of D + 1 columns that does not
depend on dL/dy:

* segment f of ``H_j``: ``x_j sum_{l != j, f_l = f} x_l V_{i_l}[f_j]``, the positions l in order;
* column D: ``x_j``.

So the row gradient coalesced over the batch is ``G_r = sum_{j: i_j = r} g_{b(j)} H_j`` with ``g_b = dL/dy_b``:
the embedding-bag backward with one bag per lookup, per-sample weights ``g_{b(j)}`` and dout H. It is multiplied by
``push_scale`` and pushed once per unique row (``None``: no push): ``default`` / ``sgd`` tables that are not
``is_sparse`` get a ``red.add`` into the owners' rows without a host synchronisation, any other table the compact
rows through one ``add_rows_async`` after one read of the unique-row count, so every stateful updater takes exactly
one step per touched row. ``values`` get no gradient; a ``values`` tensor that requires grad is refused. Reads follow
``get_rows``' rule: the caller orders a call after the Adds it wants to see (barrier / ``flush``). Under
``torch.no_grad()`` the forward computes ``y`` only and keeps nothing.

On the device, the forward checks ids, offsets and fields in one host read, then ``mvb_ffm_fwd``
(``csrc/cuda/ffm.cu``) runs one CTA per bag: the bag's rows are staged in shared memory straight from the owners'
shards, its positions grouped by field, and every (lookup, 4 columns) item of H summed by one thread; ``y_b =
sum_j x_j w_{i_j} + (1/2) sum_j <H_j[0:D], W[i_j, 0:D]>`` (every pair is met from both sides). In training the kernel
also writes H, ``[L, round4(D + 1)]`` floats: the only per-lookup output, 4 bytes x L x round4(D + 1) (B = 8192
one-hot bags of 39 fields at k = 16: 0.8 GB), freed after the backward. Nothing of size bag length squared is
written. ``y`` and H are bitwise reproducible, the same for every sharding and every batch a bag comes in, and the
forward without H is bitwise the forward with it.

Over a :class:`~multiverso_b200.tables.device.HashMatrixTable` the ids are keys, as in ``PSFactorizationMachine``:
training mode inserts missing keys, eval mode reads them as the zero row (and a backward after such a forward
raises), and keys not yet admitted under ``admit_after`` read the zero row, add 0 to ``y`` and are never pushed. On
the host backend the same maths runs in torch fp32 over ``get_rows`` of the unique ids, and the gradient goes out in
one coalesced ``add_rows``.

Accuracy of the device results against exact arithmetic, to first order in ``u = 2^-24``. For lookup j of bag b
and factor column c of segment f, let ``n_jf = #{l != j: f_l = f}`` (at most n_b - 1 for a bag of n_b lookups) and
``A_jc = sum_{l != j, f_l = f} |x_j x_l V_{i_l}[f_j]_c|``; let ``nq = round4(D + 1) / 4`` and
``N_b = 4 ceil(n_b nq / 256)``, the longest chain of terms one thread sums for the bag:

* ``H_jc``: an fma chain over the n_jf positions from 0, then the product by x_j: ``|dH_jc| <= (n_jf + 1) u A_jc``;
  column D is x_j exactly;
* ``y``: each thread sums its items' terms ``x_j w`` and ``H_jc W[i_j, c]`` (exact products of rounded H) in at
  most N_b fmas, then a 5-level warp butterfly and a sum over 8 warps (7 adds), then ``lin + 0.5 pair``:
  ``|dy_b| <= u ((N_b + 12) Lam_b + (1/2) sum_{j, c < D} (n_jf + N_b + 13) A_jc |W[i_j, c]| + |y_b|)`` with
  ``Lam_b = sum_j |x_j w_{i_j}|``. The pair sum meets every pair twice, from rounded H rows of each side, so for
  a bag whose pair terms cancel the error is of order ``u`` times the sum of their absolute values;
* ``G_r`` over the m lookups of row r (the embedding-bag backward: ``g H_j`` with one rounding each, the pieces of a
  run summed in chunk order): ``|dG_rc| <= u sum_j |g_b(j)| (n_jf + 1) A_jc + (2 m + 4) u sum_j |g_b(j) H_jc|``;
* the fused push adds ``scale * G_r`` with ``red.add``: one more rounding, ``u |W_rc + scale G_rc|``, and
  ``u |scale G_rc|`` for the product when ``|scale| != 1``.

``tests/test_gpu_field_aware_factorization_machine.py`` checks ``y`` and ``G`` against fp64 within these bounds.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _native as N
from ..tables.device import HashMatrixTable
from ..tables.options import AddOption
from ..utils import monitor
from .embedding import _bag_index, _bags, _check_values, _device_of, _dtype_of, _host_rows, _prepare, _push_device
from .topk import _rowmap_of

_WHAT = "PSFieldAwareFactorizationMachine"


def _ffm_y(rows: torch.Tensor, f: torch.Tensor, x: torch.Tensor, bag: torch.Tensor, B: int, F: int,
           k: int) -> torch.Tensor:
    """y [B] from the row of every lookup ``rows`` [L, >= D + 1], the fields f [L], the values x [L] and the bag of
    every lookup (non-decreasing), pair by pair: lookup j meets j + d for d = 1, 2, ... while they share a bag."""
    L, D = rows.shape[0], F * k
    V = rows[:, :D].reshape(L, F, k)
    y = torch.zeros(B, dtype=rows.dtype, device=rows.device).index_add(0, bag, x * rows[:, D])
    lens = torch.bincount(bag, minlength=B) if L else torch.zeros(1, dtype=torch.int64)
    for d in range(1, int(lens.max()) if L else 0):
        j = torch.nonzero(bag[:-d] == bag[d:]).view(-1)
        lk = j + d
        t = x[j] * x[lk] * (V[j, f[lk]] * V[lk, f[j]]).sum(1)
        y = y.index_add(0, bag[j], t)
    return y


def _fields_of(fields, shape, what: str) -> torch.Tensor:
    fields = torch.as_tensor(fields)
    if fields.is_floating_point() or fields.is_complex() or fields.dtype == torch.bool:
        raise TypeError(f"{what}: fields must be integers, got {fields.dtype}")
    if fields.shape != shape:
        raise ValueError(f"{what}: fields must have the shape of ids {tuple(shape)}, got {tuple(fields.shape)}")
    return fields.reshape(-1)


def _checks(f: torch.Tensor, F: int, what: str, info: dict):
    """The extra part of the id / offset check: the field range and the longest bag, in the same host read."""
    def extra(ids, offsets):
        L = ids.numel()
        parts = list(torch.aminmax(f)) if L else []
        parts.append(torch.cat([offsets[1:] - offsets[:-1], L - offsets[-1:]]).max())

        def check(v):
            if L and (v[0] < 0 or v[1] >= F):
                raise ValueError(f"{what}: fields must be in [0, {F}), got min {v[0]} max {v[1]}")
            info["max_len"] = v[-1]
        return parts, check
    return extra


def field_aware_factorization_machine_reference(weights, ids, fields, offsets=None, values=None, *, num_fields: int,
                                                num_factors: int) -> torch.Tensor:
    """Host implementation in fp64: y [B] of the bags over ``weights`` [num_row, >= D + 1] (segment f of the factors
    in columns f k .. (f + 1) k - 1, the linear weight in column D = F k). Differentiable in ``weights``."""
    w = torch.as_tensor(weights)
    F, k = int(num_fields), int(num_factors)
    if w.dim() != 2 or w.shape[1] < F * k + 1:
        raise ValueError(f"field_aware_factorization_machine_reference: weights must be [num_row, >= {F * k + 1}], "
                         f"got {tuple(w.shape)}")
    shape = torch.as_tensor(ids).shape
    f = _fields_of(fields, shape, "field_aware_factorization_machine_reference")
    ids, offsets, x = _bags(ids, offsets, values, "sum")
    info = {}
    _check_values(ids, offsets, w.shape[0], extra=_checks(f.to(ids.device), F,
                                                          "field_aware_factorization_machine_reference", info))
    ids, offsets, f = ids.to(w.device), offsets.to(w.device), f.to(w.device)
    x = torch.ones(ids.numel(), dtype=torch.float64, device=w.device) if x is None else \
        x.to(device=w.device, dtype=torch.float64)
    bag, _ = _bag_index(offsets, ids.numel())
    return _ffm_y(w.to(torch.float64)[ids], f, x, bag, offsets.numel(), F, k)


class PSFieldAwareFactorizationMachine(torch.nn.Module):
    """Field-aware factorization-machine layer whose factors and linear weights are the rows of a MatrixTable (see
    the module docstring). ``num_fields`` F, ``num_factors`` k (>= 4, a multiple of 4); ``push_scale``: the row
    gradient is multiplied by it before the push (``None``: no push); ``option``: the AddOption of the push."""

    def __init__(self, table, num_fields: int, num_factors: int, push_scale: Optional[float] = 1.0,
                 option: Optional[AddOption] = None):
        super().__init__()
        if isinstance(table, torch.Tensor):
            raise TypeError(f"{_WHAT}: the weight must be a MatrixTable (a tensor has no updater to push to)")
        if _dtype_of(table) != torch.float32:
            raise TypeError(f"{_WHAT}: the table must be float32, got {_dtype_of(table)}")
        F, k = int(num_fields), int(num_factors)
        if F != num_fields or F < 1:
            raise ValueError(f"{_WHAT}: num_fields must be a positive integer, got {num_fields}")
        if k != num_factors or k < 4 or k % 4:
            raise ValueError(f"{_WHAT}: num_factors must be a positive multiple of 4, got {num_factors}")
        D = F * k
        if D + 1 > N.FFM_MAX_DIM:
            raise ValueError(f"{_WHAT}: num_fields * num_factors + 1 must be at most {N.FFM_MAX_DIM}, got {D + 1}")
        if int(table.num_col) < D + 1:
            raise ValueError(f"{_WHAT}: the table's width ({table.num_col}) must be at least num_fields * "
                             f"num_factors + 1 = {D + 1}")
        self.table, self.push_scale, self.option = table, push_scale, option
        self.num_fields, self.num_factors, self.dim = F, k, D
        self._device = _device_of(table)
        if self._device is not None:
            self._rm = _rowmap_of(table, _WHAT)[0]
            if self._rm.num_col % 4 != 0:
                raise ValueError(f"{_WHAT}: the table's row pitch ({self._rm.num_col} floats) must be a multiple "
                                 "of 4 (16-byte row loads)")
        # ids never require grad: without an input that does, autograd would skip the backward and so the push
        self.anchor = torch.nn.Parameter(torch.zeros(0))

    def forward(self, ids, fields, offsets=None, values=None) -> torch.Tensor:
        shape = torch.as_tensor(ids).shape
        if values is not None:
            values = torch.as_tensor(values)
            if not values.is_floating_point():
                raise TypeError(f"{_WHAT}: values must be floating point, got {values.dtype}")
            if values.requires_grad:
                raise ValueError(f"{_WHAT}: values get no gradient; pass values.detach()")
            if values.shape != shape:
                raise ValueError(f"{_WHAT}: values must have the shape of ids {tuple(shape)}, got "
                                 f"{tuple(values.shape)}")
        f = _fields_of(fields, shape, _WHAT)
        f = f.to(self._device if self._device is not None else torch.device("cpu"))
        info = {}
        # over a HashMatrixTable the ids are keys: training inserts the missing ones, eval reads them as zeros
        frozen = isinstance(self.table, HashMatrixTable) and not self.training
        ids, offsets, x = _prepare(self.table, ids, offsets, values, "sum", insert=self.training,
                                   extra=_checks(f, self.num_fields, _WHAT, info))
        if self._device is None:
            return self._forward_host(ids, offsets, f, x)
        x = None if x is None else x.to(device=self._device, dtype=torch.float32).contiguous()
        f = f.to(torch.int32).contiguous()
        max_len = info.get("max_len", 0)
        if not torch.is_grad_enabled():
            return self._launch(ids, offsets, f, x, max_len, grad=False)[0]
        return _FfmFn.apply(self.anchor, ids, offsets, f, x, max_len, frozen, self)

    # ------------------------------------------------------------------------------------------------ device
    def _launch(self, ids, offsets, f, x, max_len: int, grad: bool):
        """mvb_ffm_fwd: y [B], and with ``grad`` H [L, round4(D + 1)]."""
        B, L, D = offsets.numel(), ids.numel(), self.dim
        a = N.Ffm()
        a.wmap, a.F, a.k = self._rm, self.num_fields, self.num_factors
        a.ids, a.fields, a.values = ids.data_ptr(), f.data_ptr(), N.ptr(x)
        a.offsets, a.L, a.B, a.max_len = offsets.data_ptr(), L, B, max_len
        y = torch.empty(B, dtype=torch.float32, device=self._device)
        a.y = y.data_ptr()
        h = None
        if grad:
            ldh = (D + 1 + 3) // 4 * 4
            h = torch.empty(L, ldh, dtype=torch.float32, device=self._device)
            a.h, a.ldh = h.data_ptr(), ldh
        with monitor("WORKER_TABLE_FIELD_AWARE_FACTORIZATION_MACHINE", cuda=True, nbytes=L * (D + 1) * 4):
            N.cuda_lib().mvb_ffm_fwd(a, N.stream_ptr())
        return y, h

    def _push(self, ids, offsets, h, dy) -> None:
        """G_r = sum_{j: i_j = r} dy[bag(j)] H_j through the embedding-bag backward, one bag per lookup."""
        L = ids.numel()
        if L == 0:
            return
        pos = torch.arange(L, dtype=torch.int64, device=ids.device)
        bag = torch.searchsorted(offsets, pos, right=True) - 1
        _push_device(self.table, self._rm, self.dim + 1, ids, pos, dy[bag].contiguous(), "sum", h,
                     float(self.push_scale), self.option)

    # ------------------------------------------------------------------------------------------------ host
    def _forward_host(self, ids, offsets, f, x) -> torch.Tensor:
        ids, offsets, f = ids.cpu(), offsets.cpu(), f.cpu()
        L, B = ids.numel(), offsets.numel()
        bag, _ = _bag_index(offsets, L)
        uniq, inv = torch.unique(ids, return_inverse=True)
        rows = _host_rows(self.table, uniq).to(torch.float32)
        x = torch.ones(L) if x is None else x.detach().cpu().to(torch.float32)
        F, k = self.num_fields, self.num_factors
        if not torch.is_grad_enabled():
            return _ffm_y(rows[inv], f, x, bag, B, F, k)
        rows.requires_grad_()
        table, scale, option = self.table, self.push_scale, self.option

        def push(grad):
            if scale is not None and uniq.numel():
                table.add_rows(uniq.numpy(), (grad * float(scale)).numpy(), option)
        rows.register_hook(push)
        return _ffm_y(rows[inv], f, x, bag, B, F, k)

    def extra_repr(self) -> str:
        return (f"fields={self.num_fields}, factors={self.num_factors}, "
                f"weight=MatrixTable#{getattr(self.table, 'table_id', '?')}")


class _FfmFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, ids, offsets, f, x, max_len, frozen, ffm):
        y, h = ffm._launch(ids, offsets, f, x, max_len, grad=True)
        ctx.ffm, ctx.frozen = ffm, frozen
        ctx.save_for_backward(ids, offsets, h)
        return y

    @staticmethod
    def backward(ctx, dy):
        ffm = ctx.ffm
        if ffm.push_scale is not None:
            if ctx.frozen:
                raise RuntimeError(f"{_WHAT}: backward after a forward that inserted no keys (eval mode): missing "
                                   "keys share the zero row, which must not be pushed to; run the forward in training "
                                   "mode")
            ids, offsets, h = ctx.saved_tensors
            ffm._push(ids, offsets, h, dy.to(torch.float32).contiguous())
        return torch.zeros_like(ffm.anchor), None, None, None, None, None, None, None
