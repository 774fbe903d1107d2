"""Embedding bags over a MatrixTable: the sparse-feature layer whose weight lives in the parameter server.

``embedding_bag(table, ids, offsets)`` returns, for every bag, the sum (``mode="mean"``: the mean) of its rows,
each scaled by its per-sample weight when given, with torch's ``embedding_bag`` conventions: ``ids`` is 1-D with
``offsets`` (bag b holds ``ids[offsets[b]:offsets[b + 1]]``, the last bag runs to the end) or a 2-D ``[B, n]``
tensor of bags of ``n`` lookups; an empty bag gives zeros.

On the device (``csrc/cuda/emb_bag.cu``) the forward gathers every bag's rows straight from their owners' shards
and sums them in registers: the ``lookups x dim`` tensor of gathered rows is never written. A call on any rank
reads the whole sharded table, with the consistency rule of ``get_rows``: the caller orders it after the Adds it
wants to see (barrier / ``flush``). The result is bitwise reproducible and the same for every sharding.

:class:`PSEmbedding` is the differentiable layer. Its backward sorts the lookups by row id and sums the gradient of
every unique row in one kernel, so each touched row gets exactly one updater step per backward, however often it
was looked up (what ``torch.nn.EmbeddingBag(sparse=True)`` gives a torch optimiser). The pushed value is the
coalesced gradient times ``push_scale``:

* ``default`` / ``sgd`` updaters on a table that is not ``is_sparse``: the kernel adds it straight into the owners'
  rows (``red.add``); no gradient tensor is written and the backward does not synchronise with the host.
* any other table: the kernel writes the unique ids and their gradients, and ``add_rows_async`` applies them (the
  stateful updaters on the owners, stale marking of ``is_sparse`` tables). Sizing that buffer reads the number of
  unique ids on the host: one synchronisation per backward.

Over a :class:`~multiverso_b200.tables.device.HashMatrixTable` the ids are int64 keys: one ``mvb_hash_rows_lookup``
translates them to rows before the input checks (its status word is read in the checks' one host read), then the
same kernels run on the rows. ``PSEmbedding`` in training mode inserts missing keys; in eval mode, and in
``embedding_bag``, they read the zero row, and a backward after such a forward raises. Over a table with
``admit_after``, keys not admitted yet read the zero row in training mode too, and the backward pushes nothing for
them (the zero row stays zero).

On the host backend the same calls run :func:`embedding_bag_reference` over ``get_rows`` of the unique ids, and the
backward pushes the gradient coalesced in torch with ``add_rows``: the same semantics.
"""
from __future__ import annotations

from typing import Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from .. import _native as N
from ..tables.device import HashMatrixTable, raise_hash_status
from ..tables.options import AddOption
from ..utils import monitor
from .topk import _rowmap_of

MODES = ("sum", "mean")
_INT = (torch.int32, torch.int64)


def _bags(ids, offsets, per_sample_weights, mode: str) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """Checks the shapes and types of a call; returns (ids [L] int64, offsets [B] int64, weights [L] or None)."""
    if mode not in MODES:
        raise ValueError(f"embedding_bag: mode must be one of {MODES}, got {mode!r}")
    ids = torch.as_tensor(ids)
    if ids.dtype not in _INT:
        raise TypeError(f"embedding_bag: ids must be int32 or int64, got {ids.dtype}")
    if ids.dim() == 2:
        if offsets is not None:
            raise ValueError("embedding_bag: offsets must be None when ids is 2-D (one bag per row)")
        B, n = ids.shape
        offsets = torch.arange(0, B * n, n, dtype=torch.int64, device=ids.device) if n else \
            torch.zeros(B, dtype=torch.int64, device=ids.device)
    elif ids.dim() == 1:
        if offsets is None:
            raise ValueError("embedding_bag: 1-D ids need offsets")
        offsets = torch.as_tensor(offsets, device=ids.device)
        if offsets.dtype not in _INT or offsets.dim() != 1:
            raise TypeError(f"embedding_bag: offsets must be a 1-D int32 or int64 tensor, got {offsets.dtype} "
                            f"{tuple(offsets.shape)}")
    else:
        raise ValueError(f"embedding_bag: ids must be 1-D or 2-D, got {tuple(ids.shape)}")
    psw = per_sample_weights
    if psw is not None:
        if mode != "sum":
            raise ValueError("embedding_bag: per_sample_weights are only supported with mode='sum'")
        psw = torch.as_tensor(psw)
        if psw.shape != ids.shape:
            raise ValueError(f"embedding_bag: per_sample_weights must have the shape of ids {tuple(ids.shape)}, "
                             f"got {tuple(psw.shape)}")
        if not psw.is_floating_point():
            raise TypeError(f"embedding_bag: per_sample_weights must be floating point, got {psw.dtype}")
        psw = psw.reshape(-1)
    return ids.reshape(-1).to(torch.int64).contiguous(), offsets.to(torch.int64).contiguous(), psw


def _check_values(ids: torch.Tensor, offsets: torch.Tensor, num_row: int, status: Optional[torch.Tensor] = None,
                  hash_table=None, extra=None) -> None:
    """ids in [0, num_row) and offsets that start at 0, never decrease and stay within the ids (one host read).
    ``status``: the status word of the hash translation that produced ``ids``, read in the same copy. ``extra``: a
    function of (ids, offsets) returning (int64 tensors to read in the same copy, a check called with their values
    after the checks above), for a caller with more to check."""
    L, B = ids.numel(), offsets.numel()
    if B == 0:
        if L:
            raise ValueError(f"embedding_bag: {L} ids but no bags (offsets is empty)")
        return
    parts = [offsets[:1], (offsets[1:] < offsets[:-1]).any().view(1).to(torch.int64), offsets[-1:]]
    if L:
        parts += list(torch.aminmax(ids))
    more, check = extra(ids, offsets) if extra is not None else ([], None)
    parts += more
    if status is not None:
        parts.append(status)
    v = torch.cat([p.view(-1).to(torch.int64) for p in parts]).tolist()
    if status is not None:
        raise_hash_status(v.pop(), [hash_table])
    if v[0] != 0:
        raise ValueError(f"embedding_bag: offsets must start at 0, got {v[0]}")
    if v[1]:
        raise ValueError("embedding_bag: offsets must be non-decreasing")
    if v[2] > L:
        raise ValueError(f"embedding_bag: offsets exceed the number of ids ({v[2]} > {L})")
    if L and (v[3] < 0 or v[4] >= num_row):
        raise ValueError(f"embedding_bag: ids must be in [0, {num_row}), got min {v[3]} max {v[4]}")
    if check is not None:
        check(v[5 if L else 3:])


def _bag_index(offsets: torch.Tensor, L: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(bag of every lookup, length of every bag)."""
    lens = torch.diff(offsets, append=torch.tensor([L], dtype=offsets.dtype, device=offsets.device))
    return torch.repeat_interleave(torch.arange(offsets.numel(), device=offsets.device), lens), lens


def embedding_bag_reference(weights, ids, offsets=None, per_sample_weights=None, mode: str = "sum") -> torch.Tensor:
    """Host implementation: the rows of the unique ids, then ``torch.nn.functional.embedding_bag`` over them.
    ``weights``: [num_row, dim] tensor. Returns [B, dim]."""
    w = torch.as_tensor(weights)
    ids, offsets, psw = _bags(ids, offsets, per_sample_weights, mode)
    _check_values(ids, offsets, w.shape[0])
    uniq, inv = torch.unique(ids, return_inverse=True)
    return F.embedding_bag(inv, w[uniq.to(w.device)], offsets.to(w.device), mode=mode,
                           per_sample_weights=psw)


# ------------------------------------------------------------------------------------------------ device
def _dtype_of(table):
    if isinstance(table, torch.Tensor) or hasattr(table, "_rowmap"):
        return table.dtype
    return torch.from_numpy(np.zeros(0, table.npdt)).dtype         # host-backend table


def _device_of(table) -> Optional[torch.device]:
    """The CUDA device a table is read on, None for a host-backend table or a CPU tensor."""
    if isinstance(table, torch.Tensor):
        return table.device if table.is_cuda else None
    return table.rt.device if hasattr(table, "_rowmap") else None


def _args(rm: N.RowMap, dim: int, ids: torch.Tensor, offsets: torch.Tensor, psw: Optional[torch.Tensor],
          mode: str) -> N.EmbBag:
    a = N.EmbBag()
    a.wmap, a.dim = rm, dim
    a.ids, a.L = ids.data_ptr(), ids.numel()
    a.offsets, a.B = offsets.data_ptr(), offsets.numel()
    a.psw, a.mean = N.ptr(psw), int(mode == "mean")
    return a


def _push_rows(table) -> int:
    """The backward's row bound: keys a table with admission has not admitted read the zero row, its last row,
    which is never pushed (0: every row is)."""
    return table.zero_row if isinstance(table, HashMatrixTable) and table.admit_after > 1 else 0


def _fwd_device(rm, dim, ids, offsets, psw, mode) -> torch.Tensor:
    ldo = (dim + 3) // 4 * 4
    out = torch.empty(offsets.numel(), ldo, dtype=torch.float32, device=ids.device)
    a = _args(rm, dim, ids, offsets, psw, mode)
    a.out, a.ldo = out.data_ptr(), ldo
    with monitor("WORKER_TABLE_EMBEDDING_BAG", cuda=True, nbytes=ids.numel() * dim * 4):
        N.cuda_lib().mvb_embedding_bag_fwd(a, N.stream_ptr())
    return out if ldo == dim else out[:, :dim]


def _dout_padded(dout: torch.Tensor, dim: int) -> Tuple[torch.Tensor, int]:
    """dout as rows of a multiple of 4 floats, 16-byte aligned (copied only when it is not already). A contiguous
    dout wider than dim whose pitch is a multiple of 4 is taken as it is: its first dim columns are the gradient."""
    dout = dout.to(torch.float32)
    ld = dout.shape[1]
    if ld >= dim and ld % 4 == 0 and dout.is_contiguous() and dout.data_ptr() % 16 == 0:
        return dout, ld
    ldd = (dim + 3) // 4 * 4
    pad = torch.zeros(dout.shape[0], ldd, dtype=torch.float32, device=dout.device)
    pad[:, :dim] = dout
    return pad, ldd


def _psw_grad_device(rm, dim, ids, offsets, mode, dout) -> torch.Tensor:
    d, ldd = _dout_padded(dout, dim)
    dpsw = torch.empty(ids.numel(), dtype=torch.float32, device=ids.device)
    a = _args(rm, dim, ids, offsets, None, mode)
    a.dout, a.ldd, a.dpsw = d.data_ptr(), ldd, dpsw.data_ptr()
    N.cuda_lib().mvb_embedding_bag_psw_grad(a, N.stream_ptr())
    return dpsw


def _push_device(table, rm, dim, ids, offsets, psw, mode, dout, push_scale: float,
                 option: Optional[AddOption]) -> None:
    L = ids.numel()
    if L == 0:
        return
    lib = N.cuda_lib()
    d, ldd = _dout_padded(dout, dim)
    sid, perm = torch.sort(ids, stable=True)               # (id, position) order
    nbytes = lib.mvb_embedding_bag_scratch_bytes(L, dim)
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=ids.device)
    a = _args(rm, dim, sid, offsets, psw, mode)
    a.dout, a.ldd, a.perm = d.data_ptr(), ldd, perm.data_ptr()
    a.scratch, a.scratch_bytes = scratch.data_ptr(), nbytes
    a.push_rows = _push_rows(table)
    st = N.stream_ptr()
    fused = table.updater in (N.UPD_DEFAULT, N.UPD_SGD) and not table.is_sparse
    with monitor("WORKER_TABLE_EMBEDDING_BAG_GRAD", cuda=True, nbytes=L * dim * 4):
        if fused:
            a.epilogue = N.EMB_PUSH
            a.scale = (-1.0 if table.updater == N.UPD_SGD else 1.0) * push_scale
            lib.mvb_embedding_bag_bwd(a, st)
            return
        a.epilogue, a.scale = N.EMB_COMPACT, push_scale
        n_unique = torch.empty(1, dtype=torch.int64, device=ids.device)
        a.n_unique = n_unique.data_ptr()
        lib.mvb_embedding_bag_bwd(a, st)     # count only
        U = int(n_unique.item())
        ldg = (table.num_col + 3) // 4 * 4             # the kernel writes whole 16-byte vectors
        alloc = torch.empty if dim == ldg else torch.zeros
        grads = alloc(U, ldg, dtype=torch.float32, device=ids.device)
        uniq = torch.empty(U, dtype=torch.int64, device=ids.device)
        a.grads, a.ldg, a.uniq = grads.data_ptr(), ldg, uniq.data_ptr()
        lib.mvb_embedding_bag_bwd(a, st)
    table.add_rows_async(uniq, grads if ldg == table.num_col else grads[:, :table.num_col], option)


# ------------------------------------------------------------------------------------------------ host
def _host_rows(table, uniq: torch.Tensor) -> torch.Tensor:
    if isinstance(table, torch.Tensor):
        return table[uniq]
    return torch.from_numpy(np.asarray(table.get_rows(uniq.numpy())))


def _host_backward(ctx, ids, offsets, psw, dout):
    uniq, inv, rows = ctx.host
    L = ids.numel()
    bag, lens = _bag_index(offsets, L)
    s = psw.detach().to(dout.dtype) if psw is not None else torch.ones(L, dtype=dout.dtype)
    if ctx.mode == "mean":
        s = s / lens[bag].to(dout.dtype)
    db = dout[bag]
    dpsw = None
    if ctx.needs_input_grad[1]:
        dtype, device = ctx.psw_like
        dpsw = (db * rows[inv].to(dout.dtype)).sum(1).to(dtype=dtype, device=device)
    if ctx.push_scale is not None and L:
        g = torch.zeros(uniq.numel(), dout.shape[1], dtype=dout.dtype).index_add_(0, inv, db * s[:, None])
        ctx.table.add_rows(uniq.numpy(), (g * ctx.push_scale).numpy(), ctx.option)
    return dpsw


# ------------------------------------------------------------------------------------------------ autograd
class _EmbeddingBagFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, psw, table, ids, offsets, mode, push_scale, option, frozen):
        ctx.table, ctx.mode, ctx.push_scale, ctx.option = table, mode, push_scale, option
        ctx.frozen = frozen
        ctx.anchor = None if anchor is None else (anchor.shape, anchor.dtype, anchor.device)
        ctx.psw_like = None if psw is None else (psw.dtype, psw.device)
        dev = _device_of(table)
        ctx.device = dev is not None
        if ctx.device:
            rm, _, dim = _rowmap_of(table, "embedding_bag")
            ids, offsets = ids.to(dev), offsets.to(dev)
            psw32 = None if psw is None else psw.detach().to(device=dev, dtype=torch.float32).contiguous()
            ctx.rm, ctx.dim = rm, dim
            out = _fwd_device(rm, dim, ids, offsets, psw32, mode)
            ctx.save_for_backward(ids, offsets, psw32)
            return out
        uniq, inv = torch.unique(ids.cpu(), return_inverse=True)
        rows = _host_rows(table, uniq)
        ctx.host = (uniq, inv, rows)
        offsets = offsets.cpu()
        p = None if psw is None else psw.detach().cpu().to(rows.dtype)
        ctx.save_for_backward(ids.cpu(), offsets, p)
        return F.embedding_bag(inv, rows, offsets, mode=mode, per_sample_weights=p)

    @staticmethod
    def backward(ctx, dout):
        ids, offsets, psw = ctx.saved_tensors
        dpsw = None
        if ctx.frozen and ctx.push_scale is not None:
            raise RuntimeError("PSEmbedding: backward after a forward that inserted no keys (eval mode): missing keys "
                               "share the zero row, which must not be pushed to; run the forward in training mode")
        if ctx.device:
            if ctx.needs_input_grad[1]:
                dpsw = _psw_grad_device(ctx.rm, ctx.dim, ids, offsets, ctx.mode, dout)
                dpsw = dpsw.to(dtype=ctx.psw_like[0], device=ctx.psw_like[1])
            if ctx.push_scale is not None:
                _push_device(ctx.table, ctx.rm, ctx.dim, ids, offsets, psw, ctx.mode, dout, float(ctx.push_scale),
                             ctx.option)
        else:
            dpsw = _host_backward(ctx, ids, offsets, psw, dout.cpu())
        da = None
        if ctx.anchor is not None:
            shape, dtype, device = ctx.anchor
            da = torch.zeros(shape, dtype=dtype, device=device)
        return da, dpsw, None, None, None, None, None, None, None


def _prepare(table, ids, offsets, per_sample_weights, mode, insert: bool = False, extra=None):
    """Checked (ids, offsets, weights) of a call; for a HashMatrixTable the ids are keys, translated to rows first
    (``insert``: missing keys get rows; otherwise they read the zero row). ``extra``: as in ``_check_values``."""
    if _dtype_of(table) != torch.float32:
        raise TypeError(f"embedding_bag: the table must be float32, got {_dtype_of(table)}")
    ids, offsets, psw = _bags(ids, offsets, per_sample_weights, mode)
    dev = _device_of(table)
    if dev is not None:
        rm, _, _ = _rowmap_of(table, "embedding_bag")
        if rm.num_col % 4 != 0:
            raise ValueError(f"embedding_bag: the table's row pitch ({rm.num_col} floats) must be a multiple of 4 "
                             "(16-byte row loads)")
        ids, offsets = ids.to(dev), offsets.to(dev)
    num_row = table.shape[0] if isinstance(table, torch.Tensor) else table.num_row
    if isinstance(table, HashMatrixTable):
        rows, status = torch.empty_like(ids), torch.empty(1, dtype=torch.int64, device=dev)
        table.lookup_call(ids, rows, status, insert)
        _check_values(rows, offsets, num_row, status, table, extra)
        return rows, offsets, psw
    _check_values(ids, offsets, num_row, extra=extra)
    return ids, offsets, psw


def embedding_bag(table, ids, offsets=None, per_sample_weights=None, mode: str = "sum") -> torch.Tensor:
    """Bags of table rows: ``[B, dim]``. ``table``: MatrixTable (device or host backend) or a 2-D fp32 tensor
    (a CUDA tensor may be a column slice of a wider pitch: only its columns are read), or a HashMatrixTable, whose
    ids are keys (a missing key adds zeros and is not inserted); ``ids``: int32 / int64,
    1-D with ``offsets`` or 2-D ``[B, n]``; ``per_sample_weights``: the shape of ``ids``, ``mode="sum"`` only.
    Differentiable in ``per_sample_weights``; nothing is pushed to the table (see :class:`PSEmbedding`)."""
    ids, offsets, psw = _prepare(table, ids, offsets, per_sample_weights, mode)
    if isinstance(table, torch.Tensor) and not table.is_cuda:
        return F.embedding_bag(ids, table, offsets, mode=mode, per_sample_weights=psw)
    return _EmbeddingBagFn.apply(None, psw, table, ids, offsets, mode, None, None, False)


class PSEmbedding(torch.nn.Module):
    """``torch.nn.EmbeddingBag`` whose weight is a MatrixTable: ``PSEmbedding(table, lr)`` with the ``sgd``
    updater (``-lr`` with ``default``) trains the table like ``EmbeddingBag(sparse=True)`` + SGD, the step being
    the table's updater, applied on the owners once per touched row. ``push_scale``: the coalesced gradient is
    multiplied by it before the push (``None``: do not push); ``option``: the AddOption of the push."""

    def __init__(self, table, push_scale: Optional[float] = 1.0, option: Optional[AddOption] = None,
                 mode: str = "sum"):
        super().__init__()
        if mode not in MODES:
            raise ValueError(f"PSEmbedding: mode must be one of {MODES}, got {mode!r}")
        if isinstance(table, torch.Tensor):
            raise TypeError("PSEmbedding: the weight must be a MatrixTable (a tensor has no updater to push to)")
        self.table, self.push_scale, self.option, self.mode = table, push_scale, option, mode
        self.num_embeddings, self.embedding_dim = table.num_row, table.num_col
        # ids never require grad: without an input that does, autograd would skip the backward and so the push
        self.anchor = torch.nn.Parameter(torch.zeros(0))

    def forward(self, ids, offsets=None, per_sample_weights=None) -> torch.Tensor:
        # over a HashMatrixTable the ids are keys: training inserts the missing ones, eval reads them as zeros
        frozen = isinstance(self.table, HashMatrixTable) and not self.training
        ids, offsets, psw = _prepare(self.table, ids, offsets, per_sample_weights, self.mode, insert=self.training)
        return _EmbeddingBagFn.apply(self.anchor, psw, self.table, ids, offsets, self.mode, self.push_scale,
                                     self.option, frozen)

    def extra_repr(self) -> str:
        return (f"{self.num_embeddings}, {self.embedding_dim}, mode={self.mode!r}, "
                f"weight=MatrixTable#{getattr(self.table, 'table_id', '?')}")
