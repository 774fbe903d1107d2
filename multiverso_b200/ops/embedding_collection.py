"""Many sparse features over several MatrixTables in one fused lookup: the embedding-bag collection.

A sparse-feature model (CTR, DLRM-style) has tens of categorical features over tens of tables, and several
features often share one table (``item`` and ``history`` over the item table). :class:`PSEmbeddingCollection`
looks all of them up in one call::

    cfgs = [EmbeddingBagConfig(user_t, features=["user"], push_scale=lr),
            EmbeddingBagConfig(item_t, features=["item", "history"], push_scale=lr, mode="mean")]
    ebc = PSEmbeddingCollection(cfgs)
    out = ebc(ids, lengths)          # [B, sum of feature dims], features in config order
    parts = ebc.split(out)           # {"user": [B, d_user], "item": ..., "history": ...} (views)

The input is the jagged layout of a batch of sparse features: ``ids`` (1-D) holds feature 0's lookups for bags
0..B-1, then feature 1's, and so on; ``lengths`` (``[F, B]``) is the number of lookups of every bag. Pooling
``mode``, ``push_scale`` and the ``AddOption`` are per table (per config); each table keeps its own updater.

On the device (``csrc/cuda/emb_bag_coll.cu``) the forward is one warp per bag over all ``F * B`` bags, summed in
exactly the order of :func:`embedding_bag`, so each feature's columns are bitwise equal to ``embedding_bag`` over its
table; the kernel writes them straight into their columns of the output. The backward coalesces every table's
gradient over *all* of its features before the push, so a row that two features touch in one step gets exactly
one updater step with the summed gradient (what ``EmbeddingBag(sparse=True)`` plus an optimiser does). Two
separate :class:`PSEmbedding` calls would give it two steps, which for momentum and AdaGrad is not the same step.
The table descriptors live in a device array built here, once: MatrixTable shards do not move.

Host synchronisation: the input checks read the device once per forward, however many features there are. The
backward does not synchronise when every pushing table takes the fused ``red.add`` push (``default`` / ``sgd``,
not ``is_sparse``); otherwise it reads the unique-row counts of all compact tables in one copy.

A config may name a ``HashMatrixTable``: its features' ids are then int64 keys, translated to rows by one launch per
call that covers every hash feature (dense features' ids pass through unchanged), before the input checks and inside
their one host read. In training mode missing keys are inserted; in eval mode they add zeros and a backward raises.
Keys that a table with ``admit_after`` has not admitted yet add zeros in training mode too, and the backward pushes
nothing for them.

On the host backend the same module runs ``get_rows`` of the unique ids of each table over all of its features,
torch's ``embedding_bag`` per feature, and in the backward one coalesced ``add_rows`` per table: the same semantics.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from .. import _native as N
from ..tables.device import HashMatrixTable, raise_hash_status
from ..tables.options import AddOption
from ..utils import monitor
from .embedding import MODES, _INT, _device_of, _dtype_of, _host_rows, _push_rows
from .topk import _rowmap_of

MAX_DIM = 512
_WHAT = "PSEmbeddingCollection"


@dataclass(eq=False)
class EmbeddingBagConfig:
    """One table and the features looked up in it. ``push_scale``: the coalesced gradient is multiplied by it
    before the push (``None``: nothing is pushed; the only choice for a plain tensor table); ``option``: the
    AddOption of the push; ``mode``: ``"sum"`` or ``"mean"`` pooling."""
    table: object
    features: Sequence[str]
    push_scale: Optional[float] = 1.0
    option: Optional[AddOption] = None
    mode: str = "sum"


def _class_of(dim: int) -> int:
    """float4 vectors per lane of the kernels for a dim (1..4)."""
    nv = (dim + 3) // 4
    return 1 if nv <= 32 else (nv + 31) // 32


def _device_array(struct_array, dev) -> torch.Tensor:
    return torch.frombuffer(bytearray(struct_array), dtype=torch.uint8).to(dev)


class PSEmbeddingCollection(torch.nn.Module):
    """``EmbeddingBag`` layers for many features over MatrixTables, in one fused lookup. See the module docstring."""

    def __init__(self, configs: Sequence[EmbeddingBagConfig]):
        super().__init__()
        configs = list(configs)
        if not configs:
            raise ValueError(f"{_WHAT}: needs at least one EmbeddingBagConfig")
        seen_tables: Dict[int, int] = {}
        names: List[str] = []
        feat_table: List[int] = []
        for i, c in enumerate(configs):
            if not isinstance(c, EmbeddingBagConfig):
                raise TypeError(f"{_WHAT}: config {i} is a {type(c).__name__}, not an EmbeddingBagConfig")
            if c.mode not in MODES:
                raise ValueError(f"{_WHAT}: config {i}: mode must be one of {MODES}, got {c.mode!r}")
            if id(c.table) in seen_tables:
                j = seen_tables[id(c.table)]
                raise ValueError(f"{_WHAT}: configs {j} and {i} use the same table; list both features in one config "
                                 f"(features={list(configs[j].features) + list(c.features)}) so that the table's "
                                 "gradient is coalesced over them")
            seen_tables[id(c.table)] = i
            if isinstance(c.features, str) or not c.features:
                raise ValueError(f"{_WHAT}: config {i}: features must be a non-empty list of names")
            for name in c.features:
                if name in names:
                    raise ValueError(f"{_WHAT}: duplicate feature name {name!r}")
                names.append(name)
                feat_table.append(i)
            if _dtype_of(c.table) != torch.float32:
                raise TypeError(f"{_WHAT}: config {i}: the table must be float32, got {_dtype_of(c.table)}")
            if isinstance(c.table, torch.Tensor):
                if c.push_scale is not None:
                    raise TypeError(f"{_WHAT}: config {i}: a tensor table has no updater to push to; use a "
                                    "MatrixTable or push_scale=None")
                if c.table.dim() != 2:
                    raise ValueError(f"{_WHAT}: config {i}: a tensor table must be 2-D, got {tuple(c.table.shape)}")
        devs = {str(_device_of(c.table)) for c in configs}
        if len(devs) > 1:
            raise ValueError(f"{_WHAT}: every table must be on the same device or backend, got {sorted(devs)}")
        self.configs = configs
        self.feature_names = names
        self._feat_table = feat_table
        self._num_rows = [c.table.shape[0] if isinstance(c.table, torch.Tensor) else c.table.num_row for c in configs]
        self._table_dims = [c.table.shape[1] if isinstance(c.table, torch.Tensor) else c.table.num_col
                            for c in configs]
        self.dims = [self._table_dims[t] for t in feat_table]
        self.cols = [sum(self.dims[:f]) for f in range(len(names))]
        self.out_dim = sum(self.dims)
        self._device = _device_of(configs[0].table)
        # ids in range are checked against the table of each lookup's own feature
        self._rows_of_feature = torch.tensor([self._num_rows[t] for t in feat_table], dtype=torch.int64,
                                             device=self._device)
        self._hash = [c.table for c in configs if isinstance(c.table, HashMatrixTable)]
        if self._device is not None:
            self._build_device()
        if self._hash:
            # one translation launch covers every hash feature: the index descriptors of the hash tables, and per
            # feature the descriptor of its table (-1: a dense table, whose ids are copied unchanged)
            slot = {id(t): k for k, t in enumerate(self._hash)}
            descs = (N.HashRows * len(self._hash))(*[t._hash for t in self._hash])
            self._d_hash = _device_array(descs, self._device)
            self._seg_table = torch.tensor([slot.get(id(configs[t].table), -1) for t in feat_table],
                                           dtype=torch.int32, device=self._device)
        # ids never require grad: without an input that does, autograd would skip the backward and so the push
        self.anchor = torch.nn.Parameter(torch.zeros(0))

    # ------------------------------------------------------------------------------------------ descriptors
    def _build_device(self) -> None:
        dev, T, Fn = self._device, len(self.configs), len(self.feature_names)
        tabs = (N.EmbTable * T)()
        key_base = 0
        self._compact = []
        for t, c in enumerate(self.configs):
            rm, nrow, dim = _rowmap_of(c.table, _WHAT)
            if rm.num_col % 4 != 0:
                raise ValueError(f"{_WHAT}: config {t}: the table's row pitch ({rm.num_col} floats) must be a "
                                 "multiple of 4 (16-byte row loads)")
            if not 1 <= dim <= MAX_DIM:
                raise ValueError(f"{_WHAT}: config {t}: table dims must be in [1, {MAX_DIM}], got {dim}")
            d = tabs[t]
            d.wmap, d.dim, d.key_base, d.mean = rm, dim, key_base, int(c.mode == "mean")
            d.push_rows = _push_rows(c.table)
            key_base += nrow
            if c.push_scale is None:
                d.epilogue = N.EMB_NO_PUSH
            elif c.table.updater in (N.UPD_DEFAULT, N.UPD_SGD) and not c.table.is_sparse:
                d.epilogue = N.EMB_PUSH
                d.scale = (-1.0 if c.table.updater == N.UPD_SGD else 1.0) * float(c.push_scale)
            else:
                d.epilogue, d.scale, d.ldg = N.EMB_COMPACT, float(c.push_scale), c.table.num_col
                self._compact.append(t)
        # output columns of the kernels: every feature starts at a multiple of 4
        self._padded = any(d % 4 for d in self.dims)
        pcols, col = [], 0
        for d in self.dims:
            pcols.append(col)
            col += (d + 3) // 4 * 4
        self._ldo = col
        feats = (N.EmbFeature * Fn)()
        for f, t in enumerate(self._feat_table):
            feats[f].table, feats[f].col = t, pcols[f]
        order = sorted(range(Fn), key=lambda f: _class_of(self.dims[f]))
        self._class_off = [sum(1 for f in range(Fn) if _class_of(self.dims[f]) <= k) for k in range(5)]
        self._d_tables = _device_array(tabs, dev)
        self._d_features = _device_array(feats, dev)
        self._d_class = torch.tensor(order, dtype=torch.int32, device=dev)
        # output column j of the result is column _unpad[j] of the kernels' padded layout
        self._unpad = torch.cat([torch.arange(p, p + d) for p, d in zip(pcols, self.dims)]).to(dev)
        self._max_dim = max(self._table_dims)

    def _call(self, ids: torch.Tensor, offsets: torch.Tensor, B: int) -> N.EmbColl:
        a = N.EmbColl()
        a.tables, a.features, a.class_feats = (self._d_tables.data_ptr(), self._d_features.data_ptr(),
                                               self._d_class.data_ptr())
        for k in range(5):
            a.class_off[k] = self._class_off[k]
        a.T, a.F, a.B = len(self.configs), len(self.feature_names), B
        a.ids, a.L, a.offsets = ids.data_ptr(), ids.numel(), offsets.data_ptr()
        return a

    # ------------------------------------------------------------------------------------------ inputs
    def _inputs(self, ids, lengths, per_sample_weights):
        ids = torch.as_tensor(ids)
        if ids.dtype not in _INT:
            raise TypeError(f"{_WHAT}: ids must be int32 or int64, got {ids.dtype}")
        if ids.dim() != 1:
            raise ValueError(f"{_WHAT}: ids must be 1-D (feature-major jagged layout), got {tuple(ids.shape)}")
        lengths = torch.as_tensor(lengths)
        if lengths.dtype not in _INT:
            raise TypeError(f"{_WHAT}: lengths must be int32 or int64, got {lengths.dtype}")
        Fn = len(self.feature_names)
        if lengths.dim() != 2 or lengths.shape[0] != Fn:
            raise ValueError(f"{_WHAT}: lengths must be [F, B] with F = {Fn} features, got {tuple(lengths.shape)}")
        psw = per_sample_weights
        if psw is not None:
            if any(c.mode != "sum" for c in self.configs):
                raise ValueError(f"{_WHAT}: per_sample_weights need every table to pool with mode='sum'")
            psw = torch.as_tensor(psw)
            if psw.shape != ids.shape:
                raise ValueError(f"{_WHAT}: per_sample_weights must have the shape of ids {tuple(ids.shape)}, "
                                 f"got {tuple(psw.shape)}")
            if not psw.is_floating_point():
                raise TypeError(f"{_WHAT}: per_sample_weights must be floating point, got {psw.dtype}")
        dev = self._device if self._device is not None else torch.device("cpu")
        ids = ids.to(device=dev, dtype=torch.int64).contiguous()
        lengths = lengths.to(device=dev, dtype=torch.int64).contiguous()
        status = None
        if self._hash:
            ids, status = self._translate(ids, lengths)
        self._check_values(ids, lengths, status)
        flat = lengths.view(-1)
        offsets = torch.cumsum(flat, 0) - flat
        return ids, lengths, offsets, psw

    def _translate(self, ids: torch.Tensor, lengths: torch.Tensor):
        """The keys of the hash features as rows (training: missing keys get rows), the other ids unchanged: one
        launch. Returns (rows, status word of the translation). The feature of a lookup comes from the lengths,
        which are checked only afterwards: lengths that do not sum to len(ids) or hold a negative value would hand
        keys to the wrong table, so with those nothing is inserted (a device-side test, no host read) and the checks
        then raise."""
        rows = torch.empty_like(ids)
        status = torch.empty(1, dtype=torch.int64, device=ids.device)
        if ids.numel():
            seg_end = torch.cumsum(lengths.sum(1), 0)
            ok = None
            if self.training:
                ok = (seg_end[-1:] == ids.numel()).to(torch.int64)
                if lengths.numel():
                    ok &= (lengths.view(-1).min().view(1) >= 0).to(torch.int64)
            self._hash[0].lookup_call(ids, rows, status, self.training, seg_end, self._seg_table, self._d_hash,
                                      insert_ok=ok, hash_tables=self._hash)
        else:
            status.zero_()
        return rows, status

    def _check_values(self, ids: torch.Tensor, lengths: torch.Tensor, status: Optional[torch.Tensor] = None) -> None:
        """Non-negative lengths that sum to len(ids), and every id inside its own feature's table: one host read.
        ``status``: the status word of the hash translation, read in the same copy."""
        L, flat = ids.numel(), lengths.view(-1)
        zero = torch.zeros(1, dtype=torch.int64, device=ids.device)
        parts = [flat.sum().view(1), flat.min().view(1) if flat.numel() else zero]
        if L:
            ends = torch.cumsum(lengths.sum(1), 0)
            feat = torch.searchsorted(ends, torch.arange(L, device=ids.device), right=True)
            feat.clamp_(max=len(self.feature_names) - 1)
            bad = (ids < 0) | (ids >= self._rows_of_feature[feat])
            first = bad.to(torch.int32).argmax().view(1)
            parts += [bad.any().view(1).to(torch.int64), feat.index_select(0, first), ids.index_select(0, first)]
        if status is not None:
            parts.append(status)
        v = torch.cat(parts).tolist()
        if status is not None:
            raise_hash_status(v.pop(), self._hash)
        if v[1] < 0:
            raise ValueError(f"{_WHAT}: lengths must be non-negative, got {v[1]}")
        if v[0] != L:
            raise ValueError(f"{_WHAT}: lengths sum to {v[0]} but ids has {L} entries")
        if L and v[2]:
            f = v[3]
            raise ValueError(f"{_WHAT}: ids of feature {self.feature_names[f]!r} must be in [0, "
                             f"{self._num_rows[self._feat_table[f]]}) (its table's rows), got {v[4]}")

    # ------------------------------------------------------------------------------------------ public
    def forward(self, ids, lengths, per_sample_weights=None) -> torch.Tensor:
        """``ids`` 1-D int32 / int64, feature-major; ``lengths`` ``[F, B]``; ``per_sample_weights`` the shape of
        ``ids`` (every table ``mode="sum"``), differentiable. Returns ``[B, sum of feature dims]``."""
        ids, lengths, offsets, psw = self._inputs(ids, lengths, per_sample_weights)
        # a hash table looked up in eval mode inserted nothing: its missing keys share the zero row, never pushed to
        frozen = not self.training and any(isinstance(c.table, HashMatrixTable) and c.push_scale is not None
                                           for c in self.configs)
        return _CollectionFn.apply(self.anchor, psw, self, ids, lengths, offsets, frozen)

    def split(self, out: torch.Tensor) -> Dict[str, torch.Tensor]:
        """The output of :meth:`forward` as ``{feature: [B, dim]}`` column views."""
        if out.dim() != 2 or out.shape[1] != self.out_dim:
            raise ValueError(f"{_WHAT}.split: expected [B, {self.out_dim}], got {tuple(out.shape)}")
        return {n: out[:, c:c + d] for n, c, d in zip(self.feature_names, self.cols, self.dims)}

    def extra_repr(self) -> str:
        return ", ".join(f"{n}: {d}" for n, d in zip(self.feature_names, self.dims)) + f", tables={len(self.configs)}"

    # ------------------------------------------------------------------------------------------ device
    def _fwd_device(self, ids, offsets, psw, B) -> torch.Tensor:
        out = torch.empty(B, self._ldo, dtype=torch.float32, device=ids.device)
        a = self._call(ids, offsets, B)
        a.psw, a.out, a.ldo = N.ptr(psw), out.data_ptr(), self._ldo
        with monitor("WORKER_TABLE_EMBEDDING_BAG_COLLECTION", cuda=True):
            N.cuda_lib().mvb_emb_coll_fwd(a, N.stream_ptr())
        return out[:, self._unpad] if self._padded else out

    def _dout_device(self, dout: torch.Tensor) -> torch.Tensor:
        """dout in the kernels' column layout, 16-byte aligned (copied only when it is not already)."""
        dout = dout.to(torch.float32)
        if not self._padded:
            dout = dout.contiguous()
            if dout.data_ptr() % 16 == 0:
                return dout
        pad = torch.zeros(dout.shape[0], self._ldo, dtype=torch.float32, device=dout.device)
        return pad.index_copy_(1, self._unpad, dout)

    def _psw_grad_device(self, ids, offsets, d, B) -> torch.Tensor:
        dpsw = torch.empty(ids.numel(), dtype=torch.float32, device=ids.device)
        a = self._call(ids, offsets, B)
        a.dout, a.ldd, a.dpsw = d.data_ptr(), self._ldo, dpsw.data_ptr()
        N.cuda_lib().mvb_emb_coll_psw_grad(a, N.stream_ptr())
        return dpsw

    def _push_device(self, ids, offsets, psw, d, B) -> None:
        L, T = ids.numel(), len(self.configs)
        if L == 0 or all(c.push_scale is None for c in self.configs):
            return
        lib, st, dev = N.cuda_lib(), N.stream_ptr(), ids.device
        nbytes = lib.mvb_emb_coll_scratch_bytes(L, T, self._max_dim)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        keys = torch.empty(L, dtype=torch.int64, device=dev)
        info = torch.empty(4 * T + 2, dtype=torch.int64, device=dev)
        a = self._call(ids, offsets, B)
        a.psw, a.dout, a.ldd = N.ptr(psw), d.data_ptr(), self._ldo
        a.keys, a.info, a.scratch, a.scratch_bytes = keys.data_ptr(), info.data_ptr(), scratch.data_ptr(), nbytes
        with monitor("WORKER_TABLE_EMBEDDING_BAG_COLLECTION_GRAD", cuda=True):
            lib.mvb_emb_coll_keys(a, st)
            skeys, perm = torch.sort(keys, stable=True)    # per table segment, (id, position) order
            a.skeys, a.perm = skeys.data_ptr(), perm.data_ptr()
            lib.mvb_emb_coll_count(a, st)
            if self._compact:
                inf = info.tolist()                         # the unique counts of every compact table: one read
                exact = all(self._table_dims[t] == self.configs[t].table.num_col for t in self._compact)
                grads = (torch.empty if exact else torch.zeros)(inf[4 * T], dtype=torch.float32, device=dev)
                uniq = torch.empty(inf[4 * T + 1], dtype=torch.int64, device=dev)
                a.grads, a.uniq = grads.data_ptr(), uniq.data_ptr()
            lib.mvb_emb_coll_bwd(a, st)
        for t in self._compact:
            U, _, go, uo = inf[4 * t:4 * t + 4]
            if U:
                c = self.configs[t]
                ncol = c.table.num_col
                c.table.add_rows_async(uniq[uo:uo + U], grads[go:go + U * ncol].view(U, ncol), c.option)

    # ------------------------------------------------------------------------------------------ host
    def _feature_span(self, offsets_list, L, B, f):
        lo = offsets_list[f * B] if B else 0
        hi = offsets_list[(f + 1) * B] if f + 1 < len(self.feature_names) and B else L
        return lo, hi

    def _fwd_host(self, ctx, ids, offsets, psw, B) -> torch.Tensor:
        if B == 0:
            ctx.host = None
            return torch.zeros(0, self.out_dim)
        L, off = ids.numel(), offsets.tolist()
        spans = [self._feature_span(off, L, B, f) for f in range(len(self.feature_names))]
        tables = []
        for t, c in enumerate(self.configs):
            fs = [f for f, tt in enumerate(self._feat_table) if tt == t]
            uniq, inv = torch.unique(torch.cat([ids[slice(*spans[f])] for f in fs]), return_inverse=True)
            tables.append((fs, uniq, inv, _host_rows(c.table, uniq)))
        outs = [None] * len(self.feature_names)
        views = [None] * len(self.feature_names)
        for t, (fs, uniq, inv, rows) in enumerate(tables):
            at = 0
            for f in fs:
                lo, hi = spans[f]
                inv_f = inv[at:at + hi - lo]
                at += hi - lo
                off_f = offsets[f * B:(f + 1) * B] - lo
                p = None if psw is None else psw[lo:hi].to(rows.dtype)
                outs[f] = F.embedding_bag(inv_f, rows, off_f, mode=self.configs[t].mode, per_sample_weights=p)
                views[f] = (inv_f, off_f, lo, hi)
        ctx.host = (tables, views)
        return torch.cat(outs, 1)

    def _bwd_host(self, ctx, psw, dout, need_dpsw):
        dpsw = torch.zeros(psw.numel() if psw is not None else 0, dtype=dout.dtype)
        if ctx.host is None:
            return dpsw
        tables, views = ctx.host
        B = dout.shape[0]
        for t, (fs, uniq, inv, rows) in enumerate(tables):
            c = self.configs[t]
            g = torch.zeros(uniq.numel(), self._table_dims[t], dtype=dout.dtype)
            for f in fs:
                inv_f, off_f, lo, hi = views[f]
                n = hi - lo
                lens = torch.diff(off_f, append=torch.tensor([n], dtype=off_f.dtype))
                bag = torch.repeat_interleave(torch.arange(B), lens)
                s = psw[lo:hi].detach().to(dout.dtype) if psw is not None else torch.ones(n, dtype=dout.dtype)
                if c.mode == "mean":
                    s = s / lens[bag].to(dout.dtype)
                db = dout[:, self.cols[f]:self.cols[f] + self.dims[f]][bag]
                if need_dpsw:
                    dpsw[lo:hi] = (db * rows[inv_f].to(dout.dtype)).sum(1)
                g.index_add_(0, inv_f, db * s[:, None])
            if c.push_scale is not None and uniq.numel():
                c.table.add_rows(uniq.numpy(), (g * c.push_scale).numpy(), c.option)
        return dpsw


class _CollectionFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, psw, coll, ids, lengths, offsets, frozen):
        ctx.coll, ctx.frozen = coll, frozen
        ctx.anchor = (anchor.shape, anchor.dtype, anchor.device)
        ctx.psw_like = None if psw is None else (psw.dtype, psw.device)
        B = lengths.shape[1]
        ctx.B = B
        if coll._device is not None:
            psw32 = None if psw is None else psw.detach().to(device=ids.device, dtype=torch.float32).contiguous()
            ctx.save_for_backward(ids, offsets, psw32)
            return coll._fwd_device(ids, offsets, psw32, B)
        p = None if psw is None else psw.detach().cpu().to(torch.float32)
        ctx.save_for_backward(ids, offsets, p)
        return coll._fwd_host(ctx, ids, offsets, p, B)

    @staticmethod
    def backward(ctx, dout):
        ids, offsets, psw = ctx.saved_tensors
        coll, need_dpsw, dpsw = ctx.coll, ctx.needs_input_grad[1], None
        if ctx.frozen:
            raise RuntimeError(f"{_WHAT}: backward after an eval-mode forward over a HashMatrixTable: it inserted no "
                               "keys, and the missing ones share the zero row, which must not be pushed to")
        if coll._device is not None:
            d = coll._dout_device(dout)
            if need_dpsw:
                dpsw = coll._psw_grad_device(ids, offsets, d, ctx.B)
            coll._push_device(ids, offsets, psw, d, ctx.B)
        else:
            dpsw = coll._bwd_host(ctx, psw, dout.cpu(), need_dpsw)
        if dpsw is not None and need_dpsw:
            dpsw = dpsw.to(dtype=ctx.psw_like[0], device=ctx.psw_like[1])
        else:
            dpsw = None
        shape, dtype, device = ctx.anchor
        return torch.zeros(shape, dtype=dtype, device=device), dpsw, None, None, None, None, None
