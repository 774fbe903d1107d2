"""Sampled softmax over a MatrixTable: the output layer of a model whose classes are the rows of a large table.

A full softmax over a table of N rows builds ``[B, N]`` logits, and its gradient touches every row. Sampled softmax
scores each example against its true row and a shared set of S rows drawn from a sampler q, so only the S + B
touched rows are read and pushed::

    ssm = mv.ops.PSSampledSoftmax(table, num_sampled=8192, sampler="log_uniform", push_scale=lr)
    loss = ssm(hidden, labels)       # [B] per-example loss; hidden [B, d] float32, labels [B] int32 / int64
    loss.mean().backward()           # dL/dhidden goes to autograd, the row gradient to the table's updater
    ids = ssm.draw(step)             # the S candidate ids of the call with that step index (ssm.steps: calls so far)

With row ``j`` of the table ``w_j`` and S candidates ``c_1..c_S`` drawn with replacement from q per call:

* true logit ``t_b = x_b . w_{y_b} - log(S q(y_b))``;
* sampled logits ``s_bj = x_b . w_{c_j} - log(S q(c_j))``, ``-inf`` where ``c_j == y_b`` (an accidental hit);
* ``loss_b = logsumexp(t_b, s_b.) - t_b``.

The log Q correction and the removal of accidental hits are always on. There is no bias term: fold a bias into the
table as one more column and append a constant 1 to ``hidden``.

Samplers: ``sampler="log_uniform"``, the Zipfian ``q(k) = log((k + 2) / (k + 1)) / log(N + 1)`` for ids ranked by
frequency; or ``counts=`` with ``power``, ``q ~ counts^power`` (word2vec's unigram^0.75). Either is turned into one
alias table (``mvb_build_alias_table``, weights in fp64 on the host) with an fp32 ``log q`` per row next to it.
Draw j of the call with step index ``step`` hashes a key derived from ``(seed, step)`` with j, takes a slot from
the high 32 bits and ``u`` from the low 24 and picks the slot or its alias (the rule of the WordEmbedding negative
pool): the draws are the same on every rank, in every run and on both backends.

The row gradient of a call is coalesced over its labels and candidates, duplicates included, multiplied by
``push_scale`` and pushed once per unique row (``None``: no push): ``default`` / ``sgd`` tables that are not
``is_sparse`` get a ``red.add`` into the owners' rows, other tables the compact rows through ``add_rows_async``, so
momentum and AdaGrad take exactly one step per touched row. Reads follow ``get_rows``' rule: the caller orders a
call after the Adds it wants to see (barrier / ``flush``).

On the device (``csrc/cuda/sampled_softmax.cu``) a call is: the S draws, ``mvb_get_rows`` of the candidate and label
rows, ``logits = X W_S^T`` on the wgmma GEMM (TF32 operands, fp32 accumulation), and a warp-per-example epilogue
(fp32 true logit, corrections, mask, logsumexp). The backward turns the logits into ``E = g softmax`` and ``E^T``,
forms ``dX = E W_S + e_true w_y`` and ``dW_S = E^T X`` on the same GEMM, and pushes through the embedding-bag push
(``mvb_embedding_bag_bwd``). It holds ``[B, S_pad]`` and ``[S_pad, B_pad]`` fp32 buffers (S and B rounded up to
multiples of 4), about 512 MB at B = S = 8192. A batch holds at most ``MAX_BATCH`` = 2,097,120 examples; S has no
such limit. The forward reads the device once (the label checks); the backward does not synchronise with the host
for the fused push and reads the unique-row count once for a compact push. The backward overwrites the saved logits,
so a call's graph is backpropagated once: a second backward through a retained graph raises. An empty batch returns an empty loss and pushes nothing.

On the host backend the same call draws the same ids, reads ``get_rows`` of the unique rows, evaluates the formula
in torch fp32 with autograd for ``dL/dhidden`` and pushes the row gradients with one coalesced ``add_rows``.

The sampled loss is an estimate for training. ``ssm.evaluate(hidden, labels, k=0)`` is the exact full softmax over
every row of the table (:func:`~multiverso_b200.ops.full_softmax`): ``r.lse``, the cross-entropy ``r.loss`` (the
perplexity is ``exp(r.loss.mean())``) and, for ``k > 0``, the top-k classes by logit in ``r.scores`` / ``r.ids``. It
has no log-Q correction and no accidental-hit mask, draws nothing, leaves ``ssm.steps`` alone, pushes nothing, and
on the device never writes the ``[B, N]`` logits.
"""
from __future__ import annotations

import math
from typing import Optional

import numpy as np
import torch

from .. import _native as N
from ..tables.options import AddOption
from ..utils import monitor
from .embedding import _INT, _device_of, _dtype_of, _host_rows, _push_device
from .full_softmax import FullSoftmaxResult, full_softmax
from .get_gemm import gemm_nt
from .topk import _rowmap_of

SAMPLERS = ("log_uniform",)
_WHAT = "PSSampledSoftmax"
_M64 = (1 << 64) - 1
# The backward epilogue tiles the batch in 32-example rows of a grid whose y extent is at most 65535
# (mvb_ss_bwd_epilogue): larger batches are refused before the forward draws or runs anything.
MAX_BATCH = 65535 * 32


def _round4(n: int) -> int:
    return (n + 3) // 4 * 4


def _hash64(x):
    """hash64 of csrc/cuda/mvb_common.cuh on Python ints or numpy uint64 arrays (arithmetic mod 2^64)."""
    if isinstance(x, np.ndarray):
        with np.errstate(over="ignore"):
            x = x ^ (x >> np.uint64(33))
            x = x * np.uint64(0xFF51AFD7ED558CCD)
            x = x ^ (x >> np.uint64(33))
            x = x * np.uint64(0xC4CEB9FE1A85EC53)
            return x ^ (x >> np.uint64(33))
    x &= _M64
    x ^= x >> 33
    x = (x * 0xFF51AFD7ED558CCD) & _M64
    x ^= x >> 33
    x = (x * 0xC4CEB9FE1A85EC53) & _M64
    return x ^ (x >> 33)


def draw_reference(prob: np.ndarray, alias: np.ndarray, seed: int, step: int, num_sampled: int) -> np.ndarray:
    """The ``num_sampled`` ids of the call ``(seed, step)`` from an alias table, replayed on the host: bitwise the
    draws of ``mvb_ss_sample``. Returns int64 [num_sampled]."""
    key = _hash64(_hash64(seed & _M64) ^ (((step + 1) * 0xD6E8FEB86659FD93) & _M64))
    with np.errstate(over="ignore"):
        j1 = np.arange(1, num_sampled + 1, dtype=np.uint64)
        r = _hash64(np.uint64(key) ^ (j1 * np.uint64(0x9E3779B97F4A7C15)))
    idx = (r >> np.uint64(32)) % np.uint64(prob.size)
    u = (r & np.uint64(0xFFFFFF)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    idx = idx.astype(np.int64)
    return np.where(u < prob[idx], idx, alias[idx].astype(np.int64))


def _sampler_weights(num_row: int, sampler: Optional[str], counts, power: float) -> np.ndarray:
    """The unnormalised fp64 weights of q over the rows."""
    if (sampler is None) == (counts is None):
        raise ValueError(f"{_WHAT}: give exactly one of sampler={SAMPLERS[0]!r} and counts=")
    if sampler is not None:
        if sampler not in SAMPLERS:
            raise ValueError(f"{_WHAT}: sampler must be one of {SAMPLERS}, got {sampler!r}")
        return np.log1p(1.0 / (np.arange(num_row, dtype=np.float64) + 1.0)) / math.log(num_row + 1.0)
    if not (math.isfinite(power) and power > 0):
        # 0^0 = 1 would make zero-count rows drawable, a negative power would give them infinite weight
        raise ValueError(f"{_WHAT}: power must be finite and > 0, got {power}")
    c = np.asarray(torch.as_tensor(counts).detach().cpu().to(torch.float64).numpy()).reshape(-1)
    if c.size != num_row:
        raise ValueError(f"{_WHAT}: counts must have one entry per table row ({num_row}), got {c.size}")
    if not np.isfinite(c).all() or (c < 0).any():
        raise ValueError(f"{_WHAT}: counts must be finite and non-negative")
    if not (c > 0).any():
        raise ValueError(f"{_WHAT}: counts are all zero")
    w = np.power(c, float(power))
    if not np.isfinite(w).all():
        raise ValueError(f"{_WHAT}: counts ** power overflows fp64 (power={power})")
    return w


class PSSampledSoftmax(torch.nn.Module):
    """Sampled-softmax output layer whose class weights are the rows of a MatrixTable (see the module docstring).
    ``num_sampled``: S draws per call; ``sampler`` / ``counts``, ``power``: the sampler q (exactly one of the two);
    ``push_scale``: the row gradient is multiplied by it before the push (``None``: no push); ``option``: the
    AddOption of the push; ``seed``: the draws of the call with step index k depend only on (seed, k)."""

    def __init__(self, table, num_sampled: int = 8192, sampler: Optional[str] = None, counts=None,
                 power: float = 0.75, push_scale: Optional[float] = 1.0, option: Optional[AddOption] = None,
                 seed: int = 0):
        super().__init__()
        if isinstance(table, torch.Tensor):
            raise TypeError(f"{_WHAT}: the weight must be a MatrixTable (a tensor has no updater to push to)")
        if _dtype_of(table) != torch.float32:
            raise TypeError(f"{_WHAT}: the table must be float32, got {_dtype_of(table)}")
        n, d = int(table.num_row), int(table.num_col)
        if d % 4 != 0:
            raise ValueError(f"{_WHAT}: the table's row width ({d} floats) must be a multiple of 4 (16-byte TMA "
                             "row pitch)")
        if int(num_sampled) < 1:
            raise ValueError(f"{_WHAT}: num_sampled must be >= 1, got {num_sampled}")
        if n >= 1 << 31:
            raise ValueError(f"{_WHAT}: the table has {n} rows; the alias table holds int32 ids (< 2^31 rows)")
        w = _sampler_weights(n, sampler, counts, float(power))
        prob, alias = np.empty(n, np.float32), np.empty(n, np.int32)
        N.cuda_lib().mvb_build_alias_table(np.ascontiguousarray(w).ctypes.data, n, prob.ctypes.data,
                                           alias.ctypes.data)
        with np.errstate(divide="ignore"):
            logq = np.log(w / w.sum()).astype(np.float32)
        self.table, self.num_sampled, self.push_scale, self.option = table, int(num_sampled), push_scale, option
        self.sampler, self.power, self.seed = sampler or "counts", float(power), int(seed)
        self.steps = 0
        self.num_classes, self.in_features = n, d
        self._log_s = np.float32(math.log(self.num_sampled))
        self._prob, self._alias = prob, alias
        self._device = _device_of(table)
        if self._device is not None:
            self._rm = _rowmap_of(table, _WHAT)[0]
            if self._rm.num_col != d:
                raise ValueError(f"{_WHAT}: the table's row pitch ({self._rm.num_col}) must equal its width ({d})")
            self._dprob = torch.from_numpy(prob).to(self._device)
            self._dalias = torch.from_numpy(alias).to(self._device)
            self._logq = torch.from_numpy(logq).to(self._device)
        else:
            self._logq = torch.from_numpy(logq)
        # labels never require grad and hidden may not: the anchor makes autograd run the backward, and so the push
        self.anchor = torch.nn.Parameter(torch.zeros(0))

    # ------------------------------------------------------------------------------------------------ draws
    def _args(self, step: int) -> N.SampledSoftmax:
        a = N.SampledSoftmax()
        a.alias_prob, a.alias_idx, a.logq, a.n = self._dprob.data_ptr(), self._dalias.data_ptr(), \
            self._logq.data_ptr(), self.num_classes
        a.seed, a.step = self.seed & _M64, int(step) & _M64
        a.S, a.S_pad, a.log_s = self.num_sampled, _round4(self.num_sampled), float(self._log_s)
        return a

    def _sample_device(self, step: int):
        S = self.num_sampled
        cand = torch.empty(S, dtype=torch.int64, device=self._device)
        logq_c = torch.empty(S, dtype=torch.float32, device=self._device)
        a = self._args(step)
        a.cand, a.logq_c = cand.data_ptr(), logq_c.data_ptr()
        N.cuda_lib().mvb_ss_sample(a, N.stream_ptr())
        return a, cand, logq_c

    def draw(self, step: int) -> torch.Tensor:
        """The candidate ids [num_sampled] (int64) of the call with step index ``step``: on the table's device, or
        on the CPU for a host-backend table."""
        if self._device is None:
            return torch.from_numpy(draw_reference(self._prob, self._alias, self.seed, int(step), self.num_sampled))
        return self._sample_device(step)[1]

    # ------------------------------------------------------------------------------------------------ checks
    def _check(self, hidden, labels):
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
        if dev is not None and hidden.shape[0] > MAX_BATCH:
            raise ValueError(f"{_WHAT}: a batch holds at most {MAX_BATCH} examples on the GPU (the backward's "
                             f"epilogue grid), got {hidden.shape[0]}")
        y = labels.to(device=dev if dev is not None else "cpu", dtype=torch.int64).contiguous()
        if y.numel():                                     # one device read: range and zero-count labels
            lo, hi = torch.aminmax(y)
            zero = torch.isneginf(self._logq[y.clamp(0, self.num_classes - 1)]).any()
            lo, hi, zero = torch.stack([lo, hi, zero.to(torch.int64)]).tolist()
            if lo < 0 or hi >= self.num_classes:
                raise ValueError(f"{_WHAT}: labels must be in [0, {self.num_classes}), got min {lo} max {hi}")
            if zero:
                raise ValueError(f"{_WHAT}: a label has count zero under the sampler, so its log Q is -inf")
        return y

    # ------------------------------------------------------------------------------------------------ forward
    def forward(self, hidden: torch.Tensor, labels) -> torch.Tensor:
        y = self._check(hidden, labels)
        step = self.steps
        self.steps += 1
        if y.numel() == 0:
            # an empty batch: an empty loss, nothing drawn, read or pushed (the anchor keeps backward() valid)
            return hidden.sum(1) + self.anchor.sum().to(hidden.device)
        if self._device is None:
            return self._forward_host(hidden, y, step)
        return _SampledSoftmaxFn.apply(self.anchor, hidden, y, self, step)

    def _forward_host(self, hidden: torch.Tensor, y: torch.Tensor, step: int) -> torch.Tensor:
        cand = self.draw(step)
        uniq, inv = torch.unique(torch.cat([y, cand]), return_inverse=True)
        rows = _host_rows(self.table, uniq).to(torch.float32).requires_grad_()
        B = y.numel()
        w_y, w_c = rows[inv[:B]], rows[inv[B:]]
        x = hidden.cpu()
        log_s = torch.tensor(self._log_s)
        t = (x * w_y).sum(1) - (log_s + self._logq[y])
        s = x @ w_c.t() - (log_s + self._logq[cand])[None, :]
        s = s.masked_fill(cand[None, :] == y[:, None], float("-inf"))
        loss = torch.logsumexp(torch.cat([t[:, None], s], 1), 1) - t
        table, scale, option, done = self.table, self.push_scale, self.option, []

        def push(g):
            _once(done)
            if scale is not None:
                table.add_rows(uniq.numpy(), (g * float(scale)).numpy(), option)
        rows.register_hook(push)
        return loss.to(hidden.device)

    # ------------------------------------------------------------------------------------------------ evaluation
    def evaluate(self, hidden: torch.Tensor, labels, k: int = 0) -> FullSoftmaxResult:
        """The exact full softmax of ``hidden`` [B, in_features] over all ``num_classes`` rows: ``lse``, ``loss`` and,
        for ``k > 0``, the top-k classes (see :func:`~multiverso_b200.ops.full_softmax`). Evaluation only: nothing
        is drawn, ``steps`` does not advance and nothing is pushed."""
        h = torch.as_tensor(hidden)
        if h.dim() == 2 and h.shape[1] != self.in_features:
            raise ValueError(f"{_WHAT}: hidden has {h.shape[1]} columns, the table rows {self.in_features}")
        if self._device is not None and isinstance(h, torch.Tensor) and not h.is_cuda:
            raise ValueError(f"{_WHAT}: the table is on the GPU, hidden must be too")
        return full_softmax(self.table, h, labels, k)

    def extra_repr(self) -> str:
        src = f"counts^{self.power}" if self.sampler == "counts" else repr(self.sampler)
        return (f"{self.in_features}, {self.num_classes}, num_sampled={self.num_sampled}, sampler={src}, "
                f"weight=MatrixTable#{getattr(self.table, 'table_id', '?')}")


def _once(done: list) -> None:
    """A call's backward pushes its row gradient and, on the device, turns its saved logits into E in place: a
    second backward through a retained graph would push again from the wrong values, so it is refused."""
    if done:
        raise RuntimeError(f"{_WHAT}: backward ran twice through one call (retain_graph=True); the call's row "
                           "gradient has been pushed already. Run the forward again for another step")
    done.append(True)


class _SampledSoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, hidden, y, ssm, step):
        lib, st = N.cuda_lib(), N.stream_ptr()
        dev, rm = ssm._device, ssm._rm
        x = hidden.detach().contiguous()
        if x.data_ptr() % 16:
            x = x.clone()
        B, d = x.shape
        S, Sp = ssm.num_sampled, _round4(ssm.num_sampled)
        a, cand, logq_c = ssm._sample_device(step)
        w_s = torch.empty(Sp, d, dtype=torch.float32, device=dev)
        if Sp > S:
            w_s[S:].zero_()
        w_y = torch.empty(B, d, dtype=torch.float32, device=dev)
        logits = torch.empty(B, Sp, dtype=torch.float32, device=dev)
        loss, lse, t = (torch.empty(B, dtype=torch.float32, device=dev) for _ in range(3))
        with monitor("WORKER_TABLE_SAMPLED_SOFTMAX", cuda=True, nbytes=(S + B) * d * 4):
            lib.mvb_get_rows(N.F32, rm, cand, S, w_s, d, st)
            lib.mvb_get_rows(N.F32, rm, y, B, w_y, d, st)
            gemm_nt(x, w_s, logits)
            a.x, a.w_y, a.B, a.B_pad, a.d, a.labels = x.data_ptr(), w_y.data_ptr(), B, _round4(B), d, y.data_ptr()
            a.logits, a.loss, a.lse, a.t_true = logits.data_ptr(), loss.data_ptr(), lse.data_ptr(), t.data_ptr()
            lib.mvb_ss_fwd_epilogue(a, st)
        ctx.ssm, ctx.args, ctx.done = ssm, a, []
        ctx.save_for_backward(x, y, cand, logq_c, w_s, w_y, logits, lse, t)
        return loss

    @staticmethod
    def backward(ctx, g):
        _once(ctx.done)
        x, y, cand, logq_c, w_s, w_y, logits, lse, t = ctx.saved_tensors
        ssm, a = ctx.ssm, ctx.args
        lib, st, dev = N.cuda_lib(), N.stream_ptr(), x.device
        B, d = x.shape
        S, Sp, Bp = ssm.num_sampled, _round4(ssm.num_sampled), _round4(B)
        g = g.to(torch.float32).contiguous()
        e_t = torch.empty(Sp, Bp, dtype=torch.float32, device=dev)
        e_true = torch.empty(B, dtype=torch.float32, device=dev)
        # the pointers of the forward's tensors: saved, so still alive
        a.x, a.w_y, a.labels, a.logits, a.lse, a.t_true = x.data_ptr(), w_y.data_ptr(), y.data_ptr(), \
            logits.data_ptr(), lse.data_ptr(), t.data_ptr()
        a.cand, a.logq_c = cand.data_ptr(), logq_c.data_ptr()
        a.g, a.e_t, a.e_true = g.data_ptr(), e_t.data_ptr(), e_true.data_ptr()
        dx = None
        with monitor("WORKER_TABLE_SAMPLED_SOFTMAX_GRAD", cuda=True, nbytes=(S + B) * d * 4):
            lib.mvb_ss_bwd_epilogue(a, st)                   # logits -> E, and E^T
            if ctx.needs_input_grad[1]:
                w_st = torch.empty(d, Sp, dtype=torch.float32, device=dev)
                lib.mvb_transpose_pad_f32(w_s, Sp, d, d, w_st, Sp, st)
                dx = gemm_nt(logits, w_st, torch.empty(B, d, dtype=torch.float32, device=dev))
                dx.addcmul_(e_true[:, None], w_y)
            if ssm.push_scale is not None:
                dout = torch.empty(B + Sp, d, dtype=torch.float32, device=dev)     # [X; dW_S]
                dout[:B].copy_(x)
                x_t = torch.empty(d, Bp, dtype=torch.float32, device=dev)
                lib.mvb_transpose_pad_f32(x, B, d, d, x_t, Bp, st)
                gemm_nt(e_t, x_t, dout[B:])
                ids = torch.cat([y, cand])
                offsets = torch.arange(B + S, dtype=torch.int64, device=dev)
                psw = torch.cat([e_true, torch.ones(S, dtype=torch.float32, device=dev)])
                _push_device(ssm.table, ssm._rm, d, ids, offsets, psw, "sum", dout[:B + S],
                             float(ssm.push_scale), ssm.option)
        return torch.zeros_like(ssm.anchor), dx, None, None, None
