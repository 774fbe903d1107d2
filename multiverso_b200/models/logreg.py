"""LogisticRegression (reference application: Applications/LogisticRegression, SURVEY A5-A8).

Objectives linear / sigmoid / softmax / FTRL, regularisers none / L1 / L2, dense or sparse
input, local model or parameter-server model (``use_ps``), blocking or pipelined (double
buffered GetAsync) pulls every ``sync_frequency`` minibatches -- the structure of Model /
PSModel / Objective / Regular / Updater (src/model/*.cpp, objective/objective.cpp,
regular/regular.cpp, updater/updater.cpp) -- with the hot loops on the GPU:

* K8 ``mvb_lr_sparse_fwd_bwd`` / ``mvb_lr_dense_fwd_bwd``: logits, sigma/softmax, loss,
  accuracy and the minibatch-averaged gradient,
* ``mvb_regularize``, ``mvb_ftrl_weights`` / ``mvb_ftrl_update``,
* the weights live in an ArrayTable (HBM shards); PSModel forces the server updater to
  ``sgd`` (w -= delta, ps_model.cpp:12-20); the AdaGrad server updater of BASELINE config 4
  is ``updater_type=adagrad`` (fused into the Add kernel).
"""
from __future__ import annotations

import os
from dataclasses import dataclass, field
from typing import Dict, Optional

import torch

from .. import _native as N
from ..ops.get_gemm import gemm_nt
from ..runtime import Runtime
from ..tables.device import ArrayDeviceTable
from ..tables.options import AddOption
from ..utils import Log

OBJECTIVES = {"default": 0, "linear": 0, "sigmoid": 1, "softmax": 2, "ftrl": 1}
REGULARS = {"default": 0, "none": 0, "L1": 1, "l1": 1, "L2": 2, "l2": 2}


@dataclass
class LogRegConfig:
    """The 26 configuration keys of the reference (src/configure.h:19-97) and their defaults."""
    input_size: int = 0
    output_size: int = 1
    sparse: bool = False
    train_epoch: int = 1
    minibatch_size: int = 20
    read_buffer_size: int = 2048
    regular_coef: float = 0.0005
    learning_rate: float = 0.8
    learning_rate_coef: float = 1e6
    alpha: float = 0.005
    beta: float = 1.0
    lambda1: float = 15.0
    lambda2: float = 0.0
    init_model_file: str = ""
    train_file: str = ""
    reader_type: str = "default"
    test_file: str = ""
    output_model_file: str = "logreg.model"
    output_file: str = "logreg.output"
    use_ps: bool = False
    pipeline: bool = True
    sync_frequency: int = 1
    updater_type: str = "default"
    objective_type: str = "default"
    regular_type: str = "default"
    show_time_per_sample: int = 10000
    server_updater: str = "sgd"         # addition: sgd | adagrad | momentum_sgd (server side)
    extra: Dict[str, str] = field(default_factory=dict)

    @classmethod
    def from_file(cls, path: str) -> "LogRegConfig":
        """key=value lines (src/configure.cpp:32-82); '#' starts a comment."""
        cfg = cls()
        with open(path) as f:
            for line in f:
                line = line.split("#", 1)[0].strip()
                if not line or "=" not in line:
                    continue
                k, v = [x.strip() for x in line.split("=", 1)]
                cfg.set(k, v)
        return cfg

    def set(self, key: str, value: str) -> None:
        if not hasattr(self, key) or key == "extra":
            self.extra[key] = value
            return
        cur = getattr(self, key)
        if isinstance(cur, bool):
            setattr(self, key, value.strip().lower() in ("1", "true", "yes"))
        elif isinstance(cur, int):
            setattr(self, key, int(float(value)))
        elif isinstance(cur, float):
            setattr(self, key, float(value))
        else:
            setattr(self, key, value)


# Dense problems whose forward / backward are real GEMMs (many classes or wide inputs) go through
# the library GEMM -- cuBLAS on the tensor cores -- instead of the CUDA-core K8 kernel, which is
# written for the reference's shapes (MNIST: 785 x 10) and holds at most 64 classes per sample.
GEMM_PATH_MIN_CLASSES = 65
GEMM_PATH_MIN_WORK = 1 << 26          # n * dim * out multiply-adds per minibatch


def dense_gemm_step(x: torch.Tensor, labels: torch.Tensor, w: torch.Tensor, grad: Optional[torch.Tensor],
                    objective: int, out: int):
    """One dense minibatch as two GEMMs: logits = X W^T, then (if ``grad`` is given)
    grad += (P - Y)^T X / n.  Same maths as K8 / Objective::Predict + Gradient
    (objective.cpp:64-233): objective 0 linear (squared loss), 1 sigmoid, 2 softmax.
    Returns (loss_sum, n_correct, predictions[n x out]).  Pure torch: runs on any device."""
    n, dim = x.shape
    W = w.view(out, dim)
    logits = x @ W.t()
    if out == 1:
        target = labels.view(n, 1).to(logits.dtype)
    else:
        target = torch.zeros_like(logits)
        target.scatter_(1, labels.view(n, 1).to(torch.int64), 1.0)
    if objective == 2 and out > 1:
        p = torch.softmax(logits, dim=1)
        loss = -torch.log(p.gather(1, labels.view(n, 1).to(torch.int64)).clamp_min(1e-30)).sum()
    elif objective >= 1:
        p = torch.sigmoid(logits)
        loss = -(target * torch.log(p.clamp_min(1e-30)) + (1 - target) * torch.log((1 - p).clamp_min(1e-30))).sum()
    else:
        p = logits
        loss = 0.5 * ((p - target) ** 2).sum()
    if out > 1:
        correct = (p.argmax(dim=1) == labels.to(torch.int64)).sum()
    elif objective >= 1:
        correct = ((p.view(-1) > 0.5) == (labels > 0.5)).sum()
    else:
        correct = ((p.view(-1) - labels).abs() < 0.5).sum()
    if grad is not None:
        grad.view(out, dim).addmm_((p - target).t(), x, alpha=1.0 / n)
    return loss, correct, p


class LogRegModel:
    """Model (local) / PSModel (``use_ps``) on the device backend."""

    def __init__(self, cfg: LogRegConfig):
        rt = Runtime.get()
        if rt.backend != "device":
            Log.fatal("LogRegModel needs the device backend (CUDA)")
        self.rt, self.cfg, self.dev = rt, cfg, rt.device
        self.dim = int(cfg.input_size) + 1                   # bias column (input_size += 1)
        self.out = max(1, int(cfg.output_size))
        self.objective = OBJECTIVES.get(cfg.objective_type, 0)
        if cfg.objective_type == "softmax" and self.out == 1:
            self.objective = 1
        self.ftrl = cfg.objective_type == "ftrl" or cfg.updater_type == "ftrl"
        self.regular = REGULARS.get(cfg.regular_type, 0)
        self.n_w = self.dim * self.out
        self.w = torch.zeros(self.n_w, device=self.dev)
        self.grad = torch.zeros(self.n_w, device=self.dev)
        self.loss = torch.zeros(1, device=self.dev)
        self.correct = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self._err = torch.empty(0, device=self.dev)
        self.updates = 0
        self.samples_seen = 0
        self.kernel_launches = 0
        self.lr = float(cfg.learning_rate)
        self.table = None
        self._w_next = None
        self._pending = None
        if self.ftrl:
            self.z = torch.zeros(self.n_w, device=self.dev)
            self.nacc = torch.zeros(self.n_w, device=self.dev)
        if cfg.use_ps:
            # PSModel: server does w -= delta (sgd) unless a stateful server updater is chosen
            upd = cfg.server_updater if cfg.server_updater in N.UPDATER_NAMES else "sgd"
            self.table = ArrayDeviceTable(self.n_w, "float32", updater=upd)
            if self.ftrl:
                self.table_n = ArrayDeviceTable(self.n_w, "float32", updater="sgd")
            self._w_next = torch.zeros(self.n_w, device=self.dev)
            self.pull(blocking=True)

    # ------------------------------------------------------------------ PS plumbing
    def pull(self, blocking: bool = True) -> None:
        """PullModel / GetPipelineTable (ps_model.cpp:205-271)."""
        if self.table is None:
            return
        if self.ftrl:
            self.table.get(self.z)
            self.table_n.get(self.nacc)
            return
        if blocking or not self.cfg.pipeline:
            self.table.get(self.w)
            return
        if self._pending is not None:                  # swap in the buffer requested last time
            self.table.wait(self._pending)
            self.w, self._w_next = self._w_next, self.w
        self._pending, _ = self.table.get_async(self._w_next)

    def _push(self, delta: torch.Tensor) -> None:
        """UpdateTable (ps_model.cpp:184-203): AddAsync of the lr-scaled averaged gradient."""
        opt = AddOption(learning_rate=max(self.lr, 1e-12), rho=self.cfg.alpha if self.cfg.server_updater == "adagrad" else 0.1)
        self.table.add_async(delta, opt)

    # ------------------------------------------------------------------ one minibatch
    def _ensure_err(self, n: int) -> None:
        if self._err.numel() < n * self.out:
            self._err = torch.empty(n * self.out, device=self.dev)

    def _weights(self) -> torch.Tensor:
        if self.ftrl:
            c = self.cfg
            N.cuda_lib().mvb_ftrl_weights(self.z, self.nacc, self.w, self.n_w, c.alpha, c.beta, c.lambda1, c.lambda2,
                                          N.stream_ptr())
            self.kernel_launches += 1
        return self.w

    def forward_backward_sparse(self, row_ptr, keys, vals, labels, weights=None, train=True, pred=None):
        n = labels.numel()
        self._ensure_err(n)
        a = N.LrSparse()
        a.row_ptr, a.keys, a.vals = row_ptr.data_ptr(), keys.data_ptr(), N.ptr(vals)
        a.labels, a.sample_w, a.n = labels.data_ptr(), N.ptr(weights), n
        a.objective, a.w, a.dim, a.out = self.objective, self._weights().data_ptr(), self.dim, self.out
        a.grad, a.loss_sum, a.correct = self.grad.data_ptr(), self.loss.data_ptr(), self.correct.data_ptr()
        a.pred, a.err, a.compute_grad = N.ptr(pred), self._err.data_ptr(), int(train)
        N.cuda_lib().mvb_lr_sparse_fwd_bwd(a, N.stream_ptr())
        self.kernel_launches += 1

    def forward_backward_dense(self, x, labels, train=True, pred=None):
        n = labels.numel()
        wide = self.out >= GEMM_PATH_MIN_CLASSES or n * self.dim * self.out >= GEMM_PATH_MIN_WORK
        if wide and self.dim % 4 == 0 and x.is_cuda and os.environ.get("MVB_LR_TC", "1") != "0":
            # GEMM-shaped minibatch: logits = X W^T and grad += E^T X both on the wgmma kernel (TF32 in,
            # fp32 accumulate), softmax / loss / error in the hand-written epilogue between them; no
            # library GEMM anywhere (Objective::Predict + Gradient, objective.cpp:113-120, 202-218)
            lib, st = N.cuda_lib(), N.stream_ptr()
            dev = x.device
            x2 = x.view(n, self.dim)
            n_pad = (n + 3) // 4 * 4
            logits = torch.empty(n, self.out, device=dev)
            gemm_nt(x2, self._weights().view(self.out, self.dim), logits)
            err_t = torch.empty(self.out, n_pad, device=dev)
            lib.mvb_lr_wide_epilogue(logits, labels, n, self.out, self.objective, err_t, n_pad, pred, self.loss,
                                     self.correct, st)
            self.kernel_launches += 2
            if train:
                x_t = torch.empty(self.dim, n_pad, device=dev)
                lib.mvb_transpose_pad_f32(x2, n, self.dim, self.dim, x_t, n_pad, st)
                dw = torch.empty(self.out, self.dim, device=dev)
                gemm_nt(err_t, x_t, dw)                      # [out x n] . [dim x n]^T
                lib.mvb_axpy_f32(self.grad, dw, self.out * self.dim, 1.0, st)
                self.kernel_launches += 3
            return
        if wide:
            loss, correct, p = dense_gemm_step(x.view(n, self.dim), labels, self._weights(),
                                               self.grad if train else None, self.objective, self.out)
            self.loss += loss
            self.correct += correct.to(torch.int32)
            if pred is not None:
                pred.view(n, self.out).copy_(p)
            self.kernel_launches += 2 if train else 1      # library GEMMs, counted like launches
            return
        self._ensure_err(n)
        a = N.LrDense()
        a.x, a.labels, a.n, a.dim, a.out = x.data_ptr(), labels.data_ptr(), n, self.dim, self.out
        a.objective, a.w = self.objective, self._weights().data_ptr()
        a.grad, a.loss_sum, a.correct = self.grad.data_ptr(), self.loss.data_ptr(), self.correct.data_ptr()
        a.pred, a.err, a.compute_grad = N.ptr(pred), self._err.data_ptr(), int(train)
        N.cuda_lib().mvb_lr_dense_fwd_bwd(a, N.stream_ptr())
        self.kernel_launches += 2 if train else 1

    def apply_gradient(self, n_samples: int) -> None:
        """Regularise, scale by the learning rate and update (local) or push (PS); then the
        SGD learning-rate schedule lr = max(1e-3, lr0 - t/(coef*minibatch)) (updater.cpp:44-71)."""
        cfg, lib, st = self.cfg, N.cuda_lib(), N.stream_ptr()
        if self.regular and not self.ftrl:
            lib.mvb_regularize(self.grad, self.w, self.n_w, self.regular, cfg.regular_coef, st)
            self.kernel_launches += 1
        if self.ftrl:
            if self.table is None:
                lib.mvb_ftrl_update(self.z, self.nacc, self.w, self.grad, self.n_w, cfg.alpha, st)
                self.kernel_launches += 1
            else:
                # FTRLObjective emits (dz, dn); the server subtracts, so the kernel emits the negatives
                if getattr(self, "_dz", None) is None:
                    self._dz, self._dn = torch.empty_like(self.grad), torch.empty_like(self.grad)
                lib.mvb_ftrl_delta(self.nacc, self.w, self.grad, self._dz, self._dn, self.n_w, cfg.alpha, st)
                self.kernel_launches += 1
                self.table.add_async(self._dz)
                self.table_n.add_async(self._dn)
        else:
            scaled = self.grad * self.lr if cfg.updater_type in ("sgd", "default") else self.grad
            if self.table is None:
                self.w.sub_(scaled)
            else:
                self._push(scaled)
        self.grad.zero_()
        self.updates += 1
        self.samples_seen += n_samples
        if cfg.updater_type == "sgd":
            self.lr = max(1e-3, cfg.learning_rate - self.updates / (cfg.learning_rate_coef * max(1, cfg.minibatch_size)))
        if self.table is not None and self.updates % max(1, cfg.sync_frequency) == 0:
            self.pull(blocking=not cfg.pipeline)

    # ------------------------------------------------------------------ model IO
    def save(self, path: str) -> None:
        """Model::Store (model.cpp:177-205): rank 0 pulls the whole model and writes it."""
        if self.table is not None:
            self.rt.barrier()
            self.pull(blocking=True)
        if self.rt.rank == 0:
            w = self._weights().cpu().numpy()
            with open(path, "wb") as f:
                f.write(w.astype("float32").tobytes())

    def load(self, path: str) -> None:
        """Model::Load / PSModel::Load (ps_model.cpp:115-154): worker 0 pushes the file through
        the PS negated, because the server subtracts."""
        import numpy as np
        w = torch.from_numpy(np.fromfile(path, dtype=np.float32).copy()).to(self.dev)
        assert w.numel() == self.n_w
        if self.table is None:
            self.w.copy_(w)
            return
        cur = self.table.get()
        delta = -(w - cur) if self.rt.worker_id() == 0 else torch.zeros_like(w)
        if self.table.updater_name != "sgd":
            delta = -delta
        self.table.add(delta)
        self.rt.barrier()
        self.pull(blocking=True)
