"""Table options and per-request options.

Reference: AddOption / GetOption (include/multiverso/updater/updater.h:10-110) and the
``*TableOption`` structs bound to worker/server types by DEFINE_TABLE_TYPE
(include/multiverso/table_interface.h:77-80, table/array_table.h:66-73,
table/matrix_table.h:116-127, table/matrix.h:14-22, table/kv_table.h:120-124).
"""
from __future__ import annotations

import math
import struct
from dataclasses import dataclass
from typing import Optional


class AddOption:
    """{worker_id, momentum, learning_rate, rho, lambda}; defaults {MV_WorkerId(), 0, .01, .1, .1}.

    Field order follows the reference *accessors* (SURVEY Q3), 20-byte wire layout kept."""

    __slots__ = ("worker_id", "momentum", "learning_rate", "rho", "lambda_")

    def __init__(self, worker_id: Optional[int] = None, momentum: float = 0.0,
                 learning_rate: float = 0.01, rho: float = 0.1, lambda_: float = 0.1):
        if worker_id is None:
            from ..runtime import Runtime
            rt = Runtime.get()
            worker_id = rt.worker_id() if rt.started else 0
        self.worker_id = int(worker_id)
        self.momentum = float(momentum)
        self.learning_rate = float(learning_rate)
        self.rho = float(rho)
        self.lambda_ = float(lambda_)

    def pack(self) -> bytes:
        return struct.pack("<iffff", self.worker_id, self.momentum, self.learning_rate, self.rho,
                           self.lambda_)

    @classmethod
    def unpack(cls, data: bytes) -> "AddOption":
        w, m, lr, rho, lam = struct.unpack("<iffff", data[:20])
        return cls(w, m, lr, rho, lam)

    def __repr__(self):
        return (f"AddOption {self.worker_id} {self.momentum} {self.learning_rate} {self.rho} "
                f"{self.lambda_}")


def _f32(x: float) -> float:
    return struct.unpack("<f", struct.pack("<f", x))[0]


def check_add_option(updater: str, opt: AddOption) -> None:
    """Raises ValueError for an AddOption the updater cannot step with, as the fp32 values it travels as: adam needs
    beta1 (``momentum``) in [0, 1), ``learning_rate > 0`` (it recovers the gradient as delta / learning_rate) and
    ``rho >= 0`` (the step size). ftrl needs finite ``learning_rate > 0``, ``rho > 0`` (alpha), ``lambda_ >= 0``
    (lambda1) and ``momentum >= 0`` (lambda2)."""
    if updater == "ftrl":
        try:
            lr, alpha, l1, l2 = (_f32(x) for x in (opt.learning_rate, opt.rho, opt.lambda_, opt.momentum))
        except OverflowError:          # beyond the fp32 range
            lr = alpha = l1 = l2 = float("inf")
        if not (math.isfinite(lr + alpha + l1 + l2) and lr > 0.0 and alpha > 0.0 and l1 >= 0.0 and l2 >= 0.0):
            raise ValueError(f"ftrl needs finite learning_rate > 0, rho (alpha) > 0, lambda_ (lambda1) >= 0 and "
                             f"momentum (lambda2) >= 0 as fp32, got learning_rate={opt.learning_rate}, "
                             f"rho={opt.rho}, lambda_={opt.lambda_}, momentum={opt.momentum}")
        return
    if updater != "adam":
        return
    b1, lr, rho = _f32(opt.momentum), _f32(opt.learning_rate), _f32(opt.rho)
    if not (0.0 <= b1 < 1.0 and lr > 0.0 and rho >= 0.0):
        raise ValueError(f"adam needs 0 <= momentum (beta1) < 1, learning_rate > 0 and rho >= 0 as fp32, got "
                         f"momentum={opt.momentum}, learning_rate={opt.learning_rate}, rho={opt.rho}")


class GetOption:
    __slots__ = ("worker_id",)

    def __init__(self, worker_id: Optional[int] = None):
        if worker_id is None:
            from ..runtime import Runtime
            rt = Runtime.get()
            worker_id = rt.worker_id() if rt.started else 0
        self.worker_id = int(worker_id)

    def pack(self) -> bytes:
        return struct.pack("<i", self.worker_id)


@dataclass
class ArrayTableOption:
    size: int
    dtype: str = "float32"


@dataclass
class MatrixTableOption:
    num_row: int
    num_col: int
    dtype: str = "float32"
    min_value: Optional[float] = None   # server-side random-uniform init (matrix_table.h:102)
    max_value: Optional[float] = None


@dataclass
class MatrixOption(MatrixTableOption):
    is_sparse: bool = False
    is_pipeline: bool = False


@dataclass
class SparseMatrixTableOption(MatrixTableOption):
    is_pipeline: bool = False


@dataclass
class KVTableOption:
    key_dtype: str = "int64"
    val_dtype: str = "float32"
