"""Table factories (MV_CreateTable, include/multiverso/multiverso.h:35-41,
include/multiverso/table_factory.h:16-26): pick the backend implementation."""
from __future__ import annotations

from ..runtime import Runtime
from .options import (AddOption, ArrayTableOption, GetOption, KVTableOption, MatrixOption,
                      MatrixTableOption, SparseMatrixTableOption)


def _device() -> bool:
    return Runtime.get().backend == "device"


def ArrayTable(size, dtype="float32", updater=None, init_value=None):
    if _device():
        from .device import ArrayDeviceTable
        return ArrayDeviceTable(size, dtype, updater, init_value)
    from ..host import HostArrayTable
    return HostArrayTable(size, dtype, init_value)


def MatrixTable(num_row, num_col, dtype="float32", updater=None, init_value=None, min_value=None,
                max_value=None, is_sparse=False, is_pipeline=False, seed=1):
    if _device():
        from .device import MatrixDeviceTable
        return MatrixDeviceTable(num_row, num_col, dtype, updater, init_value, min_value, max_value,
                                 is_sparse, is_pipeline, seed)
    from ..host import HostMatrixTable
    return HostMatrixTable(num_row, num_col, dtype, init_value, min_value, max_value, is_sparse,
                           is_pipeline)


def SparseMatrixTable(num_row, num_col, dtype="float32", is_pipeline=False, **kw):
    return MatrixTable(num_row, num_col, dtype, is_sparse=True, is_pipeline=is_pipeline, **kw)


def KVTable(key_dtype="int64", val_dtype="float32", capacity=None):
    if _device():
        from .device import KVDeviceTable
        return KVDeviceTable(key_dtype, val_dtype, capacity)
    from ..host import HostKVTable
    return HostKVTable(key_dtype, val_dtype)


def HashMatrixTable(capacity, num_col, dtype="float32", updater=None, init_value=None, min_value=None,
                    max_value=None, seed=1, track_access=False, admit_after=1):
    """fp32 rows keyed by any int64, allocated on first lookup (device backend only; see
    :class:`multiverso_b200.tables.device.HashMatrixTable`)."""
    from .device import check_admit_after
    check_admit_after(admit_after)
    if not _device():
        raise NotImplementedError("HashMatrixTable needs the device backend (a CUDA device): its index is a GPU "
                                  "hash table; the host backend has no counterpart")
    from .device import HashMatrixTable as _Hash
    return _Hash(capacity, num_col, dtype, updater, init_value, min_value, max_value, seed, track_access, admit_after)


def create_table(option):
    """MV_CreateTable(option)."""
    if isinstance(option, MatrixOption):
        return MatrixTable(option.num_row, option.num_col, option.dtype, min_value=option.min_value,
                           max_value=option.max_value, is_sparse=option.is_sparse,
                           is_pipeline=option.is_pipeline)
    if isinstance(option, SparseMatrixTableOption):
        return SparseMatrixTable(option.num_row, option.num_col, option.dtype, option.is_pipeline)
    if isinstance(option, MatrixTableOption):
        return MatrixTable(option.num_row, option.num_col, option.dtype, min_value=option.min_value,
                           max_value=option.max_value)
    if isinstance(option, ArrayTableOption):
        return ArrayTable(option.size, option.dtype)
    if isinstance(option, KVTableOption):
        return KVTable(option.key_dtype, option.val_dtype)
    if hasattr(option, "create"):
        # application-defined table types (DEFINE_TABLE_TYPE, table_interface.h:77-80): the option knows its table
        return option.create()
    raise TypeError(f"unknown table option {type(option)}")


def SparseTable(size, width=1):
    """LogisticRegression's application table (sparse_table.h) on the device extension point."""
    from .custom import SparseDeviceTable
    return SparseDeviceTable(size, width)


def FTRLTable(size):
    from .custom import FTRLDeviceTable
    return FTRLDeviceTable(size)


__all__ = ["SparseTable", "FTRLTable", "ArrayTable", "MatrixTable", "HashMatrixTable", "SparseMatrixTable",
           "KVTable", "create_table", "AddOption", "GetOption", "ArrayTableOption", "MatrixTableOption", "MatrixOption",
           "SparseMatrixTableOption", "KVTableOption"]
