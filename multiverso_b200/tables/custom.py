"""Application-defined tables on the device plane -- the extension point.

Reference: a user table subclasses ``WorkerTable`` / ``ServerTable``, implements ``Partition`` /
``ProcessReplyGet`` / ``ProcessAdd`` / ``ProcessGet`` and binds the pair to an option type with
``DEFINE_TABLE_TYPE`` (include/multiverso/table_interface.h:24-80); the LogisticRegression application
ships two such tables (Applications/LogisticRegression/src/util/sparse_table.h:16-302 ``SparseTable<T>`` and
util/ftrl_sparse_table.h:11-86 ``FTRLTable<T>``).

On the device plane the same contract is :class:`CustomDeviceTable`: the base class owns what every table
needs -- positional table id, symmetric (peer-mapped) shard storage, the range-partition rule of the reference
(``size / num_servers`` per server, the last one takes the remainder), checkpoint plumbing, registration with
the runtime -- and a subclass supplies the data-plane ops as kernels over the peer pointers (``self.shard_ptrs``,
one-sided like every built-in table) and, if it needs owner-side work, a ``serve()`` hook that the runtime calls
at the table's collective points.  ``create_table(option)`` accepts any option object with a ``create()`` method,
which is the ``DEFINE_TABLE_TYPE`` binding.

:class:`SparseDeviceTable` and :class:`FTRLDeviceTable` are the reference's two application tables built on
this base with the key-addressed kernels of csrc/cuda/keys.cu.
"""
from __future__ import annotations

import struct
from typing import List, Optional, Tuple

import torch

from .. import _native as N
from ..runtime import Runtime
from ..utils import Log


class CustomDeviceTable:
    """Base class of application-defined device tables (see the module docstring).

    Subclass contract:
      * call ``super().__init__(size, bytes_per_key)`` -- collective, like every table constructor;
      * implement the ops (``add`` / ``get`` ...) as kernels over ``self.shard_ptrs`` (peer mapped);
      * optionally override ``serve()`` (owner-side work at collective points), ``store`` / ``load``.
    """

    def __init__(self, size: int, bytes_per_key: int, extra_symm_bytes_per_shard: int = 0):
        rt = Runtime.get()
        if not rt.started:
            Log.fatal("MV_Init must be called before creating tables")
        if rt.backend != "device":
            Log.fatal("CustomDeviceTable needs the device backend")
        self.rt = rt
        self.size = int(size)
        S = max(rt.num_servers(), 1)
        self.S = S
        # SparseServerTable ctor (sparse_table.h:176-192): size/num_server each, last takes the remainder
        if self.size >= S:
            self.per = self.size // S
            self.lo = [s * self.per for s in range(S)]
            self.hi = [(s + 1) * self.per for s in range(S)]
            self.hi[-1] = self.size
        else:
            self.per = 1
            self.lo = [min(s, self.size) for s in range(S)]
            self.hi = [min(s + 1, self.size) for s in range(S)]
        self.sid = rt.server_id()
        self.max_keys = max(h - l for l, h in zip(self.lo, self.hi))
        self.bytes_per_key = int(bytes_per_key)
        self.shard_buf = rt.alloc_symm(max(self.max_keys * self.bytes_per_key, 16))
        self.shard_buf.tensor(torch.uint8).zero_()
        self.extra_buf = rt.alloc_symm(max(extra_symm_bytes_per_shard, 16)) if extra_symm_bytes_per_shard else None
        if self.extra_buf is not None:
            self.extra_buf.tensor(torch.uint8).zero_()
        ranks = [rt.server_id_to_rank(s) if rt.num_servers() else rt.rank for s in range(S)]
        self.shard_ptrs: List[int] = [self.shard_buf.ptrs[r] for r in ranks]
        self.extra_ptrs: List[int] = [self.extra_buf.ptrs[r] for r in ranks] if self.extra_buf is not None else []
        self.table_id = rt.register_table(self)
        if rt.size > 1:
            rt.barrier_hooks.append(self._barrier_hook)
        torch.cuda.synchronize()
        rt.barrier()                      # MV_CreateTable ends with a barrier (multiverso.h:35-41)

    def _barrier_hook(self, final: bool) -> None:
        if final:
            self.serve()

    def serve(self) -> None:
        """Owner-side work of the table at a collective point (default: nothing -- one-sided tables)."""

    def peer_tensor(self, server: int, dtype=torch.float32) -> torch.Tensor:
        """Server ``server``'s shard as a torch tensor over the PEER MAPPING (zero-copy): a subclass can express its
        ops with torch indexing / its own kernels on it; writes land in that server's HBM over NVLink."""
        from ..runtime import _CudaView
        n = (self.hi[server] - self.lo[server]) * self.bytes_per_key
        view = _CudaView(self.shard_ptrs[server], max(n, 1), self)
        t = torch.as_tensor(view, device=self.rt.device)
        return t[:n].view(dtype)

    def my_keys(self) -> Tuple[int, int]:
        return (self.lo[self.sid], self.hi[self.sid]) if self.sid >= 0 else (0, 0)

    # Serializable (table_interface.h:61-75): raw dump of the local shard
    def store(self, stream) -> None:
        lo, hi = self.my_keys()
        n = (hi - lo) * self.bytes_per_key
        torch.cuda.synchronize()
        stream.write(struct.pack("<q", n))
        stream.write(self.shard_buf.tensor(torch.uint8, n).cpu().numpy().tobytes())

    def load(self, stream) -> None:
        import numpy as np
        (n,) = struct.unpack("<q", stream.read(8))
        lo, hi = self.my_keys()
        if n != (hi - lo) * self.bytes_per_key:
            raise ValueError(f"checkpoint shard has {n} bytes, table shard {(hi - lo) * self.bytes_per_key}")
        data = np.frombuffer(stream.read(n), dtype=np.uint8).copy()
        self.shard_buf.tensor(torch.uint8, n).copy_(torch.from_numpy(data))


class SparseDeviceTable(CustomDeviceTable):
    """``SparseTable<float>`` (sparse_table.h): ``size`` keys x ``width`` fp32 values, range partitioned; the
    server SUBTRACTS what is added (``storage_[key] -= val``, sparse_table.h:206-218) and remembers which keys
    were ever written; ``get()`` without keys returns only those (sparse_table.h:220-257)."""

    def __init__(self, size: int, width: int = 1):
        self.width = int(width)
        words = lambda n: (n + 31) // 32 * 4          # noqa: E731
        super().__init__(size, 4 * self.width, extra_symm_bytes_per_shard=words(max(size, 1)) + 16)
        m = N.KeyMap()
        m.size, m.per_server, m.nservers, m.width = self.size, self.per, self.S, self.width
        for s in range(self.S):
            m.shard_ptrs[s] = self.shard_ptrs[s]
            m.touched_ptrs[s] = self.extra_ptrs[s]
        self._map = m
        self._count = torch.zeros(1, dtype=torch.int64, device=self.rt.device)

    def _keys(self, keys) -> torch.Tensor:
        return torch.as_tensor(keys, dtype=torch.int64).to(self.rt.device).contiguous().view(-1)

    def add(self, keys, vals) -> None:
        """One-sided, asynchronous: shard[key] -= val (component-wise for width > 1)."""
        k = self._keys(keys)
        v = torch.as_tensor(vals, dtype=torch.float32).to(self.rt.device).contiguous().view(-1)
        assert v.numel() == k.numel() * self.width
        N.cuda_lib().mvb_keys_add(self._map, k, v, k.numel(), -1.0, N.stream_ptr())
        self._keep = (k, v)

    def get(self, keys=None):
        """``get(keys)`` -> values [n, width]; ``get()`` -> (keys, values) of every key ever written."""
        lib = N.cuda_lib()
        if keys is not None:
            k = self._keys(keys)
            out = torch.empty(k.numel(), self.width, device=self.rt.device)
            lib.mvb_keys_get(self._map, k, out, k.numel(), N.stream_ptr())
            self._keep_get = k
            return out if self.width > 1 else out.view(-1)
        cap = self.size
        ok = torch.empty(cap, dtype=torch.int64, device=self.rt.device)
        ov = torch.empty(cap, self.width, device=self.rt.device)
        lib.mvb_keys_collect(self._map, ok, ov, self._count, cap, N.stream_ptr())
        n = int(self._count.item())
        order = torch.argsort(ok[:n])
        vals = ov[:n][order]
        return ok[:n][order], (vals if self.width > 1 else vals.view(-1))


class FTRLDeviceTable(SparseDeviceTable):
    """``FTRLTable<float>`` (ftrl_sparse_table.h): a SparseTable whose values are the FTRL pairs {z, n}; the
    worker pushes (delta z, delta n), the server subtracts both."""

    def __init__(self, size: int):
        super().__init__(size, width=2)


class SparseTableOption:
    """``SparseTableOption`` / ``DEFINE_TABLE_TYPE`` analogue: ``mv.create_table(SparseTableOption(n))``."""

    def __init__(self, size: int):
        self.size = size

    def create(self):
        return SparseDeviceTable(self.size)


class FTRLTableOption:
    def __init__(self, size: int):
        self.size = size

    def create(self):
        return FTRLDeviceTable(self.size)
