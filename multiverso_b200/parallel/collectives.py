"""MV_Aggregate and friends on the device backend (K6).

Reference: MV_Aggregate<T> -> net::Allreduce -> MPI_Allreduce(MPI_IN_PLACE, SUM)
(src/multiverso.cpp:53-56, include/multiverso/net/mpi_net.h:147-151), available in
model-averaging mode (``-ma=true``) where no parameter server is started.  Here it is a
hand-written P2P kernel over symmetric staging: one-shot for latency-bound sizes,
two-shot (reduce own slice, write back to all) above ``TWO_SHOT_BYTES``.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Tuple

import torch

from .. import _native as N
from ..runtime import Runtime
from ..utils import FLAGS, monitor

TWO_SHOT_BYTES = 512 * 1024
FUSED_BYTES = 1 << 20            # <= this: one launch (stage-in + handshake + reduce), no done-handshake
FUSED_CHANNEL = 3                # signal-pad channel of the fused path (0 barrier, 1-2 staged paths)


class _AggregateState:
    def __init__(self):
        self.staging = None
        self.cap = 0
        self.epoch = 0
        self.counter = None
        # fused latency path: double-buffered staging, own channel / epoch / grid counter, cached descriptor
        self.f_staging = None
        self.f_epoch = 0
        self.f_desc = None


_state = _AggregateState()
_symm_user: Dict[int, Tuple[object, int]] = {}       # local base ptr -> (buffer, nbytes) of symm_tensor() allocations


def reset() -> None:
    global _state
    _state = _AggregateState()
    _symm_user.clear()


def symm_tensor(numel: int, dtype=torch.float32) -> torch.Tensor:
    """A tensor in symmetric (peer-mapped, and multicast-mapped when NVLS is available) memory.
    ``aggregate`` reduces such a tensor in place with NO staging copy (model-averaging mode: keep the
    model / gradient buffer here).  Collective: every rank must allocate the same sizes in the same order."""
    rt = Runtime.get()
    nbytes = int(numel) * torch.empty(0, dtype=dtype).element_size()
    if rt.size == 1:
        return torch.empty(int(numel), dtype=dtype, device=rt.device)
    buf = rt.alloc_multicast(nbytes) or rt.alloc_symm(nbytes)
    _symm_user[buf.ptrs[rt.rank]] = (buf, nbytes)
    return buf.tensor(dtype, int(numel))


def _find_symm(ptr: int, nbytes: int):
    for base, (buf, cap) in _symm_user.items():
        if base <= ptr and ptr + nbytes <= base + cap:
            return buf, ptr - base
    return None, 0


def _aggregate_fused(rt, lib, st, data: torch.Tensor, nbytes: int) -> torch.Tensor:
    """<= 1 MB: stage-in, ready-handshake and one-shot reduction in a single launch (the whole cost
    of a small MV_Aggregate is launch latency, so it is one kernel and almost no host work)."""
    a = st.f_desc
    if a is None:
        st.f_staging = rt.alloc_symm(2 * FUSED_BYTES)
        a = N.Allreduce()
        for r in range(rt.size):
            a.bufs[r] = st.f_staging.ptrs[r]
        st.f_pads = rt.pads_array()                      # keep the ctypes array alive
        a.pads = C.cast(st.f_pads, C.POINTER(C.c_void_p))
        a.me, a.world, a.ch = rt.rank, rt.size, FUSED_CHANNEL
        a.err_flag = rt.err_flag.data_ptr()
        a.done_counter = rt.done_counter_ptr()
        a.timeout_s = float(FLAGS.get("barrier_timeout_s"))
        st.f_desc = a
        rt.barrier()                                     # everybody's staging is mapped before the first flag
    st.f_epoch += 1
    a.dtype, a.n, a.out, a.epoch = N.dtype_code(data.dtype), data.numel(), data.data_ptr(), st.f_epoch
    lib.mvb_allreduce_fused(a, data, (st.f_epoch & 1) * FUSED_BYTES, N.stream_ptr())
    return data


def _aggregate_in_place(rt, lib, st, data, nbytes, buf, off, algo) -> torch.Tensor:
    """``data`` lives in symmetric memory: two-shot (or NVLS) directly on it, no staging copy.
    Uses the staged path's channels / epochs, so the two may be mixed freely."""
    ch = 1
    stream = N.stream_ptr()
    if st.counter is None:
        st.counter = rt.done_counter_ptr()
    if st.epoch > 0:
        lib.mvb_wait(rt.pads_array(), rt.rank, rt.size, ch + 1, st.epoch, (1 << rt.size) - 1, rt.err_flag,
                     float(FLAGS.get("barrier_timeout_s")), stream)
    st.epoch += 1
    a = N.Allreduce()
    a.dtype, a.n = N.dtype_code(data.dtype), data.numel()
    for r in range(rt.size):
        a.bufs[r] = buf.ptrs[r] + off
    a.out = data.data_ptr()
    pads = rt.pads_array()
    a.pads = C.cast(pads, C.POINTER(C.c_void_p))
    a.me, a.world, a.ch, a.epoch = rt.rank, rt.size, ch, st.epoch
    a.err_flag = rt.err_flag.data_ptr()
    a.done_counter = st.counter
    a.timeout_s = float(FLAGS.get("barrier_timeout_s"))
    mc = getattr(buf, "multicast_ptr", 0)
    # in-switch reduction pays when it removes traffic: n/W instead of (W-1)/W * n per GPU (measured at
    # 2 GPUs: 686 us vs 444 us two-shot for 256 MB, so P2P below 4 ranks)
    use_nvls = bool(mc) and data.dtype == torch.float32 and (algo == "nvls" or (algo == "auto" and rt.size >= 4))
    with monitor("MV_AGGREGATE", cuda=True, nbytes=nbytes):
        if use_nvls:
            lib.mvb_allreduce_nvls(a, mc + off, stream)
        else:
            lib.mvb_allreduce_twoshot(a, stream)
    return data


def aggregate(data: torch.Tensor, algo: str = "auto") -> torch.Tensor:
    """In-place SUM all-reduce of a CUDA tensor across all ranks; returns ``data``."""
    rt = Runtime.get()
    assert data.is_cuda and data.is_contiguous()
    if rt.size == 1:
        return data
    lib = N.cuda_lib()
    nbytes = data.numel() * data.element_size()
    st = _state
    if algo in ("auto", "fused") and nbytes <= FUSED_BYTES:
        return _aggregate_fused(rt, lib, st, data, nbytes)
    user_buf, user_off = _find_symm(data.data_ptr(), nbytes) if _symm_user else (None, 0)
    if user_buf is not None and (user_off % 16 == 0):
        return _aggregate_in_place(rt, lib, st, data, nbytes, user_buf, user_off, algo)
    if st.cap < nbytes:
        if st.staging is not None:
            rt.barrier()
            rt.release_symm(st.staging)
        st.cap = max(nbytes, 1 << 20)
        st.staging = rt.alloc_multicast(st.cap) or rt.alloc_symm(st.cap)
        st.counter = rt.done_counter_ptr()
    ch = 1  # channels 1 (ready) and 2 (done) are reserved for aggregate
    stream = N.stream_ptr()
    if st.epoch > 0:
        # nobody may still be reading our staging buffer from the previous call
        lib.mvb_wait(rt.pads_array(), rt.rank, rt.size, ch + 1, st.epoch, (1 << rt.size) - 1, rt.err_flag,
                     float(FLAGS.get("barrier_timeout_s")), stream)
    stage = st.staging.tensor(data.dtype, data.numel())
    stage.copy_(data.view(-1))
    st.epoch += 1
    a = N.Allreduce()
    a.dtype, a.n = N.dtype_code(data.dtype), data.numel()
    for r in range(rt.size):
        a.bufs[r] = st.staging.ptrs[r]
    a.out = data.data_ptr()
    pads = rt.pads_array()
    a.pads = C.cast(pads, C.POINTER(C.c_void_p))
    a.me, a.world, a.ch, a.epoch = rt.rank, rt.size, ch, st.epoch
    a.err_flag = rt.err_flag.data_ptr()
    a.done_counter = st.counter
    a.timeout_s = float(FLAGS.get("barrier_timeout_s"))
    two = (algo == "twoshot") or (algo in ("auto", "nvls") and nbytes > TWO_SHOT_BYTES)
    mc = getattr(st.staging, "multicast_ptr", 0)
    use_nvls = bool(mc) and data.dtype == torch.float32 and (algo == "nvls" or (algo == "auto" and two and rt.size >= 4))
    with monitor("MV_AGGREGATE", cuda=True, nbytes=nbytes):
        if use_nvls:
            lib.mvb_allreduce_nvls(a, mc, stream)
        else:
            fn = lib.mvb_allreduce_twoshot if two else lib.mvb_allreduce_oneshot
            fn(a, stream)
    return data
