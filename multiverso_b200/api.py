"""Public API: the reference's MV_* surface (include/multiverso/multiverso.h:9-65) and the
Python binding's names (binding/python/multiverso/api.py:12-75).

The same calls work on both backends: ``device`` (CUDA present: HBM tables + sm_90a
kernels) and ``host`` (no CUDA: the C++ runtime in libmultiverso.so, TCP control plane).
"""
from __future__ import annotations

from typing import List, Optional

from .runtime import Runtime
from .utils import FLAGS, Dashboard, Log


def _rt() -> Runtime:
    return Runtime.get()


def init(argv: Optional[List[str]] = None, sync: Optional[bool] = None, **flags) -> List[str]:
    """MV_Init. ``sync=True`` selects the BSP server like ``mv.init(sync=True)`` in the
    reference binding (api.py:12-35). Extra keyword flags are MV_SetFlag'ed first.
    Returns argv with the recognised ``-key=value`` flags removed."""
    if sync is not None:
        flags["sync"] = bool(sync)
    return _rt().start(argv, **flags)


def shutdown(finalize_net: bool = True) -> None:
    """MV_ShutDown(finalize_net): ``False`` keeps the process group alive so the process
    can MV_Init again (Test/unittests/multiverso_env.h:15-17)."""
    rt = _rt()
    if rt.backend == "device":
        from .parallel import collectives
        collectives.reset()
    rt.stop(finalize_net)


def barrier() -> None:
    """MV_Barrier."""
    _rt().barrier()


def rank() -> int: return _rt().rank
def size() -> int: return _rt().size
def num_workers() -> int: return _rt().num_workers()
def num_servers() -> int: return _rt().num_servers()
def workers_num() -> int: return _rt().num_workers()   # python binding name
def worker_id() -> int: return _rt().worker_id()
def server_id() -> int: return _rt().server_id()
def worker_id_to_rank(wid: int) -> int: return _rt().worker_id_to_rank(wid)
def server_id_to_rank(sid: int) -> int: return _rt().server_id_to_rank(sid)
def is_master_worker() -> bool: return _rt().worker_id() == 0


def set_flag(name: str, value) -> None:
    """MV_SetFlag<T>(name, value)."""
    FLAGS.set(name, value)


def aggregate(data):
    """MV_Aggregate: in-place SUM all-reduce (model-averaging mode)."""
    rt = _rt()
    import torch
    if rt.backend == "device":
        from .parallel import aggregate as _agg
        t = data if torch.is_tensor(data) and data.is_cuda else torch.as_tensor(data).to(rt.device)
        _agg(t)
        if t is not data:
            if torch.is_tensor(data):
                data.copy_(t.cpu())
            else:
                import numpy as np
                np.copyto(data, t.cpu().numpy())
        return data
    from . import host
    return host.aggregate(data)


def symm_tensor(numel: int, dtype="float32"):
    """A tensor that ``aggregate`` reduces in place without a staging copy: symmetric (peer-mapped, NVLS
    multicast when available) device memory on the device backend, a plain tensor on the host backend.
    Collective on the device backend."""
    import torch
    rt = _rt()
    dt = getattr(torch, dtype) if isinstance(dtype, str) else dtype
    if rt.backend == "device":
        from .parallel import symm_tensor as _st
        return _st(numel, dt)
    return torch.empty(int(numel), dtype=dt)


def net_bind(rank_: int, endpoint: str) -> None:
    """MV_NetBind (explicit-endpoint bootstrap of the control plane, C# path)."""
    from . import host
    host.net_bind(rank_, endpoint)


def net_connect(ranks: List[int], endpoints: List[str]) -> None:
    """MV_NetConnect."""
    from . import host
    host.net_connect(ranks, endpoints)


def net_finalize() -> None:
    """MV_NetFinalize."""
    from . import host
    host.net_finalize()


def save_table(table, uri: str) -> bool:
    """MV_SaveTable: every server writes its shard of ``table`` (and the updater state) to
    ``<uri>.shard<server_id>``; collective, ends with a barrier.  Layout: the raw shard dump (which is
    all the reference writes, array_table.cpp:143-151) followed by the updater state slabs.  Files of
    stateless tables are interchangeable between the host and the device backend; for stateful updaters the
    device pads the per-worker state stride to a multiple of 4 elements, so those checkpoints must be loaded
    by the backend (and the number of servers) that wrote them."""
    rt = _rt()
    if rt.backend == "host":
        return bool(table.store(uri))
    ok = True
    if rt.server_id() >= 0:
        try:
            with open(f"{uri}.shard{rt.server_id()}", "wb") as f:
                table.store(f)
        except OSError as e:
            Log.error("save_table: %s", e)
            ok = False
    rt.barrier()
    return ok


def load_table(table, uri: str) -> bool:
    """MV_LoadTable: the inverse of ``save_table`` (same number of servers)."""
    rt = _rt()
    if rt.backend == "host":
        return bool(table.load(uri))
    ok = True
    if rt.server_id() >= 0:
        try:
            with open(f"{uri}.shard{rt.server_id()}", "rb") as f:
                table.load(f)
        except OSError as e:
            Log.error("load_table: %s", e)
            ok = False
    rt.barrier()
    return ok


def dashboard_display() -> None:
    Dashboard.display()
