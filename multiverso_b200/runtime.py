"""The Zoo of the device runtime: one process per GPU, every rank worker + server.

Reference: Zoo (src/zoo.cpp:41-186) parses flags, initialises the net, decides the role
from ``-ps_role``, starts the controller / communicator / server / worker actors and
implements Barrier / RegisterNode / FinishTrain.  On the GPU data path the actors do not
move data any more -- the "server" is the owner-side half of a fused kernel and the
"communicator" is a peer mapping -- so the Zoo keeps only what still has meaning:

* rank / size / roles / dense worker and server ids (Controller::RegisterController,
  src/controller.cpp:38-80: ids are assigned in rank order),
* the control plane (``torch.distributed``: gloo for handle exchange, NCCL only for the
  comparator baseline),
* the symmetric allocations, the signal pads + epoch counters (K11) and the watchdog flag,
* table registration (positional table ids, src/zoo.cpp:178-186).

Without CUDA the same API is served by the C++ host runtime (``multiverso_b200.host``).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, List, Optional

from . import _native as N
from .utils import FLAGS, Log

ROLE_NONE, ROLE_WORKER, ROLE_SERVER, ROLE_ALL = 0, 1, 2, 3  # include/multiverso/node.h:6-27


def parse_ps_role(s: str) -> int:
    return {"none": ROLE_NONE, "worker": ROLE_WORKER, "server": ROLE_SERVER,
            "default": ROLE_ALL}.get(s, ROLE_ALL)


class _CudaView:
    """Expose raw device memory to torch through __cuda_array_interface__."""

    def __init__(self, ptr: int, nbytes: int, owner):
        self.__cuda_array_interface__ = {
            "shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3,
            "strides": None,
        }
        self._owner = owner


class SymmBuffer:
    """A symmetric allocation: the same-sized slab on every rank, peer-mapped everywhere.

    ``ptrs[r]`` is rank r's slab as seen from this process (cudaIpc mapping for r != me).
    Replaces Blob + Allocator + NetInterface::Send on the data path (SURVEY 5.8).
    """

    def __init__(self, rt: "Runtime", nbytes: int):
        import torch
        self.rt = rt
        self.nbytes = max(int(nbytes), 16)
        lib = N.cuda_lib()
        p = C.c_void_p()
        lib.mvb_symm_alloc(self.nbytes, p)
        self.local_ptr = p.value
        self.ptrs: List[int] = [0] * rt.size
        self.ptrs[rt.rank] = self.local_ptr
        self._opened: List[int] = []
        if rt.size > 1:
            h = (C.c_char * 64)()
            lib.mvb_ipc_get_handle(self.local_ptr, C.addressof(h))
            handles = rt.all_gather_object(bytes(h.raw))
            for r, hb in enumerate(handles):
                if r == rt.rank:
                    continue
                q = C.c_void_p()
                buf = C.create_string_buffer(hb, 64)
                lib.mvb_ipc_open_handle(C.addressof(buf), q)
                self.ptrs[r] = q.value
                self._opened.append(q.value)
        self._view = _CudaView(self.local_ptr, self.nbytes, self)
        self._base = torch.as_tensor(self._view, device=rt.device)

    def tensor(self, dtype, numel: Optional[int] = None, offset_bytes: int = 0):
        """Typed torch view of the local slab (zero-copy)."""
        import torch
        esz = torch.empty((), dtype=dtype).element_size()
        if numel is None:
            numel = (self.nbytes - offset_bytes) // esz
        return self._base[offset_bytes:offset_bytes + numel * esz].view(dtype)

    def ptr_array(self):
        """ctypes void*[MAX_RANKS] of the peer mappings."""
        arr = N.VP8()
        for r in range(N.MAX_RANKS):
            arr[r] = self.ptrs[r] if r < len(self.ptrs) else None
        return arr

    def close_peers(self):
        """Phase 1 of a release: unmap the peers' slabs from this process."""
        lib = N.cuda_lib()
        for q in self._opened:
            lib.mvb_ipc_close_handle(q)
        self._opened = []

    def free_local(self):
        """Phase 2: free the exported slab -- only after EVERY rank has finished phase 1 (a peer that still
        has the slab mapped must never see it freed; same ordering as csrc/device_rt/device_rt.cpp)."""
        if self.local_ptr:
            self._base = None
            N.cuda_lib().mvb_symm_free(self.local_ptr)
            self.local_ptr = 0

    def free(self):
        """Collective release: close peer mappings, rendezvous, free the local slab."""
        self.close_peers()
        if self.rt.size > 1 and self.rt.started:
            self.rt.control_barrier()
        self.free_local()


class McBuffer:
    """A symmetric allocation that is ALSO bound to an NVLS multicast object, so kernels can use
    ``multimem.ld_reduce`` / ``multimem.st`` on ``multicast_ptr`` (in-switch reduction / broadcast).
    Allocated through torch.distributed._symmetric_memory (CUDA VMM + cuMulticast*); same
    ``ptrs`` / ``tensor`` interface as SymmBuffer. Raises if the platform has no multicast."""

    def __init__(self, rt: "Runtime", nbytes: int):
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        self.rt = rt
        self.nbytes = max(int(nbytes), 16)
        self._t = symm_mem.empty(self.nbytes, dtype=torch.uint8, device=rt.device)
        self._hdl = symm_mem.rendezvous(self._t, dist.group.WORLD.group_name)
        self.ptrs = [int(p) for p in self._hdl.buffer_ptrs]
        self.local_ptr = self.ptrs[rt.rank]
        self.multicast_ptr = int(self._hdl.multicast_ptr or 0)
        if not self.multicast_ptr:
            raise RuntimeError("no NVLS multicast support")
        self._t.zero_()

    def tensor(self, dtype, numel: Optional[int] = None, offset_bytes: int = 0):
        import torch
        esz = torch.empty((), dtype=dtype).element_size()
        if numel is None:
            numel = (self.nbytes - offset_bytes) // esz
        return self._t[offset_bytes:offset_bytes + numel * esz].view(dtype)

    def ptr_array(self):
        arr = N.VP8()
        for r in range(N.MAX_RANKS):
            arr[r] = self.ptrs[r] if r < len(self.ptrs) else None
        return arr

    def free(self):
        self._t = None
        self._hdl = None


class Runtime:
    """Singleton process state (``Zoo::Get()``)."""

    _inst: Optional["Runtime"] = None

    @classmethod
    def get(cls) -> "Runtime":
        if cls._inst is None:
            cls._inst = Runtime()
        return cls._inst

    def __init__(self):
        self.started = False
        self.rank = 0
        self.size = 1
        self.local_rank = 0
        self.device = None
        self.backend = "none"       # "device" | "host"
        self.roles: List[int] = [ROLE_ALL]
        self.worker_ranks: List[int] = [0]
        self.server_ranks: List[int] = [0]
        self.tables: List = []
        self._own_pg = False
        self._gloo = None
        self.pads: Optional[SymmBuffer] = None
        self.err_flag = None
        self.barrier_hooks = []      # callables(final: bool): served while a barrier waits (row-mailbox drains)
        self._epochs: Dict[int, int] = {}
        self._next_channel = 4       # channels 0..3 reserved (barrier, aggregate)
        self._symm: List[SymmBuffer] = []

    # ------------------------------------------------------------------ bring-up
    def start(self, argv: Optional[List[str]] = None, **flags) -> List[str]:
        """MV_Init: parse flags, bootstrap, assign roles/ids, create signal pads, barrier."""
        import torch
        rest = FLAGS.parse(list(argv) if argv else [])
        for k, v in flags.items():
            FLAGS.set(k, v)
        if self.started:
            return rest
        self.rank = int(os.environ.get("RANK", "0"))
        self.size = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", str(self.rank)))
        Log.rank = self.rank if self.size > 1 else None
        Log.to_stderr = bool(FLAGS.get("logtostderr"))
        if self.size > N.MAX_RANKS:
            Log.fatal("multiverso_b200 supports up to %d ranks on one NVSwitch domain (got %d)",
                      N.MAX_RANKS, self.size)
        if torch.cuda.is_available():
            self.backend = "device"
            ndev = torch.cuda.device_count()
            self.device = torch.device("cuda", self.local_rank % ndev)
            torch.cuda.set_device(self.device)
            N.cuda_lib()  # fail loudly if the kernel library is missing on a GPU box
        else:
            self.backend = "host"
            self.device = torch.device("cpu")
        if self.backend == "host":
            # the C++ runtime (TcpNet + controller) does bootstrap, roles and ids itself
            from . import host
            host.init_backend(self)
            self.started = True
            return rest
        if self.size > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
                os.environ.setdefault("MASTER_PORT", str(FLAGS.get("port")))
                if self.backend == "device":
                    dist.init_process_group("cpu:gloo,cuda:nccl", rank=self.rank,
                                            world_size=self.size, device_id=self.device)
                else:
                    dist.init_process_group("gloo", rank=self.rank, world_size=self.size)
                self._own_pg = True
        # ---- RegisterNode: roles + dense ids in rank order ------------------------------
        my_role = parse_ps_role(str(FLAGS.get("ps_role")))
        self.roles = self.all_gather_object(my_role)
        self.worker_ranks = [r for r, ro in enumerate(self.roles) if ro & ROLE_WORKER]
        self.server_ranks = [r for r, ro in enumerate(self.roles) if ro & ROLE_SERVER]
        if FLAGS.get("ma"):
            # model-averaging mode: no parameter server at all (src/zoo.cpp:49)
            self.server_ranks = []
        if self.backend == "device":
            self.pads = SymmBuffer(self, N.PAD_WORDS * 8)
            self.err_flag = torch.zeros(1, dtype=torch.int32, device=self.device)
            self._done_counters = torch.zeros(256, dtype=torch.int32, device=self.device)
            self._n_counters = 0
        self.started = True
        self.barrier()
        return rest

    def stop(self, finalize_net: bool = True) -> None:
        """MV_ShutDown: FinishTrain in sync mode, barrier, free tables and mappings."""
        if not self.started:
            return
        if self.backend == "host":
            from . import host
            host.shutdown_backend(self, finalize_net)
            self.tables = []
            self.started = False
            Runtime._inst = None
            return
        import torch
        self._finish_train()
        self.barrier()
        for t in list(self.tables):
            if self.backend != "device" and hasattr(t, "free"):
                t.free()
        self.tables = []          # device tables: every symmetric slab is released below, in two phases
        if self.backend == "device":
            torch.cuda.synchronize()
            # two-phase release of every symmetric allocation: all ranks unmap their peers' slabs, meet on
            # the control plane, and only then free the slabs they exported
            bufs = list(self._symm) + ([self.pads] if self.pads is not None else [])
            for b in bufs:
                if hasattr(b, "close_peers"):
                    b.close_peers()
            if self.size > 1:
                self.control_barrier()
            for b in bufs:
                if hasattr(b, "free_local"):
                    b.free_local()
                else:
                    b.free()
            self._symm = []
            self.pads = None
        if finalize_net and self._own_pg:
            import torch.distributed as dist
            if dist.is_initialized():
                dist.destroy_process_group()
            self._own_pg = False
        self.started = False
        self._epochs = {}
        self._next_channel = 4
        Runtime._inst = None

    def _finish_train(self) -> None:
        """Zoo::FinishTrain (src/zoo.cpp:152-161) for the BSP device tables. A rank that is
        done must (1) stop gating the others -- FIN on every table's ready channel -- and
        (2) keep serving as an owner: it polls the ready slots of all its tables and runs the
        fused Add for any epoch every still-active worker has published, until all workers
        of all tables have finished. Polling (never a blocking wait) keeps multi-table
        shutdown deadlock-free when ranks finish at different times."""
        import time
        import torch
        bsp = [t for t in self.tables if getattr(t, "needs_drain", lambda: False)()]
        if not bsp or self.size == 1:
            return
        lib = N.cuda_lib()
        for t in bsp:
            t.publish_finish()
        torch.cuda.current_stream().synchronize()
        pending = list(bsp)
        deadline = time.time() + 4 * float(FLAGS.get("barrier_timeout_s"))
        while pending and time.time() < deadline:
            pads = self.pads.tensor(torch.int64).cpu()
            progressed = False
            for t in list(pending):
                st = t.drain_step(pads)
                if st == "done":
                    pending.remove(t)
                    progressed = True
                elif st == "served":
                    progressed = True
            if not progressed:
                time.sleep(0.0005)
        if pending:
            Log.error("FinishTrain: %d table(s) still waiting for peers at shutdown", len(pending))

    # ------------------------------------------------------------------ identity
    def num_workers(self) -> int:
        return len(self.worker_ranks)

    def num_servers(self) -> int:
        return len(self.server_ranks)

    def worker_id(self) -> int:
        return self.worker_ranks.index(self.rank) if self.rank in self.worker_ranks else -1

    def server_id(self) -> int:
        return self.server_ranks.index(self.rank) if self.rank in self.server_ranks else -1

    def worker_id_to_rank(self, wid: int) -> int:
        return self.worker_ranks[wid]

    def server_id_to_rank(self, sid: int) -> int:
        return self.server_ranks[sid]

    def is_worker(self) -> bool:
        return self.rank in self.worker_ranks

    def is_server(self) -> bool:
        return self.rank in self.server_ranks

    # ------------------------------------------------------------------ control plane
    def control_barrier(self) -> None:
        """Host-side rendezvous on the control plane (no device work involved)."""
        if self.size > 1:
            self.all_gather_object(0)

    def all_gather_object(self, obj):
        if self.size == 1:
            return [obj]
        import torch.distributed as dist
        out = [None] * self.size
        dist.all_gather_object(out, obj, group=self._cpu_group())
        return out

    def _cpu_group(self):
        import torch.distributed as dist
        if self.backend != "device":
            return None
        if self._gloo is None:
            # a dedicated gloo group keeps pickled control traffic off the NCCL stream
            self._gloo = dist.new_group(backend="gloo")
        return self._gloo

    def host_barrier(self) -> None:
        if self.size > 1:
            import torch.distributed as dist
            dist.barrier(group=self._cpu_group())

    # ------------------------------------------------------------------ signal pads
    def new_channels(self, n: int) -> int:
        """Reserve n consecutive signal-pad channels (collective: same order on all ranks)."""
        ch = self._next_channel
        self._next_channel += n
        if self._next_channel > N.PAD_CHANNELS:
            Log.fatal("out of signal-pad channels (%d)", N.PAD_CHANNELS)
        return ch

    def next_epoch(self, channel: int) -> int:
        e = self._epochs.get(channel, 0) + 1
        self._epochs[channel] = e
        return e

    def done_counter_ptr(self) -> int:
        i = self._n_counters
        self._n_counters += 1
        return self._done_counters.data_ptr() + 4 * (i % 256)

    def pads_array(self):
        return self.pads.ptr_array()

    def alloc_symm(self, nbytes: int) -> SymmBuffer:
        b = SymmBuffer(self, nbytes)
        self._symm.append(b)
        return b

    def alloc_multicast(self, nbytes: int):
        """Symmetric + NVLS multicast allocation, or None when NVLS is unavailable / disabled.
        Collective: every rank must call it in the same order (all succeed or all fail)."""
        if self.size == 1 or not bool(FLAGS.get("nvls")) or getattr(self, "_nvls_broken", False):
            return None
        try:
            b = McBuffer(self, nbytes)
        except Exception as e:   # no multicast object / rendezvous unsupported: fall back to P2P
            self._nvls_broken = True
            Log.info("NVLS multicast unavailable (%s): using the P2P kernels", repr(e)[:120])
            return None
        ok = all(self.all_gather_object(True))
        self._symm.append(b)
        return b if ok else None

    def release_symm(self, b: SymmBuffer) -> None:
        if b in self._symm:
            self._symm.remove(b)
        b.free()

    def barrier(self) -> None:
        """MV_Barrier. Device backend: K11 flag barrier on the current stream, then the
        host waits for it (the reference's barrier is a host rendezvous, so callers expect
        all prior table ops of every rank to be complete and visible afterwards)."""
        if not self.started or self.size == 1:
            if self.backend == "device":
                import torch
                torch.cuda.synchronize()
            return
        if self.backend == "device":
            import torch
            lib = N.cuda_lib()
            ep = self.next_epoch(0)
            lib.mvb_barrier(self.pads_array(), self.rank, self.size, 0, ep, self.err_flag,
                            float(FLAGS.get("barrier_timeout_s")), N.stream_ptr())
            if self.barrier_hooks:
                # Row mailboxes: a rank waiting here still serves the pushes of the ranks that have not
                # arrived yet (they may be spinning for its ack), then -- every rank has rung its doorbells
                # before it entered -- applies what is left and meets the others once more.
                import time
                ev = torch.cuda.Event()
                ev.record()
                while not ev.query():
                    for h in self.barrier_hooks:
                        h(False)
                    time.sleep(2e-4)
                for h in self.barrier_hooks:
                    h(True)
                ep = self.next_epoch(0)
                lib.mvb_barrier(self.pads_array(), self.rank, self.size, 0, ep, self.err_flag,
                                float(FLAGS.get("barrier_timeout_s")), N.stream_ptr())
            torch.cuda.current_stream().synchronize()
            self.check_watchdog()
        else:
            from . import host
            host.barrier()

    def check_watchdog(self) -> None:
        if self.err_flag is None:
            return
        code = int(self.err_flag.item())
        if code:
            self.err_flag.zero_()
            if code == 5003:
                Log.fatal("KVTable: key INT64_MIN is reserved for empty slots (code 5003: kv-bad-key); the other "
                          "keys of the batch were added")
            if code // 100 == 31:
                Log.fatal("row mailbox overflow (code %d): a push named more rows of owner %d than a mailbox slot "
                          "holds; those rows were dropped", code, code % 100)
            Log.fatal("device watchdog: wait on peer timed out (code %d: %s, peer index %d)", code,
                      {1: "wait", 2: "barrier", 3: "add-ready", 4: "get-done", 5: "kv-full",
                       6: "allreduce"}.get(code // 1000, "?"), code % 1000)

    def register_table(self, table) -> int:
        self.tables.append(table)
        return len(self.tables) - 1
