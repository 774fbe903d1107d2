"""HBM-resident distributed tables (device backend).

Reference layer L3/L4: WorkerTable / ServerTable (include/multiverso/table_interface.h:24-75,
src/table.cpp), ArrayWorker/ArrayServer (src/table/array_table.cpp), MatrixWorkerTable /
MatrixServerTable (src/table/matrix_table.cpp), MatrixWorker/MatrixServer with sparse
delta-pull (src/table/matrix.cpp), SparseMatrixTable (src/table/sparse_matrix_table.cpp),
KVWorkerTable/KVServerTable (include/multiverso/table/kv_table.h).

Device design: every rank holds its shard (and updater state) in a symmetric, peer-mapped
HBM slab.  There is no worker half / server half exchanging messages:

* ``add`` (whole table, BSP or stateful):  K1 ``mvb_add_dense_fused`` -- the owner pulls its
  slice of every worker's staging buffer over NVLink and applies the updater in registers;
  the ready/done "messages" are signal-pad flags handled inside the kernel.
* ``add`` (async + stateless updater): one-sided ``red.global.add`` push into the owners.
* ``get`` (whole): K2 pull all-gather straight from the owners' shards.
* row ops: K4 gather / K3 scatter-add through the peer mappings.
* handles: ``*_async`` returns an int id backed by a CUDA event; ``wait(id)`` synchronises it
  (multiple Gets may be in flight, SURVEY Q6; ids are recycled, Q7).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence

import torch

from .. import _native as N
from ..runtime import Runtime
from ..utils import FLAGS, Log, monitor
from .options import AddOption, GetOption, check_add_option

_DT = {"float32": torch.float32, "float": torch.float32, "float64": torch.float64,
       "double": torch.float64, "int32": torch.int32, "int": torch.int32, "int64": torch.int64}


def _torch_dtype(d):
    return d if isinstance(d, torch.dtype) else _DT[str(d)]


def _opt_struct(o: AddOption) -> N.AddOpt:
    return N.AddOpt(o.worker_id, o.momentum, o.learning_rate, o.rho, o.lambda_)


class _AsyncOps:
    """msg-id -> CUDA event bookkeeping (WorkerTable::Wait/Reset/Notify, src/table.cpp:84-111)."""

    def __init__(self):
        self._events: Dict[int, torch.cuda.Event] = {}
        self._next = 0

    def _record(self) -> int:
        ev = torch.cuda.Event()
        ev.record()
        i = self._next
        self._next += 1
        self._events[i] = ev
        return i

    def wait(self, handle: int) -> None:
        ev = self._events.pop(handle, None)
        if ev is not None:
            ev.synchronize()
        Runtime.get().check_watchdog()


class DenseDeviceTable(_AsyncOps):
    """Range-partitioned dense storage; base of ArrayTable and MatrixTable."""

    def __init__(self, num_row: int, num_col: int, dtype="float32", updater: Optional[str] = None,
                 init_value=None, min_value=None, max_value=None, seed: int = 1):
        super().__init__()
        rt = Runtime.get()
        if not rt.started:
            Log.fatal("MV_Init must be called before creating tables")
        self.rt = rt
        self.num_row, self.num_col = int(num_row), int(num_col)
        self.size = self.num_row * self.num_col
        self.dtype = _torch_dtype(dtype)
        if self.dtype not in (torch.float32, torch.float64, torch.int32):
            # the dense, push and row kernels serve these three (as the host backend and the reference do)
            Log.fatal("device tables support float32/float64/int32, got %s", dtype)
        self.dcode = N.dtype_code(self.dtype)
        self.esz = torch.empty((), dtype=self.dtype).element_size()
        name = updater or str(FLAGS.get("updater_type"))
        if self.dtype in (torch.int32, torch.int64):
            name = "default"      # Updater<int> is always the plain add (updater.cpp:40-43)
        if name not in N.UPDATER_NAMES:
            Log.fatal("unknown updater_type '%s'", name)
        self.updater_name = name
        self.updater = N.UPDATER_NAMES[name]
        self.sync = bool(FLAGS.get("sync"))
        S = max(rt.num_servers(), 1)
        W = max(rt.num_workers(), 1)
        self.S, self.W = S, W
        # ---- partition: contiguous row ranges, last server takes the remainder ------------
        # (array_table.cpp:15-19, matrix_table.cpp:26-45; fewer rows than servers => one row
        # per server for the first num_row servers)
        if self.num_row >= S:
            self.rps = self.num_row // S
            self.row_lo = [s * self.rps for s in range(S)]
            self.row_hi = [(s + 1) * self.rps for s in range(S)]
            self.row_hi[-1] = self.num_row
        else:
            self.rps = 1
            self.row_lo = [min(s, self.num_row) for s in range(S)]
            self.row_hi = [min(s + 1, self.num_row) for s in range(S)]
        self.offs = [lo * self.num_col for lo in self.row_lo]
        self.lens = [(hi - lo) * self.num_col for lo, hi in zip(self.row_lo, self.row_hi)]
        self.sid = rt.server_id()
        self.my_len = self.lens[self.sid] if self.sid >= 0 else 0
        self.my_off = self.offs[self.sid] if self.sid >= 0 else 0
        # ---- storage ---------------------------------------------------------------------
        self.shard_buf = rt.alloc_symm(max(self.my_len, 1) * self.esz)
        self.shard = self.shard_buf.tensor(self.dtype, max(self.my_len, 1))[: self.my_len]
        if min_value is not None and max_value is not None and self.my_len:
            g = torch.Generator(device=rt.device)
            g.manual_seed(seed + 7919 * max(self.sid, 0))
            self.shard.uniform_(float(min_value), float(max_value), generator=g)
        elif init_value is not None and self.my_len:
            self.shard.fill_(init_value)
        # server s's shard as seen from here (indexed by server id)
        self.shard_ptrs = [self.shard_buf.ptrs[rt.server_id_to_rank(s)] for s in range(S)] \
            if rt.num_servers() else [self.shard_buf.local_ptr]
        # (state slabs, one slab per worker, state element per row rather than per element, a step count per row)
        nst, per_worker, per_row, row_count = {
            "default": (0, False, False, False), "sgd": (0, False, False, False),
            "momentum_sgd": (1, False, False, False), "adagrad": (1, True, False, False),
            "dcasgd": (1, True, False, False), "dcasgda": (2, True, False, False),
            "rowwise_adagrad": (1, True, True, False), "adam": (2, False, False, True),
            "ftrl": (2, False, False, False)}[name]
        self.n_states, self.state_per_worker, self.state_per_row = nst, per_worker, per_row
        # a slab holds one element per shard element, or per shard row; slabs start at multiples of 4 elements
        gran = self.num_col if per_row else 1
        self.state_stride = (self.my_len // gran + 3) // 4 * 4
        slab = self.state_stride * (W if per_worker else 1)
        # adam's step counts (one per shard row) follow v's slab in the last state array, at state_stride
        self.state_row_count = (self.my_len // self.num_col + 3) // 4 * 4 if row_count else 0
        sizes = [slab] * nst
        if row_count:
            sizes[-1] += self.state_row_count
        # state slabs are symmetric (peer-mapped) too: the async one-sided push of a stateful
        # updater updates the owner's state remotely
        self._state_bufs = [rt.alloc_symm(max(n, 1) * self.esz) for n in sizes]
        self.state = [b.tensor(self.dtype, max(n, 1)) for b, n in zip(self._state_bufs, sizes)]
        self.state_strides = [(l // gran + 3) // 4 * 4 for l in self.lens]
        # collective path resources (lazy)
        self._stage: List = []
        self._stage_idx = 0
        self.ch_ready = rt.new_channels(2)
        self.ch_done = self.ch_ready + 1
        self.add_epoch = 0
        self._done_counter = rt.done_counter_ptr()
        self._fin = torch.zeros(1, dtype=torch.int32, device=rt.device)
        self._finished = False
        self._replica = None          # fused Add -> Get: full-table replica on every rank
        self._replica_epoch = -1
        # staleness instrumentation (-staleness=true): one version counter per shard in its owner's memory
        self._ver = None
        if bool(FLAGS.get("staleness")):
            self._ver = rt.alloc_symm(64)
            self._ver.tensor(torch.int64).zero_()
            self._ver_ptrs = (C.c_void_p * N.MAX_RANKS)(*[self._ver.ptrs[rt.server_id_to_rank(s)] if s < S else None
                                                          for s in range(N.MAX_RANKS)])
            self._ver_last = torch.zeros(N.MAX_RANKS, dtype=torch.int64, device=rt.device)
            self._ver_adds = torch.zeros(N.MAX_RANKS, dtype=torch.int32, device=rt.device)
            self.staleness_hist = torch.zeros(64, dtype=torch.int64, device=rt.device)
        self._opt_box = None
        if rt.size > 1 and self.sync:
            # option boxes of the collective Add (the worker's AddOption travels with its request)
            self._opt_box = rt.alloc_symm(2 * N.MAX_RANKS * 32)
            self._opt_box.tensor(torch.uint8).zero_()
        self.table_id = rt.register_table(self)
        rt.barrier()   # MV_CreateTable ends with a barrier (multiverso.h:35-41)

    # ------------------------------------------------------------------ helpers
    def _stage_buf(self):
        if not self._stage:
            linear = (self.updater in (N.UPD_DEFAULT, N.UPD_SGD) and self.dtype == torch.float32
                      and bool(FLAGS.get("nvls_add")))
            self._stage = [(self.rt.alloc_multicast(self.size * self.esz) if linear else None)
                           or self.rt.alloc_symm(self.size * self.esz) for _ in range(2)]
        b = self._stage[self._stage_idx]
        self._stage_idx ^= 1
        return b

    def enable_replica(self) -> None:
        """Fused Add -> Get for BSP whole-table traffic: every collective Add also pushes the
        updated shard into a full-table replica on every rank (one NVLS ``multimem.st`` per tile,
        or a store per peer), so the following ``get`` is a flag wait + local copy instead of a
        second trip over NVLink. Valid for tables updated ONLY through whole-table Adds
        (ArrayTable semantics); row Adds from other ranks do not reach the replicas.
        Collective: call on every rank."""
        if self._replica is None and self.rt.size > 1:
            self._replica = self.rt.alloc_multicast(self.size * self.esz) or self.rt.alloc_symm(self.size * self.esz)

    def staging(self) -> torch.Tensor:
        """Zero-copy Add: write your delta into the returned full-size tensor, then call
        ``add(staged=True)``; the fused kernel reads it in place over NVLink."""
        self._cur_stage = self._stage_buf()
        return self._cur_stage.tensor(self.dtype, self.size)

    def _as_device(self, data) -> torch.Tensor:
        t = torch.as_tensor(data)
        if t.dtype != self.dtype:
            t = t.to(self.dtype)
        if t.device != self.rt.device:
            t = t.to(self.rt.device, non_blocking=True)
        return t.contiguous().view(-1)

    def _collective(self) -> bool:
        """BSP (or one process): owner-side fused reduce-scatter + updater. Async: one-sided
        pushes (red.add for stateless updaters, remote read-modify-write for stateful ones), so
        workers need not call add() in lockstep -- the reference's async-server contract."""
        if self.rt.size == 1 or self.sync:
            return True
        return not bool(FLAGS.get("async_one_sided"))

    # ------------------------------------------------------------------ Add (whole table)
    def add(self, delta=None, option: Optional[AddOption] = None, staged: bool = False) -> None:
        self.wait(self.add_async(delta, option, staged))

    def add_async(self, delta=None, option: Optional[AddOption] = None, staged: bool = False) -> int:
        rt, lib = self.rt, N.cuda_lib()
        opt = option or AddOption()
        check_add_option(self.updater_name, opt)
        nbytes = self.size * self.esz
        with monitor("WORKER_TABLE_ADD", cuda=True, nbytes=nbytes):
            if rt.size == 1:
                src = self._cur_stage.tensor(self.dtype, self.size) if staged else self._as_device(delta)
                self._launch_fused([src.data_ptr()], [opt], pads=False)
                self._keep = src
            elif self._collective():
                if not staged:
                    buf = self._stage_buf()
                    if rt.is_worker():
                        buf.tensor(self.dtype, self.size).copy_(self._as_device(delta))
                else:
                    buf = self._cur_stage
                # The option travels with the request (reference: last Blob of Request_Add): this worker's
                # AddOption is published through the symmetric option boxes inside the fused kernel, right
                # before its ready flag; every owner applies worker w's delta with worker w's option.
                opts = [opt] * self.W
                ptrs = [buf.ptrs[rt.worker_id_to_rank(w)] for w in range(self.W)]
                # NVLS: when the staging is multicast-bound and every rank is a worker the owner
                # reduces its slice inside the switch instead of pulling W copies
                mc = getattr(buf, "multicast_ptr", 0) if rt.num_workers() == rt.size else 0
                self._launch_fused(ptrs, opts, pads=True, multicast=mc)
            else:
                src = self._as_device(delta)
                sp = (C.c_void_p * self.S)(*self.shard_ptrs)
                so = (C.c_int64 * self.S)(*self.offs)
                sl = (C.c_int64 * self.S)(*self.lens)
                if self.updater in (N.UPD_DEFAULT, N.UPD_SGD) or self.dtype in (torch.int32, torch.int64):
                    sign = -1.0 if self.updater == N.UPD_SGD else 1.0
                    lib.mvb_push_dense_red(self.dcode, src, self.S, sp, so, sl, sign, N.stream_ptr())
                else:
                    ranks = [rt.server_id_to_rank(s) for s in range(self.S)]
                    s0 = (C.c_void_p * self.S)(*[self._state_bufs[0].ptrs[r] for r in ranks])
                    s1 = (C.c_void_p * self.S)(*[(self._state_bufs[1].ptrs[r] if self.n_states > 1 else 0)
                                                  for r in ranks])
                    ss = (C.c_int64 * self.S)(*self.state_strides)
                    ao = _opt_struct(opt)
                    ao.worker_id = max(rt.worker_id(), 0)
                    if self.updater == N.UPD_ADAM:
                        lib.mvb_push_dense_adam(self.dcode, self.updater, src, self.S, sp, s0, s1, so, sl, ss,
                                                self.num_col, ao, rt.rank, N.stream_ptr())
                    elif self.state_per_row:
                        lib.mvb_push_dense_rowwise(self.dcode, self.updater, src, self.S, sp, s0, so, sl, ss,
                                                   self.num_col, ao, rt.rank, N.stream_ptr())
                    else:
                        lib.mvb_push_dense_stateful(self.dcode, self.updater, src, self.S, sp, s0, s1, so, sl, ss, ao,
                                                    rt.rank, N.stream_ptr())
                self._keep = src
            if rt.is_worker():
                self._note_add()
        return self._record()

    def _note_add(self) -> None:
        if self._ver is not None:
            N.cuda_lib().mvb_stale_on_add(self._ver_ptrs, self.S, self._ver_last, self._ver_adds,
                                          self.staleness_hist, 64, N.stream_ptr())

    def _note_get(self) -> None:
        if self._ver is not None:
            N.cuda_lib().mvb_stale_on_get(self._ver_ptrs, self.S, self._ver_last, self._ver_adds, N.stream_ptr())

    def _opt_box_buf(self):
        """Symmetric option boxes (2 generations x MAX_RANKS AddOptions per rank); allocated at the first
        collective Add, which every rank reaches together."""
        b = self._opt_box
        if b is None:                       # async table used collectively (e.g. an explicit staged Add)
            b = self.rt.alloc_symm(2 * N.MAX_RANKS * 32)
            b.tensor(torch.uint8).zero_()
            torch.cuda.synchronize()
            self.rt.barrier()
            self._opt_box = b
        return b

    def _launch_fused(self, delta_ptrs: Sequence[int], opts: Sequence[AddOption], pads: bool,
                      serve_only: bool = False, multicast: int = 0) -> None:
        rt, lib = self.rt, N.cuda_lib()
        a = N.DenseAdd()
        a.dtype, a.updater = self.dcode, self.updater
        a.shard = self.shard_buf.local_ptr
        a.state0 = self.state[0].data_ptr() if self.n_states >= 1 else None
        a.state1 = self.state[1].data_ptr() if self.n_states >= 2 else None
        a.shard_len, a.shard_off, a.state_stride = self.my_len, self.my_off, self.state_stride
        a.num_col = self.num_col
        nw = len(delta_ptrs)
        a.nworkers = nw
        a.worker_mask = (1 << nw) - 1
        for w in range(nw):
            a.delta_ptrs[w] = delta_ptrs[w]
            a.opts[w] = _opt_struct(opts[w])
            a.opts[w].worker_id = w
            a.worker_rank[w] = rt.worker_id_to_rank(w) if rt.size > 1 else 0
        a.scale, a.clip = 1.0, 0.0
        a.my_worker = rt.worker_id() if rt.size > 1 else 0
        if pads and rt.size > 1:
            box = self._opt_box_buf()
            for r in range(rt.size):
                a.opt_box[r] = box.ptrs[r]
        a.delta_multicast = multicast or None
        if pads and self._replica is not None:
            for r in range(rt.size):
                a.replica_ptrs[r] = self._replica.ptrs[r]
            a.replica_multicast = getattr(self._replica, "multicast_ptr", 0) or None
            self._replica_epoch = self.add_epoch + 1
        self._pads_arr = rt.pads_array() if pads else None
        a.pads = C.cast(self._pads_arr, C.POINTER(C.c_void_p)) if pads else None
        a.me, a.world = rt.rank, rt.size
        a.ch_ready, a.ch_done = self.ch_ready, self.ch_done
        if pads:
            self.add_epoch += 1
        a.epoch = self.add_epoch
        a.is_worker = 1 if (rt.is_worker() and not serve_only and not self._finished) else 0
        a.err_flag = rt.err_flag.data_ptr()
        a.fin_flag = self._fin.data_ptr()
        a.done_counter = self._done_counter
        a.timeout_s = float(FLAGS.get("barrier_timeout_s"))
        lib.mvb_add_dense_fused(a, N.stream_ptr())

    # ------------------------------------------------------------------ Get (whole table)
    def get(self, out: Optional[torch.Tensor] = None, option: Optional[GetOption] = None) -> torch.Tensor:
        h, out = self._get_async(out)
        self.wait(h)
        return out

    def get_async(self, out: Optional[torch.Tensor] = None, option: Optional[GetOption] = None):
        return self._get_async(out)

    def _get_async(self, out):
        rt, lib = self.rt, N.cuda_lib()
        if self._replica is not None and self._replica_epoch == self.add_epoch and self.add_epoch > 0:
            # fused Add -> Get: the owners already pushed epoch `add_epoch` into our replica
            mask = 0
            for s_ in range(self.S):
                mask |= 1 << rt.server_id_to_rank(s_)
            with monitor("WORKER_TABLE_GET", cuda=True, nbytes=self.size * self.esz):
                lib.mvb_wait(rt.pads_array(), rt.rank, rt.size, self.ch_done, self.add_epoch, mask, rt.err_flag,
                             float(FLAGS.get("barrier_timeout_s")), N.stream_ptr())
                rep = self._replica.tensor(self.dtype, self.size)
                if out is None:
                    out = rep.clone()
                else:
                    out.view(-1).copy_(rep)
            return self._record(), out
        if out is None:
            out = torch.empty(self.size, dtype=self.dtype, device=rt.device)
        flat = out.view(-1)
        assert flat.numel() == self.size and flat.dtype == self.dtype and flat.is_cuda
        g = N.DenseGet()
        g.dtype, g.out, g.nservers = self.dcode, flat.data_ptr(), self.S
        for s in range(self.S):
            g.shard_ptrs[s] = self.shard_ptrs[s]
            g.shard_offs[s] = self.offs[s]
            g.shard_lens[s] = self.lens[s]
            g.server_rank[s] = rt.server_id_to_rank(s) if rt.size > 1 else 0
        use_pads = rt.size > 1 and self._collective() and self.add_epoch > 0
        self._gpads = rt.pads_array() if use_pads else None
        g.pads = C.cast(self._gpads, C.POINTER(C.c_void_p)) if use_pads else None
        g.me, g.world, g.ch_done, g.epoch = rt.rank, rt.size, self.ch_done, self.add_epoch
        g.err_flag = rt.err_flag.data_ptr()
        g.timeout_s = float(FLAGS.get("barrier_timeout_s"))
        self._note_get()        # versions as of the start of the pull (a conservative read point)
        with monitor("WORKER_TABLE_GET", cuda=True, nbytes=self.size * self.esz):
            lib.mvb_get_dense(g, N.stream_ptr())
        return self._record(), out

    # ------------------------------------------------------------------ BSP shutdown
    def needs_drain(self) -> bool:
        return self.sync and self.rt.size > 1 and bool(self._stage) and not self._finished

    def finish_train(self) -> None:
        self.rt._finish_train()

    def publish_finish(self) -> None:
        """Server_Finish_Train: leave EPOCH_FIN in this worker's ready slot on every rank so
        it never gates a BSP epoch again (src/server.cpp:190-213)."""
        rt, lib = self.rt, N.cuda_lib()
        self._finished = True
        if rt.is_worker() and any(getattr(b, "multicast_ptr", 0) for b in self._stage):
            # NVLS adds sum EVERY rank's staging in the switch and cannot mask a finished worker:
            # once all owners have consumed our last Add, leave zeros behind.
            if self.add_epoch > 0:
                mask = 0
                for s_ in range(self.S):
                    mask |= 1 << rt.server_id_to_rank(s_)
                lib.mvb_wait(rt.pads_array(), rt.rank, rt.size, self.ch_done, self.add_epoch, mask, rt.err_flag,
                             float(FLAGS.get("barrier_timeout_s")), N.stream_ptr())
            for b in self._stage:
                b.tensor(torch.uint8).zero_()
        if rt.is_worker():
            lib.mvb_signal(rt.pads_array(), rt.rank, rt.size, self.ch_ready, N.EPOCH_FIN, N.stream_ptr())

    def drain_step(self, pads_host) -> str:
        """One polling step of the owner-side drain: 'done' when every worker finished,
        'served' after applying one more epoch for the still-active workers, else 'wait'."""
        rt = self.rt
        flags = [int(pads_host[self.ch_ready * N.MAX_RANKS + rt.worker_id_to_rank(w)])
                 for w in range(self.W)]
        if all(f >= N.EPOCH_FIN for f in flags):
            return "done"
        nxt = self.add_epoch + 1
        if all(f >= nxt for f in flags):
            buf = self._stage[self.add_epoch % 2]   # staging parity of epoch nxt
            ptrs = [buf.ptrs[rt.worker_id_to_rank(w)] for w in range(self.W)]
            self._launch_fused(ptrs, [AddOption(0)] * self.W, pads=True, serve_only=True)
            torch.cuda.current_stream().synchronize()
            rt.check_watchdog()
            return "served"
        return "wait"

    def free(self) -> None:
        for b in [self.shard_buf] + list(self._stage) + list(self._state_bufs) + \
                ([self._replica] if self._replica is not None else []):
            self.rt.release_symm(b)
        self._stage = []
        self.shard = None

    # ------------------------------------------------------------------ checkpoint
    def store(self, stream) -> None:
        """Serializable::Store: raw dump of the local shard (array_table.cpp:143-151), followed
        by the updater state slabs (not saved by the reference, SURVEY Q14)."""
        torch.cuda.current_stream().synchronize()
        stream.write(self.shard.cpu().numpy().tobytes())
        for st in self.state:
            stream.write(st.cpu().numpy().tobytes())

    def load(self, stream) -> None:
        import numpy as np
        npdt = {torch.float32: np.float32, torch.float64: np.float64, torch.int32: np.int32,
                torch.int64: np.int64}[self.dtype]
        raw = stream.read(self.my_len * self.esz)
        if self.my_len:
            self.shard.copy_(torch.from_numpy(np.frombuffer(raw, dtype=npdt).copy()).to(self.rt.device))
        for st in self.state:
            raw = stream.read(st.numel() * self.esz)
            if len(raw) == st.numel() * self.esz:
                st.copy_(torch.from_numpy(np.frombuffer(raw, dtype=npdt).copy()).to(self.rt.device))


class RowMailbox:
    """Row mailboxes of one fp32 matrix table (csrc/cuda/rowbox.cu): the device-side row Add with
    owner-side apply.  One slot per (owner, source) in the owner's HBM, doorbell + ack flags in
    symmetric memory.  ``push_*`` is one-sided and asynchronous; ``drain`` applies, on the owner,
    every push that has arrived (``wait=True``: the next push of every source) through the table's
    updater with the SOURCE's AddOption -- exactly once per (worker,row), no host barrier, workers
    may push different numbers of times (reference: Server::ProcessAdd, src/server.cpp:48-58).

    Construction is collective (symmetric allocation); everything afterwards is not."""

    def __init__(self, table: "MatrixDeviceTable"):
        rt = table.rt
        assert table.dtype == torch.float32 and table.num_col % 4 == 0
        assert table.S == rt.size and table.W == rt.size, "row mailboxes need every rank to be worker + server"
        self.t, self.rt = table, rt
        S = table.S
        self.cap = max(hi - lo for lo, hi in zip(table.row_lo, table.row_hi))
        lib = N.cuda_lib()
        self.slot_bytes = (lib.mvb_rowbox_slot_bytes(self.cap, table.num_col) + 255) // 256 * 256
        self.nslots = lib.mvb_rowbox_slots()
        self.box = rt.alloc_symm(S * self.nslots * self.slot_bytes)
        self.ack = rt.alloc_symm(8 * N.MAX_RANKS)
        self.box.tensor(torch.uint8)[:S * self.nslots * self.slot_bytes].zero_()   # seq = 0, and no stale rows
        self.ack.tensor(torch.int64).zero_()
        dev = rt.device
        self.seg = torch.zeros(S + 1, dtype=torch.int32, device=dev)
        self.done = torch.zeros(2, dtype=torch.int32, device=dev)
        self.applied = torch.zeros(S, dtype=torch.int64, device=dev)
        self.go = torch.zeros(S, dtype=torch.int32, device=dev)
        self.epoch = 0                       # my pushes so far
        self.drain_stream = torch.cuda.Stream(device=dev)
        b = N.RowBox()
        b.map = table._rowmap
        b.me, b.cap, b.slot_bytes = rt.rank, self.cap, self.slot_bytes
        b.box, b.ack = self.box.ptr_array(), self.ack.ptr_array()
        b.seg, b.done = self.seg.data_ptr(), self.done.data_ptr()
        b.applied, b.go = self.applied.data_ptr(), self.go.data_ptr()
        b.err_flag = rt.err_flag.data_ptr()
        b.timeout_s = float(FLAGS.get("barrier_timeout_s"))
        self.c = b
        torch.cuda.synchronize()
        rt.barrier()
        rt.barrier_hooks.append(self._barrier_hook)

    def _barrier_hook(self, final: bool) -> None:
        # final: every rank's pushes are complete (they synchronised their streams before the barrier):
        # one more drain applies the at most one outstanding push per source, and the host waits for it
        for _ in range(self.nslots if final else 1):       # at most `nslots` outstanding pushes per source
            self.drain(wait=False)
        if final:
            self.drain_stream.synchronize()

    def push_delta(self, ids32: torch.Tensor, n_ptr: int, n_max: int, cur: torch.Tensor, old: torch.Tensor,
                   scale: float, option: Optional[AddOption] = None, ctas_per_sm: int = 1) -> None:
        """rows[ids] += (cur - old) * scale at their owners (ids ascending int32; count read on the device)."""
        self.epoch += 1
        ao = _opt_struct(option or AddOption())
        N.cuda_lib().mvb_rowbox_push_delta(self.c, ids32, n_ptr, n_max, cur, old, cur.stride(0), scale, self.epoch, ao,
                                           ctas_per_sm, N.stream_ptr())

    def push_vals(self, ids32: torch.Tensor, vals: torch.Tensor, option: Optional[AddOption] = None,
                  scale: float = 1.0, ctas_per_sm: int = 1) -> None:
        check_add_option(self.t.updater_name, option or AddOption())
        self.epoch += 1
        ao = _opt_struct(option or AddOption())
        N.cuda_lib().mvb_rowbox_push_vals(self.c, ids32, None, ids32.numel(), vals, vals.stride(0), scale, self.epoch,
                                          ao, ctas_per_sm, N.stream_ptr())

    def drain(self, wait: bool = False, ctas_per_sm: int = 1, stream=None) -> None:
        """Owner side: apply what has arrived (wait=False) or the next push of every source (wait=True).
        Enqueued on ``stream`` (default: the mailbox's own drain stream, so that a push spinning for an
        ack on the caller's stream can never block the drain that produces the peer's ack)."""
        t, lib = self.t, N.cuda_lib()
        st = stream if stream is not None else self.drain_stream
        sp = st.cuda_stream
        lib.mvb_rowbox_poll(self.c, -1, 1 if wait else 0, sp)
        for w in range(t.S):
            lib.mvb_rowbox_apply(self.c, t.updater, t.shard_buf.local_ptr, t._sp(0), t._sp(1), t.state_stride,
                                 t.row_lo[t.sid], w, ctas_per_sm, sp)

    def launches_per_drain(self) -> int:
        return 1 + self.t.S


class ArrayDeviceTable(DenseDeviceTable):
    """ArrayTable<T>: dense 1-D, whole-table ops (any size >= 1, SURVEY Q5)."""

    def __init__(self, size: int, dtype="float32", updater=None, init_value=None):
        super().__init__(int(size), 1, dtype, updater, init_value)
        # whole-table ops only => the fused Add -> Get replica is always coherent in BSP mode
        if self.sync and self.rt.size > 1 and bool(FLAGS.get("replicate_get")):
            self.enable_replica()
            self.rt.barrier()


class MatrixDeviceTable(DenseDeviceTable):
    """MatrixTable<T> / Matrix<T> / SparseMatrixTable<T>: dense 2-D, row addressable.

    ``is_sparse`` enables the reference's delta-pull protocol (src/table/matrix.cpp:421-572):
    every Add marks the touched rows stale for all workers (T4 behaviour, Q13) and
    ``get_stale()`` returns only the rows that changed since this worker's last pull; an
    explicit empty result replaces the reference's row-0 placeholder (Q12).  Whole-table adds
    skip all-zero rows when marking (matrix.cpp:151-164)."""

    def __init__(self, num_row: int, num_col: int, dtype="float32", updater=None, init_value=None,
                 min_value=None, max_value=None, is_sparse: bool = False, is_pipeline: bool = False,
                 seed: int = 1):
        self.is_sparse, self.is_pipeline = bool(is_sparse), bool(is_pipeline)
        super().__init__(num_row, num_col, dtype, updater, init_value, min_value, max_value, seed)
        rt = self.rt
        self._rowmap = N.RowMap()
        self._rowmap.num_row, self._rowmap.num_col = self.num_row, self.num_col
        self._rowmap.nservers = self.S
        self._rowmap.rows_per_server = self.rps
        for s in range(self.S):
            self._rowmap.shard_ptrs[s] = self.shard_ptrs[s]
        self._mailbox = None
        # async + stateful updater: row Adds go through the row mailboxes (owner-side apply on the device,
        # one-sided, no lockstep).  Collective allocation, hence decided here, at table creation.
        if (rt.size > 1 and not self.sync and self.updater not in (N.UPD_DEFAULT, N.UPD_SGD)
                and self.dtype == torch.float32 and self.num_col % 4 == 0 and self.S == rt.size and self.W == rt.size
                and str(FLAGS.get("row_mailbox")).lower() not in ("0", "false")):
            self.enable_row_mailbox()
        self._stale = None
        if self.is_sparse:
            nslots = self.W * (2 if self.is_pipeline else 1)
            # the stale bitmap is replicated: each rank tracks rows it has itself seen change
            # through Adds issued anywhere (marks are pushed by the adder to every rank's copy)
            self._stale_buf = rt.alloc_symm(nslots * self.num_row)
            self._stale = self._stale_buf.tensor(torch.uint8, nslots * self.num_row)
            self._stale.fill_(1)           # everything is stale before the first Get
            self._nslots = nslots
            rt.barrier()

    def enable_row_mailbox(self) -> "RowMailbox":
        """Collective: allocate the row mailboxes of this table (idempotent)."""
        if self._mailbox is None:
            self._mailbox = RowMailbox(self)
        return self._mailbox

    def drain_rows(self, wait: bool = False) -> None:
        """Owner side of the mailbox protocol: apply the row Adds that have arrived from any worker."""
        if self._mailbox is not None:
            self._mailbox.drain(wait=wait)

    def wait(self, handle: int) -> None:
        if self._mailbox is None:
            return super().wait(handle)
        # a push may be spinning for a peer's ack while that peer spins for mine: keep serving my
        # mailboxes while waiting (the reference's server actor never stops either)
        import time
        ev = self._events.pop(handle, None)
        while ev is not None and not ev.query():
            self._mailbox.drain(wait=False)
            time.sleep(1e-4)
        Runtime.get().check_watchdog()

        # ---- ids helper --------------------------------------------------------------------
    def _ids(self, row_ids) -> torch.Tensor:
        t = torch.as_tensor(row_ids)
        if t.dtype != torch.int64:
            t = t.to(torch.int64)
        if t.device != self.rt.device:
            t = t.to(self.rt.device, non_blocking=True)
        return t.contiguous().view(-1)

    # ---- row Get -----------------------------------------------------------------------
    def get_rows(self, row_ids, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        h, out = self.get_rows_async(row_ids, out)
        self.wait(h)
        return out

    def get_rows_async(self, row_ids, out: Optional[torch.Tensor] = None):
        lib = N.cuda_lib()
        ids = self._ids(row_ids)
        k = ids.numel()
        if out is None:
            out = torch.empty(k, self.num_col, dtype=self.dtype, device=self.rt.device)
        assert out.is_cuda and out.dtype == self.dtype and out.stride(-1) == 1
        ld = out.stride(0) if out.dim() == 2 else self.num_col
        with monitor("WORKER_TABLE_GET_ROWS", cuda=True, nbytes=k * self.num_col * self.esz):
            lib.mvb_get_rows(self.dcode, self._rowmap, ids, k, out, ld, N.stream_ptr())
        self._keep_ids = ids
        return self._record(), out

    def get_row(self, row_id: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self.get_rows([row_id], None if out is None else out.view(1, -1)).view(-1)

    # ---- row Add -----------------------------------------------------------------------
    def add_rows(self, row_ids, values, option: Optional[AddOption] = None) -> None:
        self.wait(self.add_rows_async(row_ids, values, option))

    def add_rows_async(self, row_ids, values, option: Optional[AddOption] = None) -> int:
        rt, lib = self.rt, N.cuda_lib()
        ids = self._ids(row_ids)
        k = ids.numel()
        vals = torch.as_tensor(values)
        if vals.dtype != self.dtype:
            vals = vals.to(self.dtype)
        if vals.device != rt.device:
            vals = vals.to(rt.device, non_blocking=True)
        vals = vals.contiguous().view(k, self.num_col)
        opt = option or AddOption()
        check_add_option(self.updater_name, opt)
        with monitor("WORKER_TABLE_ADD_ROWS", cuda=True, nbytes=k * self.num_col * self.esz):
            if self.updater in (N.UPD_DEFAULT, N.UPD_SGD):
                sign = -1.0 if self.updater == N.UPD_SGD else 1.0
                lib.mvb_add_rows_red(self.dcode, self._rowmap, ids, k, vals, self.num_col, sign, N.stream_ptr())
            else:
                self._add_rows_stateful(ids, vals, opt)
            if self.is_sparse:
                self._mark_stale(ids)
        self._keep_rows = (ids, vals)
        return self._record()

    def add_rows_delta(self, row_ids: torch.Tensor, cur: torch.Tensor, old: torch.Tensor, scale: float) -> None:
        """Fused AddDeltaParameter: rows += (cur - old) * scale, pushed one-sided into the owners
        (default/sgd updaters, fp32, num_col % 4 == 0). No delta tensor is materialised."""
        assert self.updater in (N.UPD_DEFAULT, N.UPD_SGD) and self.dtype == torch.float32
        ids = self._ids(row_ids)
        k = ids.numel()
        sign = -1.0 if self.updater == N.UPD_SGD else 1.0
        with monitor("WORKER_TABLE_ADD_ROWS", cuda=True, nbytes=k * self.num_col * self.esz):
            N.cuda_lib().mvb_add_rows_delta(self._rowmap, ids, k, cur, old, cur.stride(0), sign * scale,
                                            N.stream_ptr())
            if self.is_sparse:
                self._mark_stale(ids)
        self._keep_rows = (ids, cur, old)

    def add_row(self, row_id: int, values, option: Optional[AddOption] = None) -> None:
        self.add_rows([row_id], torch.as_tensor(values).view(1, -1), option)

    def _add_rows_stateful(self, ids, vals, opt: AddOption) -> None:
        """Stateful updaters must be applied by the owner exactly once per (worker,row): the
        request (ids, values) is published in symmetric staging, every owner scans all
        workers' requests in worker order (collective, like the dense fused path)."""
        rt, lib = self.rt, N.cuda_lib()
        k = ids.numel()
        if self._mailbox is not None:
            # device-side path: ids outside the table become -1 (an id >= 2^31 must not wrap to a row in the int32
            # list), then a stable sort makes each owner's entries one contiguous range and keeps the entries of a
            # repeated row in list order; one-sided pushes into the owners' mailboxes, then serve my own mailboxes
            ids = torch.where((ids >= 0) & (ids < self.num_row), ids, -1)
            ids, order = torch.sort(ids, stable=True)
            ids32, vals = ids.to(torch.int32), vals[order]
            # a slot holds `cap` entries per source, so a longer list goes in pushes of at most `cap` entries, in
            # order. The push of chunk c waits on the device for every owner's ack of chunk c - 2, and this rank's
            # own ack comes only from its own drain: wait() serves this rank's mailboxes until chunk c's push has
            # completed, so chunk c - 2 (complete before chunk c starts, same stream) is drained before it is needed
            cap = self._mailbox.cap
            for c0 in range(0, k, cap):
                if c0:
                    self.wait(self._record())
                self._mailbox.push_vals(ids32[c0:c0 + cap], vals[c0:c0 + cap], opt)
                self._mailbox.drain(wait=False)
            self._keep_push = (ids32, vals)
            return
        # a repeated row is applied once per occurrence, in list order (MatrixServerTable::ProcessAdd): the
        # owner kernel walks each run of equal ids on one warp, so make the runs adjacent without reordering
        # them (stable sort); staged requests are sorted too, so every owner sees the same order
        ids, order = torch.sort(ids, stable=True)
        vals = vals[order]
        self._keep_sorted = (ids, vals)
        st = N.stream_ptr()
        ao = _opt_struct(opt)
        if rt.size == 1:
            ao.worker_id = 0
            lib.mvb_add_rows_owner(self.dcode, self.updater, self.shard_buf.local_ptr, self._sp(0), self._sp(1),
                                   self.row_lo[0], self.row_hi[0], self.num_col, self.state_stride, ids, k, vals,
                                   self.num_col, ao, st)
            return
        counts = rt.all_gather_object(int(k))
        cap = max(max(counts), 1)
        if getattr(self, "_row_stage_cap", 0) < cap:
            self._row_stage_ids = rt.alloc_symm(cap * 8)
            self._row_stage_vals = rt.alloc_symm(cap * self.num_col * self.esz)
            self._row_stage_cap = cap
        else:
            rt.barrier()   # previous round's readers are done before we overwrite staging
        if k:
            self._row_stage_ids.tensor(torch.int64, k).copy_(ids)
            self._row_stage_vals.tensor(self.dtype, k * self.num_col).copy_(vals.view(-1))
        rt.barrier()
        if self.sid >= 0:
            for w in range(self.W):
                r = rt.worker_id_to_rank(w)
                if counts[r] == 0:
                    continue
                ao.worker_id = w
                lib.mvb_add_rows_owner(self.dcode, self.updater, self.shard_buf.local_ptr, self._sp(0), self._sp(1),
                                       self.row_lo[self.sid], self.row_hi[self.sid], self.num_col, self.state_stride,
                                       self._row_stage_ids.ptrs[r], counts[r], self._row_stage_vals.ptrs[r],
                                       self.num_col, ao, st)
        rt.barrier()

    def _sp(self, i):
        return self.state[i] if self.n_states > i else None

    # ---- whole-table ops honour the sparse bookkeeping ----------------------------------
    def add_async(self, delta=None, option=None, staged=False) -> int:
        if self.is_sparse and not staged and delta is not None:
            lib = N.cuda_lib()
            d = self._as_device(delta)
            mask = torch.empty(self.num_row, dtype=torch.uint8, device=self.rt.device)
            lib.mvb_row_nonzero_mask(self.dcode, d, self.num_row, self.num_col, self.num_col, mask, N.stream_ptr())
            h = super().add_async(d, option, False)
            self._mark_stale(mask.nonzero().view(-1))
            return h
        return super().add_async(delta, option, staged)

    def _mark_stale(self, ids: torch.Tensor) -> None:
        lib = N.cuda_lib()
        k = ids.numel()
        if k == 0:
            return
        for r in range(self.rt.size):
            lib.mvb_stale_mark(self._stale_buf.ptrs[r], self.num_row, self._nslots, ids, k, N.stream_ptr())
        self._keep_mark = ids

    def get_stale(self, option: Optional[GetOption] = None, slot: int = 0):
        """Delta pull: (row_ids, rows) that changed since this worker's previous pull.
        ``option.worker_id == -1`` returns every row (matrix.cpp:460-514)."""
        lib = N.cuda_lib()
        wid = (option.worker_id if option else self.rt.worker_id())
        if not self.is_sparse or wid < 0:
            ids = torch.arange(self.num_row, device=self.rt.device)
            return ids, self.get_rows(ids)
        w = wid + (self.W if (self.is_pipeline and slot) else 0)
        mine = self._stale[w * self.num_row:(w + 1) * self.num_row]
        mask = torch.empty(self.num_row, dtype=torch.uint8, device=self.rt.device)
        lib.mvb_stale_take(mine, self.num_row, None, -1, mask, N.stream_ptr())
        ids = mask.nonzero().view(-1)
        if ids.numel() == 0:
            return ids, torch.empty(0, self.num_col, dtype=self.dtype, device=self.rt.device)
        return ids, self.get_rows(ids)


INT64_MIN = -(1 << 63)


def raise_hash_status(code: int, tables: Sequence["HashMatrixTable"]) -> None:
    """Raise the error of a non-zero status word of ``mvb_hash_rows_lookup`` (``tables``: by descriptor index)."""
    if not code:
        return
    kind, t, server = code >> 40, (code >> 8) & 0xFFFFFFFF, code & 0xFF
    tid = tables[t].table_id if t < len(tables) else "?"
    if kind == N.HASH_BAD_KEY:
        raise ValueError(f"HashMatrixTable #{tid}: key {INT64_MIN} (INT64_MIN) is reserved for empty slots")
    if kind == N.HASH_FULL:
        tab = tables[t] if t < len(tables) else None
        limit = f" (at most {7 * tab.slots // 8} keys per server)" if tab is not None else ""
        raise RuntimeError(f"HashMatrixTable #{tid}: table full on server {server}{limit}; keys inserted before "
                           "stay valid")
    if kind == N.HASH_TIMEOUT:
        raise RuntimeError(f"HashMatrixTable #{tid}: timed out waiting for a row of server {server} to be "
                           "initialised (-barrier_timeout_s)")
    raise RuntimeError(f"HashMatrixTable #{tid}: lookup status {code:#x}")


def check_admit_after(admit_after) -> None:
    """``admit_after`` of a HashMatrixTable: an int in [1, 2^31) (TypeError / ValueError otherwise)."""
    if isinstance(admit_after, bool) or not isinstance(admit_after, int):
        raise TypeError(f"HashMatrixTable: admit_after must be an int, got {type(admit_after).__name__}")
    if not 1 <= admit_after < 1 << 31:
        raise ValueError(f"HashMatrixTable: admit_after must be in [1, 2^31), got {admit_after}")


class HashMatrixTable(MatrixDeviceTable):
    """Rows keyed by any int64 (but INT64_MIN), one row per distinct key, allocated on first lookup.

    A ``MatrixDeviceTable`` of ``S P + 1`` fp32 rows plus a device hash index (``csrc/cuda/hash_rows.cu``): server
    ``s = key mod S`` owns the key, and the ``P`` slots of server ``s`` are rows ``[s P, (s + 1) P)``. The last row is
    the zero row, which every missing key reads and which no key ever gets. ``P`` is the smallest power of two with
    ``floor(7 P / 8) >= ceil(capacity / S)``, so each server holds at most ``floor(7 P / 8)`` keys; an insert beyond
    that raises "table full" and leaves the keys inserted before valid.

    ``lookup`` translates keys to rows; the inherited row ops (``get_rows``, ``add_rows``, the updaters, row
    mailboxes) then work on them unchanged. ``get`` and ``add`` take keys, like the KVTable's; the whole-table
    dense ``get`` / ``add`` are not offered, because their layout is the slot layout.

    A key's initial row depends on the key only: ``init_value`` (default 0) in every column, or, with
    ``min_value`` and ``max_value``, ``lo + u (hi - lo)`` with ``u`` drawn from ``(key, seed, column)``. Which slot
    (row id) a key gets depends on the order in which keys arrive, which may depend on timing; nothing else does.

    ``track_access=True`` keeps a last-seen stamp per key: every lookup that inserts (a training forward of
    ``PSEmbedding`` / ``PSEmbeddingCollection``, ``lookup(insert=True)``, ``add``) raises the stamp of each key it
    touches to this rank's ``clock``, a user-defined int64 time (a step, an hour, ...). Reads (``get``,
    ``lookup(insert=False)``, eval-mode layers) stamp nothing. ``evict`` removes idle keys (``older_than``) or listed
    keys and frees their slots, so a table of fixed capacity can serve a stream of new ids. It costs one int64 per
    slot and an atomic per key and clock value.

    ``admit_after=n >= 2`` turns on count-based admission: an inserting lookup gives a missing key a slot only once
    the key's estimated count reaches ``n``. Until then the key behaves as a missing key does in eval mode: it reads
    the zero row, takes no slot, initial row, updater state or stamp, and is not an error; ``PSEmbedding`` and
    ``PSEmbeddingCollection`` push nothing for it, ``add`` drops its values. Every occurrence of a missing key in an
    inserting call (a training forward, ``lookup(insert=True)``, ``add``) counts once; keys holding a slot and
    lookups that do not insert count nothing. A call counts all its occurrences before it admits any, so a key at
    ``n - 2`` seen twice in a batch is admitted in that batch, and on one rank every occurrence of a key in a call
    gets the same row. While other ranks count concurrently, an occurrence may read zeros (and push nothing) in the
    call in which another occurrence of the same key is admitted. The count is a count-min sketch per server
    (4 rows of ``slots`` uint32 counters, 16 bytes per slot, in symmetric memory): it never under-counts, so no key
    is admitted below ``n``; a key never seen before reads at least 1 too many with probability below 2.5 %. Every
    server halves its counters once ``slots / 2`` occurrences have been counted there since the last halving, so
    counts of keys that stopped arriving fade. ``admit_after=1`` (the default) is the table without admission."""

    def __init__(self, capacity: int, num_col: int, dtype="float32", updater: Optional[str] = None,
                 init_value=None, min_value=None, max_value=None, seed: int = 1, track_access: bool = False,
                 admit_after: int = 1):
        check_admit_after(admit_after)
        rt = Runtime.get()
        if not rt.started:
            Log.fatal("MV_Init must be called before creating tables")
        if _torch_dtype(dtype) != torch.float32:
            raise TypeError(f"HashMatrixTable: rows are float32, got {dtype}")
        capacity, num_col = int(capacity), int(num_col)
        if capacity < 1:
            raise ValueError(f"HashMatrixTable: capacity must be >= 1, got {capacity}")
        if num_col < 1 or num_col % 4:
            raise ValueError(f"HashMatrixTable: num_col must be a positive multiple of 4 (16-byte row "
                             f"initialisation), got {num_col}")
        S = max(rt.num_servers(), 1)
        per_server = -(-capacity // S)
        P = 2
        while 7 * P // 8 < per_server:
            P *= 2
        self.capacity, self.slots = capacity, P
        super().__init__(S * P + 1, num_col, "float32", updater)
        lib = N.cuda_lib()
        self._keys_buf = rt.alloc_symm(P * 8)
        self._ready_buf = rt.alloc_symm(P * 4)
        self._count_buf = rt.alloc_symm(8)
        lib.mvb_hash_rows_init(self._keys_buf.local_ptr, self._ready_buf.local_ptr, self._count_buf.local_ptr, P,
                               N.stream_ptr())
        h = N.HashRows()
        h.nservers, h.slots = self.S, P
        for s in range(self.S):
            r = rt.server_id_to_rank(s) if rt.num_servers() else rt.rank
            h.keys[s], h.ready[s], h.count[s] = self._keys_buf.ptrs[r], self._ready_buf.ptrs[r], self._count_buf.ptrs[r]
        h.map = self._rowmap
        if min_value is not None and max_value is not None:
            h.init, h.lo, h.hi = N.HASH_INIT_UNIFORM, float(min_value), float(max_value)
        else:
            h.init, h.init_value = N.HASH_INIT_CONST, float(init_value or 0.0)
        h.seed = int(seed) & ((1 << 64) - 1)
        self.track_access = bool(track_access)
        self._ls_buf = None
        if self.track_access:
            # P stamps per server plus one word that stays 0: the stamp of the zero row for last_seen()
            self._ls_buf = rt.alloc_symm((P + 1) * 8)
            self._ls_buf.tensor(torch.int64, P + 1).zero_()
            self._clock = torch.zeros(1, dtype=torch.int64, device=rt.device)
            self._clock_value = 0
            self._ls_map = N.RowMap()
            self._ls_map.num_row, self._ls_map.num_col = self.num_row, 2
            self._ls_map.nservers, self._ls_map.rows_per_server = self.S, self.rps
            for s in range(self.S):
                r = rt.server_id_to_rank(s) if rt.num_servers() else rt.rank
                h.last_seen[s] = self._ls_map.shard_ptrs[s] = self._ls_buf.ptrs[r]
            h.clock = self._clock.data_ptr()
        self.admit_after = admit_after
        self._sketch_buf = None
        if admit_after > 1:
            # per server: 4 rows of W = P uint32 counters, then the uint64 total; the aging step's scratch is local
            self._sketch_buf = rt.alloc_symm(16 * P + 8)
            self._sketch_buf.tensor(torch.uint8).zero_()
            self._age = torch.zeros(N.MAX_RANKS, dtype=torch.int32, device=rt.device)
            for s in range(self.S):
                r = rt.server_id_to_rank(s) if rt.num_servers() else rt.rank
                h.sketch[s] = self._sketch_buf.ptrs[r]
                h.total[s] = self._sketch_buf.ptrs[r] + 16 * P
            h.age, h.width, h.admit_after = self._age.data_ptr(), P, admit_after
        self._hash = h
        self._d_hash = torch.frombuffer(bytearray(h), dtype=torch.uint8).to(rt.device)
        self.zero_row = self.S * P
        torch.cuda.synchronize()
        rt.barrier()            # every index is initialised before any rank inserts into it

    # ---- keys -> rows ------------------------------------------------------------------
    def _key_tensor(self, keys) -> torch.Tensor:
        t = torch.as_tensor(keys)
        if t.dtype not in (torch.int32, torch.int64):
            raise TypeError(f"HashMatrixTable: keys must be int32 or int64, got {t.dtype}")
        return t.to(device=self.rt.device, dtype=torch.int64).contiguous().view(-1)

    def lookup_call(self, keys: torch.Tensor, rows: torch.Tensor, status: torch.Tensor, insert: bool,
                    seg_end: Optional[torch.Tensor] = None, seg_table: Optional[torch.Tensor] = None,
                    tables: Optional[torch.Tensor] = None, insert_ok: Optional[torch.Tensor] = None,
                    hash_tables: Optional[Sequence["HashMatrixTable"]] = None) -> None:
        """Launch one translation of int64 device ``keys`` into ``rows`` (no host read). ``status`` (device int64,
        zeroed here) receives the first error; ``raise_hash_status`` interprets it. ``seg_end`` / ``seg_table`` /
        ``tables``: several indexes in one launch (see ``MvbHashLookup``), ``hash_tables`` the tables of ``tables``
        in order (default: this table). ``insert_ok``: device int64; when it holds 0 nothing is inserted (nor
        counted). An inserting call over tables with admission counts its keys before the translation and runs each
        such table's aging step after it."""
        a = N.HashLookup()
        a.tables = (self._d_hash if tables is None else tables).data_ptr()
        a.keys, a.n, a.rows, a.status = keys.data_ptr(), keys.numel(), rows.data_ptr(), status.data_ptr()
        a.seg_end, a.seg_table = N.ptr(seg_end), N.ptr(seg_table)
        a.G = 0 if seg_end is None else seg_end.numel()
        a.insert, a.insert_ok = int(bool(insert)), N.ptr(insert_ok)
        a.timeout_s = float(FLAGS.get("barrier_timeout_s"))
        admitting = [t for t in (hash_tables or [self]) if t.admit_after > 1] if insert else []
        a.admit = int(bool(admitting))
        status.zero_()
        lib, st = N.cuda_lib(), N.stream_ptr()
        with monitor("WORKER_TABLE_HASH_LOOKUP", cuda=True):
            lib.mvb_hash_rows_lookup(a, st)
            for t in admitting:
                if keys.numel():
                    lib.mvb_hash_rows_age(t._hash, st)

    def lookup(self, keys, insert: bool = True) -> torch.Tensor:
        """int64 rows of ``keys`` (device tensor). ``insert``: a missing key gets a row, initialised (with
        ``admit_after``: once admitted); otherwise it reads the zero row. INT64_MIN raises ValueError before anything
        is inserted."""
        k = self._key_tensor(keys)
        rows = torch.empty_like(k)
        if k.numel():
            if bool((k == INT64_MIN).any()):
                raise ValueError(f"HashMatrixTable #{self.table_id}: key {INT64_MIN} (INT64_MIN) is reserved for "
                                 "empty slots")
            status = torch.empty(1, dtype=torch.int64, device=self.rt.device)
            self.lookup_call(k, rows, status, insert)
            raise_hash_status(int(status.item()), [self])
        return rows

    def get(self, keys, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Rows of ``keys`` ``[n, num_col]``; a missing key reads zeros and is not inserted."""
        return self.get_rows(self.lookup(keys, insert=False), out)

    def add(self, keys, values, option: Optional[AddOption] = None) -> None:
        """Insert the missing keys, then ``add_rows`` of their rows (the table's updater, ``option``). With
        ``admit_after``, the values of keys not admitted are dropped."""
        rows = self.lookup(keys, insert=True)
        if self.admit_after > 1:
            keep = rows != self.zero_row
            rows, values = rows[keep], self._as_device(values).view(-1, self.num_col)[keep]
        self.add_rows(rows, values, option)

    def get_async(self, *args, **kwargs):
        raise TypeError("HashMatrixTable: the whole-table get is not offered (its layout is the slot layout); "
                        "use get(keys) or export()")

    def add_async(self, *args, **kwargs):
        raise TypeError("HashMatrixTable: the whole-table add is not offered (its layout is the slot layout); "
                        "use add(keys, values)")

    # ---- access clock and eviction ----------------------------------------------------------
    def _need_tracking(self, what: str) -> None:
        if not self.track_access:
            raise ValueError(f"HashMatrixTable #{self.table_id}: {what} needs track_access=True")

    @property
    def clock(self) -> int:
        """This rank's access clock: inserting lookups stamp the keys they touch with it (default 0)."""
        self._need_tracking("the access clock")
        return self._clock_value

    @clock.setter
    def clock(self, value: int) -> None:
        self._need_tracking("the access clock")
        value = int(value)
        if not INT64_MIN <= value < -INT64_MIN:
            raise ValueError(f"HashMatrixTable #{self.table_id}: clock {value} is not an int64")
        self._clock.fill_(value)          # in stream order: lookups enqueued before still read the old value
        self._clock_value = value

    def last_seen(self, keys) -> torch.Tensor:
        """int64 stamp of each key (the largest clock of an inserting lookup that touched it), -1 for a missing key."""
        self._need_tracking("last_seen")
        rows = self.lookup(keys, insert=False)
        out = torch.empty(rows.numel(), 2, dtype=torch.int32, device=self.rt.device)
        if rows.numel():
            N.cuda_lib().mvb_get_rows(N.I32, self._ls_map, rows, rows.numel(), out, 2, N.stream_ptr())
        return torch.where(rows == self.zero_row, -1, out.view(torch.int64).view(-1))

    def evict(self, older_than: Optional[int] = None, keys=None) -> int:
        """Collective (every rank calls it at the same point): remove the keys with ``last_seen < older_than`` (the
        same value on every rank; needs ``track_access``), the ``keys`` given on any rank (missing keys and
        INT64_MIN are ignored) and the slots refused at the capacity limit, and free their slots. Returns the
        number of keys removed over all servers.

        Survivors keep their values, updater state and stamp bit for bit, but may move to another slot: row ids that
        ``lookup`` returned before are stale afterwards. A removed key reads zeros, and when it comes back it is
        inserted like a new key (initial row from the key, zero updater state). ``PSEmbedding`` and
        ``PSEmbeddingCollection`` translate keys on every call and keep working. Each server rebuilds its index in
        place (csrc/cuda/hash_rows.cu) with a scratch of ``(slots // 2 + 2) * 8`` bytes."""
        rt, lib = self.rt, N.cuda_lib()
        if older_than is not None:
            self._need_tracking("evict(older_than=...)")
            older_than = int(older_than)
            if not INT64_MIN < older_than < -INT64_MIN:
                raise ValueError(f"HashMatrixTable #{self.table_id}: older_than {older_than} is not an int64 above "
                                 "INT64_MIN")
        if len(set(rt.all_gather_object(older_than))) != 1:
            raise ValueError(f"HashMatrixTable #{self.table_id}: evict(older_than=...) differs between ranks")
        k = self._key_tensor(keys) if keys is not None else torch.empty(0, dtype=torch.int64, device=rt.device)
        for handle in list(self._events):         # this table's outstanding async ops
            self.wait(handle)
        rt.barrier()                              # every lookup and push has landed (row mailboxes drained)
        if k.numel():
            lib.mvb_hash_rows_mark(self._hash, k, k.numel(), N.stream_ptr())
        rt.barrier()
        removed = 0
        if self.sid >= 0:
            counts = torch.empty(2, dtype=torch.int64, device=rt.device)
            work = torch.empty(self.slots // 2 + 2, dtype=torch.int64, device=rt.device)
            older = INT64_MIN if older_than is None else older_than
            if self.state_row_count:
                # adam: m and v rows of num_col elements, and the step count (one element per slot) after v's slab
                lib.mvb_hash_rows_evict_ex(self._hash, self.sid, older, self._sp(0), self._sp(1), 1,
                                           self.state_stride, self.num_col, counts, work, N.stream_ptr(),
                                           self.state[1][self.state_stride:], 1)
            else:
                lib.mvb_hash_rows_evict(self._hash, self.sid, older, self._sp(0), self._sp(1),
                                        self.W if self.state_per_worker else 1, self.state_stride,
                                        1 if self.state_per_row else self.num_col, counts, work, N.stream_ptr())
            removed = int(counts[0].item())
        rt.barrier()
        return sum(rt.all_gather_object(removed))

    def num_keys(self) -> int:
        """Keys held over all servers (reads the device)."""
        out = torch.empty(1, dtype=torch.int64, device=self.rt.device)
        N.cuda_lib().mvb_hash_rows_count(self._hash, out, N.stream_ptr())
        return int(out.item())

    def _dump(self, server: int):
        keys = torch.empty(self.slots, dtype=torch.int64, device=self.rt.device)
        rows = torch.empty_like(keys)
        cnt = torch.empty(1, dtype=torch.int64, device=self.rt.device)
        N.cuda_lib().mvb_hash_rows_dump(self._hash, server, keys, rows, cnt, N.stream_ptr())
        n = int(cnt.item())
        return keys[:n], rows[:n]

    def export(self):
        """(keys ascending [K] int64, their rows' values [K, num_col]) over all servers, on the device."""
        parts = [self._dump(s) for s in range(self.S)]
        keys = torch.cat([k for k, _ in parts])
        rows = torch.cat([r for _, r in parts])
        keys, order = torch.sort(keys)
        return keys, self.get_rows(rows[order])

    _ADMIT_TAG = b"MVBADMIT"

    def store(self, stream) -> None:
        """This rank's shard and updater state (the slot layout), then its server's keys, then, with
        ``track_access``, their last-seen stamps, then, with ``admit_after``, a tag, ``admit_after`` and its
        server's sketch and total. A table of the same capacity, width, number of servers, ``track_access`` and
        ``admit_after`` loads it back with every key in its slot, and then counts and admits as this one would. The
        clock is not stored."""
        super().store(stream)
        torch.cuda.current_stream().synchronize()
        stream.write(self._keys_buf.tensor(torch.int64, self.slots).cpu().numpy().tobytes())
        stream.write(self._ready_buf.tensor(torch.int32, self.slots).cpu().numpy().tobytes())
        if self.track_access:
            stream.write(self._ls_buf.tensor(torch.int64, self.slots).cpu().numpy().tobytes())
        if self.admit_after > 1:
            stream.write(self._ADMIT_TAG + int(self.admit_after).to_bytes(8, "little"))
            stream.write(self._sketch_buf.tensor(torch.uint8).cpu().numpy().tobytes())

    def load(self, stream) -> None:
        import numpy as np
        super().load(stream)
        raw = stream.read(self.slots * 12)
        if len(raw) != self.slots * 12:
            raise ValueError(f"HashMatrixTable #{self.table_id}: the stream holds no index of {self.slots} slots")
        arr = np.frombuffer(raw, dtype=np.uint8)
        keys = torch.from_numpy(arr[:self.slots * 8].view(np.int64).copy()).to(self.rt.device)
        ready = torch.from_numpy(arr[self.slots * 8:].view(np.int32).copy()).to(self.rt.device)
        self._keys_buf.tensor(torch.int64, self.slots).copy_(keys)
        self._ready_buf.tensor(torch.int32, self.slots).copy_(ready)
        self._count_buf.tensor(torch.int64, 1).fill_(int((ready == 1).sum()))     # refused slots hold no row
        if self.track_access:
            raw = stream.read(self.slots * 8)
            if len(raw) != self.slots * 8:
                raise ValueError(f"HashMatrixTable #{self.table_id}: the stream holds no last-seen stamps of "
                                 f"{self.slots} slots (stored without track_access?)")
            ls = torch.from_numpy(np.frombuffer(raw, dtype=np.int64).copy()).to(self.rt.device)
            self._ls_buf.tensor(torch.int64, self.slots).copy_(ls)
        self._load_sketch(stream)
        torch.cuda.synchronize()

    def _load_sketch(self, stream) -> None:
        """The admission part of a stream: required with ``admit_after``, refused without it (a seekable stream is
        peeked at and left where it was)."""
        tid = self.table_id
        if self.admit_after == 1:
            if hasattr(stream, "seekable") and stream.seekable():
                at = stream.tell()
                tag = stream.read(len(self._ADMIT_TAG))
                stream.seek(at)
                if tag == self._ADMIT_TAG:
                    raise ValueError(f"HashMatrixTable #{tid}: the stream was stored with admit_after >= 2; this "
                                     "table has admission off")
            return
        head = stream.read(16)
        if len(head) != 16 or head[:8] != self._ADMIT_TAG:
            raise ValueError(f"HashMatrixTable #{tid}: the stream holds no admission sketch (stored with "
                             f"admit_after=1?); this table has admit_after={self.admit_after}")
        stored = int.from_bytes(head[8:], "little")
        if stored != self.admit_after:
            raise ValueError(f"HashMatrixTable #{tid}: the stream was stored with admit_after={stored}; this table "
                             f"has admit_after={self.admit_after}")
        n = 16 * self.slots + 8
        raw = stream.read(n)
        if len(raw) != n:
            raise ValueError(f"HashMatrixTable #{tid}: the stream holds no sketch of {self.slots} counters per row")
        self._sketch_buf.tensor(torch.uint8).copy_(torch.frombuffer(bytearray(raw), dtype=torch.uint8))

    def free(self) -> None:
        super().free()
        for b in (self._keys_buf, self._ready_buf, self._count_buf, self._ls_buf, self._sketch_buf):
            if b is not None:
                self.rt.release_symm(b)


class KVDeviceTable(_AsyncOps):
    """KVTable<K,V>: hash-partitioned map (key % num_servers) as per-shard GPU hash tables.

    The reference's server side is an unbounded ``unordered_map`` (kv_table.h:86-106).  Here every shard is an
    open-addressing table in symmetric HBM that GROWS: at every collective point of the table (``MV_Barrier``,
    ``reserve``) the ranks agree on the fullest shard's load factor and, above 1/2, every owner re-inserts its
    shard into a table of twice (or more) the capacity in a freshly allocated symmetric slab; the old slab is
    released in two phases.  Between two collective points a shard therefore accepts at least as many new keys as it
    already holds slots in use ("kv-full" is reported by the watchdog if even that is exceeded). In a single process
    ``add`` grows the table before a batch that could take it above 1/2, so one batch of any size fits.
    INT64_MIN marks empty slots and is not a key: ``add`` skips it (the batch's other keys are added) and flags
    "kv-bad-key", which the next watchdog check raises; ``get`` returns 0 for it.
    ``add`` / ``get`` are asynchronous device operations (no stream synchronisation, no D2H per call): ``get``
    returns a device tensor; the worker-side cache ``raw()`` (kv_table.h:30) is refreshed lazily from the batches
    that were pulled."""

    MAX_LOAD = 0.5

    def __init__(self, key_dtype="int64", val_dtype="float32", capacity: Optional[int] = None):
        super().__init__()
        rt = Runtime.get()
        self.rt = rt
        self.vdtype = _torch_dtype(val_dtype)
        self.vcode = N.dtype_code(self.vdtype)
        self.vsz = torch.empty((), dtype=self.vdtype).element_size()
        cap = int(capacity or FLAGS.get("kv_capacity"))
        cap = 1 << (cap - 1).bit_length()
        self.S = max(rt.num_servers(), 1)
        self._alloc(cap)
        self._cache: Dict[int, object] = {}
        self._pending = []                      # (keys, values) device batches not yet folded into the cache
        self._count = torch.zeros(1, dtype=torch.int64, device=rt.device)
        self.growths = 0
        self._added_ub = 0                      # upper bound of the keys this worker may have inserted since the last count
        self.table_id = rt.register_table(self)
        if rt.size > 1:
            rt.barrier_hooks.append(self._barrier_hook)
        rt.barrier()

    def _alloc(self, cap: int) -> None:
        rt, lib = self.rt, N.cuda_lib()
        self.capacity = cap
        self.keys_buf = rt.alloc_symm(cap * 8)
        self.vals_buf = rt.alloc_symm(cap * self.vsz)
        lib.mvb_kv_init(self.keys_buf.local_ptr, cap, N.stream_ptr())
        self.vals_buf.tensor(torch.uint8).zero_()
        kv = N.KV()
        kv.vtype, kv.nservers, kv.capacity = self.vcode, self.S, cap
        for s in range(self.S):
            r = rt.server_id_to_rank(s) if rt.num_servers() else rt.rank
            kv.keys[s] = self.keys_buf.ptrs[r]
            kv.vals[s] = self.vals_buf.ptrs[r]
        self._kv = kv

    # ---- growth -------------------------------------------------------------------------------
    def live_keys(self) -> int:
        """Keys stored in this rank's shard (synchronises the stream)."""
        N.cuda_lib().mvb_kv_count(self.keys_buf.local_ptr, self.capacity, self._count, N.stream_ptr())
        return int(self._count.item())

    def reserve(self, keys_per_shard: int = 0) -> None:
        """Collective: grow every shard until max(load, keys_per_shard / capacity) <= 1/2."""
        rt, lib = self.rt, N.cuda_lib()
        torch.cuda.synchronize()
        live = self.live_keys()
        self._added_ub = live
        need = max(rt.all_gather_object(max(live, int(keys_per_shard))))
        cap = self.capacity
        while need > self.MAX_LOAD * cap:
            cap *= 2
        if cap == self.capacity:
            return
        if rt.size > 1:
            rt.control_barrier()                 # nobody is still pushing into the old slabs
        old_keys, old_vals, old_cap = self.keys_buf, self.vals_buf, self.capacity
        self._alloc(cap)
        lib.mvb_kv_rehash(self.vcode, old_keys.local_ptr, old_vals.local_ptr, old_cap, self.keys_buf.local_ptr,
                          self.vals_buf.local_ptr, cap, rt.err_flag, N.stream_ptr())
        torch.cuda.synchronize()
        rt.release_symm(old_keys)                # two-phase, collective
        rt.release_symm(old_vals)
        self.growths += 1
        rt.check_watchdog()

    def _barrier_hook(self, final: bool) -> None:
        if final:
            self.reserve()

    # ---- ops ----------------------------------------------------------------------------------
    def raw(self) -> Dict[int, object]:
        for k, v in self._pending:
            for kk, vv in zip(k.cpu().tolist(), v.cpu().tolist()):
                self._cache[kk] = vv
        self._pending = []
        return self._cache

    def _keys(self, keys) -> torch.Tensor:
        t = torch.as_tensor(keys, dtype=torch.int64)
        return t.to(self.rt.device).contiguous().view(-1)

    def add(self, keys, vals) -> None:
        """One-sided, asynchronous on the current stream (the reference's Add is a blocking round trip;
        ``mv.barrier()`` is the completion / visibility point here, as for every async table op)."""
        lib = N.cuda_lib()
        scalar = not hasattr(keys, "__len__") and not torch.is_tensor(keys)
        k = self._keys([keys] if scalar else keys)
        v = torch.as_tensor([vals] if scalar else vals).to(self.vdtype).to(self.rt.device).contiguous().view(-1)
        assert k.numel() == v.numel()
        n = k.numel()
        if self.rt.size == 1 and self._added_ub + n > self.MAX_LOAD * self.capacity:
            # single process: every point is a collective point, so grow for this batch's distinct keys before it
            # runs (reserve synchronises anyway)
            n = int(torch.unique(k).numel())
            self.reserve(self.live_keys() + n)
        lib.mvb_kv_add(self._kv, k, v, k.numel(), self.rt.err_flag, N.stream_ptr())
        self._keep_add = (k, v)
        self._added_ub += n

    def get(self, keys):
        """Batched lookup; returns a device tensor (a Python scalar for a scalar key)."""
        lib = N.cuda_lib()
        scalar = not hasattr(keys, "__len__") and not torch.is_tensor(keys)
        k = self._keys([keys] if scalar else keys)
        out = torch.empty(k.numel(), dtype=self.vdtype, device=self.rt.device)
        lib.mvb_kv_get(self._kv, k, out, k.numel(), N.stream_ptr())
        self._pending.append((k, out))
        if len(self._pending) > 64:
            self.raw()
        if scalar:
            return out.cpu()[0].item()
        return out

    def free(self) -> None:
        self.rt.release_symm(self.keys_buf)
        self.rt.release_symm(self.vals_buf)

    def store(self, stream) -> None:
        """KV checkpoint (the reference's is Fatal("Not implemented"), kv_table.h:108-114)."""
        import struct
        lib = N.cuda_lib()
        ok = torch.empty(self.capacity, dtype=torch.int64, device=self.rt.device)
        ov = torch.empty(self.capacity, dtype=self.vdtype, device=self.rt.device)
        cnt = torch.zeros(1, dtype=torch.int64, device=self.rt.device)
        lib.mvb_kv_dump(self.vcode, self.keys_buf.local_ptr, self.vals_buf.local_ptr, self.capacity, ok, ov, cnt,
                        N.stream_ptr())
        n = int(cnt.item())
        stream.write(struct.pack("<q", n))
        stream.write(ok[:n].cpu().numpy().tobytes())
        stream.write(ov[:n].cpu().numpy().tobytes())

    def load(self, stream) -> None:
        import struct
        import numpy as np
        (n,) = struct.unpack("<q", stream.read(8))
        if n == 0:
            return
        keys = np.frombuffer(stream.read(8 * n), dtype=np.int64).copy()
        npdt = {torch.float32: np.float32, torch.float64: np.float64, torch.int32: np.int32,
                torch.int64: np.int64}[self.vdtype]
        vals = np.frombuffer(stream.read(self.vsz * n), dtype=npdt).copy()
        self.add(torch.from_numpy(keys), torch.from_numpy(vals))
