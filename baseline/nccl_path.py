"""The NCCL-only comparator (BASELINE.md section 2): what a straightforward port would do.

    Add  = ncclReduceScatter(delta) -> stand-alone updater kernel on the shard
    Get  = ncclAllGather(shards)
    Aggregate = ncclAllReduce

"A path that only calls NCCL for Add/Get is the baseline, not the product": every fused
kernel is measured against this on the same box and shapes (bench/matrix_bw.py)."""
from __future__ import annotations

import torch
import torch.distributed as dist

from multiverso_b200 import _native as N


class NcclDenseTable:
    def __init__(self, size: int, updater: str = "sgd"):
        self.world = dist.get_world_size() if dist.is_initialized() else 1
        self.rank = dist.get_rank() if dist.is_initialized() else 0
        assert size % self.world == 0
        self.size, self.shard_len = size, size // self.world
        self.shard = torch.zeros(self.shard_len, device="cuda")
        self.recv = torch.empty(self.shard_len, device="cuda")
        self.state = torch.zeros(self.shard_len, device="cuda")
        self.updater = N.UPDATER_NAMES[updater]
        self.opt = N.AddOpt(0, 0.9, 0.01, 0.1, 0.1)

    def add(self, delta: torch.Tensor) -> None:
        if self.world > 1:
            dist.reduce_scatter_tensor(self.recv, delta, op=dist.ReduceOp.SUM)
            src = self.recv
        else:
            src = delta
        N.cuda_lib().mvb_updater_apply(N.F32, self.updater, self.shard, src, self.state, None, self.shard_len, self.opt,
                                       1.0, N.stream_ptr())

    def get(self, out: torch.Tensor) -> torch.Tensor:
        if self.world > 1:
            dist.all_gather_into_tensor(out, self.shard)
        else:
            out.copy_(self.shard)
        return out
