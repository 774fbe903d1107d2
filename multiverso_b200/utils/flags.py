"""Flag registry with the reference's ``-key=value`` command-line syntax.

Reference: MV_DEFINE_* / ParseCMDFlags / SetCMDFlag
(include/multiverso/util/configure.h:13-115, src/util/configure.cpp:9-54).  Same flag names and
defaults (SURVEY 2.3 U2); parsing compacts argv (recognised flags are removed, everything else
is left in place).  Unlike the reference (Q10) an argument containing '-' but no '=' is simply
left alone instead of aborting, and doubles are parsed from the value, not the whole argument.
"""
from __future__ import annotations

from typing import Any, Dict, List, Optional

_DEFAULTS: Dict[str, Any] = {
    # src/zoo.cpp:23-24
    "ps_role": "default", "ma": False,
    # src/server.cpp:20-21
    "sync": False, "backup_worker_ratio": 0,
    # src/updater/updater.cpp:18-19
    "updater_type": "default", "omp_threads": 4,
    # src/util/allocator.cpp:10,153
    "allocator_alignment": 16, "allocator_type": "smart",
    # src/util/log.cpp:11
    "logtostderr": False,
    # include/multiverso/net/zmq_net.h:20-21
    "machine_file": "", "port": 55555,
    # --- device additions -------------------------------------------------------------------
    "barrier_timeout_s": 120.0,   # watchdog on device-side spins (SURVEY 5.3)
    "request_stall_warn_s": 60.0,  # host backend: log a line whenever a table request has waited this long
    "kv_capacity": 1 << 20,       # slots per KV shard
    "async_one_sided": True,      # async mode: stateless updaters push with red.add
    "nvls": True,                 # use NVSwitch multicast (multimem.*) for MV_Aggregate when available
    "replicate_get": False,       # BSP ArrayTables: fused Add -> Get (updated shards pushed to replicas);
                                  # measured at 2 GPUs: multimem.st push costs +3.0 ms/GB, a net loss there
    "staleness": False,           # per-table version counters + staleness histogram (Dashboard.staleness())
    "row_mailbox": True,          # async stateful row Adds: device-side mailboxes + owner-side apply (rowbox.cu)
    "nvls_add": False,            # also reduce dense Adds in the switch (egress-bound either way;
                                  # measured slower than the P2P pull at 2 GPUs: 3.18 vs 1.71 ms)
}

_TEXT: Dict[str, str] = {
    "ps_role": "none / worker / server / default", "ma": "model average, will not start server",
    "sync": "sync or async", "backup_worker_ratio": "ratio% of backup workers, set 20 means 20%",
    "updater_type": "multiverso server updater type", "omp_threads": "#threads used by host updaters",
    "logtostderr": "log to stderr", "machine_file": "machine file path", "port": "control-plane port",
}


class FlagRegister:
    def __init__(self):
        self._values: Dict[str, Any] = dict(_DEFAULTS)

    def define(self, name: str, default: Any, text: str = "") -> None:
        self._values.setdefault(name, default)
        if text:
            _TEXT[name] = text

    def get(self, name: str) -> Any:
        return self._values[name]

    def set(self, name: str, value: Any) -> None:
        """MV_SetFlag: the flag must exist (reference CHECKs this)."""
        if name not in self._values:
            raise KeyError(f"unknown flag '{name}'")
        self._values[name] = _coerce(value, self._values[name])

    def parse(self, argv: Optional[List[str]]) -> List[str]:
        """Consume ``-key=value`` arguments; return the compacted argv."""
        if not argv:
            return []
        rest: List[str] = []
        for arg in argv:
            if arg.startswith("-") and "=" in arg:
                key, val = arg.lstrip("-").split("=", 1)
                if key in self._values:
                    self._values[key] = _coerce(val, self._values[key])
                    continue
            rest.append(arg)
        return rest

    def reset(self) -> None:
        self._values = dict(_DEFAULTS)

    def items(self):
        return self._values.items()


def _coerce(value: Any, like: Any) -> Any:
    if isinstance(like, bool):
        if isinstance(value, str):
            return value.strip().lower() in ("1", "true", "yes", "on")
        return bool(value)
    if isinstance(like, int) and not isinstance(like, bool):
        return int(value)
    if isinstance(like, float):
        return float(value)
    return str(value)


FLAGS = FlagRegister()
