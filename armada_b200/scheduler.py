"""Reference-shaped entry point for one scheduling round, backed ONLY by the CUDA library.

Mirrors `scheduling.NewPreemptingQueueScheduler(...).Schedule(ctx)`
(scheduling/preempting_queue_scheduler.go:50-84,84-285): the caller hands over the round's
SchedulingContext / NodeDb / job view (already flattened into an `ArmadaRoundInput`) and gets
back scheduled / preempted jobs plus the updated accounting.  There is no CPU fallback: if
libarmada_b200.so or a CUDA device is missing this raises.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

from . import abi
from .model import RoundResult, excluded_nodes_by_reason


def _check(lib, status: int) -> None:
    if status != abi.OK:
        raise abi.ArmadaError(status, f"{lib.armada_strerror(status).decode()}: {lib.armada_last_error().decode()}")


class DeviceRound:
    """Owns one `ArmadaRound*` (device context).  upload → run → download, like
    populateNodeDb → Schedule → result read-back in scheduling_algo.go:740-840."""

    def __init__(self, device: int = 0, lib=None):
        # `lib` is for tests only (tests/emu_lib.py steps the same kernel source through a CPU SIMT
        # emulator); the product always loads the CUDA library and fails loudly without it.
        self.lib = lib if lib is not None else abi.load_product()
        self.h = C.c_void_p()
        _check(self.lib, self.lib.armada_round_create(device, C.byref(self.h)))
        self._input: Optional[abi.RoundInput] = None

    def upload(self, inp: abi.RoundInput) -> None:
        _check(self.lib, self.lib.armada_round_upload(self.h, C.byref(inp)))
        self._input = inp

    def upload_cluster(self, inp: abi.RoundInput, cs: abi.ClusterState) -> None:
        """upload() with the pool's node set, total and caps derived on the device from the cluster as reported
        (populateNodeDb + NewSchedulingConstraints; armada_round_upload_cluster)."""
        _check(self.lib, self.lib.armada_round_upload_cluster(self.h, C.byref(inp), C.byref(cs)))
        self._input = inp

    def download_snapshot(self) -> dict:
        """What the last upload_cluster derived, in the caller's node numbering: node_state [N] (abi.NODE_*),
        node_allocatable [D][N], node_static_class [N], total_resources [D], max_resources_to_schedule [D],
        queue_limit [Q][PC][D]."""
        import numpy as np
        inp = self._input
        N, D, Q, PC = inp.num_nodes, inp.num_resources, inp.num_queues, inp.num_priority_classes
        out = {"node_state": np.zeros(N, np.uint8), "node_allocatable": np.zeros((D, N), np.int64),
               "node_static_class": np.zeros(N, np.uint32), "total_resources": np.zeros(D, np.int64),
               "max_resources_to_schedule": np.zeros(D, np.int64), "queue_limit": np.zeros((Q, PC, D), np.int64)}
        p = {k: v.ctypes.data_as(abi.u8p if v.dtype == np.uint8 else abi.u32p if v.dtype == np.uint32 else abi.i64p) for k, v in out.items()}
        _check(self.lib, self.lib.armada_round_download_snapshot(self.h, p["node_state"], p["node_allocatable"], p["node_static_class"],
                                                                 p["total_resources"], p["max_resources_to_schedule"], p["queue_limit"]))
        return out

    def run(self, budget_ns: int = 0) -> abi.RoundStats:
        """`budget_ns` > 0: the cycle's maxSchedulingDuration (scheduling_algo.go:115-118); raises
        ArmadaError(E_DEADLINE) when it runs out — nothing of the round is committed."""
        stats = abi.RoundStats()
        _check(self.lib, self.lib.armada_round_run_deadline(self.h, C.byref(stats), int(budget_ns)))
        return stats

    def download(self, res: Optional[RoundResult] = None) -> RoundResult:
        if res is None:
            res = RoundResult(self._input)
        _check(self.lib, self.lib.armada_round_download(self.h, C.byref(res.out)))
        return res

    def schedule(self, inp: abi.RoundInput, res: Optional[RoundResult] = None) -> RoundResult:
        """Host buffers in, host buffers out (the end-to-end call a Go shim makes per pool)."""
        if res is None:
            res = RoundResult(inp)
        self._input = inp
        _check(self.lib, self.lib.armada_round_schedule(self.h, C.byref(inp), C.byref(res.out), C.byref(res.stats)))
        return res

    def close(self):
        if self.h:
            self.lib.armada_round_destroy(self.h)
            self.h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PreemptingQueueScheduler:
    """`sch := NewPreemptingQueueScheduler(sctx, constraints, …, jobRepo, nodeDb, …); sch.Schedule(ctx)`"""

    def __init__(self, round_input: abi.RoundInput, device: int = 0):
        self.round_input = round_input
        self.device = device

    def schedule(self) -> RoundResult:
        with DeviceRound(self.device) as r:
            return r.schedule(self.round_input)


def round_schedule(inp: abi.RoundInput, device: int = 0) -> RoundResult:
    return PreemptingQueueScheduler(inp, device).schedule()


def _gang_csr(gangs):
    """A dry-run call's gangs (lists of job-class indices) as CSR arrays: member offsets, members, and a
    cleared ok per gang and node per member for the library to fill."""
    import numpy as np
    start = np.zeros(len(gangs) + 1, np.uint32)
    start[1:] = np.cumsum([len(g) for g in gangs])
    members = np.asarray([c for g in gangs for c in g] or [0], dtype=np.uint32)
    ok = np.zeros(max(len(gangs), 1), np.uint8)
    node = np.full(max(int(start[-1]), 1), abi.NONE, np.uint32)
    return start, members, ok, node


class DeviceNodeDb:
    """`NodeDb` on an empty cluster for dry-run gang checks — what SubmitChecker builds per executor
    (internal/scheduler/submitcheck.go:302-422).  `schedule_many(gangs)` = one
    `ScheduleManyWithTxn` + `Abort` per gang (gangs are lists of job-class indices), all gangs of the
    call in one kernel launch."""

    def __init__(self, inp: abi.RoundInput, device: int = 0, lib=None):
        self.lib = lib if lib is not None else abi.load_product()
        self.h = C.c_void_p()
        self._input = inp
        _check(self.lib, self.lib.armada_nodedb_create(device, C.byref(inp), C.byref(self.h)))

    def schedule_many(self, gangs):
        start, members, ok, node = _gang_csr(gangs)
        _check(self.lib, self.lib.armada_nodedb_schedule_many(self.h, len(gangs), start.ctypes.data_as(abi.u32p), members.ctypes.data_as(abi.u32p),
                                                              ok.ctypes.data_as(abi.u8p), node.ctypes.data_as(abi.u32p)))
        out_nodes = [node[int(start[g]):int(start[g + 1])].copy() for g in range(len(gangs))]
        return ok[: len(gangs)].astype(bool), out_nodes

    def explain(self, gangs, capacity: int = 1024, builder=None):
        """`schedule_many` that also says why, in one launch (armada_nodedb_explain).  Per gang:
        `(ok, member_node, num_placed, away, records)` — `records` is a list of abi.ExcludedReason, the
        NumExcludedNodesByReason of a failed gang of one, empty otherwise; with the db's `builder`
        (RoundInputBuilder) it is that map itself, {reason string: count}.  The record buffer starts at
        `capacity` and is grown once, to the size the library reports, when it was too small."""
        import numpy as np
        G = len(gangs)
        start, members, ok, node = _gang_csr(gangs)
        placed = np.zeros(max(G, 1), np.uint32)
        away = np.zeros(max(G, 1), np.uint8)
        rstart = np.zeros(G + 1, np.uint32)
        needed = C.c_uint32(0)
        cap = max(int(capacity), 1)
        for _ in range(2):
            recs = (abi.ExcludedReason * cap)()
            _check(self.lib, self.lib.armada_nodedb_explain(self.h, G, start.ctypes.data_as(abi.u32p), members.ctypes.data_as(abi.u32p),
                                                            ok.ctypes.data_as(abi.u8p), node.ctypes.data_as(abi.u32p), placed.ctypes.data_as(abi.u32p),
                                                            away.ctypes.data_as(abi.u8p), rstart.ctypes.data_as(abi.u32p), recs, cap, C.byref(needed)))
            if needed.value <= cap:
                break
            cap = needed.value
        out = []
        for g in range(G):
            lo, hi = int(start[g]), int(start[g + 1])
            rec = list(recs[int(rstart[g]):int(rstart[g + 1])])
            if builder is not None:
                rec = excluded_nodes_by_reason(builder, int(gangs[g][0]), rec) if rec else {}
            out.append((bool(ok[g]), node[lo:hi].copy(), int(placed[g]), bool(away[g]), rec))
        return out

    def select_nodes(self, classes):
        """One independent job per entry (its job class): the node it would be bound to on the empty
        cluster, abi.NONE if it fits nowhere (SelectNodeForJobWithTxn, nodedb.go:431-512)."""
        import numpy as np
        cls = np.asarray(list(classes) or [0], dtype=np.uint32)
        node = np.full(len(cls), abi.NONE, np.uint32)
        _check(self.lib, self.lib.armada_nodedb_select_nodes(self.h, len(list(classes)), cls.ctypes.data_as(abi.u32p), node.ctypes.data_as(abi.u32p)))
        return node[: len(list(classes))]

    def add_classes(self, class_request, class_pc, class_static_row, class_away_row, static_match, type_match) -> int:
        """armada_nodedb_add_classes: append job classes ([n][D] requests, [n] priority-class indices, [n] home
        rows, [n][MAX_AWAY] away rows) and bitmap rows ([m][sw] static_match, [m][tw] type_match, against the
        db's static classes and node types).  Returns the id of the first new class; raises ArmadaError and
        leaves the db as it was when the library refuses them."""
        import numpy as np
        inp = self._input
        pc = np.ascontiguousarray(class_pc, np.uint32).reshape(-1)
        n = len(pc)
        # the library reads these widths from raw pointers: a wrong shape is refused here
        shapes = {"class_request": (n, inp.num_resources), "class_static_row": (n,), "class_away_row": (n, abi.MAX_AWAY)}
        req = np.ascontiguousarray(class_request, np.int64)
        row = np.ascontiguousarray(class_static_row, np.uint32)
        away = np.ascontiguousarray(class_away_row, np.uint32)
        sm = np.ascontiguousarray(static_match, np.uint32)
        tm = np.ascontiguousarray(type_match, np.uint32)
        shapes.update(static_match=(len(sm), (inp.num_static_classes + 31) // 32), type_match=(len(sm), (inp.num_node_types + 31) // 32))
        for name, a in (("class_request", req), ("class_static_row", row), ("class_away_row", away), ("static_match", sm), ("type_match", tm)):
            if a.shape != shapes[name]:
                raise ValueError(f"{name} has shape {a.shape}, the db needs {shapes[name]}")
        valid = np.ones(max(n, 1), np.uint8)
        first = C.c_uint32(0)
        ptr = lambda a, t: a.ctypes.data_as(t) if a.size else None  # noqa: E731
        _check(self.lib, self.lib.armada_nodedb_add_classes(self.h, n, ptr(req.reshape(-1), abi.i64p), ptr(pc, abi.u32p), ptr(row, abi.u32p),
                                                            ptr(away.reshape(-1), abi.u32p), valid.ctypes.data_as(abi.u8p), len(sm), ptr(sm, abi.u32p),
                                                            ptr(tm, abi.u32p), C.byref(first)))
        return first.value

    def close(self):
        if self.h:
            self.lib.armada_nodedb_destroy(self.h)
            self.h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
