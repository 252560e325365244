"""SubmitChecker (internal/scheduler/submitcheck.go:57-460) over the device's dry-run NodeDb.

`SubmitChecker(cfg, pools, executors, queues).check(jobs)` returns, per job id, the reference's
`schedulingResult{isSchedulable, pools, reason}`: every single job is checked alone, every gang first
member by member and then as a whole (`Check`, `getGangSchedulingResult`, :210-296), against the pools
in configuration order with their away pools and submission groups (`getSchedulingResult`, :302-422).
`reason` is assembled exactly like the reference's, from `armada_nodedb_explain`.

The home / away / gang-away toggles and the disallowed resources are part of an `ArmadaNodeDb` (they come
from the `ArmadaRoundInput` it is created from), where the reference flips them on one NodeDb per executor
before each check (:350-369).  So this restatement keeps one db per (executor, the pool its nodes are in,
the toggles of the pool being checked): pools with equal settings share a db.  All the checks a db has to
answer in one `check` call go out as one launch.

Inherent differences: the reference ranges over Go maps for the executors of a pool and for the lines of
`pctx.String()`, so their order in `reason` is random there; here executors come in id order and lines in
reason order.  Not restated: the per-queue and global time budgets of `SubmitCheckConfig` (wall clock),
the job-result cache (:275-283, it caches what would be recomputed identically) and the gRPC plumbing.
"""
from __future__ import annotations

import copy
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi
from .model import (FloatingResource, JobSpec, NodeSpec, QueueSpec, RoundInputBuilder, SchedulingConfig, excluded_nodes_by_reason,
                    multiply_resource, pod_scheduling_context_string, quantity_string)
from .scheduler import DeviceNodeDb


@dataclass
class PoolConfig:
    """configuration.PoolConfig: the fields SubmitChecker reads."""
    name: str
    away_pools: Tuple[str, ...] = ()
    disable_home_scheduling: bool = False
    disable_away_scheduling: bool = False
    disable_gang_away_scheduling: bool = False
    unscheduled_resources: Tuple[str, ...] = ()  # ExperimentalUnscheduledResources (disallowed resources)
    submission_group: str = ""  # ExperimentalSubmissionGroup

    def get_submission_group(self) -> str:  # configuration.go:421-426
        return self.submission_group or self.name


@dataclass
class Executor:
    id: str
    nodes: List[Tuple[str, NodeSpec]] = field(default_factory=list)  # (pool, node)


@dataclass
class SchedulingResult:
    is_schedulable: bool
    pools: List[str] = field(default_factory=list)
    reason: str = ""


def resource_list_string(factory, values) -> str:
    """ResourceList.String() (internaltypes/resource_list.go:28-41): the non-zero entries in factory order."""
    parts = [f"{name}={quantity_string(int(v), factory.scales[d])}" for d, (name, v) in enumerate(zip(factory.names, values)) if int(v) != 0]
    return "(" + ",".join(parts) + ")"


class SubmitChecker:
    """`cfg` is the SchedulingConfig without floating resources; `floating` maps a floating resource name to
    (resolution, {pool: quantity}) (FloatingResourceConfig)."""

    def __init__(self, cfg: SchedulingConfig, pools: Sequence[PoolConfig], executors: Sequence[Executor], queues: Sequence[QueueSpec] = (),
                 floating: Optional[Dict[str, Tuple[str, Dict[str, object]]]] = None, device: int = 0, lib=None):
        self.floating = dict(floating or {})
        self.cfg = copy.copy(cfg)
        self.cfg.floating_resources = [FloatingResource(n, res) for n, (res, _) in sorted(self.floating.items())]
        self.factory = self.cfg.factory()
        self.pools = list(pools)
        self.executors = sorted(executors, key=lambda e: e.id)
        self.queues = {q.name: q for q in queues}
        self.device, self.lib = device, lib
        self.pools_by_group: Dict[str, List[str]] = {}  # NewSubmitChecker :81-87
        for p in self.pools:
            self.pools_by_group.setdefault(p.get_submission_group(), []).append(p.name)
        D = self.factory.D
        # totalResourcesByPool (:151-185): allocatable of the pool's nodes, plus its floating resources
        self.pool_total: Dict[str, np.ndarray] = {}
        for e in self.executors:
            for pool, n in e.nodes:
                tot = self.pool_total.setdefault(pool, np.zeros(D, np.int64))
                tot += self.factory.from_node(n.allocatable if n.allocatable is not None else n.total)
        for name, (_, by_pool) in self.floating.items():
            for pool, q in by_pool.items():
                tot = self.pool_total.setdefault(pool, np.zeros(D, np.int64))
                tot[self.factory.index[name]] += self.factory.scaled_value(name, q)

    # -- the pre-checks of getSchedulingResult --------------------------------------------------------
    def _floating_within_limits(self, pool: str, req: np.ndarray) -> Tuple[bool, str]:
        """FloatingResourceTypes.WithinLimits (floatingresources/floating_resource_types.go:60-72)."""
        avail = np.zeros(self.factory.D, np.int64)
        for name, (_, by_pool) in self.floating.items():
            if pool in by_pool:
                avail[self.factory.index[name]] = self.factory.scaled_value(name, by_pool[pool])
        if not avail.any():
            return False, f"floating resources not configured for pool {pool}"
        for name in self.factory.names:  # ExceedsAvailable over the floating part of the request, factory order
            d = self.factory.index[name]
            if name in self.floating and req[d] > avail[d]:
                return False, f"not enough floating resource {name} in pool {pool}"
        return True, ""

    def _queue_limit(self, pool: str, queue: str, pc_name: str) -> Optional[np.ndarray]:
        """constraints.GetQueueResourceLimit (calculatePerQueueLimits, constraints.go:218-256); None when the
        pool has no constraints or the queue is unknown (an empty ResourceList)."""
        if pool not in self.pool_total or queue not in self.queues:
            return None
        fractions = dict(self.cfg.priority_classes[pc_name].maximum_resource_fraction_per_queue)
        fractions.update(self.queues[queue].resource_limits_by_pc.get(pc_name, {}))
        tot = self.pool_total[pool]
        return np.asarray([multiply_resource(int(tot[d]), fractions.get(n, math.inf)) for d, n in enumerate(self.factory.names)], np.int64)

    # -- the dry runs -----------------------------------------------------------------------------------
    def _run_dry(self, jobs: Sequence[JobSpec], items: List[List[int]]):
        """Every item (a list of job indices: a single job, or a gang) on every (executor, node pool, pool
        setting) db a pool may consult.  Returns {(executor id, node pool, setting): [explain result per item]}
        and the builder of each db."""
        settings = {}
        for p in self.pools:
            settings[p.name] = (p.disable_home_scheduling, p.disable_away_scheduling, p.disable_gang_away_scheduling, tuple(sorted(p.unscheduled_resources)))
        results, builders = {}, {}
        qnames = sorted({j.queue for j in jobs})
        queues = [self.queues.get(q, QueueSpec(q)) for q in qnames]
        for e in self.executors:
            by_pool: Dict[str, List[NodeSpec]] = {}
            for pool, n in e.nodes:
                by_pool.setdefault(pool, []).append(n)
            for node_pool, nodes in sorted(by_pool.items()):
                for s in sorted(set(settings.values())):
                    cfg = copy.copy(self.cfg)
                    cfg.disable_home_scheduling, cfg.disable_away_scheduling, cfg.disable_gang_away_scheduling = s[0], s[1], s[2]
                    cfg.disallowed_resources = list(s[3])
                    b = RoundInputBuilder(cfg, nodes, jobs, queues)
                    with DeviceNodeDb(b.input, self.device, self.lib) as db:
                        res = db.explain([[int(b.job_class[j]) for j in it] for it in items])
                    results[(e.id, node_pool, s)] = res
                    builders[(e.id, node_pool, s)] = b
        return results, builders, settings

    def check(self, jobs: Sequence[JobSpec]) -> Dict[str, SchedulingResult]:
        """SubmitChecker.Check (:210-267) without its time budgets."""
        jobs = list(jobs)
        # the items: each job alone (getIndividualSchedulingResult strips the gang info, :270-271), each gang whole
        gangs: Dict[Tuple[str, str], List[int]] = {}
        for i, j in enumerate(jobs):
            if j.gang_id is not None and j.gang_cardinality > 1:
                gangs.setdefault((j.queue, j.gang_id), []).append(i)
        items = [[i] for i in range(len(jobs))] + list(gangs.values())
        single = [copy.copy(j) for j in jobs]
        for j in single:  # one class table for all dbs: gang membership plays no part in a job's class
            j.gang_id, j.gang_cardinality = None, 1
        dry, builders, settings = self._run_dry(single, items)
        item_result = [self._scheduling_result(items[k], k, single, dry, builders, settings) for k in range(len(items))]
        out: Dict[str, SchedulingResult] = {}
        for i, j in enumerate(jobs):
            if (j.queue, j.gang_id) in gangs and j.gang_cardinality > 1:
                continue
            out[j.id] = item_result[i]
        for k, members in enumerate(gangs.values()):  # getGangSchedulingResult (:287-296)
            res = next((item_result[i] for i in members if not item_result[i].is_schedulable), None)
            if res is None:
                res = item_result[len(jobs) + k]
            for i in members:
                out[jobs[i].id] = res
        return out

    def _scheduling_result(self, members: List[int], k: int, jobs, dry, builders, settings) -> SchedulingResult:
        """getSchedulingResult (:302-422) of one item."""
        f = self.factory
        req = np.sum([f.from_job(jobs[i].requests) for i in members], axis=0)
        floating_req = np.asarray([req[d] if f.names[d] in self.floating else 0 for d in range(f.D)], np.int64)
        first = jobs[members[0]]
        successful: List[str] = []
        sb = []
        for pool in self.pools:
            if pool.name in successful or any(a in successful for a in pool.away_pools):
                continue
            if floating_req.any():
                ok, why = self._floating_within_limits(pool.name, req)
                if not ok:
                    sb.append(f"pool {pool.name}:\n")
                    sb.append(f"job/gang requests floating resources {resource_list_string(f, floating_req)} but {why}\n")
                    sb.append("\n---\n")
                    continue
            limit = self._queue_limit(pool.name, first.queue, first.priority_class)
            if limit is not None and bool((req > limit).any()):
                sb.append(f"pool {pool.name}:\n")
                sb.append(f"job/gang requests resources {resource_list_string(f, req)} which exceeds the total limit of "
                          f"{resource_list_string(f, limit)} for its queue/priority class\n")
                sb.append("\n---\n")
                continue
            node_pools = (pool.name,) + tuple(pool.away_pools)
            for node_pool in node_pools:
                for e in self.executors:
                    key = (e.id, node_pool, settings[pool.name])
                    if key not in dry:
                        continue
                    ok, _, placed, away, recs = dry[key][k]
                    sb.append(e.id)
                    if ok:
                        if not away or pool.away_pools:
                            for p in self.pools_by_group[pool.get_submission_group()]:
                                if p not in successful:
                                    successful.append(p)
                        continue
                    if len(members) == 1:
                        b = builders[key]
                        excluded = excluded_nodes_by_reason(b, int(b.job_class[members[0]]), recs)
                        sb.append(":\n" + pod_scheduling_context_string(b.input.num_nodes, excluded) + "\n---\n")
                    else:
                        sb.append(f": {placed} out of {len(members)} pods schedulable\n")
        if successful:
            return SchedulingResult(True, successful)
        return SchedulingResult(False, [], "".join(sb))
