"""SubmitChecker (internal/scheduler/submitcheck.go:57-460) over the device's dry-run NodeDb.

`SubmitChecker(cfg, pools, executors, queues).check(jobs)` returns, per job id, the reference's
`schedulingResult{isSchedulable, pools, reason}`: every single job is checked alone, every gang first
member by member and then as a whole (`Check`, `getGangSchedulingResult`, :210-296), against the pools
in configuration order with their away pools and submission groups (`getSchedulingResult`, :302-422).
`reason` is assembled exactly like the reference's, from `armada_nodedb_explain`.  `check_with_durations`
also returns the time spent per queue, as `Check` does.

Lifecycle (`updateExecutors`, :128-204): `update_executors` builds the NodeDbs once and starts an empty
result cache; `check` adds the scheduling keys it has not seen to every live db
(`armada_nodedb_add_classes`).  A db's static classes tell nodes apart only by the labels its keys so far
look at (a label unique to every node, such as the hostname, would otherwise make one static class, and
one explain record, per node).  So a key that looks at a label the db does not tell apart yet (a selector
on a new label, a job pinned to a node) rebuilds that one db with its keys so far; this happens at most
once per distinct label key between two `update_executors`.  Individual results are cached by scheduling key in an
LRU of 10 000 entries (`jobSchedulingResultsCache`, :139, :269-285), gang results are not.  The reference
caches whatever the key, EmptySchedulingKey included, and so does this one (every job has a key here).
`close()` (or a `with` block) frees the dbs.

The home / away / gang-away toggles and the disallowed resources are part of an `ArmadaNodeDb` (they come
from the `ArmadaRoundInput` it is created from), where the reference flips them on one NodeDb per executor
before each check (:350-369).  So this restatement keeps one db per (executor, the pool its nodes are in,
the toggles of the pool being checked): pools with equal settings share a db.  All the checks a db has to
answer in one `check` call go out as one launch.

Time budgets (`SubmitCheckConfig.MaxDuration` / `MaxDurationPerQueue`, :211-264): the clock is read at the
reference's `Now()` call sites, in its order, and a zero limit means no limit; the jobs the walk does not
reach are absent from the result, and a gang is reached whole or not at all.  The reference checks job by
job between its clock reads; here the device answers the whole batch first, in one launch per db right
after `start`, so with a real clock that launch's wall time counts against the global budget and the walk
over the answers then applies the budgets in reference order.  With a stepping clock (tests) the results
are exact, since only the `Now()` call sites matter.

Inherent differences: the reference ranges over Go maps for the queues of a check (`jobsByQueue`), for the
executors of a pool and for the lines of `pctx.String()`, so their order is random there; here queues come
in name order, executors in id order and lines in reason order.  Not restated: the gRPC plumbing.
"""
from __future__ import annotations

import copy
import math
import time
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi
from .model import (FloatingResource, JobSpec, NodeSpec, QueueSpec, RoundInputBuilder, SchedulingConfig, excluded_nodes_by_reason,
                    UnresolvedLabels, multiply_resource, pod_scheduling_context_string, quantity_string, scheduling_key)
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


@dataclass
class SubmitCheckConfig:
    """configuration.SubmitCheckConfig: the time budgets of one check, in seconds; zero (or less) means none."""
    max_duration: float = 0.0
    max_duration_per_queue: float = 0.0


class RealClock:
    """The clock `check` reads: `now()` and `since(t)` in seconds (a test substitutes a stepping clock)."""

    def now(self) -> float:
        return time.monotonic()

    def since(self, t: float) -> float:
        return time.monotonic() - t


def _deadline(limit: float, now: float) -> Optional[float]:  # newDeadline (:35-40)
    return None if limit <= 0 else now + limit


def _exceeded(deadline: Optional[float], now: float) -> bool:  # deadline.exceeded (:42-44)
    return deadline is not None and now > deadline


RESULT_CACHE_SIZE = 10000  # lru.New(10000), :139


class SubmitChecker:
    """`cfg` is the SchedulingConfig without floating resources; `floating` maps a floating resource name to
    (resolution, {pool: quantity}) (FloatingResourceConfig)."""

    def __init__(self, cfg: SchedulingConfig, pools: Sequence[PoolConfig], executors: Sequence[Executor], queues: Sequence[QueueSpec] = (),
                 floating: Optional[Dict[str, Tuple[str, Dict[str, object]]]] = None, device: int = 0, lib=None,
                 submit_check: Optional[SubmitCheckConfig] = None, clock=None):
        self.floating = dict(floating or {})
        self.cfg = copy.copy(cfg)
        self.cfg.floating_resources = [FloatingResource(n, res) for n, (res, _) in sorted(self.floating.items())]
        self.factory = self.cfg.factory()
        self.pools = list(pools)
        self.device, self.lib = device, lib
        self.submit_check = submit_check or SubmitCheckConfig()
        self.clock = clock or RealClock()
        self.pools_by_group: Dict[str, List[str]] = {}  # NewSubmitChecker :81-87
        for p in self.pools:
            self.pools_by_group.setdefault(p.get_submission_group(), []).append(p.name)
        self.settings = {p.name: (p.disable_home_scheduling, p.disable_away_scheduling, p.disable_gang_away_scheduling, tuple(sorted(p.unscheduled_resources)))
                         for p in self.pools}
        self.dbs: Dict[Tuple[str, str, tuple], Tuple[RoundInputBuilder, DeviceNodeDb]] = {}
        self.update_executors(executors, queues)

    # -- state ---------------------------------------------------------------------------------------------
    def update_executors(self, executors: Sequence[Executor], queues: Optional[Sequence[QueueSpec]] = None) -> None:
        """updateExecutors (:128-204): one NodeDb per (executor, node pool, pool setting), the per-pool totals
        the queue limits are fractions of, and an empty result cache.  `queues` None keeps the current ones."""
        executors = sorted(executors, key=lambda e: e.id)
        D = self.factory.D
        # totalResourcesByPool (:151-185): allocatable of the pool's nodes, plus its floating resources
        pool_total: Dict[str, np.ndarray] = {}
        for e in executors:
            for pool, n in e.nodes:
                tot = pool_total.setdefault(pool, np.zeros(D, np.int64))
                tot += self.factory.from_node(n.allocatable if n.allocatable is not None else n.total)
        for name, (_, by_pool) in self.floating.items():
            for pool, q in by_pool.items():
                tot = pool_total.setdefault(pool, np.zeros(D, np.int64))
                tot[self.factory.index[name]] += self.factory.scaled_value(name, q)
        dbs = {}
        try:
            for e in executors:
                by_pool: Dict[str, List[NodeSpec]] = {}
                for pool, n in e.nodes:
                    by_pool.setdefault(pool, []).append(n)
                for node_pool, nodes in sorted(by_pool.items()):
                    for s in sorted(set(self.settings.values())):
                        cfg = copy.copy(self.cfg)
                        cfg.disable_home_scheduling, cfg.disable_away_scheduling, cfg.disable_gang_away_scheduling = s[0], s[1], s[2]
                        cfg.disallowed_resources = list(s[3])
                        b = RoundInputBuilder(cfg, nodes, [], [QueueSpec("")])
                        dbs[(e.id, node_pool, s)] = (b, DeviceNodeDb(b.input, self.device, self.lib))
        except BaseException:
            for _, db in dbs.values():
                db.close()
            raise
        self.close()
        self.executors, self.dbs, self.pool_total = executors, dbs, pool_total
        if queues is not None:
            self.queues = {q.name: q for q in queues}
        self.cache: "OrderedDict[object, SchedulingResult]" = OrderedDict()

    def close(self) -> None:
        for _, db in getattr(self, "dbs", {}).values():
            db.close()
        self.dbs = {}

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

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
    def _run_dry(self, items: List[List[int]], job_class) -> Dict[Tuple[str, str, tuple], list]:
        """Every item (a list of job indices: a single job, or a gang) on every db, one launch per db.
        Returns {(executor id, node pool, setting): [explain result per item]}."""
        return {key: db.explain([[int(job_class[key][j]) for j in it] for it in items]) for key, (_, db) in self.dbs.items()} if items else {}

    def _register(self, key, jobs: List[JobSpec]) -> np.ndarray:
        """The classes of `jobs` on db `key`, the keys it has not seen appended to it (armada_nodedb_add_classes).
        A key whose rows look at a node label the db's static classes do not tell apart (they tell apart only
        the labels its keys so far look at) needs finer static classes: the db is then rebuilt with its classes
        so far and the new ones.  If the library refuses an append, builder and db stay as they were."""
        b, db = self.dbs[key]
        n_classes, n_rows = b.input.num_classes, b.input.num_static_rows
        try:
            job_class, new_classes, new_rows = b.add_jobs(jobs)
        except UnresolvedLabels:
            keyed = [copy.copy(j) for j in b.class_jobs + list(jobs)]
            for j in keyed:  # (the queue plays no part in a class; the builder wants every job in one of its queues)
                j.queue = ""
            nb = RoundInputBuilder(b.cfg, b.nodes, keyed, [QueueSpec("")])
            self.dbs[key] = (nb, DeviceNodeDb(nb.input, self.device, self.lib))
            db.close()
            return nb.job_class[len(b.class_jobs):]
        if len(new_classes) or len(new_rows):
            try:
                first = db.add_classes(b.class_request[new_classes.start:], b.class_pc[new_classes.start:], b.class_static_row[new_classes.start:],
                                       b.class_away_row[new_classes.start:], b.static_match[new_rows.start:], b.type_match[new_rows.start:])
                if first != new_classes.start:
                    raise abi.ArmadaError(abi.E_INTERNAL, f"the db numbered the new classes from {first}, the builder from {new_classes.start}")
            except BaseException:
                b.rollback(n_classes, n_rows)
                raise
        return job_class

    def check(self, jobs: Sequence[JobSpec]) -> Dict[str, SchedulingResult]:
        """SubmitChecker.Check (:210-267): the result of every job the budgets let it reach."""
        return self.check_with_durations(jobs)[0]

    def check_with_durations(self, jobs: Sequence[JobSpec]) -> Tuple[Dict[str, SchedulingResult], Dict[str, float]]:
        """SubmitChecker.Check (:210-267): the results and the seconds spent per queue."""
        clock, budget = self.clock, self.submit_check
        start = clock.now()
        global_deadline = _deadline(budget.max_duration, start)
        jobs = list(jobs)
        single = [copy.copy(j) for j in jobs]
        for j in single:  # getIndividualSchedulingResult strips the gang info (:270-271); it plays no part in a job's class
            j.gang_id, j.gang_cardinality = None, 1
        keys = [scheduling_key(j, self.factory.from_job(self.cfg.job_requests(j.requests))) for j in single]
        job_class = {key: self._register(key, single) for key in list(self.dbs)}
        by_queue: Dict[str, List[int]] = {}
        gangs: Dict[Tuple[str, str], List[int]] = {}
        for i, j in enumerate(jobs):
            by_queue.setdefault(j.queue, []).append(i)
            if j.gang_id is not None and j.gang_cardinality > 1:  # job.IsInGang()
                gangs.setdefault((j.queue, j.gang_id), []).append(i)
        # the launch: one job per scheduling key the cache does not hold, every gang whole
        first_of_key: Dict[object, int] = {}
        at_start: Dict[object, SchedulingResult] = {}  # the cached results, for the keys the walk may evict before it reaches them
        for i, k in enumerate(keys):
            if k in self.cache:
                at_start[k] = self.cache[k]
            else:
                first_of_key.setdefault(k, i)
        items = [[i] for i in first_of_key.values()] + list(gangs.values())
        dry = self._run_dry(items, job_class)
        item_of = {("job", k): n for n, k in enumerate(first_of_key)}
        item_of.update({("gang", g): len(first_of_key) + n for n, g in enumerate(gangs)})

        def individual(i: int) -> SchedulingResult:  # getIndividualSchedulingResult (:269-285)
            k = keys[i]
            if k in self.cache:
                self.cache.move_to_end(k)
                return self.cache[k]
            if ("job", k) in item_of:
                res = self._scheduling_result([i], item_of[("job", k)], single, dry, job_class)
            else:  # evicted since the check began: the reference recomputes it, to the same result
                res = at_start[k]
            self.cache[k] = res
            if len(self.cache) > RESULT_CACHE_SIZE:
                self.cache.popitem(last=False)
            return res

        results: Dict[str, SchedulingResult] = {}
        durations: Dict[str, float] = {}
        for queue in sorted(by_queue):
            if _exceeded(global_deadline, clock.now()):
                break
            queue_start = clock.now()
            queue_deadline = _deadline(budget.max_duration_per_queue, queue_start)
            processed = set()
            for i in by_queue[queue]:
                if _exceeded(queue_deadline, clock.now()) or _exceeded(global_deadline, clock.now()):
                    break
                j = jobs[i]
                g = (j.queue, j.gang_id)
                if g not in gangs:
                    results[j.id] = individual(i)
                    continue
                if g in processed:
                    continue
                res = next((r for r in (individual(m) for m in gangs[g]) if not r.is_schedulable), None)  # getGangSchedulingResult (:287-296)
                if res is None:
                    res = self._scheduling_result(gangs[g], item_of[("gang", g)], single, dry, job_class)
                for m in gangs[g]:
                    results[jobs[m].id] = res
                processed.add(g)
            durations[queue] = clock.since(queue_start)
        return results, durations

    def _scheduling_result(self, members: List[int], k: int, jobs, dry, job_class) -> SchedulingResult:
        """getSchedulingResult (:302-422) of one item: the k-th of the launch `dry`."""
        f = self.factory
        req = np.sum([f.from_job(self.cfg.job_requests(jobs[i].requests)) for i in members], axis=0)
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
                    key = (e.id, node_pool, self.settings[pool.name])
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
                        b = self.dbs[key][0]
                        cls = int(job_class[key][members[0]])
                        excluded = excluded_nodes_by_reason(b, cls, recs)
                        sb.append(":\n" + pod_scheduling_context_string(b.input.num_nodes, excluded) + "\n---\n")
                    else:
                        sb.append(f": {placed} out of {len(members)} pods schedulable\n")
        if successful:
            return SchedulingResult(True, successful)
        return SchedulingResult(False, [], "".join(sb))
