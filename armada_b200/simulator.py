"""cmd/simulator on the device path: YAML specs in, state transitions and parquet rows out.

Host-side mirror of `internal/scheduler/simulator` (SURVEY §8 f4).  The event loop, the workload
bootstrap, the accounting between rounds and the sink rows follow the reference:

  specs       ClusterSpec / WorkloadSpec / SchedulingConfig from YAML files of the reference's schema
              (simulator/runner.go:14-87, simulator.proto; testdata/{clusters,workloads,configs}/*.yaml)
  event loop  a heap of (time, sequence number) events: schedule events every cycle period and event
              sequences (submit, leased, succeeded, preempted) — simulator.go:206-250, 494-536
  a round     per pool: queue contexts for the queues with demand, one PreemptingQueueScheduler round
              (simulator.go:538-714) — HERE the round is `armada_round_schedule` on the GPU
              (`DeviceRound.schedule`); there is no CPU path in this module
  handlers    submit / leased / succeeded / preempted (simulator.go:716-1014)
  sinks       jobs.parquet rows (sink/job_writer.go:17-32,76-104) and queue_stats.parquet rows
              (sink/queue_stats_writer.go:15-76)

Deviations, all deterministic stand-ins for things that are random in the reference: job ids are
zero-padded counters (the reference's ULIDs sort by creation time, these do too); pools of a cycle
are visited in name order (the reference ranges over a Go map); the shifted-exponential tails use a
PCG64 stream seeded with WorkloadSpec.randomSeed (the reference uses math/rand — a run with
tailMean = 0 everywhere is comparable row for row, others in distribution only).  Gang jobs carry the
template's node-uniformity label, by default the cluster name (simulator.go:456-462): a gang lands
on ONE cluster of its pool (the round's node-uniformity search, gang_scheduler.go:154-223).
"""
from __future__ import annotations

import heapq
import math
import re
from dataclasses import dataclass, field
from fractions import Fraction
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi
from .model import (AwayNodeType, JobSpec, NodeSpec, PriorityClass, QueueSpec, ResourceType, RoundInputBuilder, RoundResult,
                    SchedulingConfig, Taint, Toleration, apply_respect_node_pod_limits, parse_quantity)

CLUSTER_LABEL = "armadaproject.io/clusterName"  # simulator.go:45
NS = 1_000_000_000


class UnsupportedSpec(ValueError):
    pass


# ------------------------------------------------------------------------------------------------
# specs (simulator.proto)
# ------------------------------------------------------------------------------------------------
_DUR = re.compile(r"([0-9]*\.?[0-9]+)(ns|us|µs|ms|s|m|h)")
_DUR_NS = {"ns": 1, "us": 1_000, "µs": 1_000, "ms": 1_000_000, "s": NS, "m": 60 * NS, "h": 3600 * NS}


def parse_duration(v) -> int:
    """Go time.ParseDuration ("5m", "1h30m", "90s"); numbers are seconds.  Returns nanoseconds."""
    if v is None:
        return 0
    if isinstance(v, (int, float)):
        return int(round(v * NS))
    s = str(v).strip()
    if s in ("", "0"):
        return 0
    pos, total = 0, Fraction(0)
    for m in _DUR.finditer(s):
        if m.start() != pos:
            raise ValueError(f"bad duration {v!r}")
        total += Fraction(m.group(1)) * _DUR_NS[m.group(2)]
        pos = m.end()
    if pos != len(s):
        raise ValueError(f"bad duration {v!r}")
    return int(total)


@dataclass
class ShiftedExponential:
    minimum: int = 0  # ns
    tail_mean: int = 0  # ns

    @staticmethod
    def parse(d) -> "ShiftedExponential":
        d = d or {}
        return ShiftedExponential(parse_duration(d.get("minimum")), parse_duration(d.get("tailMean")))


@dataclass
class NodeTemplate:
    number: int
    total_resources: Dict[str, object]
    labels: Dict[str, str] = field(default_factory=dict)
    taints: Tuple[Taint, ...] = ()


@dataclass
class Cluster:
    name: str
    pool: str
    node_templates: List[NodeTemplate]


@dataclass
class ClusterSpec:
    name: str
    clusters: List[Cluster]
    workflow_manager_delay: ShiftedExponential = field(default_factory=ShiftedExponential)
    pending_delay: ShiftedExponential = field(default_factory=ShiftedExponential)


@dataclass
class JobTemplate:
    id: str
    queue: str
    number: int
    job_set: str = ""
    queue_priority: int = 0
    priority_class_name: str = ""
    requests: Dict[str, object] = field(default_factory=dict)
    tolerations: Tuple[Toleration, ...] = ()
    node_selector: Dict[str, str] = field(default_factory=dict)
    earliest_submit_time: int = 0
    earliest_submit_time_from_dependency_completion: int = 0
    dependencies: List[str] = field(default_factory=list)
    runtime: ShiftedExponential = field(default_factory=ShiftedExponential)
    gang_cardinality: int = 0
    gang_node_uniformity_label: str = ""
    repeat: Optional[Tuple[int, int]] = None  # (numTimes, period ns)
    number_successful: int = 0


@dataclass
class Queue:
    name: str
    weight: float
    job_templates: List[JobTemplate]


@dataclass
class WorkloadSpec:
    name: str
    queues: List[Queue]
    random_seed: int = 0


def _taints(lst) -> Tuple[Taint, ...]:
    return tuple(Taint(t.get("key", ""), str(t.get("value", "")), t.get("effect", "NoSchedule")) for t in (lst or []))


def _tolerations(lst) -> Tuple[Toleration, ...]:
    return tuple(Toleration(key=t.get("key", ""), operator=t.get("operator", "Equal"), value=str(t.get("value", "")),
                            effect=t.get("effect", "")) for t in (lst or []))


def cluster_spec_from_dict(d: dict, default_name: str = "") -> ClusterSpec:
    """ClusterSpecFromFilePath (runner.go:30-50)."""
    clusters = []
    for c in d.get("clusters") or []:
        nts = [NodeTemplate(int(t.get("number", 0)), dict(((t.get("totalResources") or {}).get("resources")) or {}),
                            dict(t.get("labels") or {}), _taints(t.get("taints"))) for t in c.get("nodeTemplates") or []]
        clusters.append(Cluster(str(c.get("name", "")), str(c.get("pool", "")), nts))
    spec = ClusterSpec(str(d.get("name") or default_name), clusters, ShiftedExponential.parse(d.get("workflowManagerDelayDistribution")),
                       ShiftedExponential.parse(d.get("pendingDelayDistribution")))
    # validateClusterSpec (simulator.go:257-274)
    names = [c.name for c in spec.clusters]
    if len(set(names)) != len(names):
        raise ValueError("duplicate cluster name")
    for c in spec.clusters:
        if not c.name or not c.pool:
            raise ValueError("cluster needs a name and a pool")
    return spec


def workload_spec_from_dict(d: dict, default_name: str = "") -> WorkloadSpec:
    """WorkloadSpecFromFilePath + initialiseWorkloadSpec (runner.go:52-87)."""
    queues = []
    for q in d.get("queues") or []:
        name = str(q["name"])
        jts = []
        for i, t in enumerate(q.get("jobTemplates") or []):
            req = t.get("requirements") or {}
            rr = (req.get("resourceRequirements") or {})
            rep = t.get("repeat")
            jts.append(JobTemplate(
                id=str(t.get("id") or f"{name}-{i}"), queue=name, number=int(t.get("number", 0)), job_set=str(t.get("jobSet", "")),
                queue_priority=int(t.get("queuePriority", 0)), priority_class_name=str(t.get("priorityClassName", "")),
                requests=dict(rr.get("requests") or {}), tolerations=_tolerations(req.get("tolerations")),
                node_selector={str(k): str(v) for k, v in (req.get("nodeSelector") or {}).items()},
                earliest_submit_time=parse_duration(t.get("earliestSubmitTime")),
                earliest_submit_time_from_dependency_completion=parse_duration(t.get("earliestSubmitTimeFromDependencyCompletion")),
                dependencies=[str(x) for x in (t.get("dependencies") or [])], runtime=ShiftedExponential.parse(t.get("runtimeDistribution")),
                gang_cardinality=int(t.get("gangCardinality", 0)), gang_node_uniformity_label=str(t.get("gangNodeUniformityLabel", "")),
                repeat=(int(rep.get("numTimes", 0)), parse_duration(rep.get("period"))) if rep else None))
        weight = float(q.get("weight", 0.0))
        queues.append(Queue(name, weight, jts))
    spec = WorkloadSpec(str(d.get("name") or default_name), queues, int(d.get("randomSeed", 0)))
    # validateWorkloadSpec (simulator.go:276-308)
    seen = set()
    for q in spec.queues:
        if q.weight <= 0:
            raise ValueError(f"queue {q.name} has a non-positive weight")
        for t in q.job_templates:
            if t.id in seen:
                raise ValueError(f"duplicate job template id {t.id}")
            seen.add(t.id)
            if t.gang_cardinality and t.number % t.gang_cardinality:
                raise ValueError(f"template {t.id}: number is not a multiple of the gang cardinality")
    return spec


def scheduling_config_from_dict(d: dict) -> Tuple[SchedulingConfig, str]:
    """The hot-path subset of configuration.SchedulingConfig (SchedulingConfigFromFilePath, runner.go:14-28).
    Returns (config, defaultPriorityClassName)."""
    key = {k.lower(): v for k, v in d.items()}

    def g(name, default=None):
        return key.get(name.lower(), default)

    def rate(v, default):
        if v is None:
            return default
        s = str(v).strip().lower()
        return math.inf if s in ("+inf", "inf") else float(s)

    supported = [ResourceType(str(r["name"]), str(r.get("resolution", "1"))) for r in g("supportedResourceTypes") or []]
    indexed = [ResourceType(str(r["name"]), str(r.get("resolution", "1"))) for r in g("indexedResources") or []]
    pcs = {}
    for name, p in (g("priorityClasses") or {}).items():
        pk = {k.lower(): v for k, v in (p or {}).items()}
        away = tuple(AwayNodeType(int(a.get("priority", 0)), str(a.get("wellKnownNodeTypeName", ""))) for a in pk.get("awaynodetypes") or [])
        pcs[str(name)] = PriorityClass(int(pk.get("priority", 0)), bool(pk.get("preemptible", False)), away,
                                       {str(k): float(v) for k, v in (pk.get("maximumresourcefractionperqueue") or {}).items()})
    wk = {str(w["name"]): _taints(w.get("taints")) for w in g("wellKnownNodeTypes") or []}
    exp = g("experimentalDominantResourceFairnessResourcesToConsider")
    if g("floatingResources"):
        raise UnsupportedSpec("floating resources")
    cfg = SchedulingConfig(
        supported_resource_types=supported, indexed_resources=indexed, priority_classes=pcs,
        indexed_taints=g("indexedTaints"), indexed_node_labels=tuple(g("indexedNodeLabels") or ()), well_known_node_types=wk,
        drf_resources=tuple(g("dominantResourceFairnessResourcesToConsider") or ()),
        drf_multipliers={str(r["name"]): float(r.get("multiplier", 1.0)) for r in exp} if exp else None,
        protected_fraction_of_fair_share=float(g("protectedFractionOfFairShare", 0.0)),
        protect_uncapped_adjusted_fair_share=bool(g("protectUncappedAdjustedFairShare", False)),
        max_queue_lookback=int(g("maxQueueLookback", 0)),
        maximum_resource_fraction_to_schedule={str(k): float(v) for k, v in (g("maximumResourceFractionToSchedule") or {}).items()} or None,
        maximum_scheduling_rate=rate(g("maximumSchedulingRate"), math.inf), maximum_scheduling_burst=int(g("maximumSchedulingBurst", 2**62)),
        maximum_per_queue_scheduling_rate=rate(g("maximumPerQueueSchedulingRate"), math.inf),
        maximum_per_queue_scheduling_burst=int(g("maximumPerQueueSchedulingBurst", 2**62)),
        enable_prefer_large_job_ordering=bool(g("enablePreferLargeJobOrdering", False)),
        disallowed_resources=(), respect_node_pod_limits=bool(g("respectNodePodLimits", False)))
    return cfg, str(g("defaultPriorityClassName", ""))


def _load_yaml(path: str) -> dict:
    import yaml
    with open(path) as f:
        return yaml.safe_load(f) or {}


def _stem(path: str) -> str:
    import os
    return os.path.splitext(os.path.basename(path))[0]


def cluster_spec_from_file(path: str) -> ClusterSpec:
    return cluster_spec_from_dict(_load_yaml(path), _stem(path))


def workload_spec_from_file(path: str) -> WorkloadSpec:
    return workload_spec_from_dict(_load_yaml(path), _stem(path))


def scheduling_config_from_file(path: str) -> Tuple[SchedulingConfig, str]:
    return scheduling_config_from_dict(_load_yaml(path))


def expand_repeating_templates(w: WorkloadSpec) -> WorkloadSpec:
    """expandRepeatingTemplates (simulator.go:1031-1053)."""
    import copy
    out = WorkloadSpec(w.name, [], w.random_seed)
    for q in w.queues:
        ts = []
        for t in q.job_templates:
            if t.repeat:
                times, period = t.repeat
                for i in range(times):
                    c = copy.deepcopy(t)
                    c.repeat = None
                    c.id = f"{t.id}-repeat-{i}"
                    c.earliest_submit_time = t.earliest_submit_time + i * period
                    ts.append(c)
            else:
                ts.append(copy.deepcopy(t))
        out.queues.append(Queue(q.name, q.weight, ts))
    return out


# ------------------------------------------------------------------------------------------------
# sink rows
# ------------------------------------------------------------------------------------------------
@dataclass
class JobRunRow:
    """sink/job_writer.go:17-32."""
    queue: str
    job_set: str
    job_id: str
    run_id: str
    priority_class: str
    cpu: float
    memory: float
    gpu: float
    ephemeral_storage: float
    exit_code: int
    state: str
    submitted_time: int
    scheduled_time: int
    finished_time: int


@dataclass
class QueueStatsRow:
    """sink/queue_stats_writer.go:15-31."""
    ts: int
    queue: str
    pool: str
    fair_share: float
    adjusted_fair_share: float
    actual_share: float
    cpu_share: float
    memory_share: float
    gpu_share: float
    allocated_cpu: int
    allocated_memory: int
    allocated_gpu: int
    num_scheduled: int
    num_preempted: int
    num_evicted: int


class MemorySink:
    """Keeps the rows (tests, callers that post-process)."""

    def __init__(self):
        self.job_rows: List[JobRunRow] = []
        self.queue_rows: List[QueueStatsRow] = []

    def on_job_rows(self, rows: Sequence[JobRunRow]):
        self.job_rows += rows

    def on_cycle_end(self, rows: Sequence[QueueStatsRow]):
        self.queue_rows += rows

    def close(self):
        pass


class ParquetSink(MemorySink):
    """jobs.parquet + queue_stats.parquet under `path`, the reference's column names and types
    (sink/sink.go:25-70)."""

    def __init__(self, path: str):
        super().__init__()
        self.path = path

    def close(self):
        import os
        import pyarrow as pa
        import pyarrow.parquet as pq
        os.makedirs(self.path, exist_ok=True)

        def table(rows, cls, i32):
            cols = {}
            for f in cls.__dataclass_fields__:
                vals = [getattr(r, f) for r in rows]
                typ = cls.__dataclass_fields__[f].type
                if typ in ("str", str):
                    cols[f] = pa.array(vals, pa.string())
                elif typ in ("float", float):
                    cols[f] = pa.array(vals, pa.float64())
                else:
                    cols[f] = pa.array(vals, pa.int32() if f in i32 else pa.int64())
            return pa.table(cols)

        pq.write_table(table(self.job_rows, JobRunRow, {"exit_code"}), os.path.join(self.path, "jobs.parquet"))
        pq.write_table(table(self.queue_rows, QueueStatsRow, {"num_scheduled", "num_preempted", "num_evicted"}),
                       os.path.join(self.path, "queue_stats.parquet"))


# ------------------------------------------------------------------------------------------------
# simulator
# ------------------------------------------------------------------------------------------------
@dataclass
class _Job:
    id: str
    queue: str
    job_set: str
    template: JobTemplate
    created: int  # logical timestamp: the job order inside a queue (simulator.go:801)
    submit_time: int  # ns
    gang_id: Optional[str]
    queued: bool = True
    node: Optional[str] = None
    pool: Optional[str] = None
    scheduled_at_priority: Optional[int] = None
    run_id: Optional[str] = None
    run_created: int = 0
    terminal: bool = False


@dataclass
class StateTransition:
    """model.StateTransition: what the sinks and `Simulator.transitions` see (kind ∈ submit, leased,
    succeeded, preempted)."""
    time: int
    kind: str
    job_id: str
    queue: str
    node: Optional[str] = None


Engine = Callable[[abi.RoundInput], RoundResult]


def device_engine(device: int = 0) -> Engine:
    """The product engine: one persistent `ArmadaRound` handle on the GPU.  Raises without the CUDA
    library / a device — there is no CPU path."""
    from .scheduler import DeviceRound
    dev = DeviceRound(device)
    return dev.schedule


class Simulator:
    """simulator.NewSimulator / Run (simulator.go:114-250)."""

    def __init__(self, cluster_spec: ClusterSpec, workload_spec: WorkloadSpec, scheduling_config: SchedulingConfig,
                 default_priority_class: str = "", engine: Optional[Engine] = None, sink=None, enable_fast_forward: bool = False,
                 hard_termination_minutes: int = 0, scheduler_cycle_period_seconds: int = 10):
        self.cluster_spec = cluster_spec
        self.workload_spec = expand_repeating_templates(workload_spec)
        self.cfg = scheduling_config
        self.default_pc = default_priority_class
        self.engine = engine if engine is not None else device_engine(0)
        self.sink = sink if sink is not None else MemorySink()
        self.enable_fast_forward = enable_fast_forward
        self.hard_termination_ns = hard_termination_minutes * 60 * NS
        self.period_ns = scheduler_cycle_period_seconds * NS
        apply_respect_node_pod_limits(self.cfg)  # NewSimulator (simulator.go:123), before the factory is made
        self.factory = scheduling_config.factory()
        self.time = 0  # epochStart
        self.seq = 0
        self.events: List[Tuple[int, int, object]] = []
        self.should_schedule = False
        self.logical_created = 0
        self.next_id = 0
        self.jobs: Dict[str, _Job] = {}  # the JobDb: queued and running jobs
        self.active_templates: Dict[str, JobTemplate] = {}
        self.templates_by_dependency: Dict[str, Dict[str, JobTemplate]] = {}
        self.demand_by_queue: Dict[str, np.ndarray] = {}
        self.alloc: Dict[str, Dict[str, Dict[str, np.ndarray]]] = {}  # pool -> queue -> pc -> int64[D]
        self.nodes_by_pool: Dict[str, List[NodeSpec]] = {}
        self.pool_of_node: Dict[str, str] = {}
        self.transitions: List[StateTransition] = []
        self.rounds = 0
        self.rng = np.random.Generator(np.random.PCG64(self.workload_spec.random_seed or 1))
        self._setup_clusters()
        self._bootstrap_workload()

    # -- setup -------------------------------------------------------------------------------
    def _setup_clusters(self):
        """setupClusters (simulator.go:310-378): node ids "<cluster>-<template>-<i>", the cluster label."""
        index = 0
        clusters_of_pool: Dict[str, int] = {}
        for c in self.cluster_spec.clusters:
            clusters_of_pool[c.pool] = clusters_of_pool.get(c.pool, 0) + 1
            for ti, t in enumerate(c.node_templates):
                labels = dict(t.labels)
                labels[CLUSTER_LABEL] = c.name
                for i in range(t.number):
                    nid = f"{c.name}-{ti}-{i}"
                    self.nodes_by_pool.setdefault(c.pool, []).append(NodeSpec(nid, index, dict(t.total_resources), t.taints, labels))
                    self.pool_of_node[nid] = c.pool
                    index += 1
        labels = list(self.cfg.indexed_node_labels)
        if CLUSTER_LABEL not in labels:
            self.cfg.indexed_node_labels = tuple(labels + [CLUSTER_LABEL])
        for pool in self.nodes_by_pool:
            self.alloc[pool] = {}

    def _new_id(self) -> str:
        self.next_id += 1
        return f"{self.next_id:026d}"  # sorts by creation, like a ULID

    def _submit_events(self, t: JobTemplate, at: int):
        evs = []
        gang_id = None
        for k in range(t.number):
            jid = self._new_id()
            if t.gang_cardinality and k % t.gang_cardinality == 0:
                gang_id = f"{self._new_id()}-0"
            evs.append(("submit", jid, t, gang_id if t.gang_cardinality else None))
        if evs:
            self._push(at, ("sequence", t.queue, t.job_set, evs))

    def _bootstrap_workload(self):
        """bootstrapWorkload (simulator.go:380-446)."""
        for q in self.workload_spec.queues:
            for t in q.job_templates:
                self.active_templates[t.id] = t
        for q in self.workload_spec.queues:
            for t in q.job_templates:
                if not t.dependencies:
                    self._submit_events(t, self.time + t.earliest_submit_time)
        for q in self.workload_spec.queues:
            for t in q.job_templates:
                for dep in t.dependencies:
                    if dep not in self.active_templates:
                        raise ValueError(f"jobTemplate {t.id} depends on jobTemplate {dep}, which does not exist")
                    self.templates_by_dependency.setdefault(dep, {})[t.id] = t

    # -- event log ---------------------------------------------------------------------------
    def _push(self, at: int, ev):
        heapq.heappush(self.events, (at, self.seq, ev))
        self.seq += 1

    def run(self) -> "Simulator":
        """Run (simulator.go:206-250)."""
        self._push(self.time, ("schedule",))
        end = self.time + (self.hard_termination_ns if self.hard_termination_ns > 0 else 100 * 365 * 24 * 3600 * NS)
        while self.events:
            at, _, ev = heapq.heappop(self.events)
            self.time = at
            if ev[0] == "schedule":
                self._handle_schedule()
            else:
                self._handle_sequence(ev)
            if self.time > end:
                break
        self.sink.close()
        return self

    def _duration(self, d: ShiftedExponential) -> int:
        """generateRandomShiftedExponentialDuration (simulator.go:855-871)."""
        tail = int(self.rng.exponential() * d.tail_mean) if d.tail_mean else 0
        return d.minimum + tail

    # -- a cycle -----------------------------------------------------------------------------
    def _job_spec(self, j: _Job) -> JobSpec:
        t = j.template
        return JobSpec(id=j.id, queue=j.queue, priority_class=t.priority_class_name or self.default_pc, requests=t.requests,
                       queue_priority=t.queue_priority, submit_time=j.created, tolerations=t.tolerations, node_selector=t.node_selector,
                       gang_id=j.gang_id, gang_cardinality=t.gang_cardinality if j.gang_id else 1,
                       gang_node_uniformity_label=(t.gang_node_uniformity_label or CLUSTER_LABEL) if j.gang_id else None, node=j.node,
                       scheduled_at_priority=j.scheduled_at_priority, active_run_timestamp=j.run_created)

    def _handle_schedule(self):
        """handleScheduleEvent (simulator.go:538-714)."""
        if self.active_templates:
            self._push(self.time + self.period_ns, ("schedule",))
        if not self.should_schedule and self.enable_fast_forward:
            return
        sequences = []
        weights = {q.name: q.weight for q in self.workload_spec.queues}
        for pool in sorted(self.nodes_by_pool):
            nodes = self.nodes_by_pool[pool]
            jobs = [j for j in self.jobs.values() if not j.terminal and (j.queued or j.pool == pool)]
            jobs.sort(key=lambda j: j.id)
            queues = []
            for q in self.workload_spec.queues:
                if q.name not in self.demand_by_queue:  # only queues that ever had a job (simulator.go:573-578)
                    continue
                dem = self.demand_by_queue[q.name]
                queues.append(QueueSpec(q.name, 1.0 / weights[q.name], False, dict(self.alloc[pool].get(q.name, {})), dem.copy(), dem.copy()))
            if not queues:
                continue
            specs = [self._job_spec(j) for j in jobs]
            b = RoundInputBuilder(self.cfg, nodes, specs, queues)
            res = self.engine(b.input)
            self.rounds += 1
            state, node = res.job_state, res.job_node
            preempted = [jobs[i] for i in range(len(jobs)) if state[i] == abi.JOB_PREEMPTED]
            scheduled = [jobs[i] for i in range(len(jobs)) if state[i] == abi.JOB_SCHEDULED]
            sched_at = {jobs[i].id: int(res.job_scheduled_at_priority[i]) for i in range(len(jobs)) if state[i] == abi.JOB_SCHEDULED}
            node_of = {jobs[i].id: nodes[int(node[i])].id for i in range(len(jobs)) if state[i] == abi.JOB_SCHEDULED}
            self._queue_stats(pool, b, res, jobs)
            key = lambda j: (j.queue, j.id)  # noqa: E731  (deterministic event order, simulator.go:627-646)
            preempted.sort(key=key)
            scheduled.sort(key=key)
            for j in preempted:
                j.queued = False
                j.terminal = True  # run failed, job failed
            for j in scheduled:
                j.queued = False
                j.node, j.pool = node_of[j.id], pool
                j.scheduled_at_priority = sched_at[j.id]
                j.run_id = self._new_id()
                j.run_created = self.time
            # sctx.AllocatedByQueueAndPriority() (simulator.go:673)
            qa = res.queue_allocated_by_pc
            self.alloc[pool] = {q.name: {pcn: qa[qi, pi].copy() for pi, pcn in enumerate(b.pc_names)} for qi, q in enumerate(b.queues)}
            for j in preempted:
                sequences.append((j.queue, j.job_set, [("preempted", j.id)]))
            for j in scheduled:
                sequences.append((j.queue, j.job_set, [("leased", j.id, pool)]))
            if self.time != 0 and not scheduled and not preempted:
                self.should_schedule = False
        for queue, job_set, evs in sequences:
            self._push(self.time, ("sequence", queue, job_set, evs))

    def _queue_stats(self, pool: str, b: RoundInputBuilder, res: RoundResult, jobs: List[_Job]):
        """QueueStatsWriter.Update (sink/queue_stats_writer.go:47-76)."""
        f = self.factory
        state = res.job_state
        D = f.D
        total_alloc = res.queue_allocated.sum(axis=0)
        drf_mult = np.array([b.input.drf_multipliers[d] for d in range(D)])
        totals = b.total_resources.astype(np.float64)

        def share(qi, name):
            if name not in f.index:
                return float("nan")
            d = f.index[name]
            return float(res.queue_allocated[qi, d]) / float(total_alloc[d]) if total_alloc[d] else float("nan")

        def units(qi, name):
            if name not in f.index:
                return 0
            d = f.index[name]
            return int(float(Fraction(int(res.queue_allocated[qi, d])) * Fraction(10) ** f.scales[d]))

        rows = []
        for qi, q in enumerate(b.queues):
            mine = [i for i, j in enumerate(jobs) if j.queue == q.name]
            cost = 0.0
            for d in range(D):  # UnweightedCostFromAllocation (fairness.go:99-105)
                if drf_mult[d] > 0 and totals[d] > 0:
                    cost = max(cost, float(res.queue_allocated[qi, d]) / totals[d] * drf_mult[d])
            rows.append(QueueStatsRow(
                ts=self.time // NS, queue=q.name, pool=pool, fair_share=float(res.queue_fair_share[qi, 0]),
                adjusted_fair_share=float(res.queue_fair_share[qi, 1]), actual_share=float(cost), cpu_share=share(qi, "cpu"),
                memory_share=share(qi, "memory"), gpu_share=share(qi, "nvidia.com/gpu"), allocated_cpu=units(qi, "cpu"),
                allocated_memory=units(qi, "memory") // (1024 * 1024), allocated_gpu=units(qi, "nvidia.com/gpu"),
                num_scheduled=sum(1 for i in mine if state[i] in (abi.JOB_SCHEDULED, abi.JOB_SCHEDULED_AND_EVICTED)),
                num_preempted=sum(1 for i in mine if state[i] == abi.JOB_PREEMPTED),
                num_evicted=sum(1 for i in mine if state[i] in (abi.JOB_PREEMPTED, abi.JOB_SCHEDULED_AND_EVICTED))))
        self.sink.on_cycle_end(rows)

    # -- event sequences -----------------------------------------------------------------------
    def _req_vector(self, t: JobTemplate) -> np.ndarray:
        return self.factory.from_job(self.cfg.job_requests(t.requests))

    def _row(self, j: _Job, state: str) -> JobRunRow:
        t = j.template

        def q(name):
            return float(parse_quantity(t.requests[name])) if name in t.requests else 0.0

        return JobRunRow(j.queue, j.job_set, j.id, j.run_id or "", t.priority_class_name or self.default_pc, q("cpu"), q("memory"),
                         q("nvidia.com/gpu"), q("ephemeral-storage"), 0, state, j.submit_time // NS, j.run_created // NS, self.time // NS)

    def _handle_sequence(self, ev):
        """handleEventSequence (simulator.go:716-776)."""
        _, queue, job_set, evs = ev
        rows = []
        for e in evs:
            kind = e[0]
            if kind == "submit":
                self.should_schedule = True
                _, jid, t, gang_id = e
                self.logical_created += 1
                j = _Job(jid, queue, job_set, t, self.logical_created, self.time, gang_id)
                self.jobs[jid] = j
                self.demand_by_queue[queue] = self.demand_by_queue.get(queue, np.zeros(self.factory.D, np.int64)) + self._req_vector(t)
                self.transitions.append(StateTransition(self.time, "submit", jid, queue))
            elif kind == "leased":  # handleJobRunLeased (simulator.go:817-849)
                _, jid, pool = e
                j = self.jobs[jid]
                done = self.time + self._duration(self.cluster_spec.pending_delay)
                if j.gang_id:  # gang members end together (simulator.go:463-464)
                    done += j.template.runtime.minimum
                else:
                    done += self._duration(j.template.runtime)
                self._push(done, ("sequence", queue, job_set, [("succeeded", jid)]))
                self.transitions.append(StateTransition(self.time, "leased", jid, queue, j.node))
            elif kind == "succeeded":  # handleJobSucceeded (simulator.go:873-944)
                self.should_schedule = True
                _, jid = e
                j = self.jobs.get(jid)
                if j is None or j.terminal:
                    continue
                del self.jobs[jid]
                t = j.template
                pcn = t.priority_class_name or self.default_pc
                a = self.alloc[j.pool].setdefault(j.queue, {})
                a[pcn] = a.get(pcn, np.zeros(self.factory.D, np.int64)) - self._req_vector(t)
                self.demand_by_queue[j.queue] = self.demand_by_queue[j.queue] - self._req_vector(t)
                rows.append(self._row(j, "SUCCEEDED"))
                self.transitions.append(StateTransition(self.time, "succeeded", jid, queue, j.node))
                t.number_successful += 1
                if t.number == t.number_successful:
                    self.active_templates.pop(t.id, None)
                    for dep in list(self.templates_by_dependency.get(t.id, {}).values()):
                        dep.dependencies.remove(t.id)
                        if dep.dependencies:
                            continue
                        at = max(self.time + dep.earliest_submit_time, self.time + dep.earliest_submit_time_from_dependency_completion)
                        self._submit_events(dep, at)
                    self.templates_by_dependency.pop(t.id, None)
            elif kind == "preempted":  # handleJobRunPreempted (simulator.go:977-1014)
                self.should_schedule = True
                _, jid = e
                j = self.jobs.pop(jid)
                self.demand_by_queue[j.queue] = self.demand_by_queue[j.queue] - self._req_vector(j.template)
                gang_id = None
                if j.gang_id and j.template.gang_cardinality > 1:
                    attempt = int(j.gang_id.split("-")[1])  # (always the first attempt's number, like the reference)
                    gang_id = f"{j.gang_id}-{attempt + 1}"
                retry = self._new_id()
                at = self.time + self._duration(self.cluster_spec.workflow_manager_delay)
                self._push(at, ("sequence", queue, job_set, [("submit", retry, j.template, gang_id)]))
                rows.append(self._row(j, "PREEMPTED"))
                self.transitions.append(StateTransition(self.time, "preempted", jid, queue, j.node))
        if rows:
            self.sink.on_job_rows(rows)


def simulate_files(cluster_path: str, workload_path: str, config_path: str, output_dir: Optional[str] = None, engine: Optional[Engine] = None,
                   **kw) -> Simulator:
    """cmd/simulator --clusters … --workloads … --configs … [--outputDir …]."""
    cfg, default_pc = scheduling_config_from_file(config_path)
    sink = ParquetSink(output_dir) if output_dir else MemorySink()
    sim = Simulator(cluster_spec_from_file(cluster_path), workload_spec_from_file(workload_path), cfg, default_pc, engine=engine, sink=sink, **kw)
    return sim.run()


def main(argv: Optional[Sequence[str]] = None) -> int:
    """cmd/simulator's command line (cmd/simulator/cmd/root.go:24-33): `python -m armada_b200.simulator --clusters C.yaml
    --workloads W.yaml --config S.yaml --outputDir out/`.  Every round runs on cuda:0 (no CPU path)."""
    import argparse
    import os
    import sys
    import time
    ap = argparse.ArgumentParser(prog="armada_b200.simulator")
    ap.add_argument("--clusters", required=True, help="Path specifying cluster configurations to simulate.")
    ap.add_argument("--workloads", required=True, help="Path specifying workloads to simulate.")
    ap.add_argument("--config", required=True, help="Path to scheduler configurations to simulate.")
    ap.add_argument("--outputDir", default="", help="Directory for jobs.parquet / queue_stats.parquet (default: a timestamped directory).")
    ap.add_argument("--overwriteOutputDir", action="store_true")
    ap.add_argument("--enableFastForward", action="store_true", help="Skips schedule events when we're in a steady state")
    ap.add_argument("--hardTerminationMinutes", type=int, default=-1, help="Limit the time simulated.  -1 for no limit.")
    ap.add_argument("--schedulerCyclePeriodSeconds", type=int, default=10)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    out = a.outputDir or time.strftime("armada_simulator_%Y_%m_%d_%H_%M_%S")
    if os.path.exists(out) and os.listdir(out) and not a.overwriteOutputDir:
        print(f"output directory {out} already exists and is not empty (use --overwriteOutputDir)", file=sys.stderr)
        return 1
    t0 = time.perf_counter()
    s = simulate_files(a.clusters, a.workloads, a.config, output_dir=out, engine=device_engine(a.device), enable_fast_forward=a.enableFastForward,
                       hard_termination_minutes=max(a.hardTerminationMinutes, 0), scheduler_cycle_period_seconds=a.schedulerCyclePeriodSeconds)
    print(f"simulated {s.time / NS:.0f} s in {s.rounds} rounds, {len(s.sink.job_rows)} job rows -> {out} ({time.perf_counter() - t0:.1f} s wall)")
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
