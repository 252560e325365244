"""Host-side mirror of the reference's scheduler-internal types for ONE round, and the
flattening of those types into the SoA `ArmadaRoundInput` the C ABI consumes.

Mirrors (names follow the reference):
  * ResourceListFactory / quantity scaling   internaltypes/resource_list_factory.go:21-109,
                                              internaltypes/quantity_util.go:7-18
  * Node, NodeType                            internaltypes/node.go:26-62, node_type.go:68-124
  * taint / toleration / selector / affinity  nodedb/nodematching.go:127-240,
    matching (static predicates)              kubernetesobjects/taint/taint.go:44-58,
                                              k8s component-helpers v0.32 (restated below)
  * PriorityClass / AwayNodeType              common/types/scheduling.go:56-109
  * per-round / per-queue limits              scheduling/constraints/constraints.go:213-256
The string logic runs on the host; the device only sees dense ids and bitmaps.
"""
from __future__ import annotations

import ctypes
import math
import operator
from dataclasses import dataclass, field, replace
from fractions import Fraction
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi

UNSCHEDULABLE_TAINT_KEY = "armadaproject.io/unschedulable"  # internaltypes/unschedulable.go:7-17
NODE_ID_LABEL = "armadaproject.io/nodeId"
WILDCARD = "*"  # configuration.WildCardWellKnownNodeTypeValue
PODS = "pods"  # armadaresource.PodsResourceName: the node's pod capacity (node.Status.Allocatable["pods"])

_SUFFIX = {
    "": Fraction(1), "n": Fraction(1, 10**9), "u": Fraction(1, 10**6), "m": Fraction(1, 1000), "k": Fraction(10**3), "M": Fraction(10**6), "G": Fraction(10**9),
    "T": Fraction(10**12), "P": Fraction(10**15), "Ki": Fraction(2**10), "Mi": Fraction(2**20),
    "Gi": Fraction(2**30), "Ti": Fraction(2**40), "Pi": Fraction(2**50), "Ei": Fraction(2**60), "E": Fraction(10**18),
}


def parse_quantity(q) -> Fraction:
    """k8s resource.Quantity → exact rational (subset: decimal number + SI/binary suffix)."""
    if isinstance(q, (int, Fraction)):
        return Fraction(q)
    s = str(q).strip()
    for suf in ("Ki", "Mi", "Gi", "Ti", "Pi", "Ei", "n", "u", "m", "k", "M", "G", "T", "P", "E"):
        if s.endswith(suf):
            return Fraction(s[: -len(suf)]) * _SUFFIX[suf]
    return Fraction(s)


@dataclass(frozen=True)
class ResourceType:
    name: str
    resolution: str  # e.g. "1m" → scale -3 ; "1" → scale 0


class ResourceListFactory:
    """internaltypes.ResourceListFactory: fixed resource order + per-resource decimal scale."""

    def __init__(self, supported: Sequence[ResourceType]):
        self.names = [r.name for r in supported]
        self.index = {n: i for i, n in enumerate(self.names)}
        # scale = floor(log10(resolution)), resource_list_factory.go:66-71
        self.scales = [int(math.floor(math.log10(float(parse_quantity(r.resolution))))) for r in supported]
        self.D = len(self.names)

    def _scaled(self, name: str, q, round_up: bool) -> int:
        i = self.index[name]
        v = parse_quantity(q) / (Fraction(10) ** self.scales[i])
        return int(math.ceil(v)) if round_up else int(math.floor(v))

    def from_node(self, res: Dict[str, object]) -> np.ndarray:  # FromNodeProto: round DOWN, ignore unknown
        out = np.zeros(self.D, dtype=np.int64)
        for k, v in res.items():
            if k in self.index:
                out[self.index[k]] = self._scaled(k, v, False)
        return out

    def from_job(self, res: Dict[str, object]) -> np.ndarray:  # FromJobResourceListIgnoreUnknown: round UP
        out = np.zeros(self.D, dtype=np.int64)
        for k, v in res.items():
            if k in self.index:
                out[self.index[k]] = self._scaled(k, v, True)
        return out

    def scaled_value(self, name: str, q) -> int:  # Quantity.ScaledValue (rounds up)
        return self._scaled(name, q, True)


@dataclass(frozen=True)
class Taint:
    key: str
    value: str = ""
    effect: str = "NoSchedule"


@dataclass(frozen=True)
class Toleration:
    key: str = ""
    operator: str = ""  # "", "Equal", "Exists"
    value: str = ""
    effect: str = ""


def toleration_tolerates_taint(t: Toleration, taint: Taint) -> bool:
    """v1.Toleration.ToleratesTaint (k8s api core/v1 toleration.go)."""
    if t.effect and t.effect != taint.effect:
        return False
    if t.key and t.key != taint.key:
        return False
    if t.operator in ("", "Equal"):
        return t.value == taint.value
    return t.operator == "Exists"


def find_untolerated(taints: Sequence[Taint], tolerations: Sequence[Toleration]) -> Optional[Taint]:
    """koTaint.FindMatchingUntoleratedTaint: ALL taints must be tolerated, whatever their effect."""
    for taint in taints:
        if not any(toleration_tolerates_taint(t, taint) for t in tolerations):
            return taint
    return None


@dataclass(frozen=True)
class MatchExpression:
    key: str
    operator: str  # In, NotIn, Exists, DoesNotExist, Gt, Lt
    values: Tuple[str, ...] = ()


def _match_expr(labels: Dict[str, str], e: MatchExpression) -> bool:
    has = e.key in labels
    v = labels.get(e.key)
    if e.operator == "In":
        return has and v in e.values
    if e.operator == "NotIn":
        return (not has) or v not in e.values
    if e.operator == "Exists":
        return has
    if e.operator == "DoesNotExist":
        return not has
    if e.operator in ("Gt", "Lt"):
        if not has or len(e.values) != 1:
            return False
        try:
            a, b = int(v), int(e.values[0])
        except ValueError:
            return False
        return a > b if e.operator == "Gt" else a < b
    return False


def match_node_selector_terms(labels: Dict[str, str], terms: Sequence[Tuple[MatchExpression, ...]]) -> bool:
    """corev1.MatchNodeSelectorTerms: terms are ORed, expressions ANDed, empty term matches nothing."""
    for term in terms:
        if len(term) == 0:
            continue
        if all(_match_expr(labels, e) for e in term):
            return True
    return False


@dataclass
class AwayNodeType:
    priority: int
    well_known_node_type: str = ""
    # extra (name, [(resource, op, value)]) entries: types.AwayTypeEntry
    node_types: Tuple[Tuple[str, Tuple[Tuple[str, str, str], ...]], ...] = ()


@dataclass
class PriorityClass:
    priority: int
    preemptible: bool
    away_node_types: Tuple[AwayNodeType, ...] = ()
    # MaximumResourceFractionPerQueue (types/scheduling.go:62-68)
    maximum_resource_fraction_per_queue: Dict[str, float] = field(default_factory=dict)


@dataclass(frozen=True)
class FloatingResource:
    name: str
    resolution: str = "1"
    quantity: Optional[object] = None  # the pool's total; None = this pool is not listed for the resource


@dataclass
class SchedulingConfig:
    """The hot-path-relevant subset of configuration.SchedulingConfig (configuration.go:186-361)."""
    supported_resource_types: Sequence[ResourceType]
    indexed_resources: Sequence[ResourceType]  # resolution in quantity units, e.g. cpu "1", memory "128Mi"
    priority_classes: Dict[str, PriorityClass]
    indexed_taints: Optional[Sequence[str]] = None  # None ⇒ all taints indexed
    indexed_node_labels: Sequence[str] = ()
    well_known_node_types: Dict[str, Tuple[Taint, ...]] = field(default_factory=dict)
    drf_resources: Sequence[str] = ()  # DominantResourceFairnessResourcesToConsider
    drf_multipliers: Optional[Dict[str, float]] = None  # Experimental…ResourcesToConsider
    protected_fraction_of_fair_share: float = 0.0
    protect_uncapped_adjusted_fair_share: bool = False
    max_queue_lookback: int = 0
    maximum_resource_fraction_to_schedule: Optional[Dict[str, float]] = None
    maximum_scheduling_rate: float = math.inf
    maximum_scheduling_burst: int = 2**62
    maximum_per_queue_scheduling_rate: float = math.inf
    maximum_per_queue_scheduling_burst: int = 2**62
    enable_prefer_large_job_ordering: bool = True
    disable_home_scheduling: bool = False
    disable_away_scheduling: bool = False
    disable_gang_away_scheduling: bool = False
    disallowed_resources: Sequence[str] = ()
    # FloatingResources of THIS pool (configuration.FloatingResourceConfig): resources no node holds, limited per pool
    floating_resources: Sequence["FloatingResource"] = ()
    # RespectNodePodLimits (configuration.go:227): every job is one pod, counted against each node's `pods` capacity.
    # Takes effect once apply_respect_node_pod_limits has added `pods` to the resource lists.
    respect_node_pod_limits: bool = False

    def job_requests(self, requests: Dict[str, object]) -> Dict[str, object]:
        """A job's requests as the JobDb records them (getResourceRequirements, jobdb.go:256-263): with
        respect_node_pod_limits the job asks for one pod, whatever its own requests say about pods."""
        return {**requests, PODS: 1} if self.respect_node_pod_limits else requests

    def factory(self) -> ResourceListFactory:
        # NewResourceListFactory: the supported (Kubernetes) types, then the floating ones (resource_list_factory.go:41-53)
        return ResourceListFactory(list(self.supported_resource_types) + [ResourceType(f.name, f.resolution) for f in self.floating_resources])

    def allowed_priorities(self) -> List[int]:
        """types.AllowedPriorities (common/types/scheduling.go:99-109): PC + away priorities, sorted, unique."""
        ps = set()
        for pc in self.priority_classes.values():
            ps.add(pc.priority)
            for a in pc.away_node_types:
                ps.add(a.priority)
        return sorted(ps)


def apply_respect_node_pod_limits(cfg: SchedulingConfig) -> bool:
    """ApplyRespectNodePodLimits (configuration.go:548-580): with the knob on, `pods` at resolution 1 becomes a
    supported and an indexed resource, so that the factory, the NodeDb's index and every resource list count pods.
    An existing `pods` entry is reset to resolution 1 in place (each job is exactly one pod slot); otherwise the
    entry is appended.  Idempotent; returns whether the knob is on (and the config was brought to that form).
    Call it before the config makes a factory, a builder, a SubmitChecker or a Simulator."""
    if not cfg.respect_node_pod_limits:
        return False

    def ensure(types: Sequence[ResourceType]) -> List[ResourceType]:  # ensurePodsResourceType
        out = list(types)
        for i, t in enumerate(out):
            if t.name == PODS:
                out[i] = ResourceType(PODS, "1")
                return out
        return out + [ResourceType(PODS, "1")]

    cfg.supported_resource_types = ensure(cfg.supported_resource_types)
    cfg.indexed_resources = ensure(cfg.indexed_resources)
    return True


@dataclass
class NodeSpec:
    id: str
    index: int
    total: Dict[str, object]
    taints: Tuple[Taint, ...] = ()
    labels: Dict[str, str] = field(default_factory=dict)
    allocatable: Optional[Dict[str, object]] = None  # default: total
    unschedulable: bool = False
    over_allocated: bool = False
    # whether the node type was made with the unschedulable taint (None: as `unschedulable` says).  A node that
    # populateNodeDb marks unschedulable keeps the type it was created with (WithSchedulable, node.go:302-310).
    type_unschedulable: Optional[bool] = None


@dataclass
class JobSpec:
    id: str
    queue: str
    priority_class: str
    requests: Dict[str, object]
    queue_priority: int = 0
    submit_time: int = 0
    tolerations: Tuple[Toleration, ...] = ()
    node_selector: Dict[str, str] = field(default_factory=dict)
    affinity: Optional[Tuple[Tuple[MatchExpression, ...], ...]] = None  # required node-affinity terms
    gang_id: Optional[str] = None
    gang_cardinality: int = 1
    gang_node_uniformity_label: Optional[str] = None  # GangInfo.NodeUniformity() (jobdb/gang.go)
    node: Optional[str] = None  # id of the node the job runs on (None = queued)
    scheduled_at_priority: Optional[int] = None
    active_run_timestamp: int = 0


@dataclass
class QueueSpec:
    name: str
    priority_factor: float = 1.0
    cordoned: bool = False
    allocated_by_pc: Dict[str, np.ndarray] = field(default_factory=dict)  # pc name -> int64[D]
    demand: Optional[np.ndarray] = None  # int64[D]
    constrained_demand: Optional[np.ndarray] = None
    short_job_penalty: Optional[np.ndarray] = None
    limiter_tokens: Optional[float] = None  # None ⇒ burst (fresh limiter)
    # per-queue overrides of MaximumResourceFraction by priority class name
    resource_limits_by_pc: Dict[str, Dict[str, float]] = field(default_factory=dict)


def multiply_resource(res: int, m: float) -> int:
    """multiplyResource, internaltypes/resource_list.go:312-331."""
    if m == 1.0:
        return int(res)
    if math.isinf(m):
        return (2**63 - 1) if ((m < 0) == (res < 0)) else -(2**63)
    v = float(res) * m
    if v >= 9.223372036854775807e18:  # Go int64(float) overflow is implementation-defined; saturate
        return 2**63 - 1
    if v <= -9.223372036854775808e18:
        return -(2**63)
    return int(v)


def _kubernetes_requirements(cfg: SchedulingConfig, f: "ResourceListFactory", requests) -> np.ndarray:
    """Job.KubernetesResourceRequirements in factory units: the floating resources left out."""
    req = f.from_job(cfg.job_requests(requests))
    for fr in cfg.floating_resources:
        req[f.index[fr.name]] = 0
    return req


def queue_limit_fractions(cfg: SchedulingConfig, pc_name: str, q: "QueueSpec") -> Dict[str, float]:
    """calculatePerQueueLimits' fractions of one (queue, priority class), constraints.go:231-256."""
    fractions = dict(cfg.priority_classes[pc_name].maximum_resource_fraction_per_queue)
    fractions.update(q.resource_limits_by_pc.get(pc_name, {}))
    return fractions


def populate_node_db(cfg: SchedulingConfig, nodes: Sequence[NodeSpec], jobs: Sequence[JobSpec], other_pool_jobs: Sequence[JobSpec],
                     queues: Sequence["QueueSpec"] = ()):
    """populateNodeDb (scheduling_algo.go:861-935), the pool's total (:455-456) and NewSchedulingConstraints
    (constraints/constraints.go:94-111, 205-256) on the specs of a pool as reported.  `jobs` are this pool's, `other_pool_jobs`
    the other pools' (running ones have `node` set; jobs on nodes outside `nodes` are skipped).  Returns
    (nodes, total, constraints): the NodeSpecs the NodeDb holds, in the given order — an unschedulable node without a job
    of this pool is dropped; a node whose jobs Exceed its allocatable is over-allocated and unschedulable (keeping its node
    type); the other pools' requests come off the allocatable, floored at zero — the total [D] (their allocatable plus the
    floating totals), and {"max_resources_to_schedule": [D], "queue_limit": {queue: {priority class: [D]}}}."""
    f = cfg.factory()
    ids = {n.id for n in nodes}
    pool_jobs: Dict[str, int] = {}
    used: Dict[str, np.ndarray] = {}
    other: Dict[str, np.ndarray] = {}
    for j in jobs:
        if j.node is None or j.node not in ids:
            continue
        pool_jobs[j.node] = pool_jobs.get(j.node, 0) + 1
        used[j.node] = used.get(j.node, np.zeros(f.D, np.int64)) + _kubernetes_requirements(cfg, f, j.requests)
    for j in other_pool_jobs:
        if j.node is None or j.node not in ids:
            continue
        req = _kubernetes_requirements(cfg, f, j.requests)
        used[j.node] = used.get(j.node, np.zeros(f.D, np.int64)) + req
        other[j.node] = other.get(j.node, np.zeros(f.D, np.int64)) + req
    kept: List[NodeSpec] = []
    total = np.zeros(f.D, np.int64)
    for n in nodes:
        if n.unschedulable and not pool_jobs.get(n.id):
            continue
        alloc = f.from_node(n.allocatable if n.allocatable is not None else n.total)
        m = replace(n, over_allocated=False)
        if n.id in used and (used[n.id] > alloc).any():
            m = replace(m, over_allocated=True, unschedulable=True, type_unschedulable=n.unschedulable)
        if n.id in other:  # MarkResourceUnallocatable, node.go:285-294
            alloc = np.maximum(alloc - other[n.id], 0)
            m = replace(m, allocatable={name: Fraction(int(alloc[i])) * Fraction(10) ** f.scales[i] for i, name in enumerate(f.names)})
        kept.append(m)
        total += alloc
    for fr in cfg.floating_resources:
        if fr.quantity is not None:
            total[f.index[fr.name]] += f.scaled_value(fr.name, fr.quantity)
    fr = cfg.maximum_resource_fraction_to_schedule or {}
    constraints = {"max_resources_to_schedule": np.array([multiply_resource(int(total[d]), fr.get(name, math.inf)) for d, name in enumerate(f.names)], np.int64),
                   "queue_limit": {q.name: {pc: np.array([multiply_resource(int(total[d]), queue_limit_fractions(cfg, pc, q).get(name, math.inf))
                                                          for d, name in enumerate(f.names)], np.int64) for pc in cfg.priority_classes}
                                   for q in queues}}
    return kept, total, constraints


class UnresolvedLabels(ValueError):
    """RoundInputBuilder.add_jobs: a new row looks at a node label the builder's static classes do not resolve."""


def scheduling_key(j: JobSpec, req: np.ndarray):
    """A job's class: the fields of its SchedulingKey (node selector, affinity, tolerations, requests, priority
    class; internaltypes/podutils.go:49-68), `req` being its requests in factory units."""
    return (tuple(sorted(j.tolerations, key=repr)), tuple(sorted(j.node_selector.items())), j.affinity, tuple(int(x) for x in req), j.priority_class)


class RoundInputBuilder:
    """Flattens (config, nodes, jobs, queues) into an ArmadaRoundInput.  Every array the input points into is the
    builder's attribute of the field's name and lives as long as the builder."""

    # NULL unless a gang of the round has a node uniformity label / the caller gives its queued order
    gang_uniformity_label = uniformity_value_start = class_uniformity_row = None
    queued_start = queued_order = None

    def __init__(self, cfg: SchedulingConfig, nodes: Sequence[NodeSpec], jobs: Sequence[JobSpec],
                 queues: Sequence[QueueSpec], total_resources: Optional[np.ndarray] = None,
                 queued_order: Optional[Dict[str, List[str]]] = None, global_limiter_tokens: Optional[float] = None,
                 other_pool_jobs: Optional[Sequence[JobSpec]] = None):
        """`other_pool_jobs` given (a list, possibly empty): the pool as reported, for armada_round_upload_cluster.  Then
        `self.cluster_state` is its ArmadaClusterState; the nodes' over_allocated is not read, and every static class without
        the unschedulable taint gets a variant with it (static_class_unschedulable), matched like the others."""
        self.cfg = cfg
        self.other_pool_jobs = None if other_pool_jobs is None else list(other_pool_jobs)
        self.factory = cfg.factory()
        self.nodes = list(nodes)
        self.jobs = list(jobs)
        self.queues = sorted(queues, key=lambda q: q.name)  # index order == name order
        self.queue_index = {q.name: i for i, q in enumerate(self.queues)}
        self.node_pos = {n.id: i for i, n in enumerate(self.nodes)}
        self.job_pos = {j.id: i for i, j in enumerate(self.jobs)}
        self._keep: List[object] = []
        self.pc_names = sorted(cfg.priority_classes.keys())
        self.pc_index = {n: i for i, n in enumerate(self.pc_names)}
        self.input = abi.RoundInput()
        self.input._keepalive = self._keep
        self._rows: Dict[object, int] = {}  # the static bitmap rows: key -> index into row_specs
        self.row_specs: List[Tuple[Tuple[Toleration, ...], Tuple[Tuple[str, str], ...], object]] = []
        self._config()
        class_meta = self._job_classes()
        class_uniformity_row = self._uniformity_rows(class_meta)  # adds rows, so it runs before anything reads the row table
        self._nodes()  # the row table → the label keys rows look at → the static classes
        self._match()
        self._jobs(class_uniformity_row)
        self._context(total_resources, global_limiter_tokens)
        self._queues()  # the per-queue limits are fractions of _context's total_resources
        if queued_order is not None:
            self._queued_order(queued_order)
        if self.other_pool_jobs is not None:
            self._cluster_state()

    # -- helpers ---------------------------------------------------------------------------
    def _attach(self, **arrays):
        vars(self).update(abi.attach(self.input, self._keep, **arrays))

    def _row(self, tolerations, selector, affinity) -> int:
        """The static row of (tolerations, node selector, affinity); a new one is appended to row_specs."""
        key = (tuple(sorted(tolerations, key=repr)), tuple(sorted(selector.items())), affinity)
        if key not in self._rows:
            self._rows[key] = len(self.row_specs)
            self.row_specs.append((tuple(tolerations), tuple(sorted(selector.items())), affinity))
        return self._rows[key]

    def _node_taints(self, n: NodeSpec) -> Tuple[Taint, ...]:
        t = tuple(n.taints)
        if n.unschedulable:  # CreateNodeAndType, node.go:120-122
            t = t + (Taint(UNSCHEDULABLE_TAINT_KEY, "true", "NoSchedule"),)
        return t

    def _node_labels(self, n: NodeSpec) -> Dict[str, str]:
        labels = dict(n.labels)
        labels[NODE_ID_LABEL] = n.id
        return labels

    def _away_tolerations(self, pc: PriorityClass, k: int, req: np.ndarray) -> Tuple[Toleration, ...]:
        """getEffectiveAwayNodeTaints + toleration synthesis, nodedb.go:532-598."""
        away = pc.away_node_types[k]
        taints: List[Taint] = []
        if away.well_known_node_type:
            taints += list(self.cfg.well_known_node_types.get(away.well_known_node_type, ()))
        for name, conditions in away.node_types:
            ok = True
            for (resource, op, value) in conditions:  # matchesCondition :514-530 (first condition decides)
                jv = int(parse_quantity(0))
                if resource in self.factory.index:
                    i = self.factory.index[resource]
                    # GetByNameZeroIfMissing(...).Value(): quantity rounded up to an integer
                    jv = int(math.ceil(Fraction(int(req[i])) * (Fraction(10) ** self.factory.scales[i])))
                v = int(math.ceil(parse_quantity(value)))
                ok = {">": jv > v, "<": jv < v, "==": jv == v}[op]
                break
            if ok:
                taints += list(self.cfg.well_known_node_types[name])
        out = []
        for t in taints:
            if t.value == WILDCARD:
                out.append(Toleration(key=t.key, operator="Exists", effect=t.effect))
            else:
                out.append(Toleration(key=t.key, value=t.value, effect=t.effect))
        return tuple(out)

    # -- stages, in the order __init__ runs them --------------------------------------------
    def _config(self):
        """Resources, the node index, priorities and priority classes."""
        cfg, f, inp = self.cfg, self.factory, self.input
        inp.abi_version = abi.ABI_VERSION
        inp.num_resources = f.D
        inp.num_indexed = len(cfg.indexed_resources)
        for i, r in enumerate(cfg.indexed_resources):
            inp.indexed_resource[i] = f.index[r.name]
            inp.indexed_resolution[i] = f.scaled_value(r.name, r.resolution)  # makeIndexedResourceResolution
        self.priorities = [-1] + cfg.allowed_priorities()
        inp.num_priorities = len(self.priorities)
        for i, p in enumerate(self.priorities):
            inp.priorities[i] = p
        well_known_names = sorted(cfg.well_known_node_types.keys())
        inp.num_priority_classes = len(self.pc_names)
        for i, name in enumerate(self.pc_names):
            pc = cfg.priority_classes[name]
            s = inp.priority_classes[i]
            s.priority = pc.priority
            s.preemptible = 1 if pc.preemptible else 0
            s.num_away = len(pc.away_node_types)
            for k, a in enumerate(pc.away_node_types):
                s.away_priority[k] = a.priority
                # (a name without a WellKnownNodeTypes entry adds no taints here; the reference fails the away attempt that reaches it)
                s.away_well_known[k] = well_known_names.index(a.well_known_node_type) if a.well_known_node_type in well_known_names else abi.NONE

    def _job_classes(self) -> List[Tuple[Tuple[Toleration, ...], Dict[str, str], object, List[Tuple[Toleration, ...]]]]:
        """Job classes with their home and away rows, and each job's class.  Returns per class its tolerations,
        selector, affinity and per away node type the tolerations it adds, from which the uniformity rows are made."""
        self._classes: Dict[object, int] = {}
        self._class_req: List[np.ndarray] = []
        self._class_pc: List[int] = []
        self._class_row: List[int] = []
        self._class_away: List[List[int]] = []
        self._class_meta: List[Tuple[Tuple[Toleration, ...], Dict[str, str], object, List[Tuple[Toleration, ...]]]] = []
        self.class_jobs: List[JobSpec] = []  # the first job of each class (none for the placeholder class)
        job_class = self._register(self.jobs)
        if not self._class_req:  # keep arrays non-empty for the C side (no jobs: no uniformity rows follow this row); no job has this class
            self._class_req, self._class_pc, self._class_row = [np.zeros(self.factory.D, np.int64)], [0], [self._row((), {}, None)]
            self._class_away = [[abi.NONE] * abi.MAX_AWAY]
        self._attach_classes()
        self._attach(job_class=job_class if self.jobs else [0])
        return self._class_meta

    def _register(self, jobs: Sequence[JobSpec]) -> np.ndarray:
        """The class of each job, registering the classes (and their rows) not seen before."""
        cfg, f = self.cfg, self.factory
        job_class = np.zeros(len(jobs), dtype=np.uint32)
        for ji, j in enumerate(jobs):
            req = f.from_job(cfg.job_requests(j.requests))
            key = scheduling_key(j, req)
            if key not in self._classes:
                self._classes[key] = len(self._class_req)
                self._class_req.append(req)
                pc = cfg.priority_classes[j.priority_class]
                self._class_pc.append(self.pc_index[j.priority_class])
                self._class_row.append(self._row(j.tolerations, j.node_selector, j.affinity))
                aw = [abi.NONE] * abi.MAX_AWAY
                extras: List[Tuple[Toleration, ...]] = []
                for k in range(len(pc.away_node_types)):
                    extra = self._away_tolerations(pc, k, req)
                    extras.append(extra)
                    if extra:
                        aw[k] = self._row(tuple(j.tolerations) + extra, j.node_selector, j.affinity)
                self._class_away.append(aw)
                self._class_meta.append((tuple(j.tolerations), dict(j.node_selector), j.affinity, extras))
                self.class_jobs.append(j)
            job_class[ji] = self._classes[key]
        return job_class

    def _attach_classes(self):
        self.input.num_classes = len(self._class_req)
        self._attach(class_request=np.stack(self._class_req), class_pc=self._class_pc, class_static_row=self._class_row,
                     class_away_row=self._class_away, class_key_valid=np.ones(len(self._class_req)))

    def add_jobs(self, jobs: Sequence[JobSpec]) -> Tuple[np.ndarray, range, range]:
        """Register the classes of `jobs` (scheduling keys) against the builder's fixed node static classes and node
        types: the class arrays, row table and bitmaps grow, the nodes stay.  Returns each job's class, the new
        classes and the new rows (what armada_nodedb_add_classes appends to a NodeDb made from this builder's
        input).  Classes and rows get the ids a builder made with all the jobs at once gives them, as long as no
        placeholder class was made.  Raises UnresolvedLabels, the builder unchanged, when a new row looks at a node
        label the static classes do not tell apart (only labels the rows so far look at do): such jobs need a
        builder made with them.  Gang node uniformity is not registered (the dry-run NodeDb has none)."""
        c0, r0 = len(self._class_req), len(self.row_specs)
        job_class = self._register(jobs)
        for r in range(r0, len(self.row_specs)):
            _, selector, affinity = self.row_specs[r]
            keys = {k for k, _ in selector} | {e.key for term in (affinity or ()) for e in term}
            unresolved = sorted(k for k in keys if k in self.node_label_keys and k not in self.static_label_keys)
            if unresolved:
                self.rollback(c0, r0)
                raise UnresolvedLabels(f"the static classes do not tell nodes apart by label(s) {unresolved}")
        if len(self._class_req) > c0:
            self._attach_classes()
        if len(self.row_specs) > r0:
            sm, tm = self._match_rows(r0, len(self.row_specs))
            self.input.num_static_rows = len(self.row_specs)
            self._attach(static_match=np.concatenate([self.static_match, sm]), type_match=np.concatenate([self.type_match, tm]))
        return job_class, range(c0, len(self._class_req)), range(r0, len(self.row_specs))

    def rollback(self, num_classes: int, num_rows: int) -> None:
        """Forget the classes and rows from `num_classes` / `num_rows` on: what add_jobs registered since the
        builder had that many (when the db they were meant for refused them)."""
        for key in [k for k, c in self._classes.items() if c >= num_classes]:
            del self._classes[key]
        for seq in (self._class_req, self._class_pc, self._class_row, self._class_away, self._class_meta):
            del seq[num_classes:]
        del self.class_jobs[len(self._classes):]  # (the placeholder class has no key and no job)
        for key in [k for k, r in self._rows.items() if r >= num_rows]:
            del self._rows[key]
        del self.row_specs[num_rows:]
        self._attach_classes()
        self.input.num_static_rows = num_rows
        self._attach(static_match=self.static_match[:num_rows], type_match=self.type_match[:num_rows])

    def _uniformity_rows(self, class_meta) -> np.ndarray:
        """Gang node uniformity (gang_scheduler.go:154-223): value slots per label, rows per (class, slot).  Adds
        rows to the row table; returns the [C][V][1 + MAX_AWAY] rows for class_uniformity_row."""
        indexed_labels = set(self.cfg.indexed_node_labels)
        uni_labels: Dict[str, int] = {}
        uni_values: List[List[str]] = []
        uni_classes: Dict[int, set] = {}
        for ji, j in enumerate(self.jobs):
            lab = j.gang_node_uniformity_label
            if not lab or j.gang_id is None or j.gang_cardinality <= 1 or lab not in indexed_labels:
                continue
            if lab not in uni_labels:  # nodeDb.IndexedNodeLabelValues(label) minus "" (:181-190)
                uni_labels[lab] = len(uni_values)
                uni_values.append(sorted({self._node_labels(n)[lab] for n in self.nodes if self._node_labels(n).get(lab)}))
            uni_classes.setdefault(uni_labels[lab], set()).add(int(self.job_class[ji]))
        uni_start = [0]
        for vals in uni_values:
            uni_start.append(uni_start[-1] + len(vals))
        class_uni = np.full((self.input.num_classes, max(1, uni_start[-1]), 1 + abi.MAX_AWAY), abi.NONE, dtype=np.uint32)
        for lab, li in uni_labels.items():
            for c in uni_classes.get(li, ()):
                tol, sel, aff, extras = class_meta[c]
                for vi, val in enumerate(uni_values[li]):
                    sel2 = dict(sel)
                    sel2[lab] = val  # jctx.AddNodeSelector
                    class_uni[c, uni_start[li] + vi, 0] = self._row(tol, sel2, aff)
                    for k, extra in enumerate(extras):
                        if extra:
                            class_uni[c, uni_start[li] + vi, 1 + k] = self._row(tol + extra, sel2, aff)
        self.uni_labels, self.uni_values, self.uni_start = uni_labels, uni_values, uni_start
        return class_uni

    def _nodes(self):
        """Node resources, id ranks, static classes, node types and flags."""
        cfg, f, inp = self.cfg, self.factory, self.input
        N, D = len(self.nodes), f.D
        inp.num_nodes = N
        node_total = np.zeros((D, N), dtype=np.int64)
        node_alloc = np.zeros((D, N), dtype=np.int64)
        for i, n in enumerate(self.nodes):
            node_total[:, i] = f.from_node(n.total)
            node_alloc[:, i] = f.from_node(n.allocatable if n.allocatable is not None else n.total)
        id_rank = np.zeros(N, dtype=np.uint32)
        for r, i in enumerate(sorted(range(N), key=lambda i: self.nodes[i].id)):
            id_rank[i] = r
        indexed_taints = None if cfg.indexed_taints is None else set(cfg.indexed_taints)
        indexed_labels = set(cfg.indexed_node_labels)
        # relevant label keys: only labels some row looks at distinguish static classes
        rel_keys = set()
        for (_, selector, affinity) in self.row_specs:
            rel_keys.update(k for k, _ in selector)
            if affinity:
                for term in affinity:
                    rel_keys.update(e.key for e in term)
        static_classes: Dict[object, int] = {}
        static_specs: List[Tuple[Tuple[Taint, ...], Dict[str, str]]] = []
        node_static = np.zeros(N, dtype=np.uint32)
        types: Dict[object, int] = {}
        type_specs: List[Tuple[Tuple[Taint, ...], Dict[str, str], set]] = []
        node_type = np.zeros(N, dtype=np.uint32)
        node_flags = np.zeros(N, dtype=np.uint8)
        for i, n in enumerate(self.nodes):
            taints = self._node_taints(n)
            labels = self._node_labels(n)
            skey = (tuple(sorted(taints, key=repr)), tuple(sorted((k, v) for k, v in labels.items() if k in rel_keys)))
            if skey not in static_classes:
                static_classes[skey] = len(static_specs)
                static_specs.append((taints, labels))
            node_static[i] = static_classes[skey]
            # NewNodeType, node_type.go:68-124
            type_taints = taints if n.type_unschedulable is None else self._node_taints(replace(n, unschedulable=n.type_unschedulable))
            ttaints = tuple(t for t in type_taints if indexed_taints is None or t.key in indexed_taints)
            tlabels = {k: v for k, v in labels.items() if k in indexed_labels}
            unset = set(k for k in indexed_labels if k not in tlabels)
            tkey = (tuple(sorted(ttaints, key=repr)), tuple(sorted(tlabels.items())), tuple(sorted(unset)))
            forced = getattr(n, "forced_type", None)  # tests only: WithNodeTypeNodes
            if forced is not None:
                tkey = ("forced", forced)
            if tkey not in types:
                types[tkey] = len(type_specs)
                type_specs.append((ttaints, tlabels, unset))
            node_type[i] = types[tkey]
            over = n.over_allocated and self.other_pool_jobs is None  # (the cluster path derives it)
            node_flags[i] = (abi.NODE_UNSCHEDULABLE if n.unschedulable else 0) | (abi.NODE_OVERALLOCATED if over else 0)
        self.static_class_unschedulable = None
        if self.other_pool_jobs is not None:  # WithSchedulable(false): the class with the unschedulable taint added
            unsched = Taint(UNSCHEDULABLE_TAINT_KEY, "true", "NoSchedule")
            scu = []
            for taints, labels in list(static_specs):
                if any(t.key == UNSCHEDULABLE_TAINT_KEY for t in taints):
                    scu.append(abi.NONE)
                    continue
                vt = tuple(taints) + (unsched,)
                skey = (tuple(sorted(vt, key=repr)), tuple(sorted((k, v) for k, v in labels.items() if k in rel_keys)))
                if skey not in static_classes:
                    static_classes[skey] = len(static_specs)
                    static_specs.append((vt, labels))
                scu.append(static_classes[skey])
            scu += [abi.NONE] * (len(static_specs) - len(scu))
            self.static_class_unschedulable = scu
        inp.num_static_classes, inp.num_node_types = max(1, len(static_specs)), max(1, len(type_specs))
        self.static_specs, self.type_specs = static_specs, type_specs
        self.static_label_keys, self.node_label_keys = rel_keys, {k for n in self.nodes for k in self._node_labels(n)}
        self.type_keys = list(types.keys())
        self._attach(node_index=[n.index for n in self.nodes] or [0], node_id_rank=id_rank if N else [0],
                     node_type=node_type if N else [0], node_static_class=node_static if N else [0],
                     node_flags=node_flags if N else [0], node_total=node_total if N else np.zeros((D, 1)),
                     node_allocatable=node_alloc if N else np.zeros((D, 1)))

    def _match(self):
        """Per row, the static classes (static_match) and node types (type_match) its requirements admit."""
        self.input.num_static_rows = len(self.row_specs)
        static_match, type_match = self._match_rows(0, len(self.row_specs))
        self._attach(static_match=static_match, type_match=type_match)

    def _match_rows(self, r0: int, r1: int) -> Tuple[np.ndarray, np.ndarray]:
        """static_match and type_match of rows [r0, r1)."""
        S, T = self.input.num_static_classes, self.input.num_node_types
        static_match = np.zeros((r1 - r0, (S + 31) // 32), dtype=np.uint32)
        type_match = np.zeros((r1 - r0, (T + 31) // 32), dtype=np.uint32)
        for r, (tolerations, selector, affinity) in enumerate(self.row_specs[r0:r1]):
            for s, (taints, labels) in enumerate(self.static_specs):
                ok = find_untolerated(taints, tolerations) is None  # NodeTolerationRequirementsMet
                ok = ok and all(labels.get(k) == v for k, v in selector)  # NodeSelectorRequirementsMet(node, nil)
                if ok and affinity is not None:
                    ok = match_node_selector_terms(labels, affinity)  # NodeAffinityRequirementsMet
                if ok:
                    static_match[r, s >> 5] |= np.uint32(1 << (s & 31))
            for t, (ttaints, tlabels, unset) in enumerate(self.type_specs):
                ok = find_untolerated(ttaints, tolerations) is None  # TolerationRequirementsMet(nodeType)
                if ok:
                    for k, v in selector:  # NodeSelectorRequirementsMet(type labels, unsetIndexedLabels)
                        if k in tlabels:
                            if tlabels[k] != v:
                                ok = False
                                break
                        elif k in unset:
                            ok = False
                            break
                if ok:
                    type_match[r, t >> 5] |= np.uint32(1 << (t & 31))
        return static_match, type_match

    def _jobs(self, class_uniformity_row: np.ndarray):
        """Per-job arrays, gangs and the gangs' uniformity labels."""
        inp = self.input
        J = len(self.jobs)
        inp.num_jobs = J
        gangs: Dict[Tuple[str, str], int] = {}
        gang_card: List[int] = []
        job_gang = np.full(max(J, 1), abi.NONE, dtype=np.uint32)
        job_queue = np.full(max(J, 1), abi.NONE, dtype=np.uint32)
        job_node = np.full(max(J, 1), abi.NONE, dtype=np.uint32)
        job_sap = np.full(max(J, 1), abi.NO_PRIORITY, dtype=np.int32)
        job_qp = np.zeros(max(J, 1), dtype=np.uint32)
        job_st = np.zeros(max(J, 1), dtype=np.int64)
        job_art = np.zeros(max(J, 1), dtype=np.int64)
        job_id_rank = np.zeros(max(J, 1), dtype=np.uint32)
        for r, i in enumerate(sorted(range(J), key=lambda i: self.jobs[i].id)):
            job_id_rank[i] = r
        for ji, j in enumerate(self.jobs):
            if j.queue in self.queue_index:
                job_queue[ji] = self.queue_index[j.queue]
            if j.gang_id is not None and j.gang_cardinality > 1:  # GangInfo.IsGang
                gk = (j.queue, j.gang_id)
                if gk not in gangs:
                    gangs[gk] = len(gang_card)
                    gang_card.append(j.gang_cardinality)
                job_gang[ji] = gangs[gk]
            if j.node is not None:
                job_node[ji] = self.node_pos[j.node]
                if j.scheduled_at_priority is not None:
                    job_sap[ji] = j.scheduled_at_priority
            job_qp[ji] = j.queue_priority
            job_st[ji] = j.submit_time
            job_art[ji] = j.active_run_timestamp
        inp.num_gangs = len(gang_card)
        self._attach(job_queue=job_queue, job_queue_priority=job_qp, job_submit_time=job_st, job_id_rank=job_id_rank,
                     job_gang=job_gang, job_node=job_node, job_scheduled_at_priority=job_sap, job_active_run_timestamp=job_art,
                     gang_cardinality=gang_card or [0])
        indexed_labels = set(self.cfg.indexed_node_labels)
        gang_label = np.full(max(1, len(gang_card)), abi.NONE, dtype=np.uint32)
        for ji, j in enumerate(self.jobs):
            if job_gang[ji] != abi.NONE and j.gang_node_uniformity_label:
                lab = j.gang_node_uniformity_label
                gang_label[job_gang[ji]] = self.uni_labels[lab] if lab in indexed_labels else abi.LABEL_NOT_INDEXED
        if (gang_label != abi.NONE).any():
            inp.num_uniformity_labels = len(self.uni_values)
            self._attach(gang_uniformity_label=gang_label, uniformity_value_start=self.uni_start,
                         class_uniformity_row=class_uniformity_row)

    def _context(self, total_resources, global_limiter_tokens):
        """Floating resources, the scheduling context's scalars, the round's limits and its rate limiter."""
        cfg, f, inp = self.cfg, self.factory, self.input
        # floating resources (floatingresources/floating_resource_types.go:19-37)
        fmask = 0
        for fr in cfg.floating_resources:
            d = f.index[fr.name]
            fmask |= 1 << d
            if fr.quantity is not None:
                inp.floating_limits_configured = 1
                inp.floating_limit[d] = f.scaled_value(fr.name, fr.quantity)
        inp.floating_resource_mask = fmask
        if total_resources is None:  # nodeDb.TotalKubernetesResources(): Σ allocatable
            total_resources = self.node_allocatable.sum(axis=1) if self.nodes else np.zeros(f.D, np.int64)
        self.total_resources = np.asarray(total_resources, dtype=np.int64)
        for d in range(f.D):
            inp.total_resources[d] = int(self.total_resources[d])
        mult = {}
        if cfg.drf_multipliers:
            mult = {k: (v if v > 0 else 1.0) for k, v in cfg.drf_multipliers.items()}
        else:
            mult = {k: 1.0 for k in cfg.drf_resources}
        for d, name in enumerate(f.names):
            inp.drf_multipliers[d] = float(mult.get(name, 0.0))
        inp.protected_fraction_of_fair_share = cfg.protected_fraction_of_fair_share
        inp.protect_uncapped_adjusted_fair_share = int(cfg.protect_uncapped_adjusted_fair_share)
        inp.prefer_large_job_ordering = int(cfg.enable_prefer_large_job_ordering)
        inp.disable_home_scheduling = int(cfg.disable_home_scheduling)
        inp.disable_away_scheduling = int(cfg.disable_away_scheduling)
        inp.disable_gang_away_scheduling = int(cfg.disable_gang_away_scheduling)
        inp.max_queue_lookback = cfg.max_queue_lookback
        mask = 0
        for r in cfg.disallowed_resources:
            if r in f.index:
                mask |= 1 << f.index[r]
        inp.disallowed_resource_mask = mask
        # calculatePerRoundLimits, constraints.go:213-229 (missing fractions default to +Inf)
        inp.has_round_limit = 1
        fr = cfg.maximum_resource_fraction_to_schedule or {}
        for d, name in enumerate(f.names):
            inp.max_resources_to_schedule[d] = multiply_resource(int(self.total_resources[d]), fr.get(name, math.inf))
        # rate limiters (golang.org/x/time/rate): fresh limiter ⇒ tokens == burst
        inp.global_limiter_is_inf = int(math.isinf(cfg.maximum_scheduling_rate))
        inp.global_limiter_burst = min(cfg.maximum_scheduling_burst, 2**62)
        inp.global_limiter_tokens = float(inp.global_limiter_burst) if global_limiter_tokens is None else global_limiter_tokens

    def _queues(self):
        """Per-queue weights, accounting, limits (from total_resources) and rate limiters."""
        cfg, f = self.cfg, self.factory
        Qn, PCn, D = len(self.queues), len(self.pc_names), f.D
        self.input.num_queues = Qn
        qw = np.zeros(max(Qn, 1), dtype=np.float64)
        qc = np.zeros(max(Qn, 1), dtype=np.uint8)
        qa = np.zeros((max(Qn, 1), PCn, D), dtype=np.int64)
        qd = np.zeros((max(Qn, 1), D), dtype=np.int64)
        qcd = np.zeros((max(Qn, 1), D), dtype=np.int64)
        qp = np.zeros((max(Qn, 1), D), dtype=np.int64)
        qhl = np.zeros((max(Qn, 1), PCn), dtype=np.uint8)
        ql = np.zeros((max(Qn, 1), PCn, D), dtype=np.int64)
        qt = np.zeros(max(Qn, 1), dtype=np.float64)
        qb = np.zeros(max(Qn, 1), dtype=np.int64)
        qi = np.zeros(max(Qn, 1), dtype=np.uint8)
        for i, q in enumerate(self.queues):
            qw[i] = 1.0 / q.priority_factor if q.priority_factor > 0 else 1.0
            qc[i] = int(q.cordoned)
            for pcn, rl in q.allocated_by_pc.items():
                qa[i, self.pc_index[pcn]] = rl
            if q.demand is not None:
                qd[i] = q.demand
            if q.constrained_demand is not None:
                qcd[i] = q.constrained_demand
            elif q.demand is not None:
                qcd[i] = q.demand
            if q.short_job_penalty is not None:
                qp[i] = q.short_job_penalty
            # calculatePerQueueLimits, constraints.go:231-256
            for pcn in cfg.priority_classes:
                fractions = queue_limit_fractions(cfg, pcn, q)
                pi = self.pc_index[pcn]
                qhl[i, pi] = 1
                for d, name in enumerate(f.names):
                    ql[i, pi, d] = multiply_resource(int(self.total_resources[d]), fractions.get(name, math.inf))
            qb[i] = min(cfg.maximum_per_queue_scheduling_burst, 2**62)
            qt[i] = float(qb[i]) if q.limiter_tokens is None else q.limiter_tokens
            qi[i] = int(math.isinf(cfg.maximum_per_queue_scheduling_rate))
        self._attach(queue_weight=qw, queue_cordoned=qc, queue_allocated_by_pc=qa, queue_demand=qd, queue_constrained_demand=qcd,
                     queue_short_job_penalty=qp, queue_has_limit=qhl, queue_limit=ql, queue_limiter_tokens=qt,
                     queue_limiter_burst=qb, queue_limiter_is_inf=qi)

    def _cluster_state(self):
        """ArmadaClusterState: the other pools' running jobs on this pool's nodes, the unschedulable variants of the
        static classes and the caps of NewSchedulingConstraints as fractions (+Inf where none is configured)."""
        cfg, f = self.cfg, self.factory
        cs = abi.ClusterState()
        cs.abi_version = abi.ABI_VERSION
        on = [j for j in self.other_pool_jobs if j.node is not None and j.node in self.node_pos]
        cs.num_other_pool_jobs = len(on)
        fr = cfg.maximum_resource_fraction_to_schedule or {}
        cs.has_round_limit = 1
        for d, name in enumerate(f.names):
            cs.max_fraction_to_schedule[d] = fr.get(name, math.inf)
        qf = np.full((max(len(self.queues), 1), len(self.pc_names), f.D), math.inf)
        for i, q in enumerate(self.queues):
            for pcn in cfg.priority_classes:
                fractions = queue_limit_fractions(cfg, pcn, q)
                for d, name in enumerate(f.names):
                    qf[i, self.pc_index[pcn], d] = fractions.get(name, math.inf)
        self.cluster_keep: List[object] = []
        self.cluster_state_arrays = abi.attach(
            cs, self.cluster_keep, other_pool_job_node=[self.node_pos[j.node] for j in on] or [0],
            other_pool_job_request=[_kubernetes_requirements(cfg, f, j.requests) for j in on] or [np.zeros(f.D)],
            static_class_unschedulable=self.static_class_unschedulable, queue_limit_fraction=qf)
        cs._keepalive = self.cluster_keep
        self.cluster_state = cs

    def _queued_order(self, queued_order: Dict[str, List[str]]):
        """The caller's order of each queue's queued jobs: queues in index order, jobs by position."""
        start = [0]
        order: List[int] = []
        for q in self.queues:
            order += [self.job_pos[jid] for jid in queued_order.get(q.name, [])]
            start.append(len(order))
        self._attach(queued_start=start, queued_order=order or [0])

    # The names the arrays had before they were named after their fields.  Each is a read-only alias of the same
    # array, so code written against it, in-place writes included, changes what the library reads.
    FORMER_NAMES = {
        "qw": "queue_weight", "qc": "queue_cordoned", "qa": "queue_allocated_by_pc", "qd": "queue_demand",
        "qcd": "queue_constrained_demand", "qp": "queue_short_job_penalty", "qhl": "queue_has_limit", "ql": "queue_limit",
        "qt": "queue_limiter_tokens", "qb": "queue_limiter_burst", "qi": "queue_limiter_is_inf",
        "job_qp": "job_queue_priority", "job_st": "job_submit_time", "job_sap": "job_scheduled_at_priority",
        "job_art": "job_active_run_timestamp", "gang_card": "gang_cardinality", "class_row": "class_static_row",
        "class_away": "class_away_row", "node_static": "node_static_class", "node_alloc": "node_allocatable",
    }


for _former, _field in RoundInputBuilder.FORMER_NAMES.items():
    setattr(RoundInputBuilder, _former, property(operator.attrgetter(_field)))


class RoundResult:
    """Caller-allocated ArmadaRoundOutput + numpy views."""

    # ask for job_seq_first_pass / job_reason_first_pass (the inputs of `queue_stats`); off by default: 5 bytes per job
    # more to bring back per round.  tests/conftest.py switches it on for every test.
    FIRST_PASS_DEFAULT = False

    def __init__(self, inp: abi.RoundInput, first_pass: Optional[bool] = None):
        J, N, Q = max(inp.num_jobs, 1), max(inp.num_nodes, 1), max(inp.num_queues, 1)
        D, PL, PC = inp.num_resources, inp.num_priorities, inp.num_priority_classes
        shape = {"node_alloc": (PL, D, N), "queue_allocated": (Q, D), "queue_allocated_by_pc": (Q, PC, D), "queue_fair_share": (Q, 3),
                 "scheduled_resources": D, "evicted_resources": D, "job_excluded_nodes": (J, abi.EXCLUDED_KINDS)}  # the others: [J]
        arrays = {n: np.zeros(shape.get(n, J), abi.field_dtype(abi.RoundOutput, n)) for n in self.ARRAYS + self.FIRST_PASS_ARRAYS}
        arrays["job_node"].fill(abi.NONE)
        vars(self).update(arrays)
        self.first_pass = RoundResult.FIRST_PASS_DEFAULT if first_pass is None else first_pass
        skip = (() if inp.collect_excluded_nodes else ("job_excluded_nodes",)) + (() if self.first_pass else self.FIRST_PASS_ARRAYS)
        self.out = abi.RoundOutput()
        abi.attach(self.out, [], **{n: a for n, a in arrays.items() if n not in skip})  # the arrays live on self
        self.stats = abi.RoundStats()
        self.num_jobs = inp.num_jobs

    ARRAYS = ("job_state", "job_node", "job_scheduled_at_priority", "job_preempted_at_priority", "job_method",
              "job_reason", "job_seq", "node_alloc", "queue_allocated", "queue_allocated_by_pc", "queue_fair_share",
              "scheduled_resources", "evicted_resources", "job_excluded_nodes")
    FIRST_PASS_ARRAYS = ("job_seq_first_pass", "job_reason_first_pass")
    SCALARS = ("num_scheduled_jobs", "num_scheduled_gangs", "num_evicted_jobs", "termination_reason",
               "num_result_scheduled", "num_result_preempted")

    def diff(self, other: "RoundResult") -> List[str]:
        """Bit-exact comparison of every output; returns a list of human-readable mismatches."""
        bad = []
        names = self.ARRAYS + (self.FIRST_PASS_ARRAYS if self.first_pass and other.first_pass else ())
        for name in names:
            x, y = getattr(self, name), getattr(other, name)
            if x.dtype.kind == "f":
                eq = x.view(np.uint64) == y.view(np.uint64)
            else:
                eq = x == y
            if not eq.all():
                idx = np.argwhere(~eq)[:5].tolist()
                bad.append(f"{name}: {int((~eq).sum())} mismatches, first at {idx}: {x[tuple(idx[0])]} vs {y[tuple(idx[0])]}")
        for name in self.SCALARS:
            if getattr(self.out, name) != getattr(other.out, name):
                bad.append(f"{name}: {getattr(self.out, name)} vs {getattr(other.out, name)}")
        return bad


def _field(inp, name: str, n: int) -> np.ndarray:
    """Pointer field `name` of an ABI struct as a copy of its first n elements."""
    ptr = getattr(inp, name)
    return np.ctypeslib.as_array(ptr, (n,)).copy() if n and ptr else np.zeros(n, np.dtype(ptr._type_))


class ClusterSnapshot:
    """populateNodeDb (scheduling_algo.go:861-935) and NewSchedulingConstraints (constraints.go:94-111, 205-256)
    restated on the ABI arrays: what armada_round_upload_cluster derives from (inp, cs).

      input     the ArmadaRoundInput armada_round_upload takes for the same round: the kept nodes in the caller's
                order with their id ranks among themselves, node flags, static classes and allocatable as derived,
                job_node renumbered, the derived total and caps
      kept      the caller's index of each node of `input`
      snapshot  what armada_round_download_snapshot returns (the names of DeviceRound.download_snapshot)"""

    def __init__(self, inp: abi.RoundInput, cs: abi.ClusterState):
        N, D, J, K = inp.num_nodes, inp.num_resources, inp.num_jobs, cs.num_other_pool_jobs
        Q, PC, S = inp.num_queues, inp.num_priority_classes, inp.num_static_classes
        self.num_nodes = N
        node_kube = np.array([not ((inp.floating_resource_mask >> d) & 1) for d in range(D)])
        alloc_in = _field(inp, "node_allocatable", D * N).reshape(D, N)
        flags_in = _field(inp, "node_flags", N)
        sclass_in = _field(inp, "node_static_class", N)
        req = _field(inp, "class_request", inp.num_classes * D).reshape(-1, D) * node_kube  # KubernetesResourceRequirements
        jn = _field(inp, "job_node", J).astype(np.int64)
        run = jn != abi.NONE
        used = np.zeros((D, N), np.int64)
        np.add.at(used.T, jn[run], req[_field(inp, "job_class", J).astype(np.int64)[run]])
        pool_jobs = np.bincount(jn[run], minlength=N)
        on = _field(cs, "other_pool_job_node", K).astype(np.int64)
        oreq = _field(cs, "other_pool_job_request", K * D).reshape(K, D) * node_kube
        other = np.zeros((D, N), np.int64)
        np.add.at(other.T, on, oreq)
        used += other
        other_jobs = np.bincount(on, minlength=N)
        unsched = (flags_in & abi.NODE_UNSCHEDULABLE) != 0
        dropped = unsched & (pool_jobs == 0)  # no job of this pool: not inserted, not counted
        exceeds = ~dropped & (pool_jobs + other_jobs > 0) & (used > alloc_in).any(axis=0)
        scu = _field(cs, "static_class_unschedulable", S)
        sclass = sclass_in.copy()
        switch = exceeds & (scu[sclass_in] != abi.NONE)  # WithSchedulable(false) adds the taint, keeps the node type
        sclass[switch] = scu[sclass_in[switch]]
        marked = ~dropped & (other_jobs > 0)  # MarkResourceUnallocatable: allocatable - other pools, floored at zero
        alloc = np.where(marked, np.maximum(alloc_in - other, 0), alloc_in)
        state = (np.where(unsched, abi.NODE_UNSCHEDULABLE, 0) | np.where(exceeds, abi.NODE_UNSCHEDULABLE | abi.NODE_OVERALLOCATED, 0)
                 | np.where(dropped, abi.NODE_DROPPED, 0)).astype(np.uint8)
        kept = np.nonzero(~dropped)[0]
        total = alloc[:, kept].sum(axis=1).astype(np.int64)
        for d in range(D):
            if (inp.floating_resource_mask >> d) & 1:
                total[d] += inp.floating_limit[d]
        max_sched = np.array([multiply_resource(int(total[d]), cs.max_fraction_to_schedule[d]) for d in range(D)], np.int64)
        qf = _field(cs, "queue_limit_fraction", Q * PC * D).reshape(Q, PC, D) if cs.queue_limit_fraction else np.full((Q, PC, D), math.inf)
        qlimit = np.array([[[multiply_resource(int(total[d]), float(qf[q, pc, d])) for d in range(D)] for pc in range(PC)] for q in range(Q)],
                          np.int64).reshape(Q, PC, D)
        self.kept = kept
        self.snapshot = {"node_state": state, "node_allocatable": alloc, "node_static_class": sclass, "total_resources": total,
                         "max_resources_to_schedule": max_sched, "queue_limit": qlimit}
        # the equivalent explicit input
        compact = np.full(N, abi.NONE, np.int64)
        compact[kept] = np.arange(len(kept))
        rank = _field(inp, "node_id_rank", N).astype(np.int64)
        new_rank = np.empty(len(kept), np.uint32)
        new_rank[np.argsort(rank[kept], kind="stable")] = np.arange(len(kept))
        out = abi.RoundInput()
        ctypes.memmove(ctypes.addressof(out), ctypes.addressof(inp), ctypes.sizeof(out))  # every field; node and job arrays replaced below
        self._keep: List[np.ndarray] = []
        out.num_nodes = len(kept)
        nk = lambda a: a[:, kept] if a.ndim == 2 else a[kept]  # noqa: E731
        abi.attach(out, self._keep, node_index=nk(_field(inp, "node_index", N)), node_id_rank=new_rank,
                   node_type=nk(_field(inp, "node_type", N)), node_static_class=nk(sclass), node_flags=nk(state),
                   node_total=nk(_field(inp, "node_total", D * N).reshape(D, N)), node_allocatable=nk(alloc),
                   job_node=np.where(run, compact[np.where(run, jn, 0)], abi.NONE), queue_limit=qlimit)
        out.has_round_limit = cs.has_round_limit
        for d in range(D):
            out.total_resources[d] = int(total[d])
            out.max_resources_to_schedule[d] = int(max_sched[d])
        out._keepalive = [inp, self._keep]
        self.input = out

    def in_caller_nodes(self, res: "RoundResult", inp: abi.RoundInput) -> "RoundResult":
        """A RoundResult of `self.input`'s round in the caller's node numbering (the RoundResult of `inp`)."""
        return result_in_caller_nodes(res, self.kept, inp)


def result_in_caller_nodes(res: "RoundResult", kept, inp: abi.RoundInput) -> "RoundResult":
    """A RoundResult over a pool's kept nodes (node k = the caller's node kept[k]) in the caller's node numbering, as
    the RoundResult of `inp`, the round as reported: job_node mapped back, node_alloc columns of dropped nodes zero
    (what armada_round_download leaves in a zeroed buffer)."""
    kept = np.asarray(kept, np.int64)
    out = RoundResult(inp, res.first_pass)
    for name in RoundResult.ARRAYS + RoundResult.FIRST_PASS_ARRAYS:
        getattr(out, name)[...] = getattr(res, name) if name != "node_alloc" else 0
    out.node_alloc[:, :, kept] = res.node_alloc[:, :, : len(kept)]
    out.job_node[...] = np.where(res.job_node == abi.NONE, abi.NONE, kept[np.where(res.job_node == abi.NONE, 0, res.job_node)])
    for name in RoundResult.SCALARS:
        setattr(out.out, name, getattr(res.out, name))
    return out


def node_preemptibility_stats(b: "RoundInputBuilder", res: "RoundResult") -> List[Tuple[str, bool, str]]:
    """EvictorResult.NodePreemptiblityStats of the round's first evictor (NewNodeEvictor with the fair-share filter,
    preempting_queue_scheduler.go:93-136; eviction.go:197-273): per node, in node-id order, (node id, can every job on
    it be preempted, the sorted reasons).  A report for operators (scheduling reports, cycle metrics), derived on the
    host from the round's inputs and the fair shares the device computed — the evictions themselves happen on the
    device (`k_evict_balance`) and `evictable_jobs` below is checked against them in the tests."""
    reasons, _ = _eviction_reasons(b, res)
    inp = b.input
    by_node: Dict[int, List[int]] = {}
    for j, n in enumerate(b.job_node[: len(b.jobs)]):
        if n != abi.NONE:
            by_node.setdefault(int(n), []).append(j)
    out = []
    for i in sorted(range(len(b.nodes)), key=lambda i: b.nodes[i].id):
        node = b.nodes[i]
        jobs = by_node.get(i, [])
        if not jobs:  # nodeFilter: "node_empty" (eviction.go:88-95, 200-210)
            rs = {"node_empty"} | ({"node_unschedulable"} if node.unschedulable else set())
            out.append((node.id, not node.unschedulable, ",".join(sorted(rs))))
            continue
        rs = {reasons[j] for j in jobs if reasons[j]}
        if node.unschedulable:
            rs.add("node_unschedulable")
        out.append((node.id, not rs, ",".join(sorted(rs)) if rs else "all_jobs_preemptible"))
    return out


def evictable_jobs(b: "RoundInputBuilder", res: "RoundResult") -> np.ndarray:
    """The running jobs the first evictor's job filter lets through (bool[J])."""
    return _eviction_reasons(b, res)[1]


def _eviction_reasons(b: "RoundInputBuilder", res: "RoundResult"):
    cfg, inp = b.cfg, b.input
    J, D = len(b.jobs), b.factory.D
    total = b.total_resources.astype(np.float64)
    mult = np.array([inp.drf_multipliers[d] for d in range(D)])
    # qctx.GetAllocation() = Allocated + ShortJobPenalty at the start of the round
    alloc = b.queue_allocated_by_pc.sum(axis=1).astype(np.float64) + b.queue_short_job_penalty.astype(np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        frac_d = np.where(total != 0, alloc / np.where(total != 0, total, 1.0), 0.0) * mult
        actual = np.maximum(frac_d.max(axis=1), 0.0) if D else np.zeros(len(b.queues))
        fs = res.queue_fair_share
        fair = fs[:, 2] if cfg.protect_uncapped_adjusted_fair_share else np.maximum(fs[:, 1], fs[:, 0])
        fraction = actual / fair[: len(actual)]
    reasons: List[str] = [""] * J
    evict = np.zeros(J, dtype=bool)
    for j, spec in enumerate(b.jobs):
        if b.job_node[j] == abi.NONE:
            continue
        q = b.job_queue[j]
        if q == abi.NONE:
            reasons[j] = "invalid_queue"
        elif not cfg.priority_classes[spec.priority_class].preemptible:
            reasons[j] = "job_not_preemptible"
        elif fraction[q] <= cfg.protected_fraction_of_fair_share:  # (NaN compares false: evicted, like the reference)
            reasons[j] = "below_protected_fair_share"
        else:
            evict[j] = True
    return reasons, evict


# constraints.go:17-55 + gang_scheduler.go:168-216: the strings behind ARMADA_REASON_*
REASON_TEXT = {
    abi.REASON_MAX_RESOURCES_SCHEDULED: "maximum resources scheduled",
    abi.REASON_MAX_RESOURCES_PER_QUEUE: "resource limit exceeded",
    abi.REASON_GLOBAL_RATE_LIMIT: "global scheduling rate limit exceeded",
    abi.REASON_QUEUE_RATE_LIMIT: "queue scheduling rate limit exceeded",
    abi.REASON_QUEUE_CORDONED: "queue cordoned",
    abi.REASON_GLOBAL_RATE_LIMIT_GANG: "gang would exceed global scheduling rate limit",
    abi.REASON_QUEUE_RATE_LIMIT_GANG: "gang would exceed queue scheduling rate limit",
    abi.REASON_GANG_EXCEEDS_GLOBAL_BURST: "gang cardinality too large: exceeds global max burst size",
    abi.REASON_GANG_EXCEEDS_QUEUE_BURST: "gang cardinality too large: exceeds queue max burst size",
    abi.REASON_GANG_DOES_NOT_FIT: "unable to schedule gang since minimum cardinality not met",
    abi.REASON_JOB_DOES_NOT_FIT: "job does not fit on any node",
    abi.REASON_UNIFORMITY_LABEL_NOT_INDEXED: "uniformity label is not indexed",
    abi.REASON_NO_NODES_WITH_UNIFORMITY_LABEL: "no nodes with uniformity label",
    abi.REASON_GANG_FITS_NO_UNIFORMITY_VALUE: "at least one job in the gang does not fit on any node",
    abi.REASON_FLOATING_RESOURCES: "floating resource limit",
}


@dataclass
class QueueStats:
    """scheduling.QueueStats (result.go:15-28) without the wall-clock `Time`."""
    gangs_considered: int = 0
    jobs_considered: int = 0
    gangs_scheduled: int = 0
    first_gang_considered_sample_job_id: str = ""
    first_gang_considered_result: str = ""
    first_gang_considered_queue_position: int = 0
    last_gang_scheduled_sample_job_id: str = ""
    last_gang_scheduled_queue_position: int = 0
    last_gang_scheduled_queue_cost: float = 0.0
    last_gang_scheduled_resources: Optional[np.ndarray] = None
    last_gang_scheduled_queue_resources: Optional[np.ndarray] = None


def queue_stats(b: "RoundInputBuilder", res: "RoundResult") -> Dict[str, QueueStats]:
    """SchedulingResult.AdditionalSchedulingInfo.StatsPerQueue: the statistics QueueScheduler.Schedule keeps per queue
    (queue_scheduler.go:190-235) for the FIRST schedule pass of the round (preempting_queue_scheduler.go:270-272), from
    the device's first-pass view (`job_seq_first_pass`, `job_reason_first_pass`).  A gang = the jobs of one loop
    iteration; its sample job = gctx.JobIds()[0], the first member in queue order; loopNumber = iteration − 1.  The
    queue's allocation and cost at its last scheduled gang are REPLAYED from the start-of-pass allocation (the
    snapshot's minus what the first evictor took) plus the first-pass successes up to that iteration."""
    if not res.first_pass:
        raise ValueError("queue_stats needs a RoundResult created with first_pass=True")
    J, f, cfg = len(b.jobs), b.factory, b.cfg
    seq, why = res.job_seq_first_pass[:J], res.job_reason_first_pass[:J]
    req = b.class_request[b.job_class[:J]] if J else np.zeros((0, f.D), np.int64)
    pcprio = np.array([cfg.priority_classes[j.priority_class].priority for j in b.jobs], np.int64)
    running = b.job_node[:J] != abi.NONE

    def order_key(j):  # SchedulingOrderCompare (jobdb/comparison.go:49-107)
        return (0 if running[j] else 1, -pcprio[j], b.job_queue_priority[j], b.job_active_run_timestamp[j] if running[j] else 0, b.job_submit_time[j], b.job_id_rank[j])

    evicted = evictable_jobs(b, res)
    total = b.total_resources.astype(np.float64)
    mult = np.array([b.input.drf_multipliers[d] for d in range(f.D)])
    out: Dict[str, QueueStats] = {}
    for qi, q in enumerate(b.queues):
        mine = np.nonzero((b.job_queue[:J] == qi) & (seq > 0))[0]
        if len(mine) == 0:
            continue
        st = QueueStats()
        gangs: Dict[int, List[int]] = {}
        for j in mine:
            gangs.setdefault(int(seq[j]), []).append(int(j))
        alloc = b.queue_allocated_by_pc[qi].sum(axis=0) + b.queue_short_job_penalty[qi]  # qctx.GetAllocation(): Allocated + ShortJobPenalty
        for j in np.nonzero((b.job_queue[:J] == qi) & evicted)[0]:
            alloc = alloc - req[j]
        for s in sorted(gangs):
            members = sorted(gangs[s], key=order_key)
            ok = all(why[j] == 0 for j in members)
            st.gangs_considered += 1
            st.jobs_considered += len(members)
            if st.first_gang_considered_sample_job_id == "":
                st.first_gang_considered_sample_job_id = b.jobs[members[0]].id
                st.first_gang_considered_queue_position = s - 1
                st.first_gang_considered_result = "scheduled" if ok else REASON_TEXT.get(int(why[members[0]]), str(int(why[members[0]])))
            if ok:
                st.gangs_scheduled += 1
                gang_total = req[members].sum(axis=0)
                alloc = alloc + gang_total
                st.last_gang_scheduled_sample_job_id = b.jobs[members[0]].id
                st.last_gang_scheduled_queue_position = s - 1
                st.last_gang_scheduled_resources = gang_total
                st.last_gang_scheduled_queue_resources = alloc.copy()
                with np.errstate(divide="ignore", invalid="ignore"):
                    frac = np.where(total != 0, alloc / np.where(total != 0, total, 1.0), 0.0) * mult
                cost = max(float(frac.max()), 0.0) if f.D else 0.0
                st.last_gang_scheduled_queue_cost = cost / float(b.queue_weight[qi])
        out[q.name] = st
    return out


# ---- the reference's exclusion reason strings (nodedb/nodematching.go:14-122, context/pod.go:58-80) ----------
_DEC_SUFFIX = {-9: "n", -6: "u", -3: "m", 0: "", 3: "k", 6: "M", 9: "G", 12: "T", 15: "P", 18: "E"}


def quantity_string(value: int, scale: int) -> str:
    """`resource.NewScaledQuantity(value, scale).String()` — how `ResourceList.asQuantity` prints
    (internaltypes/resource_list.go:292-297).  Restated from apimachinery's Quantity.CanonicalizeBytes and
    int64Amount.AsCanonicalBytes (read, not executed): a DecimalSI quantity strips trailing zeros of the
    value into the exponent, then multiplies back until the exponent is a multiple of 3, and prints the
    integer with the SI suffix of that exponent; zero is "0".  Exponents outside n…E never arise from an
    int64 at the factory's scales and are refused."""
    value, exp = int(value), int(scale)
    if value == 0:
        return "0"
    while value % 10 == 0:
        value //= 10
        exp += 1
    r = exp % 3  # Python's modulo is non-negative: 1 ↔ Go's {1, -2}, 2 ↔ {2, -1}
    value *= 10 ** r
    exp -= r
    if exp not in _DEC_SUFFIX:
        raise ValueError(f"quantity {value}e{exp} has no DecimalSI suffix")
    return f"{value}{_DEC_SUFFIX[exp]}"


def untolerated_taint_reason(t: Taint) -> str:  # UntoleratedTaint.String
    return f"taint {t.key}={t.value}:{t.effect} not tolerated"


def missing_label_reason(label: str) -> str:  # MissingLabel.String
    return f"node does not match pod NodeSelector: label {label} not set"


def unmatched_label_reason(label: str, pod_value: str, node_value: str) -> str:  # UnmatchedLabel.String
    return f"node does not match pod NodeSelector: required label {label} = {pod_value}, but node has {node_value}"


def node_selector_string(terms: Sequence[Tuple[MatchExpression, ...]]) -> str:
    """`(*v1.NodeSelector).String()` as printed by UnmatchedNodeSelector (`%s`): the gogo-protobuf
    generated String of k8s.io/api/core/v1 (generated.pb.go; restated from reading it)."""
    def req(e: MatchExpression) -> str:
        return f"NodeSelectorRequirement{{Key:{e.key},Operator:{e.operator},Values:[{' '.join(e.values)}],}}"
    out = "&NodeSelector{NodeSelectorTerms:[]NodeSelectorTerm{"
    for term in terms:
        out += "NodeSelectorTerm{MatchExpressions:[]NodeSelectorRequirement{" + "".join(req(e) + "," for e in term) + "},"
        out += "MatchFields:[]NodeSelectorRequirement{},},"
    return out + "},}"


def insufficient_resources_reason(name: str, required: str, available: str) -> str:  # InsufficientResources.String
    return f"pod requires {required} {name}, but only {available} is available"


def _selector_reason(selector: Sequence[Tuple[str, str]], labels: Dict[str, str], unset: Optional[set]) -> Optional[str]:
    """NodeSelectorRequirementsMet (nodematching.go:215-240).  The reference ranges over the selector MAP, so
    when several labels fail it reports one at random; this restatement takes them in label order."""
    for label, pod_value in selector:
        if label in labels:
            if labels[label] != pod_value:
                return unmatched_label_reason(label, pod_value, labels[label])
        elif unset is None or label in unset:
            return missing_label_reason(label)
    return None


def excluded_reason_string(b: "RoundInputBuilder", row: int, cls: int, rec) -> str:
    """The reason string of one ExcludedReason record of a job of class `cls` probed with static row `row`."""
    kind = int(rec.kind)
    if kind == abi.EXCL_IMPLICIT:
        return "insufficient resources available"  # PodRequirementsNotMetReasonInsufficientResources
    if kind == abi.EXCL_DISALLOWED:
        return "job requests disallowed resource and therefore cannot be scheduled"  # disallowedResourceRequested, nodedb.go:26
    tolerations, selector, affinity = b.row_specs[row]
    if kind == abi.EXCL_NODE_TYPE:  # NodeTypeJobRequirementsMet (:127-139)
        taints, labels, unset = b.type_specs[int(rec.sub)]
        t = find_untolerated(taints, tolerations)
        if t is not None:
            return untolerated_taint_reason(t)
        r = _selector_reason(selector, labels, unset)
        if r is None:
            raise ValueError(f"node type {int(rec.sub)} matches row {row}")
        return r
    if kind == abi.EXCL_STATIC:  # StaticJobRequirementsMet's string predicates (:161-181)
        taints, labels = b.static_specs[int(rec.sub)]
        t = find_untolerated(taints, tolerations)
        if t is not None:
            return untolerated_taint_reason(t)
        r = _selector_reason(selector, labels, None)
        if r is not None:
            return r
        if affinity is not None and not match_node_selector_terms(labels, affinity):
            return "node does not match pod NodeAffinity " + node_selector_string(affinity)
        raise ValueError(f"static class {int(rec.sub)} matches row {row}")
    # ARMADA_EXCL_STATIC_TOTAL / ARMADA_EXCL_RESOURCES: InsufficientResources (resource_list.go:167-191)
    d = int(rec.sub)
    f = b.factory
    return insufficient_resources_reason(f.names[d], quantity_string(int(b.class_request[cls, d]), f.scales[d]),
                                         quantity_string(int(rec.quantity), f.scales[d]))


def pod_scheduling_context_string(num_nodes: int, excluded: Dict[str, int], node_id: str = "") -> str:
    """PodSchedulingContext.String (context/pod.go:62-81) through text/tabwriter(minwidth 1, tabwidth 1,
    padding 1, ' ', 0): each column of a run of lines that have a cell there is as wide as its widest
    cell plus one.  The reference ranges over the excluded-nodes MAP, so its lines come in random order;
    here they come in reason-string order."""
    head = [("Node:", node_id or "none"), ("Number of nodes in cluster:", str(num_nodes))]
    if not excluded:
        head.append(("Excluded nodes:", "none"))  # a cell of the first column too
    w0 = max(len(a) for a, _ in head) + 1
    out = "".join(a.ljust(w0) + v + "\n" for a, v in head)
    if not excluded:
        return out
    out += "Excluded nodes:\n"
    items = sorted(excluded.items())
    w1 = max(len(f"{c}:") for _, c in items) + 1
    return out + "".join(" " + f"{c}:".ljust(w1) + reason + "\n" for reason, c in items)


def last_probe_row(b: "RoundInputBuilder", cls: int) -> Optional[int]:
    """The static row of the last probe SelectNodeForJobWithTxn runs for a single job of class `cls` that
    fits nowhere (nodedb.go:431-512): the last away node type that adds taints when away scheduling is
    on, else the home row when home scheduling is on; None when no probe runs."""
    if not b.cfg.disable_away_scheduling:
        for k in reversed(range(abi.MAX_AWAY)):
            if int(b.class_away_row[cls, k]) != abi.NONE:
                return int(b.class_away_row[cls, k])
    return None if b.cfg.disable_home_scheduling else int(b.class_static_row[cls])


def excluded_nodes_by_reason(b: "RoundInputBuilder", cls: int, records) -> Dict[str, int]:
    """NumExcludedNodesByReason of a failed single job of class `cls` from its explain records: records
    whose strings coincide (two node types with the same untolerated taint, a total and an allocatable of
    the same quantity, …) add up, as they do under the reference's string keys."""
    row = last_probe_row(b, cls)
    out: Dict[str, int] = {}
    for r in records:
        s = excluded_reason_string(b, row, cls, r)
        out[s] = out.get(s, 0) + int(r.count)
    return out
