"""Deterministic synthetic rounds: BASELINE.json configs C1–C5 (SURVEY.md §8d) and a small
random-scenario generator for parity fuzzing.  Everything is built directly as SoA numpy
arrays (1M jobs do not go through per-job Python objects).

Generator: numpy PCG64 seeded with 20240601 (SURVEY names PCG32; numpy ships PCG64 — the
stream only has to be deterministic and identical for the oracle and the device).
Shapes follow the reference's fixtures: Test32CpuNode / Test8GpuNode
(testfixtures.go:1030-1073), N1Cpu4GiJobs… (:615-694), TestPriorityClasses (:78-105),
TestResources index resolutions (:108-112), factory order memory, cpu, gpu (:1249-1255).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import abi

SEED = 20240601
GI = 2**30
MI = 2**20
I64_MAX = 2**63 - 1

# factory order (GetTestSupportedResourceTypes): memory [bytes], cpu [milli], gpu [milli]
MEM, CPU, GPU = 0, 1, 2
D = 3
INDEXED = [CPU, MEM, GPU]                 # TestResources order: cpu, memory, nvidia.com/gpu
RESOLUTION = [1000, 128 * MI, 1000]
PRIORITIES = [-1, 0, 1, 2, 3, 28000, 29000, 30000]
# (priority, preemptible): PriorityClass0..3 of the fixtures
PCS = [(0, True), (1, True), (2, True), (3, False)]


def rl(cpu=0, mem_gi=0, gpu=0) -> np.ndarray:
    v = np.zeros(D, np.int64)
    v[CPU] = int(cpu * 1000)
    v[MEM] = int(mem_gi * GI)
    v[GPU] = int(gpu * 1000)
    return v


NODE_CPU32 = rl(32, 256)
NODE_GPU8 = rl(64, 1024, 8)
SHAPES = [rl(1, 4), rl(1, 16), rl(8, 64), rl(16, 128), rl(8, 128, 1)]  # C3 job shapes; last needs gpu toleration


@dataclass
class RawRound:
    """SoA arrays of one round + conversion to the C ABI struct."""
    node_total: np.ndarray            # [D][N]
    node_allocatable: np.ndarray      # [D][N]
    node_type: np.ndarray
    node_static_class: np.ndarray
    class_request: np.ndarray         # [C][D]
    class_pc: np.ndarray
    class_static_row: np.ndarray
    static_match: np.ndarray          # [rows][sw]
    type_match: np.ndarray
    job_class: np.ndarray
    job_queue: np.ndarray
    job_submit_time: np.ndarray
    queue_weight: np.ndarray
    num_node_types: int = 1
    num_static_classes: int = 1
    job_gang: Optional[np.ndarray] = None
    gang_cardinality: Optional[np.ndarray] = None
    job_node: Optional[np.ndarray] = None
    job_scheduled_at_priority: Optional[np.ndarray] = None
    job_active_run_timestamp: Optional[np.ndarray] = None
    job_queue_priority: Optional[np.ndarray] = None
    node_flags: Optional[np.ndarray] = None
    node_index: Optional[np.ndarray] = None
    node_id_rank: Optional[np.ndarray] = None
    class_away_row: Optional[np.ndarray] = None
    pcs: Sequence[Tuple[int, bool]] = tuple(PCS)
    pc_away: Optional[Dict[int, List[int]]] = None     # pc index -> away priorities
    priorities: Sequence[int] = tuple(PRIORITIES)
    protected_fraction: float = 0.0
    max_queue_lookback: int = 0
    prefer_large: bool = True
    round_limit: Optional[np.ndarray] = None
    queue_limit: Optional[np.ndarray] = None            # [Q][PC][D]
    queue_allocated_by_pc: Optional[np.ndarray] = None  # [Q][PC][D]; default: Σ running jobs
    global_tokens: Optional[float] = None
    global_burst: int = 2**62
    global_inf: bool = True
    indexed: Optional[Sequence[int]] = None             # indexed resources (default: all of them)
    resolution: Optional[Sequence[int]] = None          # index resolution per entry of `indexed` (default: TestResources)
    drf_multipliers: Optional[Sequence[float]] = None   # [D] (default: every resource counts with weight 1)
    name: str = ""
    _keep: list = field(default_factory=list)

    def to_input(self) -> abi.RoundInput:
        inp = abi.RoundInput()
        inp.abi_version = abi.ABI_VERSION
        D = self.node_total.shape[0]
        inp.num_resources = D
        indexed = list(self.indexed) if self.indexed is not None else INDEXED
        inp.num_indexed = len(indexed)
        res = list(self.resolution) if self.resolution is not None else [RESOLUTION[INDEXED.index(d)] for d in indexed]
        for i, (d, r) in enumerate(zip(indexed, res)):
            inp.indexed_resource[i] = d
            inp.indexed_resolution[i] = r
        inp.num_priorities = len(self.priorities)
        for i, p in enumerate(self.priorities):
            inp.priorities[i] = p
        inp.num_priority_classes = len(self.pcs)
        for i, (p, pre) in enumerate(self.pcs):
            inp.priority_classes[i].priority = p
            inp.priority_classes[i].preemptible = int(pre)
            aw = (self.pc_away or {}).get(i, [])
            inp.priority_classes[i].num_away = len(aw)
            for k, ap in enumerate(aw):
                inp.priority_classes[i].away_priority[k] = ap
                inp.priority_classes[i].away_well_known[k] = k
        N = self.node_total.shape[1]
        J = len(self.job_class)
        Q = len(self.queue_weight)
        Cn = self.class_request.shape[0]
        PCn = len(self.pcs)
        total = self.node_allocatable.sum(axis=1)
        for d in range(D):
            inp.total_resources[d] = int(total[d])
            inp.drf_multipliers[d] = float(self.drf_multipliers[d]) if self.drf_multipliers is not None else 1.0
            inp.max_resources_to_schedule[d] = int(self.round_limit[d]) if self.round_limit is not None else I64_MAX
        inp.has_round_limit = 1
        inp.prefer_large_job_ordering = int(self.prefer_large)
        inp.protected_fraction_of_fair_share = self.protected_fraction
        inp.max_queue_lookback = self.max_queue_lookback
        inp.global_limiter_is_inf = int(self.global_inf)
        inp.global_limiter_burst = self.global_burst
        inp.global_limiter_tokens = float(self.global_burst) if self.global_tokens is None else self.global_tokens
        inp.num_nodes, inp.num_node_types, inp.num_static_classes = N, self.num_node_types, self.num_static_classes
        inp.num_classes = Cn
        inp.num_static_rows = self.static_match.shape[0]
        inp.num_jobs = J
        inp.num_gangs = 0 if self.gang_cardinality is None else len(self.gang_cardinality)
        inp.num_queues = Q
        job_node = self.job_node if self.job_node is not None else np.full(J, abi.NONE)
        # queue accounting derived from the job arrays (calculateJobSchedulingInfo, scheduling_algo.go:522-632)
        jq = np.asarray(self.job_queue).astype(np.int64)
        req = np.asarray(self.class_request)[np.asarray(self.job_class).astype(np.int64)]  # [J][D]
        has_q = jq != abi.NONE
        running = (np.asarray(job_node).astype(np.int64) != abi.NONE) & has_q
        demand = np.zeros((Q, D), np.int64)
        np.add.at(demand, jq[has_q], req[has_q])
        if self.queue_allocated_by_pc is not None:
            alloc_pc = self.queue_allocated_by_pc
        else:
            alloc_pc = np.zeros((Q, PCn, D), np.int64)
            jpc = np.asarray(self.class_pc)[np.asarray(self.job_class).astype(np.int64)].astype(np.int64)
            np.add.at(alloc_pc, (jq[running], jpc[running]), req[running])
        self._keep = []  # the struct only holds raw pointers into these arrays
        abi.attach(
            inp, self._keep,
            node_index=self.node_index if self.node_index is not None else np.arange(N),
            node_id_rank=self.node_id_rank if self.node_id_rank is not None else np.arange(N),
            node_type=self.node_type, node_static_class=self.node_static_class,
            node_flags=self.node_flags if self.node_flags is not None else np.zeros(N),
            node_total=self.node_total, node_allocatable=self.node_allocatable,
            class_request=self.class_request, class_pc=self.class_pc, class_static_row=self.class_static_row,
            class_away_row=self.class_away_row if self.class_away_row is not None else np.full((Cn, abi.MAX_AWAY), abi.NONE),
            class_key_valid=np.ones(Cn), static_match=self.static_match, type_match=self.type_match,
            job_class=self.job_class, job_queue=self.job_queue,
            job_queue_priority=self.job_queue_priority if self.job_queue_priority is not None else np.full(J, 1000),
            job_submit_time=self.job_submit_time, job_id_rank=np.arange(J),
            job_gang=self.job_gang if self.job_gang is not None else np.full(J, abi.NONE), job_node=job_node,
            job_scheduled_at_priority=(self.job_scheduled_at_priority if self.job_scheduled_at_priority is not None
                                       else np.full(J, abi.NO_PRIORITY)),
            job_active_run_timestamp=self.job_active_run_timestamp if self.job_active_run_timestamp is not None else np.zeros(J),
            gang_cardinality=self.gang_cardinality if self.gang_cardinality is not None else np.zeros(1),
            queue_weight=self.queue_weight, queue_cordoned=np.zeros(Q), queue_allocated_by_pc=alloc_pc,
            queue_demand=demand, queue_constrained_demand=demand, queue_short_job_penalty=np.zeros((Q, D)),
            queue_has_limit=np.ones((Q, PCn)) if self.queue_limit is not None else np.zeros((Q, PCn)),
            queue_limit=self.queue_limit if self.queue_limit is not None else np.zeros((Q, PCn, D)),
            queue_limiter_tokens=np.full(Q, float(2**62)), queue_limiter_burst=np.full(Q, 2**62), queue_limiter_is_inf=np.ones(Q))
        inp._keepalive = self._keep
        self.input = inp
        return inp

    def h2d_bytes(self) -> int:
        return int(sum(a.nbytes for a in self._keep))


def _bitmap(rows: List[List[int]], ncols: int) -> np.ndarray:
    w = (ncols + 31) // 32
    m = np.zeros((len(rows), w), np.uint32)
    for r, cols in enumerate(rows):
        for c in cols:
            m[r, c >> 5] |= np.uint32(1 << (c & 31))
    return m


def _nodes(n_cpu: int, n_gpu: int, rng: Optional[np.random.Generator] = None):
    """n_cpu Test32CpuNode + n_gpu Test8GpuNode (gpu taint + label ⇒ static class / node type 1),
    interleaved deterministically so that id order mixes both kinds."""
    N = n_cpu + n_gpu
    kind = np.zeros(N, np.uint32)
    if n_gpu:
        idx = np.floor(np.arange(n_gpu) * (N / n_gpu)).astype(np.int64)
        kind[idx] = 1
    total = np.where(kind[None, :] == 1, NODE_GPU8[:, None], NODE_CPU32[:, None]).astype(np.int64)
    return total, kind


def _classes(pc: int = 0):
    """One job class per C3 shape at priority class `pc`; the gpu shape tolerates the gpu taint."""
    class_request = np.stack(SHAPES)
    class_pc = np.full(len(SHAPES), pc, np.uint32)
    class_row = np.array([0, 0, 0, 0, 1], np.uint32)
    # row 0: no tolerations → only untainted nodes (static class 0); row 1: tolerates gpu=true
    static_match = _bitmap([[0], [0, 1]], 2)
    type_match = _bitmap([[0], [0, 1]], 2)
    return class_request, class_pc, class_row, static_match, type_match


def config_c1() -> RawRound:
    """C1: simulator clusters/cpu_1_1_100.yaml — 100 × (32 cpu, 1024Gi), 1 queue, 1000 × (1 cpu, 10Gi)."""
    N, J = 100, 1000
    total = np.repeat(rl(32, 1024)[:, None], N, axis=1)
    return RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=np.zeros(N), node_static_class=np.zeros(N),
        class_request=rl(1, 10)[None, :], class_pc=np.zeros(1), class_static_row=np.zeros(1),
        static_match=_bitmap([[0]], 1), type_match=_bitmap([[0]], 1),
        job_class=np.zeros(J), job_queue=np.zeros(J), job_submit_time=np.arange(J), queue_weight=np.ones(1), name="C1")


def config_c2(n_nodes=10_000, n_queues=16, n_jobs=100_000) -> RawRound:
    """C2: 10k × Test32CpuNode, 16 equal-weight queues, 100k × N1Cpu4GiJobs, empty cluster."""
    rng = np.random.default_rng(SEED)
    total = np.repeat(NODE_CPU32[:, None], n_nodes, axis=1)
    return RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=np.zeros(n_nodes), node_static_class=np.zeros(n_nodes),
        class_request=rl(1, 4)[None, :], class_pc=np.zeros(1), class_static_row=np.zeros(1),
        static_match=_bitmap([[0]], 1), type_match=_bitmap([[0]], 1),
        job_class=np.zeros(n_jobs), job_queue=rng.integers(0, n_queues, n_jobs), job_submit_time=np.arange(n_jobs),
        queue_weight=np.ones(n_queues), name="C2")


def _weights(n_queues: int) -> np.ndarray:
    return np.array([1.0, 0.5, 0.25])[np.arange(n_queues) % 3]


def config_c3(n_nodes=100_000, n_queues=64, n_jobs=1_000_000, seed=SEED) -> RawRound:
    """C3: 80 % Test32CpuNode + 20 % tainted Test8GpuNode, 64 queues (weights 1, ½, ¼), 1M jobs of 5 shapes."""
    rng = np.random.default_rng(seed)
    n_gpu = n_nodes // 5
    total, kind = _nodes(n_nodes - n_gpu, n_gpu)
    cr, cpc, crow, sm, tm = _classes()
    return RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=kind, node_static_class=kind,
        num_node_types=2, num_static_classes=2,
        class_request=cr, class_pc=cpc, class_static_row=crow, static_match=sm, type_match=tm,
        job_class=rng.integers(0, len(SHAPES), n_jobs), job_queue=rng.integers(0, n_queues, n_jobs),
        job_submit_time=np.arange(n_jobs), queue_weight=_weights(n_queues), name="C3")


def config_c4(n_nodes=100_000, n_queues=64, n_jobs=1_000_000, seed=SEED) -> RawRound:
    """C4: C3 with 10 % of the jobs in gangs of 2–64 contiguous members (atomic placement)."""
    rng = np.random.default_rng(seed)
    r = config_c3(n_nodes, n_queues, n_jobs, seed)
    job_class = np.asarray(r.job_class).copy()
    job_queue = np.asarray(r.job_queue).copy()
    gang = np.full(n_jobs, abi.NONE, np.uint32)
    cards: List[int] = []
    target = n_jobs // 10
    # gang starts are spread uniformly; members are consecutive submit times in ONE queue/shape
    sizes = []
    tot = 0
    while tot < target:
        s = int(rng.integers(2, 65))
        sizes.append(s)
        tot += s
    starts = np.sort(rng.choice(n_jobs - 64, size=len(sizes), replace=False))
    pos = 0
    for s, st in zip(sizes, starts):
        st = max(int(st), pos)
        if st + s > n_jobs:
            break
        g = len(cards)
        cards.append(s)
        gang[st:st + s] = g
        job_class[st:st + s] = job_class[st]
        job_queue[st:st + s] = job_queue[st]
        pos = st + s
    r.job_class, r.job_queue, r.job_gang, r.gang_cardinality, r.name = job_class, job_queue, gang, np.array(cards, np.uint32), "C4"
    return r


def config_c5(n_nodes=100_000, n_queues=64, n_new_jobs=400_000, seed=SEED) -> RawRound:
    """C5: C3 nodes pre-filled to ~90 % cpu by running preemptible jobs of the first half of the
    queues (far over their fair share); the other half of the queues has queued demand;
    ProtectedFractionOfFairShare = 0.5 ⇒ evict → re-schedule → oversubscribed-evict round."""
    rng = np.random.default_rng(seed)
    n_gpu = n_nodes // 5
    total, kind = _nodes(n_nodes - n_gpu, n_gpu)
    cr, cpc, crow, sm, tm = _classes()
    half = n_queues // 2
    # running jobs per node: cpu32 node: 16c + 8c + 4×1c = 28c ; gpu node: 3×16c + 8c + 1c = 57c
    per_cpu = [3, 2, 0, 0, 0, 0]
    per_gpu = [3, 3, 3, 2, 0]
    counts = np.where(kind == 1, len(per_gpu), len(per_cpu))
    jn = np.repeat(np.arange(n_nodes), counts)
    offs = np.concatenate([[0], np.cumsum(counts)[:-1]])
    within = np.arange(len(jn)) - np.repeat(offs, counts)
    pat = np.array([per_cpu, per_gpu + [0]])
    jc = pat[np.repeat((kind == 1).astype(np.int64), counts), within]
    n_run = len(jn)
    run_q = rng.integers(0, half, n_run)
    new_c = rng.integers(0, len(SHAPES), n_new_jobs)
    new_q = rng.integers(half, n_queues, n_new_jobs)
    J = n_run + n_new_jobs
    job_node = np.concatenate([jn, np.full(n_new_jobs, abi.NONE)])
    return RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=kind, node_static_class=kind,
        num_node_types=2, num_static_classes=2,
        class_request=cr, class_pc=cpc, class_static_row=crow, static_match=sm, type_match=tm,
        job_class=np.concatenate([jc, new_c]), job_queue=np.concatenate([run_q, new_q]),
        job_submit_time=np.arange(J), job_node=job_node,
        job_scheduled_at_priority=np.concatenate([np.zeros(n_run), np.full(n_new_jobs, abi.NO_PRIORITY)]),
        job_active_run_timestamp=np.concatenate([np.arange(n_run), np.zeros(n_new_jobs)]),
        queue_weight=_weights(n_queues), protected_fraction=0.5, name="C5")


def with_pod_limits(r: RawRound, pods) -> RawRound:
    """`r` with RespectNodePodLimits on (model.apply_respect_node_pod_limits): a `pods` resource after the others,
    indexed last at resolution 1, `pods` per node (a number or one per node) and one pod per job.  Pods play no part
    in DRF (they are not among its resources) and have no round or queue limit.  A node never starts above its pod
    capacity: one with more running jobs than `pods` gets a capacity of its running jobs."""
    D, N = r.node_total.shape
    cap = np.broadcast_to(np.asarray(pods, np.int64), (N,)).copy()
    if r.job_node is not None:
        jn = np.asarray(r.job_node).astype(np.int64)
        cap = np.maximum(cap, np.bincount(jn[jn != abi.NONE], minlength=N)[:N])
    indexed = list(r.indexed) if r.indexed is not None else list(INDEXED)
    res = list(r.resolution) if r.resolution is not None else [RESOLUTION[INDEXED.index(d)] for d in indexed]
    drf = list(r.drf_multipliers) if r.drf_multipliers is not None else [1.0] * D
    r.node_total = np.vstack([r.node_total, cap[None, :]])
    r.node_allocatable = np.vstack([r.node_allocatable, cap[None, :]])
    r.class_request = np.hstack([np.asarray(r.class_request, np.int64), np.ones((len(r.class_request), 1), np.int64)])
    r.indexed, r.resolution, r.drf_multipliers = indexed + [D], res + [1], drf + [0.0]
    if r.round_limit is not None:
        r.round_limit = np.append(r.round_limit, I64_MAX)
    if r.queue_limit is not None:
        r.queue_limit = np.concatenate([r.queue_limit, np.full(r.queue_limit.shape[:2] + (1,), I64_MAX, np.int64)], axis=2)
    r.name += "+pods"
    return r


def unfeasible_runs_round(n_nodes: int) -> RawRound:
    """Edge case: runs of jobs whose scheduling key is already known to be unfeasible
    (queue_scheduler.go:339-349), shorter and longer than the iterator's 128-record fast-forward
    step, ending in the middle of a step and at the end of a queue.  The oversized request (64 cpu)
    fits no node and does not fit the packed key either."""
    small, huge = rl(1, 4), rl(64, 4)
    total = np.repeat(NODE_CPU32[:, None], n_nodes, axis=1)
    runs = [(0, 3), (1, 700), (0, 5), (1, 130), (0, 2), (1, 127), (0, 1), (1, 129)]
    cls = np.concatenate([np.full(n, c) for c, n in runs] + [np.zeros(40, np.int64)])
    queue = np.concatenate([np.zeros(len(cls) - 40, np.int64), np.ones(40, np.int64)])  # + a queue of plain jobs
    return RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=np.zeros(n_nodes), node_static_class=np.zeros(n_nodes),
        class_request=np.stack([small, huge]), class_pc=np.zeros(2), class_static_row=np.zeros(2),
        static_match=_bitmap([[0]], 1), type_match=_bitmap([[0]], 1),
        job_class=cls, job_queue=queue, job_submit_time=np.arange(len(cls)), queue_weight=np.ones(2), name="unfeasible-runs")


def scaled(name: str, scale: float) -> RawRound:
    """A geometrically similar, smaller instance of a named config (parity tests)."""
    f = {"C2": lambda: config_c2(max(8, int(10_000 * scale)), 16, max(64, int(100_000 * scale))),
         "C3": lambda: config_c3(max(10, int(100_000 * scale)), 64, max(100, int(1_000_000 * scale))),
         "C4": lambda: config_c4(max(70, int(100_000 * scale)), 64, max(700, int(1_000_000 * scale))),
         "C5": lambda: config_c5(max(10, int(100_000 * scale)), 64, max(100, int(400_000 * scale)))}[name]
    return f()


def random_round(seed: int, n_nodes=60, n_queues=5, n_jobs=400, n_running=120, gangs=True, priorities=True,
                 protected_fraction=0.0, lookback=0, round_limit=False, queue_limits=False, away=False,
                 unaligned=False) -> RawRound:
    """Small random round inside the device fast-path domain exercising every mechanism:
    several node kinds, priority classes 0–3 (incl. non-preemptible), running jobs at various
    priorities (⇒ eviction, fair-share and urgency preemption), gangs, limits, lookback."""
    rng = np.random.default_rng(seed)
    n_gpu = n_nodes // 4
    total, kind = _nodes(n_nodes - n_gpu, n_gpu)
    # shuffle which nodes are small to get more distinct keys
    small = rng.random(n_nodes) < 0.3
    total = total.copy()
    total[CPU, small & (kind == 0)] = 16_000
    total[MEM, small & (kind == 0)] = 128 * GI
    npc = len(PCS) if priorities else 1
    shapes = [rl(1, 4), rl(1, 16), rl(2, 8), rl(4, 16), rl(8, 64), rl(16, 128), rl(8, 128, 1), rl(32, 256), rl(1, 1, 1)]
    resolution = None
    if unaligned:
        # the reference's default index resolutions (config/scheduler/config.yaml:116-124: cpu 100m, memory
        # 100Mi, gpu 1) with requests and node sizes that are NOT multiples of them (250m, 4Gi, 256Gi …),
        # node sizes that differ by less than one resolution step, allocatable below total
        resolution = [100, 100 * MI, 1000]
        shapes = [rl(0.25, 4), rl(1, 4), rl(1.5, 16), rl(2, 8.5), rl(3.75, 16), rl(8, 64), rl(16, 128), rl(8, 128, 1), rl(30.25, 250), rl(1, 1, 1)]
        jitter = rng.integers(0, 4, n_nodes)
        total[CPU] -= jitter * 30           # 30m steps: several nodes per rounded cpu bucket
        total[MEM] -= rng.integers(0, 5, n_nodes) * 37 * MI
    rows = [0, 0, 0, 0, 0, 0, 1, 0, 1] if not unaligned else [0, 0, 1, 0, 0, 0, 0, 1, 0, 1]
    cls_req, cls_pc, cls_row = [], [], []
    pc_away = None
    away_rows = []
    for pc in range(npc):
        for s, rw in zip(shapes, rows):
            cls_req.append(s)
            cls_pc.append(pc)
            cls_row.append(rw)
            away_rows.append([abi.NONE] * abi.MAX_AWAY)
    pcs = list(PCS[:npc])
    prios = list(PRIORITIES)
    if away:  # PriorityClass4PreemptibleAway-like: home 30000, away 29000 on gpu-tainted nodes
        pcs.append((30000, True))
        pc_away = {len(pcs) - 1: [29000]}
        for s, rw in zip(shapes[:6], rows[:6]):
            cls_req.append(s)
            cls_pc.append(len(pcs) - 1)
            cls_row.append(rw)
            away_rows.append([1] + [abi.NONE] * (abi.MAX_AWAY - 1))  # + toleration gpu=true
    Cn = len(cls_req)
    static_match = _bitmap([[0], [0, 1]], 2)
    J = n_jobs + n_running
    job_class = rng.integers(0, Cn, J)
    job_queue = rng.integers(0, n_queues, J)
    # a few jobs of unknown queues among the running ones
    job_node = np.full(J, abi.NONE, np.int64)
    sap = np.full(J, abi.NO_PRIORITY, np.int64)
    art = np.zeros(J, np.int64)
    # place running jobs greedily so nodes are not over-allocated
    free = total.copy()
    placed = 0
    for j in range(n_jobs, J):
        c = job_class[j]
        req = cls_req[c]
        cand = np.nonzero((free >= req[:, None]).all(axis=0) & ((kind == 0) | (cls_row[c] == 1) | (away_rows[c][0] != abi.NONE)))[0]
        if len(cand) == 0:
            job_class[j] = 0
            c = 0
            req = cls_req[0]
            cand = np.nonzero((free >= req[:, None]).all(axis=0) & (kind == 0))[0]
            if len(cand) == 0:
                continue
        n = int(cand[rng.integers(0, len(cand))])
        free[:, n] -= req
        job_node[j] = n
        pcp = pcs[cls_pc[c]][0]
        sap[j] = pcp if rng.random() < 0.8 else abi.NO_PRIORITY
        if away and cls_pc[c] == len(pcs) - 1 and kind[n] == 1:
            sap[j] = 29000
        art[j] = placed
        placed += 1
    # drop running jobs that could not be placed (turn them into queued jobs)
    gang = np.full(J, abi.NONE, np.int64)
    cards: List[int] = []
    if gangs:
        j = 0
        while j < n_jobs - 8:
            if rng.random() < 0.05:
                s = int(rng.integers(2, 7))
                g = len(cards)
                cards.append(s)
                gang[j:j + s] = g
                job_class[j:j + s] = job_class[j]
                job_queue[j:j + s] = job_queue[j]
                j += s
            else:
                j += 1
        # one running gang (members on nodes) to exercise gang eviction
        run_idx = np.nonzero(job_node != abi.NONE)[0]
        if len(run_idx) >= 3:
            g = len(cards)
            cards.append(3)
            members = run_idx[:3]
            gang[members] = g
            job_queue[members] = job_queue[members[0]]
    unknown = (rng.random(J) < 0.02) & (gang == abi.NONE)
    job_queue = np.where(unknown & (job_node != abi.NONE), abi.NONE, job_queue)
    limit = None
    if round_limit:
        limit = (total.sum(axis=1) * 0.3).astype(np.int64)
    qlimit = None
    if queue_limits:
        qlimit = np.full((n_queues, len(pcs), D), I64_MAX, np.int64)
        qlimit[:, :, CPU] = int(total[CPU].sum() * 0.2)
    allocatable = total.copy()
    node_index = None
    if unaligned:
        allocatable[MEM] -= rng.integers(0, 3, n_nodes) * 512 * MI   # kubelet reservations: allocatable < total
        allocatable = np.maximum(allocatable, free * 0 + (total - free))  # never below what already runs
        node_index = rng.permutation(n_nodes)                         # NodeFactory index order != node id order
    return RawRound(
        node_total=total, node_allocatable=allocatable, node_type=kind, node_static_class=kind,
        num_node_types=2, num_static_classes=2, node_index=node_index, resolution=resolution,
        class_request=np.stack(cls_req), class_pc=np.array(cls_pc), class_static_row=np.array(cls_row),
        class_away_row=np.array(away_rows, np.uint32), static_match=static_match, type_match=static_match.copy(),
        job_class=job_class, job_queue=job_queue, job_submit_time=rng.permutation(J), job_node=job_node,
        job_scheduled_at_priority=sap, job_active_run_timestamp=art,
        job_queue_priority=rng.integers(0, 3, J), job_gang=gang if gangs else None,
        gang_cardinality=np.array(cards, np.uint32) if gangs and cards else None,
        queue_weight=np.array([1.0, 0.5, 0.25, 2.0])[np.arange(n_queues) % 4], pcs=tuple(pcs), pc_away=pc_away,
        priorities=tuple(prios), protected_fraction=protected_fraction, max_queue_lookback=lookback,
        round_limit=limit, queue_limit=qlimit, name=f"random-{seed}")


def rounding_round() -> RawRound:
    """gang_scheduler_test.go:244-262 ("jobs of size not a multiple of the resolution blocks scheduling
    new jobs"): 3 × Test32CpuNode, index resolutions cpu 17 / memory 128Mi, four 16-cpu / 128Gi jobs.
    A node with 16 cpu left has a ROUNDED quantity of 0 and the iterator's lower bound (16) skips it,
    so only three jobs are placed although the fourth would fit."""
    N, J = 3, 4
    total = np.repeat(NODE_CPU32[:, None], N, axis=1)
    return RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=np.zeros(N), node_static_class=np.zeros(N),
        class_request=rl(16, 128)[None, :], class_pc=np.zeros(1), class_static_row=np.zeros(1),
        static_match=_bitmap([[0]], 1), type_match=_bitmap([[0]], 1),
        job_class=np.zeros(J), job_queue=np.zeros(J), job_submit_time=np.arange(J), queue_weight=np.ones(1),
        indexed=[CPU, MEM], resolution=[17000, 128 * MI], name="rounding")


def many_classes_round(seed: int = 9, n_classes: int = 300, n_nodes: int = 80, n_queues: int = 6, n_jobs: int = 1500) -> RawRound:
    """More distinct scheduling keys than the shared-memory class table holds (256): the table moves
    to global memory and only the first classes get best-fit windows."""
    rng = np.random.default_rng(seed)
    shapes = []
    c = 0
    while len(shapes) < n_classes:
        shapes.append(rl(1 + c % 12, 2 + 2 * (c // 12)))
        c += 1
    total = np.repeat(NODE_CPU32[:, None], n_nodes, axis=1)
    return RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=np.zeros(n_nodes), node_static_class=np.zeros(n_nodes),
        class_request=np.stack(shapes), class_pc=np.zeros(n_classes), class_static_row=np.zeros(n_classes),
        static_match=_bitmap([[0]], 1), type_match=_bitmap([[0]], 1),
        job_class=rng.integers(0, n_classes, n_jobs), job_queue=rng.integers(0, n_queues, n_jobs), job_submit_time=np.arange(n_jobs),
        queue_weight=np.ones(n_queues), name=f"many-classes-{n_classes}")
