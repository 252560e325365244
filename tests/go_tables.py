"""Evaluate the JSON ASTs extracted from the reference's Go test tables
(tests/golden/extract_go_tables.py) against the Python fixtures, and drive the round /
NodeDb entry points the way the reference's test drivers do."""
from __future__ import annotations

import copy
import json
import math
import os
from typing import Callable, Dict, List, Optional

import numpy as np

import fixtures as fx
from armada_b200 import abi
from armada_b200.model import (AwayNodeType, JobSpec, MatchExpression, NodeSpec, PriorityClass, QueueSpec, ResourceType,
                               RoundInputBuilder, SchedulingConfig, Taint, Toleration, parse_quantity)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class UnsupportedCase(Exception):
    pass


def load_cases(name: str) -> Dict[str, dict]:
    with open(os.path.join(GOLDEN, f"{name}.json")) as f:
        cases = json.load(f)["cases"]
    if name == "preempting_queue_scheduler":
        for manual in MANUAL_PQS:
            assert manual in cases, manual
            cases[manual] = {"manual": manual}
    return cases


class Rl(dict):
    """A quantity map (resource name → quantity string/number)."""


class _Fresh:
    """An identifier whose value is rebuilt on every use (config objects are mutated by With…Config)."""

    def __init__(self, make):
        self.make = make


class Env:
    """Evaluation environment: Go identifier / function name → Python value."""

    def __init__(self):
        self.fx = fx.Fixtures()
        F = self.fx
        self.ids = {
            "testfixtures.TestPriorities": fx.TestPriorities,
            "testfixtures.PriorityClass0": fx.PriorityClass0,
            "testfixtures.PriorityClass1": fx.PriorityClass1,
            "testfixtures.PriorityClass2": fx.PriorityClass2,
            "testfixtures.PriorityClass2NonPreemptible": fx.PriorityClass2NonPreemptible,
            "testfixtures.PriorityClass3": fx.PriorityClass3,
            "testfixtures.PriorityClass4PreemptibleAway": fx.PriorityClass4PreemptibleAway,
            "testfixtures.PriorityClass5PreemptibleAwayLowPriority": fx.PriorityClass5PreemptibleAwayLowPriority,
            "testfixtures.PriorityClass6Preemptible": fx.PriorityClass6Preemptible,
            "testfixtures.PriorityClass7PreemptibleAwayConditional": fx.PriorityClass7PreemptibleAwayConditional,
            "testfixtures.TestPool": "pool",
            "v1.TaintEffectNoSchedule": "NoSchedule",
            "v1.NodeSelectorOpNotIn": "NotIn",
            "v1.NodeSelectorOpIn": "In",
            "armadaconfiguration.GangIdAnnotation": "armadaproject.io/gangId",
            "armadaconfiguration.GangCardinalityAnnotation": "armadaproject.io/gangCardinality",
            # queue_scheduler_test.go:33-34 (a local of the test function): the reference's DEFAULT
            # ordering (config.yaml:85 enablePreferLargeJobOrdering: false); a fresh copy per use
            "schedulingConfigWithPreferLargeJobDisabled": _Fresh(lambda: fx.test_scheduling_config(enable_prefer_large_job_ordering=False)),
        }
        self.calls: Dict[str, Callable] = {
            "testfixtures.IntRange": lambda a, b: list(range(a, b + 1)),
            "testfixtures.Repeat": lambda v, n: [v] * n,
            "armadaslices.Concatenate": lambda *ls: [x for l in ls for x in l],
            # Go `append(l, x...)`: the parser drops the spread marker; elements are never lists
            # themselves in these tables, so list arguments are spread.
            "append": lambda l, *xs: list(l or []) + [y for x in xs for y in (x if isinstance(x, list) else [x])],
            "testfixtures.TestSchedulingConfig": lambda: fx.test_scheduling_config(),
            "testfixtures.N32CpuNodes": lambda n, p: F.n_cpu32(n),
            "testfixtures.NTainted32CpuNodes": lambda n, p: F.n_tainted_cpu32(n),
            "testfixtures.N8GpuNodes": lambda n, p: F.n_gpu8(n),
            "testfixtures.N1Cpu4GiJobs": lambda q, pc, n: F.n_1cpu_4gi(q, pc, n),
            "testfixtures.N1Cpu16GiJobs": lambda q, pc, n: F.n_1cpu_16gi(q, pc, n),
            "testfixtures.N16Cpu128GiJobs": lambda q, pc, n: F.n_16cpu_128gi(q, pc, n),
            "testfixtures.N32Cpu256GiJobs": lambda q, pc, n: F.n_32cpu_256gi(q, pc, n),
            "testfixtures.N32Cpu256GiJobsWithLargeJobToleration": lambda q, pc, n: F.n_32cpu_256gi_large_toleration(q, pc, n),
            "testfixtures.N1GpuJobs": lambda q, pc, n: F.n_1gpu(q, pc, n),
            "testfixtures.WithGangAnnotationsJobs": lambda jobs: fx.with_gang(jobs),
            "testfixtures.WithGangJobDetails": self._with_gang_details,
            "testfixtures.WithAnnotationsJobs": self._with_annotations,
            "testfixtures.WithNodeSelectorJobs": lambda sel, jobs: fx.with_node_selector(jobs, sel),
            "testfixtures.WithNodeAffinityJobs": self._with_affinity,
            "testfixtures.WithPriorityJobs": lambda p, jobs: fx.with_priority(jobs, p),
            "testfixtures.WithRequestsJobs": self._with_requests,
            "testfixtures.TestNodeFactory.AddLabels": self._add_labels,
            "testfixtures.TestNodeFactory.AddTaints": self._add_taints,
            "testfixtures.WithUsedResourcesNodes": self._with_used,
            "testfixtures.WithNodeTypeNodes": self._with_node_type,
            "testfixtures.Cpu": lambda c: Rl(cpu=c),
            "testfixtures.CpuMem": lambda c, m: Rl(cpu=c, memory=m),
            "testfixtures.CpuMemGpu": lambda c, m, g: Rl({"cpu": c, "memory": m, "nvidia.com/gpu": g}),
            "testfixtures.TestResourceListFactory.MakeAllZero": lambda: Rl(),
            "resource.MustParse": lambda s: s,
            "pointer.MustParseResource": lambda s: s,
            "testfixtures.SingleQueuePriorityOne": lambda name: [{"Name": name, "PriorityFactor": 1.0}],
            "testfixtures.WithProtectedFractionOfFairShareConfig": lambda v, c: self._cfg(c, protected_fraction_of_fair_share=float(v)),
            "testfixtures.WithRoundLimitsConfig": lambda l, c: self._round_limits(c, dict(l)),
            # MaximumResourceFractionToScheduleByPool: the pool's own map REPLACES the global one (constraints.go:208-214);
            # the drivers schedule the pool "pool" (gang_scheduler_test.go:626,651)
            "testfixtures.WithRoundLimitsPoolConfig": lambda by_pool, c: self._round_limits_pool(c, by_pool),
            "testfixtures.WithPerPriorityLimitsConfig": self._per_priority_limits,
            "testfixtures.WithGlobalSchedulingRateLimiterConfig": lambda r, b, c: self._cfg(c, maximum_scheduling_rate=float(r), maximum_scheduling_burst=int(b)),
            "testfixtures.WithPerQueueSchedulingLimiterConfig": lambda r, b, c: self._cfg(c, maximum_per_queue_scheduling_rate=float(r), maximum_per_queue_scheduling_burst=int(b)),
            "testfixtures.WithMaxLookbackPerQueueConfig": lambda n, c: self._cfg(c, max_queue_lookback=int(n)),
            "testfixtures.WithMaxQueueLookbackConfig": lambda n, c: self._cfg(c, max_queue_lookback=int(n)),
            "testfixtures.WithIndexedTaintsConfig": lambda ts, c: self._cfg(c, indexed_taints=list(c.indexed_taints) + list(ts)),
            "testfixtures.WithIndexedNodeLabelsConfig": lambda ls, c: self._cfg(c, indexed_node_labels=list(c.indexed_node_labels) + list(ls)),
            "testfixtures.WithIndexedResourcesConfig": lambda rs, c: self._cfg(c, indexed_resources=[ResourceType(r["Name"], str(r["Resolution"])) for r in rs]),
        }

    # ---- helpers backing Go fixture functions ----------------------------------------------
    def _round_limits(self, c, limits):
        pool = getattr(c, "_pool_round_limits", None)
        c2 = self._cfg(c, maximum_resource_fraction_to_schedule=dict(pool) if pool is not None else limits)
        c2._pool_round_limits = pool
        return c2

    def _round_limits_pool(self, c, by_pool):
        pool = by_pool.get("pool")
        c2 = self._cfg(c, maximum_resource_fraction_to_schedule=dict(pool)) if pool is not None else self._cfg(c)
        c2._pool_round_limits = dict(pool) if pool is not None else None
        return c2

    @staticmethod
    def _cfg(c: SchedulingConfig, **kw) -> SchedulingConfig:
        for k, v in kw.items():
            setattr(c, k, v)
        return c

    @staticmethod
    def _per_priority_limits(limits, c: SchedulingConfig):
        for pcn, lim in limits.items():
            pc = c.priority_classes[pcn]
            c.priority_classes[pcn] = PriorityClass(pc.priority, pc.preemptible, (), dict(lim))
        return c

    @staticmethod
    def _with_gang_details(jobs, gang_id, card, uniformity):
        if uniformity:
            raise UnsupportedCase("node uniformity label")
        for j in jobs:
            j.gang_id, j.gang_cardinality = gang_id, int(card)
        return jobs

    def _with_annotations(self, ann, jobs):
        gid = ann.get("armadaproject.io/gangId")
        card = ann.get("armadaproject.io/gangCardinality")
        if gid is not None and card is not None:
            for j in jobs:
                j.gang_id, j.gang_cardinality = gid, int(card)
        return jobs

    @staticmethod
    def _with_affinity(terms, jobs):
        conv = []
        for t in terms:
            exprs = tuple(MatchExpression(e["Key"], e["Operator"], tuple(e.get("Values", []))) for e in t.get("MatchExpressions", []))
            conv.append(exprs)
        for j in jobs:
            j.affinity = tuple(j.affinity or ()) + tuple(conv)
        return jobs

    @staticmethod
    def _with_requests(rl, jobs):
        res = rl.get("Resources", rl)
        for j in jobs:
            j.requests.update(res)
        return jobs

    @staticmethod
    def _add_labels(nodes, labels):
        for n in nodes:
            n.labels.update(labels)
        return nodes

    @staticmethod
    def _add_taints(nodes, taints):
        for n in nodes:
            n.taints = tuple(n.taints) + tuple(Taint(t["Key"], t.get("Value", ""), t.get("Effect", "")) for t in taints)
        return nodes

    @staticmethod
    def _with_used(p, rl, nodes):
        for n in nodes:
            if not hasattr(n, "used"):
                n.used = []
            n.used.append((int(p), dict(rl)))
        return nodes

    @staticmethod
    def _with_node_type(node_type, nodes):
        for n in nodes:
            n.forced_type = node_type
        return nodes

    # ---- evaluator ----------------------------------------------------------------------------
    def ev(self, n):
        if isinstance(n, (int, float, str, bool)) or n is None:
            return n
        if isinstance(n, list):
            return [self.ev(x) for x in n]
        if "unsupported" in n:
            raise UnsupportedCase(n["unsupported"])
        if "id" in n:
            if n["id"] in self.ids:
                v = self.ids[n["id"]]
                return v.make() if isinstance(v, _Fresh) else v
            raise UnsupportedCase(f"identifier {n['id']}")
        if "neg" in n:
            return -self.ev(n["neg"])
        if "op" in n:
            # Go constant expressions are exact (arbitrary precision) and rounded once
            from fractions import Fraction
            l, r = self.ev(n["l"]), self.ev(n["r"])
            if isinstance(l, (int, float, Fraction)) and isinstance(r, (int, float, Fraction)):
                both_int = isinstance(l, int) and isinstance(r, int)
                fl, fr = Fraction(l), Fraction(r)
                v = {"+": lambda: fl + fr, "-": lambda: fl - fr, "*": lambda: fl * fr, "/": lambda: fl / fr}[n["op"]]()
                if both_int and n["op"] != "/":
                    return int(v)
                if both_int and v.denominator == 1:
                    return int(v)  # Go integer constant division of exact multiples
                return v
            return {"+": lambda: l + r, "-": lambda: l - r, "*": lambda: l * r, "/": lambda: l / r}[n["op"]]()
        if "call" in n:
            name = n["call"]
            if name not in self.calls:
                if name and (name.startswith("[]") or name in ("float64", "int", "int32", "uint", "int64", "uint32")):
                    return self.ev(n["args"][0])
                raise UnsupportedCase(f"function {name}")
            return self.calls[name](*[self.ev(a) for a in n["args"]])
        if "lit" in n:
            typ = n["lit"]
            elems = n["elems"]
            keyed = any(k is not None for k, _ in elems)
            if not elems and typ in ("", "case"):
                return {}
            if typ.startswith("[]") or (not keyed and typ in ("", "case")):
                return [self.ev(v) for _, v in elems]
            out = {}
            for k, v in elems:
                if isinstance(k, dict) and "id" in k and k["id"] not in self.ids:
                    key = k["id"]  # struct field name
                else:
                    key = self.ev(k)
                out[key] = self.ev(v)
            return out
        raise UnsupportedCase(f"node {list(n.keys())}")


# =================================================================================================
# Builders shared by the drivers
# =================================================================================================
SYNTH_QUEUE = None


def materialize_used(cfg: SchedulingConfig, nodes: List[NodeSpec], F: fx.Fixtures) -> List[JobSpec]:
    """WithUsedResourcesNodes → synthetic running jobs (preemptible, bound at priority p, no queue
    context) so that AllocatableByPriority[p'] -= rl for all p' <= p (MarkAllocated)."""
    jobs = []
    for n in nodes:
        for (p, rl) in getattr(n, "used", []):
            if not rl:
                continue
            pcn = f"zz-used-{p}"
            if pcn not in cfg.priority_classes:
                if p not in cfg.allowed_priorities():
                    raise UnsupportedCase(f"used resources at priority {p} not in allowed priorities")
                cfg.priority_classes[pcn] = PriorityClass(p, True)
            j = F.job("zz-no-queue", pcn, rl)
            j.node = n.id
            j.scheduled_at_priority = p
            jobs.append(j)
    return jobs


def expected_states(n_jobs: int, scheduled: List[int], never: List[int]) -> np.ndarray:
    st = np.full(n_jobs, abi.JOB_FAILED, np.uint8)
    st[never] = abi.JOB_NONE
    st[scheduled] = abi.JOB_SCHEDULED
    return st


# =================================================================================================
# TestQueueScheduler driver (queue_scheduler_test.go:480-680)
# =================================================================================================
def run_queue_scheduler_case(case: dict, run_round: Callable) -> None:
    env = Env()
    tc = env.ev(case)
    cfg: SchedulingConfig = tc["SchedulingConfig"]
    nodes: List[NodeSpec] = tc["Nodes"]
    jobs: List[JobSpec] = tc["Jobs"]
    queues_in = tc["Queues"]
    synth = materialize_used(cfg, nodes, env.fx)
    f = cfg.factory()
    qspecs = []
    initial = tc.get("InitialAllocatedByQueueAndPriorityClass") or {}
    for q in queues_in:
        name = q["Name"]
        demand = np.zeros(f.D, np.int64)
        for j in jobs:
            if j.queue == name:
                demand += f.from_job(j.requests)
        limits = {}
        for pcn, lim in (q.get("ResourceLimitsByPriorityClassName") or {}).items():
            limits[pcn] = dict(lim.get("MaximumResourceFraction") or {})
            by_pool = (lim.get("MaximumResourceFractionByPool") or {}).get("pool")
            if by_pool:  # util.MergeMaps(fractions, queuePoolConfig), constraints.go:244-249
                limits[pcn].update(by_pool.get("MaximumResourceFraction") or {})
        alloc = {pcn: f.from_job(rl) for pcn, rl in (initial.get(name) or {}).items()}
        qspecs.append(QueueSpec(name=name, priority_factor=float(q.get("PriorityFactor", 1.0)), demand=demand,
                                constrained_demand=demand, allocated_by_pc=alloc, resource_limits_by_pc=limits))
    b = RoundInputBuilder(cfg, nodes, list(jobs) + synth, qspecs)
    res = run_round(b.input)
    nj = len(jobs)
    exp_sched = sorted(tc.get("ExpectedScheduledIndices") or [])
    never = tc.get("ExpectedNeverAttemptedIndices") or []
    got_sched = sorted(int(i) for i in np.nonzero(res.job_state[:nj] == abi.JOB_SCHEDULED)[0])
    assert got_sched == exp_sched, f"scheduled {got_sched} != expected {exp_sched}"
    exp = expected_states(nj, exp_sched, never)
    got = res.job_state[:nj]
    assert (got == exp).all(), f"job states {got.tolist()} != expected {exp.tolist()}"
    assert res.out.termination_reason != 0
    # scheduled jobs must be on a node that statically matches
    for i in got_sched:
        assert res.job_node[i] != abi.NONE


# =================================================================================================
# TestPreemptingQueueScheduler driver (preempting_queue_scheduler_test.go:2046-2377)
# =================================================================================================
def _gpu_taint():
    return Taint("gpu", "true", "NoSchedule")


def _home_away_cfg(lower: bool = False, **kw) -> SchedulingConfig:
    pcs = {"armada-preemptible-away": PriorityClass(30000, True, (AwayNodeType(29000, "gpu"),)), "armada-preemptible": PriorityClass(30000, True)}
    if lower:
        pcs["armada-preemptible-away-lower"] = PriorityClass(30000, True, (AwayNodeType(28000, "gpu"),))
    return fx.test_scheduling_config(priority_classes=pcs, well_known_node_types={"gpu": (_gpu_taint(),)}, **kw)


def _away_jobs(F, queue, n, pc="armada-preemptible-away"):
    return F.n_1cpu_4gi(queue, pc, n)


def _home_gpu_jobs(F, queue, n):  # Test1GpuPodReqs + the gpu toleration, priority class armada-preemptible
    return F.n_1gpu(queue, "armada-preemptible", n)


def _pqs_away_first(F, mixed):
    nodes = (F.n_cpu32(1) + [F.gpu8_tainted()]) if mixed else [F.gpu8_tainted(), F.gpu8_tainted()]
    return {"SchedulingConfig": _home_away_cfg() if mixed else fx.test_scheduling_config(well_known_node_types={"gpu": (_gpu_taint(),)}),
            "Nodes": nodes, "PriorityFactorByQueue": {"A": 1.0, "B": 1.0},
            "Rounds": [{"JobsByQueue": {"A": _away_jobs(F, "A", 96)}, "ExpectedScheduledIndices": {"A": list(range(96))}},
                       {"JobsByQueue": {"B": _home_gpu_jobs(F, "B", 12)}, "ExpectedScheduledIndices": {"B": list(range(8 if mixed else 12))},
                        "ExpectedPreemptedIndices": {"A": {0: list(range(32, 96))}}}]}


def _pqs_home_first(F, mixed):
    nodes = (F.n_cpu32(1) + [F.gpu8_tainted()]) if mixed else [F.gpu8_tainted(), F.gpu8_tainted()]
    return {"SchedulingConfig": _home_away_cfg(), "Nodes": nodes, "PriorityFactorByQueue": {"A": 1.0, "B": 1.0},
            "Rounds": [{"JobsByQueue": {"B": _home_gpu_jobs(F, "B", 12)}, "ExpectedScheduledIndices": {"B": list(range(8 if mixed else 12))}},
                       {"JobsByQueue": {"A": _away_jobs(F, "A", 96)}, "ExpectedScheduledIndices": {"A": list(range(32))}}]}


def _pqs_multiple_levels(F):
    node = F.cpu32()
    node.taints = node.taints + (_gpu_taint(),)
    c_jobs = F.n_jobs("C", "armada-preemptible", 17, {"cpu": "1", "memory": "4Gi"}, (Toleration("gpu", "", "true"),))
    return {"SchedulingConfig": _home_away_cfg(lower=True, protected_fraction_of_fair_share=5.0), "Nodes": [node],
            "PriorityFactorByQueue": {"A": 1.0, "B": 1.0, "C": 1.0},
            "Rounds": [{"JobsByQueue": {"A": _away_jobs(F, "A", 16, "armada-preemptible-away-lower"), "B": _away_jobs(F, "B", 16)},
                        "ExpectedScheduledIndices": {"A": list(range(16)), "B": list(range(16))}},
                       {"JobsByQueue": {"C": c_jobs}, "ExpectedScheduledIndices": {"C": list(range(17))},
                        "ExpectedPreemptedIndices": {"A": {0: list(range(16))}, "B": {0: [15]}}}]}


# TestPreemptingQueueScheduler cases whose config / nodes / jobs are built in closures in the table
# (preempting_queue_scheduler_test.go:1707-2045): transcribed by hand
MANUAL_PQS = {
    "home-away preemption, away jobs first": lambda F: _pqs_away_first(F, False),
    "home-away preemption, home jobs first": lambda F: _pqs_home_first(F, False),
    "home-away preemption, mixed nodes, away jobs first": lambda F: _pqs_away_first(F, True),
    "home-away preemption, mixed nodes, home jobs first": lambda F: _pqs_home_first(F, True),
    "home-away preemption through multiple levels": _pqs_multiple_levels,
}


def run_pqs_case(case: dict, run_round: Callable, check_expected: bool = True, on_round: Optional[Callable] = None) -> None:
    env = Env()
    tc = MANUAL_PQS[case["manual"]](env.fx) if "manual" in case else env.ev(case)
    cfg: SchedulingConfig = tc["SchedulingConfig"]
    nodes: List[NodeSpec] = tc["Nodes"]
    rounds = tc["Rounds"]
    pf_by_queue: Dict[str, float] = tc["PriorityFactorByQueue"]
    f = cfg.factory()
    synth = materialize_used(cfg, nodes, env.fx)
    running: List[JobSpec] = []  # jobs with an active run
    run_ts = [0]

    def start_run(job: JobSpec, node_id: str, priority: int):
        j = copy.copy(job)
        j.node = node_id
        j.scheduled_at_priority = priority
        run_ts[0] += 1
        j.active_run_timestamp = run_ts[0]
        return j

    for node_idx, jobs in (tc.get("InitialRunningJobs") or {}).items():
        for job in jobs:
            running.append(start_run(job, nodes[int(node_idx)].id, cfg.priority_classes[job.priority_class].priority))

    alloc_by_queue_pc: Dict[str, Dict[str, np.ndarray]] = {}
    demand_by_queue: Dict[str, np.ndarray] = {}
    node_of_job: Dict[str, str] = {}
    round_of_job: Dict[str, int] = {}
    index_of_job: Dict[str, int] = {}
    tokens_global = None
    tokens_queue: Dict[str, Optional[float]] = {q: None for q in pf_by_queue}
    cordoned = set()

    for ri, rnd in enumerate(rounds):
        if rnd.get("OptimiserEnabled"):
            raise UnsupportedCase("optimiser")
        if rnd.get("IndicesToUnbind"):
            raise UnsupportedCase("IndicesToUnbind")
        queued: List[JobSpec] = []
        for queue, jobs in (rnd.get("JobsByQueue") or {}).items():
            for k, job in enumerate(jobs):
                assert job.queue == queue
                queued.append(job)
                round_of_job[job.id] = ri
                index_of_job[job.id] = k
                demand_by_queue[queue] = demand_by_queue.get(queue, np.zeros(f.D, np.int64)) + f.from_job(job.requests)
        for idx in rnd.get("NodeIndicesToCordon") or []:
            cordoned.add(int(idx))
        rnodes = []
        for i, n in enumerate(nodes):
            n2 = copy.copy(n)
            if i in cordoned:  # taints += UnschedulableTaint (test driver :2150-2160)
                n2.taints = tuple(n.taints) + (Taint("armadaproject.io/unschedulable", "true", "NoSchedule"),)
            rnodes.append(n2)
        qspecs = []
        for qn, pf in pf_by_queue.items():
            d = demand_by_queue.get(qn, np.zeros(f.D, np.int64))
            qspecs.append(QueueSpec(name=qn, priority_factor=pf, demand=d, constrained_demand=d,
                                    allocated_by_pc=dict(alloc_by_queue_pc.get(qn, {})), limiter_tokens=tokens_queue[qn]))
        all_jobs = running + queued + synth
        # rate limiters persist between rounds; 1 s passes between rounds (test driver :2071-2083)
        b = RoundInputBuilder(cfg, rnodes, all_jobs, qspecs, global_limiter_tokens=tokens_global)
        res = run_round(b.input)
        if on_round is not None:
            on_round(ri, b, res)
        pos = b.job_pos
        states = {j.id: int(res.job_state[pos[j.id]]) for j in all_jobs}
        sched = [j for j in queued + running if states[j.id] == abi.JOB_SCHEDULED]
        preempted = [j for j in running + queued if states[j.id] == abi.JOB_PREEMPTED]

        # accounting identity checked by the reference driver (:2213-2236)
        for j in preempted:
            m = alloc_by_queue_pc.setdefault(j.queue, {})
            m[j.priority_class] = m.get(j.priority_class, np.zeros(f.D, np.int64)) - f.from_job(j.requests)
        for j in sched:
            m = alloc_by_queue_pc.setdefault(j.queue, {})
            m[j.priority_class] = m.get(j.priority_class, np.zeros(f.D, np.int64)) + f.from_job(j.requests)
        for qn in pf_by_queue:
            qi = b.queue_index[qn]
            for pcn, pi in b.pc_index.items():
                want = alloc_by_queue_pc.get(qn, {}).get(pcn, np.zeros(f.D, np.int64))
                got = res.queue_allocated_by_pc[qi, pi]
                assert (got == want).all(), f"round {ri}: queue {qn} pc {pcn} allocation {got} != {want}"

        for j in preempted:
            nid = rnodes[int(res.job_node[pos[j.id]])].id
            assert nid == node_of_job[j.id], f"round {ri}: job preempted from unexpected node"
        for j in sched:
            nid = rnodes[int(res.job_node[pos[j.id]])].id
            if j.id in node_of_job:
                assert node_of_job[j.id] == nid
            node_of_job[j.id] = nid

        if check_expected:
            exp_s = {q: sorted(v) for q, v in (rnd.get("ExpectedScheduledIndices") or {}).items() if v}
            got_s: Dict[str, List[int]] = {}
            for j in sched:
                got_s.setdefault(j.queue, []).append(index_of_job[j.id])
            got_s = {q: sorted(v) for q, v in got_s.items()}
            assert got_s == exp_s, f"round {ri}: scheduled {got_s} != expected {exp_s}"
            exp_p = {}
            for q, m in (rnd.get("ExpectedPreemptedIndices") or {}).items():
                mm = {int(r): sorted(v) for r, v in m.items() if v}
                if mm:
                    exp_p[q] = mm
            got_p: Dict[str, Dict[int, List[int]]] = {}
            for j in preempted:
                got_p.setdefault(j.queue, {}).setdefault(round_of_job[j.id], []).append(index_of_job[j.id])
            got_p = {q: {r: sorted(v) for r, v in m.items()} for q, m in got_p.items()}
            assert got_p == exp_p, f"round {ri}: preempted {got_p} != expected {exp_p}"
            # no oversubscribed nodes at real priorities (:2301-2310)
            for p in range(1, res.node_alloc.shape[0]):
                assert (res.node_alloc[p][:, : len(rnodes)] >= 0).all(), f"round {ri}: oversubscribed node at level {p}"

        # carry state into the next round (:2312-2370)
        pre_ids = {j.id for j in preempted}
        running = [j for j in running if j.id not in pre_ids]
        for j in sorted(sched, key=lambda j: j.submit_time):
            if j.node is None:
                running.append(start_run(j, node_of_job[j.id], int(res.job_scheduled_at_priority[pos[j.id]])))
        # limiter state: tokens consumed this round, then +rate*1s capped at burst
        nsched_new = sum(1 for j in queued if states[j.id] == abi.JOB_SCHEDULED)
        if not math.isinf(cfg.maximum_scheduling_rate):
            cur = float(b.input.global_limiter_tokens) - nsched_new
            tokens_global = min(float(b.input.global_limiter_burst), cur + cfg.maximum_scheduling_rate * 1.0)
        if not math.isinf(cfg.maximum_per_queue_scheduling_rate):
            for qn in pf_by_queue:
                used = sum(1 for j in queued if j.queue == qn and states[j.id] == abi.JOB_SCHEDULED)
                cur = float(b.queue_limiter_tokens[b.queue_index[qn]]) - used
                tokens_queue[qn] = min(float(b.queue_limiter_burst[b.queue_index[qn]]), cur + cfg.maximum_per_queue_scheduling_rate * 1.0)
