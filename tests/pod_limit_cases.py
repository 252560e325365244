"""RespectNodePodLimits (configuration.go:548-580, jobdb.go:256-263): every job is one pod, counted against each
node's `pods` capacity.  Bodies shared by the emulator and GPU modules (tests/test_pod_limits_emu.py,
tests/test_pod_limits_gpu.py), each round compared bit for bit with the oracle:

  * the reference's TestPreemptingQueueScheduler_RespectNodePodLimits table (preempting_queue_scheduler_test.go:3018-3250,
    tests/golden/respect_node_pod_limits.json) and TestPreemptingQueueScheduler_NonPreemptibleOverPack (:3252-3330),
    restated through RoundInputBuilder;
  * seeded rounds where the pod capacity binds, in each form of the assignment loop a pods field can give;
  * the SubmitChecker's reason for a job refused on pods, and simulator runs whose pod capacity binds before cpu.

Pods are one more resource at resolution 1, indexed last; nothing in the kernels knows them by name."""
from __future__ import annotations

import json
import os
from dataclasses import dataclass
from typing import Callable, Dict, List

import numpy as np

import fixtures as fx
import go_tables as gt
import oracle_lib
import shape_cases
from armada_b200 import abi, synth
from armada_b200 import simulator as sim
from armada_b200.model import (PODS, JobSpec, QueueSpec, ResourceType, RoundInputBuilder, apply_respect_node_pod_limits)
from armada_b200.submitcheck import Executor, PoolConfig, SubmitChecker

with open(os.path.join(gt.GOLDEN, "respect_node_pod_limits.json")) as _f:
    TABLE = json.load(_f)["cases"]


def pod_limits_config(**overrides):
    """TestSchedulingConfig with RespectNodePodLimits on and applied."""
    cfg = fx.test_scheduling_config(respect_node_pod_limits=True, **overrides)
    assert apply_respect_node_pod_limits(cfg)
    return cfg


# ---- the reference's tables ----------------------------------------------------------------------------
@dataclass
class TableRound:
    builder: RoundInputBuilder
    incumbents: List[JobSpec]
    challengers: List[JobSpec]
    tc: dict


def _table_round(cfg, node_resources: List[Dict[str, str]], incumbent_pc: str, n_incumbents: int, n_challengers: int,
                 gang: bool, tc: dict) -> TableRound:
    """The drivers' common set-up: queue A; incumbents bound to the first node at their priority class's priority;
    PriorityClass3 challengers; allocatedByPriorityClass from the incumbents; demand = constrained demand = the
    challengers' requests (AllResourceRequirements, pods included)."""
    F = fx.Fixtures()
    nodes = [F.node(res) for res in node_resources]
    incumbents = F.n_1cpu_4gi("A", incumbent_pc, n_incumbents)
    for k, j in enumerate(incumbents):
        j.node, j.scheduled_at_priority, j.active_run_timestamp = nodes[0].id, cfg.priority_classes[incumbent_pc].priority, k + 1
    challengers = F.n_1cpu_4gi("A", fx.PriorityClass3, n_challengers)
    if gang:
        for j in challengers:
            j.gang_id, j.gang_cardinality = "gang-1", n_challengers
    f = cfg.factory()
    alloc: Dict[str, np.ndarray] = {}
    for j in incumbents:
        alloc[j.priority_class] = alloc.get(j.priority_class, np.zeros(f.D, np.int64)) + f.from_job(cfg.job_requests(j.requests))
    demand = np.zeros(f.D, np.int64)
    for j in challengers:
        demand += f.from_job(cfg.job_requests(j.requests))
    q = QueueSpec("A", 1.0, allocated_by_pc=alloc, demand=demand, constrained_demand=demand.copy())
    return TableRound(RoundInputBuilder(cfg, nodes, incumbents + challengers, [q]), incumbents, challengers, tc)


def respect_node_pod_limits_round(name: str) -> TableRound:
    """One case of TestPreemptingQueueScheduler_RespectNodePodLimits: nodes of 10 cpu / 64Gi / the case's pod capacity."""
    tc = gt.Env().ev(TABLE[name])
    caps = [tc["nodePodCapacity"]] + list(tc.get("extraNodePodCapacities") or [])
    pc = tc.get("incumbentPriorityClass") or fx.PriorityClass0  # ("" only where there are no incumbents)
    return _table_round(pod_limits_config(), [{"cpu": "10", "memory": "64Gi", PODS: str(c)} for c in caps], pc,
                        tc.get("incumbentCount", 0), tc.get("challengerCount", 0), tc.get("challengerIsGang", False), tc)


def non_preemptible_over_pack_round() -> TableRound:
    """TestPreemptingQueueScheduler_NonPreemptibleOverPack: the knob off, a 5 cpu node held by five non-preemptible
    PriorityClass2 jobs, one PriorityClass3 challenger."""
    tc = {"incumbentPriorityClass": fx.PriorityClass2NonPreemptible, "expectedPreemptions": 0, "expectedNewlyScheduled": 0}
    return _table_round(fx.test_scheduling_config(), [{"cpu": "5", "memory": "64Gi"}], fx.PriorityClass2NonPreemptible, 5, 1, False, tc)


def check_table_expectations(t: TableRound, res) -> None:
    """The reference's assertions: counts, the preempted and scheduled jobs' classes, the node the challenger takes."""
    ni = len(t.incumbents)
    state = np.asarray(res.job_state)[: ni + len(t.challengers)]
    preempted = [t.builder.jobs[i] for i in np.nonzero(state == abi.JOB_PREEMPTED)[0]]
    scheduled = [int(i) for i in np.nonzero(state == abi.JOB_SCHEDULED)[0]]
    assert len(preempted) == t.tc["expectedPreemptions"], state.tolist()
    assert len(scheduled) == t.tc["expectedNewlyScheduled"], state.tolist()
    assert all(j.priority_class == t.tc["incumbentPriorityClass"] for j in preempted)
    for i in scheduled:
        assert t.builder.jobs[i].priority_class == fx.PriorityClass3
        if t.tc.get("extraNodePodCapacities"):
            assert int(res.job_node[i]) != 0, "the challenger should land on an extra node, not the saturated one"


def table_on_the_oracle(t: TableRound) -> None:
    check_table_expectations(t, oracle_lib.round_schedule(t.builder.input))


def table_against_the_oracle(schedule: Callable, t: TableRound) -> None:
    want = oracle_lib.round_schedule(t.builder.input)
    got = schedule(t.builder.input)
    bad = got.diff(want)
    assert not bad, "device != oracle:\n  " + "\n  ".join(bad)
    check_table_expectations(t, got)


def releases_pod_slot() -> None:
    """TestNodeBindingEvictionUnbinding_ReleasesPodSlot (nodedb/nodedb_test.go:240-305) on the oracle's NodeDb: cpu 1m,
    memory 1 and pods 1 both supported and indexed; a 10 cpu / 64Gi node with one pod slot.  Binding a PriorityClass0
    job uses the slot, evicting and unbinding it frees the slot, a second job binds and uses it again."""
    types = [ResourceType("cpu", "1m"), ResourceType("memory", "1"), ResourceType(PODS, "1")]
    cfg = fx.test_scheduling_config(supported_resource_types=types, indexed_resources=types, respect_node_pod_limits=True)
    assert apply_respect_node_pod_limits(cfg)
    F = fx.Fixtures()
    node = F.node({"cpu": "10", "memory": "64Gi", PODS: "1"})
    jobs = [F.job("queue", fx.PriorityClass0, {"cpu": "1", "memory": "1Gi"}) for _ in range(2)]
    b = RoundInputBuilder(cfg, [node], jobs, [QueueSpec("queue")])
    pods = b.factory.index[PODS]
    level = b.priorities.index(cfg.priority_classes[fx.PriorityClass0].priority)
    db = oracle_lib.OracleNodeDb(b.input)
    try:
        assert db.get_alloc(0)[level, pods] == 1
        ok, nodes, *_ = db.schedule_many([0])
        assert ok and nodes[0] == 0
        assert db.get_alloc(0)[level, pods] == 0, "bind should consume the pod slot"
        db.evict(0)
        db.unbind(0)
        assert db.get_alloc(0)[level, pods] == 1, "evict + unbind should free the pod slot"
        ok, nodes, *_ = db.schedule_many([1])
        assert ok and nodes[0] == 0, "the second job should bind after the slot is freed"
        assert db.get_alloc(0)[level, pods] == 0, "the second bind should also consume the pod slot"
    finally:
        db.close()


# ---- seeded rounds where the pod capacity binds ---------------------------------------------------------
@dataclass(frozen=True)
class PodCase:
    form: str       # the assignment loop's form: k32 | k64 | unguarded | exact
    kind: str       # "batch": queued jobs only; "eviction": running jobs, priorities, protected fraction 0.5
    caps: str       # "one": 1 pod per node; "small": 1-8 (pods bind first); "wide": 110 (cpu or memory binds first)
    seed: int
    n_nodes: int = 60

    @property
    def id(self) -> str:
        return f"{self.form}-{self.kind}-{self.caps}-s{self.seed}" + (f"-n{self.n_nodes}" if self.n_nodes != 60 else "")


def pod_round(case: PodCase) -> synth.RawRound:
    """synth.random_round (node kinds, gangs, and for "eviction" running jobs, priority classes, away node types on odd
    seeds) with pod limits.  The "unguarded" form measures memory in units of 2**k bytes, the least k for which the
    key's fields and the node index fit 63 bits (62 or 63 of them): the key fits only without guard bits.  "exact" has
    cpu quantities off the index resolution."""
    evict = case.kind == "eviction"
    r = synth.random_round(case.seed, n_nodes=case.n_nodes, n_queues=5, n_jobs=12 * case.n_nodes, n_running=3 * case.n_nodes if evict else 0,
                           gangs=True, priorities=evict, protected_fraction=0.5 if evict else 0.0, away=evict and case.seed % 2 == 1,
                           unaligned=case.form == "exact")
    N = r.node_total.shape[1]
    rng = np.random.default_rng(case.seed)
    caps = {"one": np.ones(N, np.int64), "small": rng.integers(1, 9, N), "wide": np.full(N, 110)}[case.caps]
    r = synth.with_pod_limits(r, caps)
    if case.form == "unguarded":
        top = r.node_allocatable.max(axis=1)
        others = sum(int(top[d] // res).bit_length() for d, res in zip(r.indexed, r.resolution) if d != synth.MEM)
        k = max(0, int(top[synth.MEM]).bit_length() - (63 - (N - 1).bit_length() - others))
        r.resolution[r.indexed.index(synth.MEM)] = 1 << k
    return r


CASES = [PodCase("k32", "batch", "one", 1), PodCase("k64", "batch", "small", 2), PodCase("k64", "eviction", "small", 3),
         PodCase("k64", "batch", "wide", 4), PodCase("k64", "eviction", "wide", 5), PodCase("unguarded", "batch", "small", 6),
         PodCase("unguarded", "eviction", "small", 7), PodCase("exact", "batch", "small", 8), PodCase("exact", "eviction", "small", 9)]


def seeded_round(dev, case: PodCase, capfd) -> None:
    """One seeded round through `dev` (a DeviceRound) against the oracle: the loop form it was built for, every output
    array, and that the binding resource is the one the case was built for."""
    inp = pod_round(case).to_input()
    want = oracle_lib.round_schedule(inp)
    got, lay, form = shape_cases.schedule_with_layout(dev, inp, capfd)
    assert form == case.form, f"{case.id}: built for {case.form}, the library chose {form} ({lay})"
    bad = got.diff(want)
    assert not bad, f"{case.id}: device != oracle:\n  " + "\n  ".join(bad)
    N, pods = inp.num_nodes, inp.num_resources - 1
    full = (np.asarray(want.node_alloc)[1:, pods, :N] == 0).any()  # a node with no pod slot left at some real priority
    assert full == (case.caps != "wide"), case.id
    assert (np.asarray(want.job_state) == abi.JOB_FAILED).any(), f"{case.id}: every job fit"


def c3_with_pods(scale: float = 1.0, pods: int = 110) -> synth.RawRound:
    """C3 with the knob on: every node holds `pods` pods (110 is the kubelet's default); one C3 round at `scale`."""
    r = synth.config_c3() if scale == 1.0 else synth.scaled("C3", scale)
    return synth.with_pod_limits(r, pods)


# ---- SubmitChecker -----------------------------------------------------------------------------------------
def _reason(excluded: str) -> str:
    return ("executor-0:\n"
            "Node:                       none\n"
            "Number of nodes in cluster: 1\n"
            "Excluded nodes:\n"
            f" 1: {excluded}\n"
            "\n---\n")


def submit_checker_refuses_on_pods(lib) -> None:
    """A job that fits on cpu and memory is refused when no node has a pod slot for it.  A node that reports no `pods`
    has 0 (FromNodeProto); pods being indexed, the node iterator never reaches it (nodeiteration.go:344-377), so it
    counts as "insufficient resources available".  A node whose allocatable reports a slot its total does not is
    reached and fails StaticJobRequirementsMet's check of the totals: InsufficientResources on pods at scale 0.  A gang
    of three on a node with two slots places two.  With the knob off the same jobs are accepted."""
    F = fx.Fixtures()
    no_pods = F.node({"cpu": "32", "memory": "256Gi"})
    slot_in_allocatable_only = F.node({"cpu": "32", "memory": "256Gi"})
    slot_in_allocatable_only.allocatable = {"cpu": "32", "memory": "256Gi", PODS: "1"}
    two = F.node({"cpu": "32", "memory": "256Gi", PODS: "2"})
    job = F.job("queue", fx.PriorityClass0, {"cpu": "1", "memory": "4Gi"})
    gang = fx.with_gang(F.n_1cpu_4gi("queue", fx.PriorityClass0, 3), "g")
    for cfg, want in ((pod_limits_config(), False), (fx.test_scheduling_config(), True)):
        for node, excluded in ((no_pods, "insufficient resources available"),
                               (slot_in_allocatable_only, "pod requires 1 pods, but only 0 is available")):
            with SubmitChecker(cfg, [PoolConfig("cpu")], [Executor("executor-0", [("cpu", node)])], [QueueSpec("queue")], lib=lib) as c:
                got = c.check([job])[job.id]
            assert got.is_schedulable == want, got
            assert got.reason == ("" if want else _reason(excluded))
        with SubmitChecker(cfg, [PoolConfig("cpu")], [Executor("executor-0", [("cpu", two)])], [QueueSpec("queue")], lib=lib) as c:
            got = c.check(gang)
        assert all(r.is_schedulable == want for r in got.values()), got
        if not want:
            assert got[gang[0].id].reason == "executor-0: 2 out of 3 pods schedulable\n"


# ---- simulator -------------------------------------------------------------------------------------------
SIM_CONFIG = {
    "defaultPriorityClassName": "armada-default",
    "priorityClasses": {"armada-default": {"priority": 30000, "preemptible": False}},
    "supportedResourceTypes": [{"name": "memory", "resolution": "1"}, {"name": "cpu", "resolution": "1m"}],
    "indexedResources": [{"name": "cpu", "resolution": "1"}, {"name": "memory", "resolution": "1Mi"}],
    "dominantResourceFairnessResourcesToConsider": ["cpu", "memory"],
    "maximumSchedulingRate": "+inf", "maximumPerQueueSchedulingRate": "+inf",
}
SIM_CLUSTER = {"name": "pods", "clusters": [{"name": "c0", "pool": "default", "nodeTemplates": [
    {"number": 3, "totalResources": {"resources": {"cpu": "32", "memory": "256Gi", PODS: "4"}}}]}]}
SIM_WORKLOAD = {"name": "w", "randomSeed": 1, "queues": [
    {"name": "A", "weight": 1, "jobTemplates": [{"id": "a", "number": 30, "jobSet": "s",
                                                 "requirements": {"resourceRequirements": {"requests": {"cpu": "1", "memory": "4Gi"}}},
                                                 "runtimeDistribution": {"minimum": "1m"}}]},
    {"name": "B", "weight": 2, "jobTemplates": [{"id": "b", "number": 12, "jobSet": "s",
                                                 "requirements": {"resourceRequirements": {"requests": {"cpu": "2", "memory": "8Gi"}}},
                                                 "runtimeDistribution": {"minimum": "90s"}}]}]}


def simulate(tmp_path, tag: str, engine, respect, pods_on_nodes: bool = True):
    """One simulator run from YAML files; `respect` None leaves the key out of the config.  Returns the run and the
    rows of its two parquet files."""
    import pyarrow.parquet as pq
    import yaml
    cfg = dict(SIM_CONFIG)
    if respect is not None:
        cfg["respectNodePodLimits"] = respect
    cluster = json.loads(json.dumps(SIM_CLUSTER))
    if not pods_on_nodes:
        del cluster["clusters"][0]["nodeTemplates"][0]["totalResources"]["resources"][PODS]
    d = tmp_path / tag
    d.mkdir()
    paths = []
    for name, doc in (("cluster", cluster), ("workload", SIM_WORKLOAD), ("config", cfg)):
        paths.append(str(d / f"{name}.yaml"))
        with open(paths[-1], "w") as f:
            yaml.safe_dump(doc, f)
    s = sim.simulate_files(*paths, output_dir=str(d / "out"), engine=engine)
    return s, [pq.read_table(str(d / "out" / n)).to_pylist() for n in ("jobs.parquet", "queue_stats.parquet")]


def _per_cycle(jobs_rows) -> List[int]:
    counts: Dict[int, int] = {}
    for r in jobs_rows:
        counts[r["scheduled_time"]] = counts.get(r["scheduled_time"], 0) + 1
    return [counts[t] for t in sorted(counts)]


def simulator_pod_cap_binds(tmp_path, engine) -> None:
    """Three 32-cpu nodes with 4 pod slots each: at most 12 jobs run at once although cpu would take 48.  The run
    driven by `engine` writes the rows the oracle-driven run writes."""
    dev, (dev_jobs, dev_queues) = simulate(tmp_path, "engine", engine, True)
    ref, (ref_jobs, ref_queues) = simulate(tmp_path, "oracle", oracle_lib.round_schedule, True)
    assert dev.rounds == ref.rounds
    assert dev_jobs == ref_jobs and len(dev_jobs) == 42
    assert repr(dev_queues) == repr(ref_queues)  # (NaN shares compare as text)
    assert max(_per_cycle(ref_jobs)) <= 12 and _per_cycle(ref_jobs)[0] == 12


def simulator_knob_off(tmp_path, engine) -> None:
    """With the knob off (or absent) a node's `pods` is an unknown resource: the rows are those of the same cluster
    without pods, and the first cycle fills every queue's demand."""
    _, rows_off = simulate(tmp_path, "off", engine, False)
    _, rows_absent = simulate(tmp_path, "absent", engine, None)
    _, rows_plain = simulate(tmp_path, "plain", engine, None, pods_on_nodes=False)
    assert repr(rows_off) == repr(rows_absent) == repr(rows_plain)  # (NaN shares compare as text)
    assert _per_cycle(rows_off[0])[0] == 42
