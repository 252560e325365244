"""Oracle pinned against the reference's unit-level known-answer tables (CPU only):
  TestNodeTypeIterator / TestNodeTypesIterator  nodedb/nodeiteration_test.go:75-690  (exact visit order)
  TestCalculateFairShares                       scheduling/context/scheduling_test.go:74-230 (exact doubles)
  TestDominantResourceFairness                  scheduling/fairness/fairness_test.go:62-170
  TestGangScheduler                             scheduling/gang_scheduler_test.go:33-760 (single-queue cases)
  TestNodeIndexKey / bind-evict-unbind vectors  nodedb/encoding_test.go, nodedb/nodedb_test.go:148-422
"""
import ctypes as C
from fractions import Fraction

import json

import numpy as np
import pytest

import fixtures as fx
import go_tables as gt
import oracle_lib
from armada_b200 import abi
from armada_b200.model import (JobSpec, NodeSpec, PriorityClass, QueueSpec, ResourceType, RoundInputBuilder,
                               SchedulingConfig)

NTI = gt.load_cases("node_type_iterator")
NTSI = gt.load_cases("node_types_iterator")
FAIR = gt.load_cases("calculate_fair_shares")
DRF = gt.load_cases("dominant_resource_fairness")
GANG = gt.load_cases("gang_scheduler")


def _iterator_case(case, multi):
    env = gt.Env()
    for name in ("nodeTypeA", "nodeTypeB", "nodeTypeC", "nodeTypeD"):
        env.ids[name] = name
        env.calls[name + ".GetId"] = (lambda n: (lambda: n))(name)
    tc = env.ev(case)
    cfg = fx.test_scheduling_config()
    nodes = tc["nodes"]
    for i, n in enumerate(nodes):  # "Set monotonically increasing node IDs" (test driver)
        n.id, n.index = str(i), i
        n.labels[fx.TestHostnameLabel] = n.id
    synth_jobs = gt.materialize_used(cfg, nodes, env.fx)
    b = RoundInputBuilder(cfg, nodes, synth_jobs, [QueueSpec("A")])
    wanted = set(tc["nodeTypeIds"] if multi else [tc["nodeTypeId"]])
    row = 0
    b.type_match[row, :] = 0
    for t, key in enumerate(b.type_keys):
        if key[0] == "forced" and key[1] in wanted:
            b.type_match[row, t >> 5] |= np.uint32(1 << (t & 31))
    f = cfg.factory()
    rr = f.from_job(dict(tc["resourceRequests"]))
    ireq = [int(rr[f.index[r.name]]) for r in cfg.indexed_resources]
    db = oracle_lib.OracleNodeDb(b.input)
    got = db.iterate(row, int(tc["priority"]), ireq)
    assert got == [int(x) for x in tc["expected"]]


@pytest.mark.parametrize("name", sorted(NTI.keys()))
def test_node_type_iterator(name):
    _iterator_case(NTI[name], multi=False)


@pytest.mark.parametrize("name", sorted(NTSI.keys()))
def test_node_types_iterator(name):
    _iterator_case(NTSI[name], multi=True)


@pytest.mark.parametrize("name", sorted(FAIR.keys()))
def test_calculate_fair_shares(name):
    env = gt.Env()
    for nm, v in (("zeroCpu", 0), ("oneCpu", 1), ("fortyCpu", 40), ("oneHundredCpu", 100), ("oneThousandCpu", 1000)):
        env.ids[nm] = {"cpu": str(v)}
    tc = env.ev(FAIR[name])
    cfg = fx.test_scheduling_config(drf_resources=["cpu"])
    f = cfg.factory()
    queues = [QueueSpec(qn, priority_factor=1.0, demand=f.from_job(q["Demand"]), constrained_demand=f.from_job(q["Demand"]))
              for qn, q in tc["queueCtxs"].items()]
    weights = {qn: float(q["Weight"]) for qn, q in tc["queueCtxs"].items()}
    total = f.from_node(tc["availableResources"])
    b = RoundInputBuilder(cfg, [fx.Fixtures().cpu32()], [], queues, total_resources=total)
    for qn, w in weights.items():  # the test passes weights directly (not 1/priorityFactor)
        b.queue_weight[b.queue_index[qn]] = w
    res = oracle_lib.round_schedule(b.input)
    for qn in weights:
        qi = b.queue_index[qn]
        for col, key in enumerate(("expectedFairShares", "expectedDemandCappedAdjustedFairShares", "expectedUncappedAdjustedFairShares")):
            want = float(tc[key][qn])
            got = float(res.queue_fair_share[qi, col])
            assert got == want, f"{key}[{qn}]: {got!r} != {want!r}"  # exact float64 equality, like assert.Equal


@pytest.mark.parametrize("name", sorted(DRF.keys()))
def test_dominant_resource_fairness(name):
    env = gt.Env()
    env.ids["rlFactory"] = None
    env.ids["poolName"] = "pool"
    env.calls["fooBarBaz"] = lambda _f, a, b_, c: {"foo": a, "bar": b_, "baz": c}
    tc = env.ev(DRF[name])
    names = ["foo", "bar", "baz"]
    scale = Fraction(1, 1000)  # unset resolution ⇒ milli (resolutionToScale)
    to_i = lambda m: np.array([int(Fraction(str(m[n])) / scale) for n in names], np.int64)  # noqa: E731
    total, alloc = to_i(tc["totalResources"]), to_i(tc["allocation"])
    cfgd = tc["config"]
    mult = {n: 0.0 for n in names}
    exp = cfgd.get("ExperimentalDominantResourceFairnessResourcesToConsider")
    pools = cfgd.get("Pools") or []
    for p in pools:  # pool override (fairness.go:46-52)
        if p.get("Name") == "pool" and p.get("DominantResourceFairnessResourcesToConsider"):
            exp = p["DominantResourceFairnessResourcesToConsider"]
    plain = cfgd.get("DominantResourceFairnessResourcesToConsider") or []
    if exp and plain and not pools:
        pytest.skip("invalid config case")
    if exp and (not plain or pools):
        for r in exp:
            nm, m = (r[0], r[1]) if isinstance(r, list) else (r["Name"], r["Multiplier"])
            mult[nm] = float(m) if float(m) > 0 else 1.0
    else:
        for nm in plain:
            mult[nm] = 1.0
    m = np.array([mult[n] for n in names], np.float64)
    lib = oracle_lib.load()
    cost = lib.armada_oracle_drf_cost(3, total.ctypes.data_as(abi.i64p), m.ctypes.data_as(abi.f64p), alloc.ctypes.data_as(abi.i64p))
    w = float(tc.get("weight", 1.0)) or 1.0
    assert cost / w == float(tc["expectedCost"])


def _single_queue(gangs):
    return len({j.queue for g in gangs for j in g}) == 1


@pytest.mark.parametrize("name", sorted(GANG.keys()))
def test_gang_scheduler(name):
    """TestGangScheduler cases whose gangs all belong to one queue are order-equivalent to a
    QueueScheduler pass over that queue (gangs in submit order), so they can be driven through the
    round entry point (tests/gang_cases.py builds the round)."""
    import gang_cases
    b, tc, gangs = gang_cases.gang_case_round(name)
    res = oracle_lib.round_schedule(b.input)
    gang_cases.check_gang_case(b, tc, gangs, res)


def test_node_index_key_bytes():
    """TestNodeIndexKey (nodedb/encoding_test.go): layout | typeId | res... | nodeIndex |, big endian,
    sign bit flipped for int64."""
    lib = oracle_lib.load()
    q = np.array([1, -2, 3], np.int64)
    res = np.array([1, 1, 1], np.int64)
    out = np.zeros(8 * 5, np.uint8)
    lib.armada_oracle_node_index_key(3, 7, q.ctypes.data_as(abi.i64p), res.ctypes.data_as(abi.i64p), 9, 1, out.ctypes.data_as(abi.u8p))
    words = [int.from_bytes(bytes(out[8 * i: 8 * i + 8]), "big") for i in range(5)]
    assert words[0] == 7 and words[4] == 9
    assert words[1] == 1 ^ (1 << 63) and words[2] == ((-2) & (2**64 - 1)) ^ (1 << 63) and words[3] == 3 ^ (1 << 63)
    # rounding (TestRoundQuantityToResolution): toward zero to a multiple of the resolution
    q = np.array([1999, -1999, 2000], np.int64)
    res = np.array([1000, 1000, 1000], np.int64)
    lib.armada_oracle_node_index_key(3, 0, q.ctypes.data_as(abi.i64p), res.ctypes.data_as(abi.i64p), 0, 1, out.ctypes.data_as(abi.u8p))
    words = [int.from_bytes(bytes(out[8 * i: 8 * i + 8]), "big") ^ (1 << 63) for i in range(1, 4)]
    signed = [w - 2**64 if w >= 2**63 else w for w in words]
    assert signed == [1000, -1000, 2000]
    # byte order == numeric order (TestNodeIndexKeyComparison)
    keys = []
    for v in (-5, -1, 0, 1, 7):
        q = np.array([v, 0, 0], np.int64)
        lib.armada_oracle_node_index_key(3, 1, q.ctypes.data_as(abi.i64p), np.ones(3, np.int64).ctypes.data_as(abi.i64p), 0, 0, out.ctypes.data_as(abi.u8p))
        keys.append(bytes(out))
    assert keys == sorted(keys)


def test_eviction_allocatable_vectors():
    """TestEviction (nodedb/nodedb_test.go:363-422): a PriorityClass0 job and a non-preemptible
    PriorityClass3 job (1 cpu / 4Gi each) on a 32 cpu / 256Gi node, then both evicted."""
    F = fx.Fixtures()
    cfg = fx.test_scheduling_config()
    node = F.cpu32()
    j0 = F.job("A", fx.PriorityClass0, {"cpu": "1", "memory": "4Gi"})
    j3 = F.job("A", fx.PriorityClass3, {"cpu": "1", "memory": "4Gi"})
    for j in (j0, j3):
        j.node = node.id
    b = RoundInputBuilder(cfg, [node], [j0, j3], [QueueSpec("A")])
    db = oracle_lib.OracleNodeDb(b.input)
    f = cfg.factory()
    prios = b.priorities  # [-1,0,1,2,3,28000,29000,30000]
    cpu, mem = f.index["cpu"], f.index["memory"]

    def vec(c, m):
        v = np.zeros(f.D, np.int64)
        v[cpu], v[mem] = c * 1000, m * 2**30
        return v

    a = db.get_alloc(0)
    for lvl, p in enumerate(prios):
        want = vec(30, 248) if p <= 0 else vec(31, 252)  # non-preemptible job deducted at every level
        assert (a[lvl] == want).all(), (p, a[lvl], want)
    db.evict(0)
    db.evict(1)
    a = db.get_alloc(0)
    for lvl, p in enumerate(prios):
        want = vec(30, 248) if p == -1 else vec(32, 256)  # evicted jobs only count at EvictedPriority
        assert (a[lvl] == want).all(), (p, a[lvl], want)
    db.unbind(0)
    db.unbind(1)
    a = db.get_alloc(0)
    assert all((a[lvl] == vec(32, 256)).all() for lvl in range(len(prios)))


# ---- TestScheduleIndividually / TestScheduleMany (nodedb/nodedb_test.go:424-588, :590-670) --------
SCHED_ONE = gt.load_cases("schedule_individually")
SCHED_MANY = gt.load_cases("schedule_many")


def _nodedb_for(nodes, job_groups, env):
    cfg = fx.test_scheduling_config()
    jobs = [j for g in job_groups for j in g]
    t = 0
    for j in jobs:
        t += 1
        j.submit_time = t
    queues = sorted({j.queue for j in jobs})
    b = RoundInputBuilder(cfg, nodes, jobs, [QueueSpec(q, 1.0) for q in queues])
    return b, oracle_lib.OracleNodeDb(b.input)


@pytest.mark.parametrize("name", sorted(SCHED_ONE.keys()))
def test_schedule_individually(name):
    """One ScheduleManyWithTxn call per job on the same NodeDb, committed when it succeeds."""
    env = gt.Env()
    try:
        tc = env.ev(SCHED_ONE[name])
    except gt.UnsupportedCase as e:
        pytest.skip(f"not modelled: {e}")
    jobs = tc["Jobs"]
    for j in jobs:
        j.gang_id, j.gang_cardinality = None, 1
    b, db = _nodedb_for(tc["Nodes"], [[j] for j in jobs], env)
    want = [bool(x) for x in tc["ExpectSuccess"]]
    got = []
    for j in jobs:
        ok, node, _, _, _ = db.schedule_many([b.job_pos[j.id]])
        got.append(ok)
        if ok:
            assert node[0] != abi.NONE
    assert got == want


@pytest.mark.parametrize("name", sorted(SCHED_MANY.keys()))
def test_schedule_many(name):
    """Gang transactions: all members or none (the failed gang leaves no trace: "correct rollback")."""
    env = gt.Env()
    # locals of the reference's test function (nodedb_test.go:591-592); fresh job objects per use
    env.ids["gangSuccess"] = gt._Fresh(lambda: fx.with_gang(env.fx.n_1cpu_4gi("A", fx.PriorityClass0, 32)))
    env.ids["gangFailure"] = gt._Fresh(lambda: fx.with_gang(env.fx.n_1cpu_4gi("A", fx.PriorityClass0, 33)))
    try:
        tc = env.ev(SCHED_MANY[name])
    except gt.UnsupportedCase as e:
        pytest.skip(f"not modelled: {e}")
    groups = tc["Jobs"]
    b, db = _nodedb_for(tc["Nodes"], groups, env)
    want = [bool(x) for x in tc["ExpectSuccess"]]
    got = []
    for g in groups:
        ok, node, _, _, _ = db.schedule_many([b.job_pos[j.id] for j in g])
        got.append(ok)
        if ok:
            assert (node != abi.NONE).all()
    assert got == want


import order_cases  # noqa: E402


@pytest.mark.parametrize("name", sorted(order_cases.CASES))
def test_job_priority_comparer(name):
    """TestJobPriorityComparer (jobdb/comparison_test.go:13-75) through the round's attempt order."""
    b, expected = order_cases.comparison_round(name)
    order_cases.check_order(b, expected, oracle_lib.round_schedule(b.input))


@pytest.mark.parametrize("name,pc_fraction,queue_fraction,want", [
    # constraints_test.go:53-63, :96-111, :131-140, :141-150 — pool total 1000 cpu / 1000Gi
    ("within-constraints", {"cpu": 0.9, "memory": 0.9}, {"cpu": 0.9, "memory": 0.9}, ("900", "900Gi")),
    ("exceeds-queue-priority-class-constraint", {}, {"cpu": 0.000001, "memory": 0.9}, ("1m", "900Gi")),
    ("exceeds-priority-class-constraint", {"cpu": 0.00000001, "memory": 0.9}, None, ("10n", "900Gi")),
    ("priority-class-constraint-ignored-if-there-is-a-queue-constraint", {"cpu": 0.00000001, "memory": 0.9}, {"cpu": 0.9, "memory": 0.9}, ("900", "900Gi")),
    ("no-constraints", {}, None, None),
])
def test_per_queue_limits(name, pc_fraction, queue_fraction, want):
    """TestConstraints' GetQueueResourceLimit expectations (constraints_test.go:32-178): calculatePerQueueLimits
    (constraints.go:231-256) as flattened by RoundInputBuilder into queue_limit[Q][PC][D]."""
    cfg = SchedulingConfig(supported_resource_types=[ResourceType("cpu", "1m"), ResourceType("memory", "1")],
                           indexed_resources=[ResourceType("cpu", "1"), ResourceType("memory", "1")],
                           priority_classes={"priority-class-1": PriorityClass(0, True, (), dict(pc_fraction))}, drf_resources=["cpu", "memory"])
    q = QueueSpec("queue-1", 1.0, resource_limits_by_pc={"priority-class-1": queue_fraction} if queue_fraction is not None else {})
    f = cfg.factory()
    total = f.from_node({"cpu": "1000", "memory": "1000Gi"})
    b = RoundInputBuilder(cfg, [], [], [q], total_resources=total)
    got = b.queue_limit[0, 0]
    if want is None:  # rlFactory.MakeAllMax()
        assert (got == 2**63 - 1).all()
    else:
        assert list(got) == list(f.from_node({"cpu": want[0], "memory": want[1]}))


@pytest.mark.parametrize("seed", range(6))
def test_node_preemptibility_stats_agree_with_the_round(seed):
    """NodePreemptiblityStats (eviction.go:38-49,197-273) derived on the host: the job filter it restates selects exactly
    the jobs the round evicted (running jobs that end RESCHEDULED or PREEMPTED when no oversubscribed eviction followed),
    and the per-node summary follows the reference's rules."""
    from armada_b200.model import evictable_jobs, node_preemptibility_stats
    import gang_cases
    b = gang_cases.uniformity_round(seed, floating=False, n_jobs=200)
    res = oracle_lib.round_schedule(b.input)
    ev = evictable_jobs(b, res)
    running = b.job_node[: len(b.jobs)] != abi.NONE
    if int(res.stats.evicted_pass2) == 0:
        touched = np.isin(res.job_state[: len(b.jobs)], (abi.JOB_RESCHEDULED, abi.JOB_PREEMPTED)) & running
        assert (touched == ev).all()
    assert int(ev.sum()) == int(res.stats.evicted_pass1)
    stats = node_preemptibility_stats(b, res)
    assert [s[0] for s in stats] == sorted(n.id for n in b.nodes)
    by_node = {}
    for j, n in enumerate(b.job_node[: len(b.jobs)]):
        if n != abi.NONE:
            by_node.setdefault(b.nodes[int(n)].id, []).append(j)
    for nid, preemptible, reason in stats:
        jobs = by_node.get(nid, [])
        if not jobs:
            assert reason == "node_empty" and preemptible
        elif preemptible:
            assert reason == "all_jobs_preemptible" and all(ev[j] for j in jobs)
        else:
            assert not all(ev[j] for j in jobs) and set(reason.split(",")) <= {"job_not_preemptible", "below_protected_fair_share", "invalid_queue"}


@pytest.mark.parametrize("seed", range(6))
def test_queue_stats_from_the_first_pass_view(seed):
    """QueueStats (queue_scheduler.go:190-235, result.go:15-28) derived from job_seq_first_pass / job_reason_first_pass:
    counts and positions are consistent with the round's outcome, and the replayed queue allocation at a queue's last
    scheduled gang ends where the round's own accounting ends when nothing happened after the first pass."""
    from armada_b200.model import queue_stats
    import gang_cases
    b = gang_cases.uniformity_round(seed, floating=False, n_jobs=220)
    res = oracle_lib.round_schedule(b.input)
    stats = queue_stats(b, res)
    J = len(b.jobs)
    seq = res.job_seq_first_pass[:J]
    assert seq.max() <= int(res.stats.loop_iterations) and (seq > 0).sum() > 0
    positions = set()
    for qi, q in enumerate(b.queues):
        mine = (b.job_queue[:J] == qi) & (seq > 0)
        if not mine.any():
            assert q.name not in stats
            continue
        st = stats[q.name]
        assert st.jobs_considered == int(mine.sum()) and st.gangs_considered == len(set(seq[mine].tolist()))
        assert st.gangs_scheduled <= st.gangs_considered
        assert st.first_gang_considered_queue_position == int(seq[mine].min()) - 1
        assert st.first_gang_considered_result == "scheduled" or st.first_gang_considered_result in gt_reason_texts()
        positions.add(st.first_gang_considered_queue_position)
        if int(res.stats.evicted_pass2) == 0 and st.gangs_scheduled:
            # nothing moved after the first pass: the replay's last allocation (incl. the short-job penalty, zero here)
            # is the queue's final allocation
            assert (st.last_gang_scheduled_queue_resources == res.queue_allocated[qi] + b.queue_short_job_penalty[qi]).all()
    assert 0 in positions  # some queue was looked at in the very first iteration


def gt_reason_texts():
    from armada_b200.model import REASON_TEXT
    return set(REASON_TEXT.values())


PQ_ORDER = {
    # queue_scheduler_test.go:699-834 — items {queue: (proposedQueueCost, currentQueueCost, queueBudget, itemSize)}, expected sort.Sort order
    "BelowFairShare_EvenCurrentCost": ({"A": (2, 0, 5, 2), "B": (3, 0, 5, 3), "C": (1, 0, 5, 1)}, ["B", "A", "C"]),
    "BelowFairShare_UnevenCurrentCost": ({"A": (4, 2, 5, 2), "B": (3, 2, 5, 1), "C": (2, 1, 5, 1)}, ["C", "A", "B"]),
    "AboveFairShare": ({"A": (8, 6, 5, 2), "B": (7, 4, 5, 3), "C": (9, 8, 5, 1)}, ["B", "A", "C"]),
    "MixedFairShare": ({"A": (8, 6, 5, 2), "B": (3, 2, 5, 1)}, ["B", "A"]),
    "Fallback": ({"B": (0, 0, 0, 0), "C": (0, 0, 0, 0), "A": (0, 0, 0, 0)}, ["A", "B", "C"]),
}


@pytest.mark.parametrize("name", sorted(PQ_ORDER))
def test_queue_candidate_gang_iterator_pq_ordering(name):
    """TestQueueCandidateGangIteratorPQ_Ordering_* / _Fallback: the oracle's Less, sorted like sort.Sort."""
    import functools
    lib = oracle_lib.load()
    lib.armada_oracle_pq_less.argtypes = [C.c_int32, C.c_int32, abi.f64p, abi.f64p]
    lib.armada_oracle_pq_less.restype = C.c_int32
    items, want = PQ_ORDER[name]
    rank = {q: i for i, q in enumerate(sorted(items))}

    def vec(q):
        return np.array(list(items[q]) + [rank[q], 0], np.float64)

    def cmp(a, b):
        if lib.armada_oracle_pq_less(1, 0, vec(a).ctypes.data_as(abi.f64p), vec(b).ctypes.data_as(abi.f64p)):
            return -1
        if lib.armada_oracle_pq_less(1, 0, vec(b).ctypes.data_as(abi.f64p), vec(a).ctypes.data_as(abi.f64p)):
            return 1
        return 0

    assert sorted(items, key=functools.cmp_to_key(cmp)) == want
