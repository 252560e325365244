"""Seeded dry-run clusters for armada_nodedb_explain and the reference it is checked against.

The reference for every output is the CPU oracle's NodeDb: `dry_run` for ok / member_node,
`schedule_many` (which commits nothing when the gang fails) for the members placed before the failure,
and `iterate` — the literal NodeTypesIterator — for the nodes the last probe of a failed single job
reaches.  Each reached node is then classified the way JobRequirementsMet words it
(nodematching.go:147-190)."""
from __future__ import annotations

import random

import numpy as np

import fixtures as fx
import oracle_lib
from armada_b200 import abi
from armada_b200.model import (MatchExpression, NodeSpec, QueueSpec, RoundInputBuilder, Taint, Toleration, excluded_nodes_by_reason,
                               last_probe_row)
from armada_b200.scheduler import DeviceNodeDb

GPU = Taint("gpu", "true", "NoSchedule")
LARGE = Taint("largeJobsOnly", "true", "NoSchedule")
SPOT = Taint("spot", "yes", "NoExecute")  # not indexed: the node type ignores it, the static class does not


def _node(rng, i, allocatable_extra, kinds=6):
    kind = rng.randrange(kinds)
    cpu = rng.choice([4, 8, 16, 32, 64])
    mem = rng.choice([16, 64, 128, 256])
    res = {"cpu": str(cpu), "memory": f"{mem}Gi"}
    taints, labels = [], {fx.ClusterNameLabel: rng.choice(["c1", "c2"])}
    if kind == 1:
        res["nvidia.com/gpu"] = str(rng.choice([1, 4, 8]))
        taints.append(GPU)
        labels["gpu"] = "true"
    elif kind == 2:
        taints.append(LARGE)
        labels["largeJobsOnly"] = "true"
    elif kind == 3:
        taints.append(SPOT)
    elif kind == 4:
        labels["zone"] = rng.choice(["a", "b"])
    alloc = None
    if rng.random() < 0.5:  # allocatable below total, in unaligned steps
        alloc = {"cpu": f"{cpu * 1000 - rng.choice([0, 150, 500, 999])}m", "memory": f"{mem * 1024 - rng.choice([0, 3, 700])}Mi"}
        if "nvidia.com/gpu" in res:  # a gpu held back: only a walk that does not index gpus rejects on it
            alloc["nvidia.com/gpu"] = str(int(res["nvidia.com/gpu"]) - rng.choice([0, 1]))
        if allocatable_extra and rng.random() < 0.3:  # allocatable above total: only the total check rejects
            alloc["cpu"] = str(cpu + 8)
    return NodeSpec(id=f"node-{rng.randrange(10**6):06d}-{i}", index=i, total=res, taints=tuple(taints), labels=labels,
                    allocatable=alloc)


def _job(rng, f, pcs, indexed_only=False):
    pc = rng.choice(pcs)
    req = {"cpu": rng.choice(["1", "3500m", "8", "17", "40", "70"]), "memory": rng.choice(["1Gi", "100Gi", "129Gi", "300Gi"])}
    if rng.random() < 0.25:
        req["nvidia.com/gpu"] = rng.choice(["1", "2", "9"])
    tol = []
    if rng.random() < 0.3:
        tol.append(Toleration("gpu", "", "true"))
    if rng.random() < 0.2:
        tol.append(Toleration("largeJobsOnly", "", "true"))
    if rng.random() < 0.15:
        tol.append(Toleration("spot", "Exists"))
    kw = {}
    if rng.random() < 0.2 and not indexed_only:
        kw["node_selector"] = {"zone": rng.choice(["a", "b", "c"])}
    if rng.random() < 0.1:
        kw["node_selector"] = {fx.ClusterNameLabel: "c2"}
    if rng.random() < 0.15 and not indexed_only:
        kw["affinity"] = ((MatchExpression(fx.ClusterNameLabel, rng.choice(["In", "NotIn"]), ("c1",)),),)
    return f.job("A", pc, req, tol, **kw)


class Case:
    """One seeded cluster and a batch of gangs (lists of job indices into `b`)."""

    def __init__(self, seed, n_nodes=40, n_gangs=40, cfg_over=None, allocatable_extra=False, gang_sizes=(1, 1, 1, 2, 3, 5), indexed_only=False):
        # indexed_only: only taints and labels the node types index, so that a failed walk reaches few nodes
        # (every node a walk reaches costs one block-wide pass over the cluster)
        rng = random.Random(seed)
        f = fx.Fixtures()
        cfg = fx.test_scheduling_config(**(cfg_over or {}))
        pcs = [fx.PriorityClass1, fx.PriorityClass4PreemptibleAway, fx.PriorityClass6Preemptible, fx.PriorityClass7PreemptibleAwayConditional]
        nodes = [_node(rng, i, allocatable_extra, 3 if indexed_only else 6) for i in range(n_nodes)]
        jobs, groups = [], []
        for g in range(n_gangs):
            size = rng.choice(gang_sizes)
            members = [_job(rng, f, pcs, indexed_only) for _ in range(size)]
            if size > 1:
                for m in members[1:]:  # gang members share the first one's class half of the time
                    if rng.random() < 0.5:
                        m.requests, m.tolerations, m.priority_class = dict(members[0].requests), members[0].tolerations, members[0].priority_class
                        m.node_selector, m.affinity = dict(members[0].node_selector), members[0].affinity
                members = fx.with_gang(members, f"gang-{g}")
            groups.append(list(range(len(jobs), len(jobs) + size)))
            jobs += members
        self.cfg, self.nodes, self.jobs, self.groups = cfg, nodes, jobs, groups
        self.b = RoundInputBuilder(cfg, nodes, jobs, [QueueSpec("A", 1.0)])
        self.classes = [[int(self.b.job_class[j]) for j in g] for g in groups]


def case_from(cfg, nodes, jobs, groups):
    case = Case.__new__(Case)
    case.cfg, case.nodes, case.jobs, case.groups = cfg, nodes, jobs, groups
    case.b = RoundInputBuilder(cfg, nodes, jobs, [QueueSpec("A", 1.0)])
    case.classes = [[int(case.b.job_class[j]) for j in g] for g in groups]
    return case


def held_back_gpus_case():
    """gpus not indexed and held back from allocatable: the walk reaches every gpu node and rejects it
    on its allocatable (ARMADA_EXCL_RESOURCES), or on its total when that is short too."""
    f = fx.Fixtures()
    cfg = fx.test_scheduling_config(indexed_resources=fx.test_resources()[:2])
    nodes = []
    for i in range(12):
        n = f.gpu8()
        n.allocatable = {"cpu": "64", "memory": "1024Gi", "nvidia.com/gpu": str(7 - i % 3)}
        if i % 4 == 0:
            n.total = dict(n.total, **{"nvidia.com/gpu": "6"})
        nodes.append(n)
    nodes += [f.cpu32() for _ in range(3)]
    jobs = [f.job("A", fx.PriorityClass1, {"cpu": "1", "memory": "1Gi", "nvidia.com/gpu": q}) for q in ("8", "7500m", "1")]
    return case_from(cfg, nodes, jobs, [[0], [1], [2]])


def reference(case):
    """Per gang (ok, member_node, num_placed, member 0 placed away, records as sorted (kind, sub, quantity,
    count) tuples)."""
    b = case.b
    inp = b.input
    N, D = inp.num_nodes, inp.num_resources
    odb = oracle_lib.OracleNodeDb(inp)
    nodes_of_type = np.bincount(b.node_type[:N], minlength=inp.num_node_types)
    sw, tw = (inp.num_static_classes + 31) // 32, (inp.num_node_types + 31) // 32
    scratch = oracle_lib.OracleNodeDb(inp)
    out = []
    for g in case.groups:
        ok, node = odb.dry_run(g)
        if ok:  # ScheduledAway of member 0: the gang once more on a scratch NodeDb, committed, then unbound
            _, _, _, _, method = scratch.schedule_many(g)
            for j in g:
                scratch.unbind(j)
            out.append((True, node, len(g), int(method[0]) == abi.METHOD_AWAY, []))
            continue
        _, partial, _, _, _ = odb.schedule_many(g)
        placed = 0
        while placed < len(g) and partial[placed] != abi.NONE:
            placed += 1
        recs = []
        if len(g) == 1:
            recs = _records(b, int(b.job_class[g[0]]), odb, N, D, nodes_of_type, sw, tw)
        out.append((False, node, placed, False, recs))
    odb.close()
    scratch.close()
    return out


def _records(b, cls, odb, N, D, nodes_of_type, sw, tw):
    inp = b.input
    req = b.class_request[cls]
    if any((inp.disallowed_resource_mask >> d) & 1 and req[d] > 0 for d in range(D)):
        return [(abi.EXCL_DISALLOWED, 0, 0, N)]
    row = last_probe_row(b, cls)
    recs = {}
    if row is not None:
        pc = inp.priority_classes[int(b.class_pc[cls])]
        sched_at = pc.priority
        for k in range(abi.MAX_AWAY):
            if int(b.class_away_row[cls, k]) == row and not b.cfg.disable_away_scheduling:
                sched_at = pc.away_priority[k]
        for t in range(inp.num_node_types):
            if not (int(b.type_match[row, t >> 5]) >> (t & 31)) & 1 and nodes_of_type[t]:
                recs[(abi.EXCL_NODE_TYPE, t, 0)] = int(nodes_of_type[t])
        ireq = [int(req[inp.indexed_resource[i]]) for i in range(inp.num_indexed)]
        for n in odb.iterate(row, sched_at, ireq):
            s = int(b.node_static_class[n])
            if not (int(b.static_match[row, s >> 5]) >> (s & 31)) & 1:
                key = (abi.EXCL_STATIC, s, 0)
            else:
                dt = [d for d in range(D) if req[d] > b.node_total[d, n]]
                da = [d for d in range(D) if req[d] > b.node_allocatable[d, n]]
                key = (abi.EXCL_STATIC_TOTAL, dt[0], int(b.node_total[dt[0], n])) if dt else (abi.EXCL_RESOURCES, da[0], int(b.node_allocatable[da[0], n]))
            recs[key] = recs.get(key, 0) + 1
    rest = N - sum(recs.values())
    if rest > 0:
        recs[(abi.EXCL_IMPLICIT, 0, 0)] = rest
    return sorted((k, s, q, c) for (k, s, q), c in recs.items())


def records_tuples(records):
    return [(int(r.kind), int(r.sub), int(r.quantity), int(r.count)) for r in records]


def kind_histogram(records):
    """The round's ARMADA_EXCL_* histogram of a record list (STATIC_TOTAL counts as RESOURCES)."""
    h = np.zeros(abi.EXCLUDED_KINDS, np.uint32)
    for k, _, _, c in records:
        h[abi.EXCL_RESOURCES if k == abi.EXCL_STATIC_TOTAL else k] += c
    return h


def round_kind_histogram(case, job):
    """The oracle round's job_excluded_nodes for `job` alone on the empty cluster."""
    b = RoundInputBuilder(case.cfg, case.nodes, [case.jobs[job]], [QueueSpec("A", 1.0)])
    b.input.collect_excluded_nodes = 1
    res = oracle_lib.round_schedule(b.input)
    return np.asarray(res.job_excluded_nodes)[0]


CONFIGS = {
    "home+away": {},
    "no-away": dict(disable_away_scheduling=True),
    "no-home": dict(disable_home_scheduling=True),
    "no-gang-away": dict(disable_gang_away_scheduling=True),
    "disallowed-gpu": dict(disallowed_resources=["nvidia.com/gpu"]),
    "gpu-not-indexed": dict(indexed_resources=fx.test_resources()[:2]),
}


def check_case(case, lib, capacity=1024, round_kinds=True):
    """explain on a db of `case` (the product library when `lib` is None) against reference(), schedule_many
    on the same db and, for failed single jobs, the oracle round's kind histogram."""
    want = reference(case)
    db = DeviceNodeDb(case.b.input, lib=lib)
    try:
        got = db.explain(case.classes, capacity=capacity)
        ok_sm, nodes_sm = db.schedule_many(case.classes)
    finally:
        db.close()
    N = case.b.input.num_nodes
    failed_single = 0
    for g, ((ok, node, placed, away, recs), (wok, wnode, wplaced, waway, wrecs)) in enumerate(zip(got, want)):
        assert ok == wok and ok == bool(ok_sm[g]), g
        assert away == waway, g
        assert (node == wnode).all() and (node == nodes_sm[g]).all(), g
        assert placed == wplaced, g
        assert records_tuples(recs) == wrecs, g
        if not ok and len(case.groups[g]) == 1:
            failed_single += 1
            assert sum(r.count for r in recs) == N
            hist = round_kind_histogram(case, case.groups[g][0]) if round_kinds else np.zeros(1)
            if hist.sum():  # the round attempted the job on the node db (no constraint stopped it first)
                assert (kind_histogram(wrecs) == hist).all(), g
            # every record renders to a reason string, and they still sum to N
            strings = excluded_nodes_by_reason(case.b, case.classes[g][0], recs)
            assert sum(strings.values()) == N
        else:
            assert recs == []
    return got, failed_single
