"""The TestSubmitChecker table (tests/golden/submit_checker.json) replayed through
armada_b200.submitcheck.SubmitChecker."""
import json
import os

import fixtures as fx
from armada_b200.model import JobSpec, NodeSpec, QueueSpec, Taint, Toleration
from armada_b200.submitcheck import Executor, PoolConfig, SubmitChecker

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "submit_checker.json")))
CASES = {c["name"]: c for c in GOLDEN["cases"]}


def build(case, lib=None):
    """(checker, jobs) of one case."""
    cfg = fx.test_scheduling_config()
    pools = [PoolConfig(p["name"], tuple(p.get("away_pools", ())), unscheduled_resources=tuple(p.get("unscheduled_resources", ())),
                        submission_group=p.get("submission_group", "")) for p in GOLDEN["pools"]]
    executors, k = [], 0
    for e, nodes in enumerate(case["executors"]):
        ex = Executor(f"executor-{e}")
        for kind, pool in nodes:
            spec = GOLDEN["node_kinds"][kind]
            node = NodeSpec(id=f"node-{k:04d}", index=k, total=dict(spec["total"]), taints=tuple(Taint(*t) for t in spec.get("taints", ())),
                            labels={fx.TestHostnameLabel: f"node-{k:04d}"})
            ex.nodes.append((pool, node))
            k += 1
        executors.append(ex)
    q = case["queue"] or {}
    queue = QueueSpec("queue", q.get("priority_factor", 1.0), resource_limits_by_pc=q.get("resource_limits_by_pc", {}))
    floating = {n: (res, by_pool) for n, (res, by_pool) in GOLDEN["floating"].items()}
    jobs = []
    for i, j in enumerate(case["jobs"]):
        spec = GOLDEN["job_kinds"][j["kind"]]
        req = dict(spec["requests"], **j.get("requests", {}))
        ncard = sum(1 for x in case["jobs"] if x.get("gang") and x.get("gang") == j.get("gang"))
        jobs.append(JobSpec(id=j["id"], queue="queue", priority_class=spec["pc"], requests=req, submit_time=i,
                            tolerations=tuple(Toleration(key, "", value) if op == "" else Toleration(key, op, value) for key, op, value in spec.get("tolerations", ())),
                            node_selector=dict(j.get("selector", {})), gang_id=j.get("gang"), gang_cardinality=max(ncard, 1)))
    return SubmitChecker(cfg, pools, executors, [queue], floating, lib=lib), jobs


def replay(name, lib=None):
    case = CASES[name]
    checker, jobs = build(case, lib)
    got = checker.check(jobs)
    assert len(got) == len(case["expected"])
    for jid, (ok, pools) in case["expected"].items():
        assert got[jid].is_schedulable == ok, (name, jid, got[jid])
        assert sorted(got[jid].pools) == pools, (name, jid, got[jid])
    return got
