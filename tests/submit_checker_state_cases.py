"""SubmitChecker across checks: NodeDbs kept alive between checks, the result cache and the time budgets.
The bodies are shared by the emulator and the GPU suites (`lib` None = the product library)."""
from __future__ import annotations

import copy
import random

import pytest

import explain_cases as ec
import fixtures as fx
import submit_checker_cases as sc
from armada_b200 import abi, submitcheck
from armada_b200.model import NODE_ID_LABEL, QueueSpec
from armada_b200.submitcheck import Executor, PoolConfig, SubmitCheckConfig, SubmitChecker


class SteppingClock:
    """testfixtures.NewSteppingClock (testfixtures.go:1193-1217): every now() returns the time and then advances
    it by `step`; since() reads it without advancing."""

    def __init__(self, step: float, start: float = 0.0):
        self.t, self.step = start, step

    def now(self) -> float:
        t = self.t
        self.t += self.step
        return t

    def since(self, t: float) -> float:
        return self.t - t


# submitcheck_test.go:294-321, 352-364: batchJobs = N1Cpu4GiJobs("queue", PriorityClass1, 20) (:46)
_BATCH = [{"id": f"batchJob{i}", "kind": "small"} for i in range(20)]
_GANG = [{"id": f"largeGangJob[{i}]", "kind": "small", "gang": "largeGangJob"} for i in range(4)]
TIME_LIMIT_CASES = {
    "Per-queue time limit stops checking jobs": dict(
        jobs=_BATCH, config=SubmitCheckConfig(max_duration_per_queue=5.0), step=1.0,
        expected={f"batchJob{i}": (True, ["cpu"]) for i in range(3)}),
    "Global time limit stops checking jobs": dict(
        jobs=_BATCH, config=SubmitCheckConfig(max_duration=8.0), step=1.0,
        expected={f"batchJob{i}": (True, ["cpu"]) for i in range(3)}),
    "Partial gang deferred when time limit splits members": dict(
        jobs=[{"id": "smallJob1", "kind": "small"}, {"id": "smallJob2", "kind": "small"}] + _GANG,
        config=SubmitCheckConfig(max_duration_per_queue=3.0), step=1.0,
        expected={"smallJob1": (True, ["cpu"]), "smallJob2": (True, ["cpu"])}),
}


def replay_time_limit(name, lib=None):
    """One of the stepping-clock cases of TestSubmitChecker on one small cpu node (Executor(SmallNode("cpu")))."""
    spec = TIME_LIMIT_CASES[name]
    case = {"executors": [[["small", "cpu"]]], "jobs": spec["jobs"], "queue": None}
    checker, jobs = sc.build(case, lib)
    with checker:
        checker.submit_check, checker.clock = spec["config"], SteppingClock(spec["step"])
        got, durations = checker.check_with_durations(jobs)
    assert {k: (r.is_schedulable, sorted(r.pools)) for k, r in got.items()} == spec["expected"]
    assert list(durations) == ["queue"]
    return got


# -- seeded sequences of checks ------------------------------------------------------------------------
def _executors(rng, n_exec=2, n_nodes=12):
    pools = ["cpu", "gpu"]
    out = []
    for e in range(n_exec):
        ex = Executor(f"executor-{e}")
        for i in range(n_nodes):
            ex.nodes.append((rng.choice(pools), ec._node(rng, e * 1000 + i, False)))
        out.append(ex)
    return out


def _jobs(rng, f, n, tag, queues=("A", "B")):
    pcs = [fx.PriorityClass1, fx.PriorityClass4PreemptibleAway, fx.PriorityClass6Preemptible]
    jobs = [ec._job(rng, f, pcs) for _ in range(n)]
    for j in jobs:
        j.queue = rng.choice(queues)
    for g in range(n // 6):  # a few gangs of 2-3 jobs of one queue
        members = [j for j in jobs if j.gang_id is None][: rng.choice([2, 3])]
        for m in members:
            m.queue = members[0].queue
        fx.with_gang(members, f"{tag}-gang-{g}")
    for i, j in enumerate(jobs):
        j.id = f"{tag}-{i}"
    return jobs


def _pools():
    return [PoolConfig("cpu"), PoolConfig("gpu"), PoolConfig("cpu-away", ("gpu",)), PoolConfig("cpu-no-home", disable_home_scheduling=True)]


class CountingNodeDb(submitcheck.DeviceNodeDb):
    """DeviceNodeDb that counts its creations and records the gangs of each of its explain launches."""
    created = 0

    def __init__(self, *a, **kw):
        type(self).created += 1
        self.launches = []
        super().__init__(*a, **kw)

    def explain(self, gangs, *a, **kw):
        self.launches.append([list(g) for g in gangs])
        return super().explain(gangs, *a, **kw)


def _single(j, jid):
    c = copy.copy(j)
    c.id, c.gang_id, c.gang_cardinality = jid, None, 1
    return c


def _rebuilds(live, jobs):
    """The dbs a check of `jobs` has to rebuild: those whose static classes do not tell apart a node label some
    job's selector or affinity looks at."""
    def keys(j):
        return {k for k in j.node_selector} | {e.key for term in (j.affinity or ()) for e in term}
    return sum(1 for b, _ in live.dbs.values() if any(k in b.node_label_keys and k not in b.static_label_keys for j in jobs for k in keys(j)))


def _same(got, want):
    assert set(got) == set(want)
    for jid in want:
        assert (got[jid].is_schedulable, got[jid].pools, got[jid].reason) == (want[jid].is_schedulable, want[jid].pools, want[jid].reason), jid


def check_state_sequence(seed, lib, monkeypatch, n_checks=7):
    """A sequence of checks with overlapping and new scheduling keys, across one update_executors, against a
    fresh SubmitChecker per check (the result a checker without state gives); a check creates dbs only to
    rebuild those whose static classes do not tell apart a label its keys look at, and a key already in the
    cache launches nothing for its individual check."""
    rng = random.Random(seed)
    f = fx.Fixtures()
    cfg = fx.test_scheduling_config()
    queues = [QueueSpec("A"), QueueSpec("B")]
    executors = _executors(rng)
    monkeypatch.setattr(submitcheck, "DeviceNodeDb", CountingNodeDb)
    earlier = _jobs(rng, f, 30, "first")  # the jobs later checks repeat keys of
    cache_hits = 0
    with SubmitChecker(cfg, _pools(), executors, queues, lib=lib) as live:
        for k in range(n_checks):
            if k == n_checks // 2:
                executors = _executors(rng)
                created = CountingNodeDb.created
                live.update_executors(executors)
                assert CountingNodeDb.created == created + len(live.dbs) and len(live.cache) == 0
            jobs = (earlier if k == 0 else _jobs(rng, f, rng.randrange(6, 14), f"c{k}"))
            jobs = jobs + [_single(rng.choice(earlier), f"c{k}-again-{i}") for i in range(4)]
            cached = set(live.cache)
            launched = {key: len(db.launches) for key, (_, db) in live.dbs.items()}
            created, rebuilds = CountingNodeDb.created, _rebuilds(live, jobs)
            got = live.check(jobs)
            assert CountingNodeDb.created == created + rebuilds
            for key, (b, db) in live.dbs.items():
                singles = {g[0] for L in db.launches[launched[key]:] for g in L if len(g) == 1}
                for j in jobs:
                    sk = submitcheck.scheduling_key(j, live.factory.from_job(j.requests))
                    if sk in cached and j.gang_id is None:
                        cache_hits += 1
                        assert b._classes[sk] not in singles, (k, j.id)
            with SubmitChecker(cfg, _pools(), executors, queues, lib=lib) as fresh:
                want = fresh.check(jobs)
            assert set(want) == {j.id for j in jobs}
            _same(got, want)
    assert cache_hits > 0


def check_pinned_job_then_more_checks(lib, monkeypatch):
    """A job pinned to one node (a selector on the node-id label, which the static classes tell apart only
    once a key looks at it), then checks of other jobs: every result as a fresh checker's, the dbs rebuilt
    once, by the check that brings the label."""
    f = fx.Fixtures()
    cfg = fx.test_scheduling_config()
    nodes = [f.cpu32() for _ in range(4)]
    executors = [Executor("executor-0", [("cpu", n) for n in nodes])]
    queues = [QueueSpec("queue")]

    def job(jid, **kw):
        j = f.job("queue", fx.PriorityClass1, {"cpu": "1", "memory": "4Gi"}, **kw)
        j.id = jid
        return j

    checks = [[job("pinned0", node_selector={NODE_ID_LABEL: nodes[0].id})],
              [job("plain0"), job("plain1", node_selector={fx.ClusterNameLabel: "nowhere"})],
              [job("pinned1", node_selector={NODE_ID_LABEL: nodes[1].id}), job("plain2"), job("gone", node_selector={NODE_ID_LABEL: "no-such-node"})]]
    monkeypatch.setattr(submitcheck, "DeviceNodeDb", CountingNodeDb)
    with SubmitChecker(cfg, _pools(), executors, queues, lib=lib) as live:
        for k, jobs in enumerate(checks):
            created, rebuilds = CountingNodeDb.created, _rebuilds(live, jobs)
            got = live.check(jobs)
            assert CountingNodeDb.created == created + rebuilds and rebuilds == (len(live.dbs) if k == 0 else 0), k
            with SubmitChecker(cfg, _pools(), executors, queues, lib=lib) as fresh:
                _same(got, fresh.check(jobs))
            assert got[jobs[0].id].is_schedulable
        assert not got["gone"].is_schedulable


def check_refused_append_rolls_back(lib, monkeypatch):
    """A db that refuses an append (here a stand-in for a failed device allocation) fails that check and leaves
    builder and db as they were: the next checks answer as a fresh checker does."""
    f = fx.Fixtures()
    cfg = fx.test_scheduling_config()
    executors = [Executor("executor-0", [("cpu", f.cpu32()) for _ in range(3)]), Executor("executor-1", [("gpu", f.cpu32())])]
    queues = [QueueSpec("queue")]

    def job(jid, cpu):
        j = f.job("queue", fx.PriorityClass1, {"cpu": cpu, "memory": "4Gi"})
        j.id = jid
        return j

    with SubmitChecker(cfg, _pools(), executors, queues, lib=lib) as live:
        b, db = live.dbs[sorted(live.dbs)[-1]]
        before = (b.input.num_classes, b.input.num_static_rows)

        def refuse(*a, **kw):
            raise abi.ArmadaError(abi.E_CUDA, "device allocation failed")
        monkeypatch.setattr(db, "add_classes", refuse)
        with pytest.raises(abi.ArmadaError):
            live.check([job("a", "1")])
        assert (b.input.num_classes, b.input.num_static_rows) == before
        monkeypatch.undo()
        for jobs in ([job("a", "1"), job("b", "40")], [job("c", "1"), job("d", "2")]):
            got = live.check(jobs)
            with SubmitChecker(cfg, _pools(), executors, queues, lib=lib) as fresh:
                _same(got, fresh.check(jobs))
