"""armada_nodedb_add_classes: a dry-run NodeDb that received job classes through appends answers exactly
like one created with all of them, and an append the library refuses leaves the db as it was.  The bodies
are shared by the emulator and the GPU suites (`lib` None = the product library)."""
from __future__ import annotations

import random

import numpy as np
import pytest

import explain_cases as ec
import fixtures as fx
from armada_b200 import abi
from armada_b200.model import NODE_ID_LABEL, MatchExpression, QueueSpec, RoundInputBuilder, UnresolvedLabels
from armada_b200.scheduler import DeviceNodeDb


def _cluster(seed, n_nodes=40, n_jobs=(4, 12, 12)):
    """Seeded nodes (unaligned allocatable ⇒ exact mode, away node types, several node types and static
    classes) and three batches of jobs K0, K1, K2."""
    rng = random.Random(seed)
    f = fx.Fixtures()
    cfg = fx.test_scheduling_config()
    pcs = [fx.PriorityClass1, fx.PriorityClass4PreemptibleAway, fx.PriorityClass6Preemptible, fx.PriorityClass7PreemptibleAwayConditional]
    nodes = [ec._node(rng, i, seed % 2 == 1) for i in range(n_nodes)]
    batches = [[ec._job(rng, f, pcs) for _ in range(n)] for n in n_jobs]
    # K0 looks at every label K1 and K2 may look at, so that the static classes made with K0 resolve their rows
    batches[0] += [f.job("A", fx.PriorityClass1, {"cpu": "1", "memory": "1Gi"}, node_selector={"zone": "a"}),
                   f.job("A", fx.PriorityClass1, {"cpu": "1", "memory": "1Gi"}, node_selector={fx.ClusterNameLabel: "c1"})]
    return rng, cfg, nodes, batches


def _groups(rng, n0, n, count=40):
    """Gangs (lists of job indices) of 1-4 members; the multi-member ones mix K0 with K1 / K2 jobs."""
    out = [[i] for i in range(n)]
    for _ in range(count):
        size = rng.choice([2, 3, 4])
        out.append([rng.randrange(n0)] + rng.sample(range(n0, n), size - 1))
    return out


def append(b: RoundInputBuilder, db: DeviceNodeDb, jobs):
    """add_jobs on the builder, the classes and rows it added onto the db; returns the jobs' classes."""
    cls, new_classes, new_rows = b.add_jobs(jobs)
    c0, r0 = new_classes.start, new_rows.start
    first = db.add_classes(b.class_request[c0:], b.class_pc[c0:], b.class_static_row[c0:], b.class_away_row[c0:], b.static_match[r0:], b.type_match[r0:])
    assert first == c0
    return cls


def explain_tuples(res):
    return [(ok, node.tolist(), placed, away, ec.records_tuples(recs)) for ok, node, placed, away, recs in res]


def check_append_parity(seed, lib, chunk):
    """db A made with K0 and given K1 then K2 in appends of `chunk` jobs (None: one per batch) against db B made
    with K0 ∪ K1 ∪ K2, and B against the oracle's dry-run NodeDb.  Returns A's class count at creation and
    after each append."""
    rng, cfg, nodes, (k0, k1, k2) = _cluster(seed)
    jobs = k0 + k1 + k2
    b_all = RoundInputBuilder(cfg, nodes, jobs, [QueueSpec("A", 1.0)])
    b_app = RoundInputBuilder(cfg, nodes, k0, [QueueSpec("A", 1.0)])
    groups = _groups(rng, len(k0), len(jobs))
    db_b = DeviceNodeDb(b_all.input, lib=lib)
    db_a = DeviceNodeDb(b_app.input, lib=lib)
    try:
        classes = list(b_app.job_class[: len(k0)])
        sizes = [b_app.input.num_classes]
        for batch in (k1, k2):
            step = chunk or len(batch)
            for lo in range(0, len(batch), step):
                classes += list(append(b_app, db_a, batch[lo:lo + step]))
                sizes.append(b_app.input.num_classes)
        # the same class ids in the same order, the same rows and bitmaps
        assert classes == list(b_all.job_class)
        for name in ("class_request", "class_pc", "class_static_row", "class_away_row", "static_match", "type_match"):
            assert np.array_equal(getattr(b_app, name), getattr(b_all, name)), name
        assert b_app.row_specs == b_all.row_specs
        gangs = [[int(b_all.job_class[j]) for j in g] for g in groups]
        got_a, got_b = db_a.explain(gangs), db_b.explain(gangs)
        assert explain_tuples(got_a) == explain_tuples(got_b)
        ok_a, nodes_a = db_a.schedule_many(gangs)
        ok_b, nodes_b = db_b.schedule_many(gangs)
        assert (ok_a == ok_b).all() and all((x == y).all() for x, y in zip(nodes_a, nodes_b))
        every = list(range(b_all.input.num_classes))
        assert (db_a.select_nodes(every) == db_b.select_nodes(every)).all()
    finally:
        db_a.close()
        db_b.close()
    case = ec.case_from(cfg, nodes, jobs, groups)
    case.b = b_all
    case.classes = [[int(b_all.job_class[j]) for j in g] for g in groups]
    got, _ = ec.check_case(case, lib, round_kinds=False)
    assert explain_tuples(got) == explain_tuples(got_a)
    return sizes


def check_failed_append_changes_nothing(lib):
    rng, cfg, nodes, (k0, k1, _) = _cluster(5)
    b = RoundInputBuilder(cfg, nodes, k0, [QueueSpec("A", 1.0)])
    gangs = [[int(c)] for c in b.job_class] + [list(map(int, b.job_class[:3]))]
    db = DeviceNodeDb(b.input, lib=lib)
    try:
        before = explain_tuples(db.explain(gangs))
        C, rows, D = b.input.num_classes, b.input.num_static_rows, b.factory.D
        sw, tw = b.static_match.shape[1], b.type_match.shape[1]
        req = np.ones((1, D), np.int64)
        away = np.full((1, abi.MAX_AWAY), abi.NONE, np.uint32)
        no_rows = np.zeros((0, sw), np.uint32), np.zeros((0, tw), np.uint32)
        attempts = {
            "row out of range": (req, [0], [rows + 1], away, np.zeros((1, sw), np.uint32), np.zeros((1, tw), np.uint32)),
            "away row out of range": (req, [0], [0], np.full((1, abi.MAX_AWAY), rows, np.uint32)) + no_rows,
            "static_match without type_match": (req, [0], [rows], away, np.full((1, sw), 0xFFFFFFFF, np.uint32), np.zeros((1, tw), np.uint32)),
            "negative request": (-req, [0], [0], away) + no_rows,
            "bad class_pc": (req, [b.input.num_priority_classes], [0], away) + no_rows,
        }
        for what, args in attempts.items():
            with pytest.raises(abi.ArmadaError) as e:
                db.add_classes(*args)
            assert e.value.status == abi.E_INVALID, what
            assert explain_tuples(db.explain(gangs)) == before, what
            with pytest.raises(abi.ArmadaError):  # the class count did not move: class C is still unknown
                db.select_nodes([C])
        assert append(b, db, k1)[0] >= C  # a valid append still takes the next ids
        assert explain_tuples(db.explain(gangs)) == before
    finally:
        db.close()


def check_unresolved_label_changes_nothing(lib):
    """A key whose row looks at a node label the static classes do not tell apart is refused by add_jobs, the
    builder unchanged, and a db made with that key answers like the oracle."""
    rng, cfg, nodes, (k0, k1, _) = _cluster(7)
    k0, k1 = ([j for j in k if not j.node_selector and j.affinity is None] for k in (k0, k1))  # rows that look at no label
    b = RoundInputBuilder(cfg, nodes, k0, [QueueSpec("A", 1.0)])
    arrays = {name: getattr(b, name).copy() for name in ("class_request", "class_pc", "class_static_row", "class_away_row", "static_match", "type_match")}
    counts = (b.input.num_classes, b.input.num_static_rows, len(b.row_specs), len(b.class_jobs))
    f = fx.Fixtures()
    for new in (f.job("A", fx.PriorityClass1, {"cpu": "1", "memory": "1Gi"}, node_selector={"zone": "b"}),
                f.job("A", fx.PriorityClass1, {"cpu": "1", "memory": "1Gi"}, affinity=((MatchExpression(fx.ClusterNameLabel, "In", ("c2",)),),)),
                f.job("A", fx.PriorityClass1, {"cpu": "1", "memory": "1Gi"}, node_selector={NODE_ID_LABEL: nodes[3].id})):
        with pytest.raises(UnresolvedLabels):
            b.add_jobs(k1[:3] + [new])
        assert (b.input.num_classes, b.input.num_static_rows, len(b.row_specs), len(b.class_jobs)) == counts
        for name, a in arrays.items():
            assert np.array_equal(getattr(b, name), a), name
        jobs = b.class_jobs + [new]
        case = ec.case_from(cfg, nodes, jobs, [[len(jobs) - 1]])
        ec.check_case(case, lib, round_kinds=False)
    assert b.add_jobs(k1[:3])[1].start == counts[0]  # keys that need no finer classes still go in
