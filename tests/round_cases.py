"""Bodies of the schedule-pass parity tests that run on both the emulator and the GPU, each output array compared
bit for bit with the CPU oracle.  A body takes what differs between the tiers as arguments:
  schedule(inp)       runs one round on the tier's shared handle and returns its RoundResult
  make_round()        a fresh DeviceRound, for tests that need a handle of their own
  make_nodedb(inp)    a dry-run DeviceNodeDb on the tier's library
and the sizes and seeds of the tier."""
from __future__ import annotations

import numpy as np
import pytest

import gang_cases
import go_tables as gt
import oracle_lib
import order_cases
from armada_b200 import abi, synth

PQS = gt.load_cases("preempting_queue_scheduler")
QS = gt.load_cases("queue_scheduler")


def assert_parity(schedule, inp, label=""):
    want = oracle_lib.round_schedule(inp)
    got = schedule(inp)
    bad = got.diff(want)
    assert not bad, f"{label}: device != oracle:\n  " + "\n  ".join(bad)
    return got, want


def round_or_skip(schedule, inp):
    """assert_parity for the reference tables: an input the device refuses as unsupported skips the case."""
    try:
        got = schedule(inp)
    except abi.ArmadaError as e:
        if e.status == abi.E_UNSUPPORTED:
            raise gt.UnsupportedCase(str(e))
        raise
    bad = got.diff(oracle_lib.round_schedule(inp))
    assert not bad, "device != oracle:\n  " + "\n  ".join(bad)
    return got


def reference_table(schedule, run_case, case):
    """One scenario of the reference's TestPreemptingQueueScheduler or TestQueueScheduler table (`run_case` is
    go_tables.run_pqs_case or run_queue_scheduler_case), driven through the device."""
    try:
        run_case(case, lambda inp: round_or_skip(schedule, inp))
    except gt.UnsupportedCase as e:
        pytest.skip(f"outside device domain / not modelled: {e}")


def _seeded_round(seed, unaligned=False):
    """The seed picks the size and which of away node types, round / queue limits, protection and lookback the round has."""
    return synth.random_round(seed, away=(seed % 4 == 1), round_limit=(seed % 6 == 3), queue_limits=(seed % 6 == 4),
                              protected_fraction=0.5 if seed % 3 == 2 else 0.0, lookback=40 if seed % 5 == 1 else 0,
                              n_nodes=40 + 13 * (seed % 7), n_jobs=300 + 50 * (seed % 5), n_running=80 + 20 * (seed % 4), unaligned=unaligned)


def random_rounds(schedule, seed):
    r = _seeded_round(seed)
    got, _ = assert_parity(schedule, r.to_input(), r.name)
    assert got.stats.gpu_launches > 0


def random_rounds_many_nodes(schedule, seed, n_nodes, n_jobs, n_running):
    r = synth.random_round(seed, n_nodes=n_nodes, n_queues=9, n_jobs=n_jobs, n_running=n_running,
                           protected_fraction=0.5 if seed % 2 else 0.0)
    assert_parity(schedule, r.to_input(), r.name)


def scaled_config(schedule, name, scale):
    r = synth.scaled(name, scale)
    got, want = assert_parity(schedule, r.to_input(), f"{name}@{scale}")
    assert got.out.num_result_scheduled == want.out.num_result_scheduled


def runs_of_known_unschedulable_jobs(schedule, n_nodes):
    """synth.unfeasible_runs_round: skipped runs around the 128-record fast-forward step; the level
    scan that proves the miss covers node counts that are not a multiple of its stride."""
    r = synth.unfeasible_runs_round(n_nodes)
    got, want = assert_parity(schedule, r.to_input(), r.name)
    assert got.out.num_result_scheduled == want.out.num_result_scheduled == 11 + 40


def partly_indexed_resources(schedule, seed, indexed):
    """Not every resource is part of the best-fit key (nodedb indexedResources ⊂ resources): the
    key no longer carries the whole row, so the SWAR shortcuts are off and the assignment table
    keeps rows beside the keys (Batch::chain_run, row-reading cursor refills)."""
    batchy = seed != 403
    r = synth.random_round(seed, n_nodes=120, n_queues=6, n_jobs=900, n_running=0 if batchy else 200, gangs=not batchy, priorities=not batchy)
    r.indexed = indexed
    got, _ = assert_parity(schedule, r.to_input(), f"{r.name} indexed={indexed}")
    if batchy:
        assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0


def exact_mode_unaligned_round(schedule, seed):
    """Inputs outside the fast domain run in exact mode: the reference's default index resolutions
    (config/scheduler/config.yaml:116-124: cpu 100m, memory 100Mi) with 250m / 4Gi-style requests, node sizes
    that are not multiples of them, allocatable < total, a NodeFactory index order that differs from the
    node-id order, classes that match several node types.  Every probe is the literal ordered walk of
    nodeiteration.go:318-382; no E_UNSUPPORTED."""
    r = _seeded_round(seed, unaligned=True)
    assert_parity(schedule, r.to_input(), r.name)


def resolution_rounding_blocks_a_feasible_node(schedule):
    """gang_scheduler_test.go:244-262 on the device path: the fourth job fits a node but the rounded
    index key hides that node from the iterator."""
    got, want = assert_parity(schedule, synth.rounding_round().to_input(), "rounding")
    assert got.out.num_result_scheduled == want.out.num_result_scheduled == 3
    assert int((got.job_state == abi.JOB_FAILED).sum()) == 1


def more_classes_than_the_shared_memory_table_holds(schedule, **sizes):
    r = synth.many_classes_round(**sizes)
    got, _ = assert_parity(schedule, r.to_input(), r.name)
    assert got.out.num_result_scheduled > 0


def time_budget(make_round, inp, budget_ns):
    """armada_round_run_deadline: a budget that cannot be met returns ARMADA_E_DEADLINE (the reference's
    cancelled context, scheduling_algo.go:115-118), download is refused, and the same handle still
    schedules the uploaded snapshot afterwards, bit-exact."""
    with make_round() as dev:
        dev.upload(inp)
        with pytest.raises(abi.ArmadaError) as ei:
            dev.run(budget_ns=budget_ns)
        assert ei.value.status == abi.E_DEADLINE
        with pytest.raises(abi.ArmadaError) as ei:
            dev.download()
        assert ei.value.status == abi.E_STATE
        dev.run(budget_ns=60_000_000_000)
        assert not dev.download().diff(oracle_lib.round_schedule(inp))


def dry_run_case(make_nodedb, r, gangs_as_jobs):
    """gangs_as_jobs: lists of job indices; the product takes the jobs' classes.  Returns the verdicts."""
    inp = r.to_input()
    jc = np.asarray(r.job_class).astype(np.int64)
    odb = oracle_lib.OracleNodeDb(inp)
    want = [odb.dry_run(g) for g in gangs_as_jobs]
    singles = [i for i, g in enumerate(gangs_as_jobs) if len(g) == 1]
    with make_nodedb(inp) as db:
        got_ok, got_nodes = db.schedule_many([[int(jc[j]) for j in g] for g in gangs_as_jobs])
        sel = db.select_nodes([int(jc[gangs_as_jobs[i][0]]) for i in singles])
    assert list(got_ok) == [ok for ok, _ in want]
    for g, (a, (_, b)) in enumerate(zip(got_nodes, want)):
        assert (a == b).all(), f"gang {g}: {a} vs {b}"
    # armada_nodedb_select_nodes: the single-job form gives the same nodes as gangs of one
    for i, n in zip(singles, sel):
        ok, nodes = want[i]
        assert (n != abi.NONE) == ok and (not ok or n == nodes[0])
    return [ok for ok, _ in want]


def dry_run_nodedb_matches_the_oracle(make_nodedb, seed, unaligned, n_nodes, n_jobs, n_singles, n_gangs, max_gang):
    """armada_nodedb_schedule_many (SubmitChecker's ScheduleManyWithTxn + Abort on an empty cluster,
    submitcheck.go:302-422): single jobs and gangs of every class in one launch, including gangs too big for
    the cluster (up to max_gang - 1 members), against the oracle's NodeDb: same verdicts, same nodes."""
    r = synth.random_round(seed, n_nodes=n_nodes, n_jobs=n_jobs, n_running=0, gangs=False, unaligned=unaligned, away=(seed == 1))
    rng = np.random.default_rng(seed)
    job_class = np.asarray(r.job_class)
    J = len(job_class)
    gangs = [[int(j)] for j in rng.choice(J, n_singles, replace=False)]
    for _ in range(n_gangs):
        size = int(rng.integers(2, max_gang))
        same = np.nonzero(job_class == job_class[int(rng.integers(0, J))])[0]
        # the oracle's jobs must be distinct inside one gang
        gangs.append(list(dict.fromkeys(int(same[i % len(same)]) for i in range(size))))
    assert any(dry_run_case(make_nodedb, r, gangs))


def dry_run_nodedb_resolution_rounding(make_nodedb):
    """The rounded index key can hide a node from the iterator even on an empty cluster: 20 cpu on a
    32-cpu node with a 17-cpu index resolution (rounded 17 < 20) is unschedulable in the reference."""
    r = synth.rounding_round()
    r.class_request = np.stack([synth.rl(16, 128), synth.rl(20, 128)])
    r.class_pc = np.zeros(2)
    r.class_static_row = np.zeros(2)
    r.job_class = np.array([0, 0, 1, 1])
    assert dry_run_case(make_nodedb, r, [[0], [2], [0, 1], [3]]) == [True, False, True, False]


def snapshot_construction(schedule, seed):
    """NULL queue_allocated_by_pc / queue_constrained_demand: the library derives the queue accounting
    from the job arrays (calculateJobSchedulingInfo + constructSchedulingContext,
    scheduling_algo.go:522-632,664-676) — on the device in the product (k_snapshot_*), restated in the
    oracle; without per-queue limits that equals what the host-side generator passes explicitly."""
    limits = seed == 4
    r = synth.random_round(seed, n_nodes=50, n_jobs=350, n_running=100, protected_fraction=0.5, queue_limits=limits)
    inp = r.to_input()
    explicit = oracle_lib.round_schedule(inp)
    inp.queue_allocated_by_pc = None
    inp.queue_constrained_demand = None
    want = oracle_lib.round_schedule(inp)
    got = schedule(inp)
    assert not got.diff(want)
    if not limits:
        assert not want.diff(explicit)


def excluded_nodes_properties(inp, res):
    """queue_scheduler_test.go:656-676: for a single job that could not be scheduled the excluded nodes
    add up to the number of nodes; jobs that were never attempted (or did not fail) and gang members report
    nothing.  Returns the number of jobs that report."""
    ex = np.asarray(res.job_excluded_nodes)
    st = np.asarray(res.job_state)
    gang = np.ctypeslib.as_array(inp.job_gang, (inp.num_jobs,))
    tot = ex.sum(axis=1)
    assert (tot[(st != abi.JOB_FAILED) | (gang != abi.NONE)] == 0).all()
    attempted = tot > 0
    assert (tot[attempted] == inp.num_nodes).all()
    return int(attempted.sum())


def excluded_nodes_by_reason_kind(schedule, seed, unaligned):
    """collect_excluded_nodes: PodSchedulingContext.NumExcludedNodesByReason of the jobs that fail, by
    reason kind (node type / taints+labels / resources on a reached node / never reached), identical to
    the oracle's restatement of nodedb.go:445-480,605-640,786-797,1102-1117."""
    r = synth.random_round(700 + seed, n_nodes=40 + 7 * seed, n_queues=4, n_jobs=600, n_running=100 if seed % 2 else 0, gangs=seed % 3 == 0,
                           priorities=seed % 2 == 1, unaligned=unaligned)
    inp = r.to_input()
    inp.collect_excluded_nodes = 1
    got, _ = assert_parity(schedule, inp, r.name)
    assert excluded_nodes_properties(inp, got) > 0


def gang_scheduler_table(schedule, name):
    """TestGangScheduler (gang_scheduler_test.go:33-760) through the kernel: node-uniformity search, floating
    resources, round / queue limits, the resolution-rounding case."""
    b, tc, gangs = gang_cases.gang_case_round(name)
    got, _ = assert_parity(schedule, b.input, name)
    gang_cases.check_gang_case(b, tc, gangs, got)


def uniformity_and_floating_round(schedule, seed):
    got, want = assert_parity(schedule, gang_cases.uniformity_round(seed).input, f"uniformity round {seed}")
    if seed == 1:  # the generator reaches every new outcome
        reasons = set(int(x) for x in want.job_reason)
        assert {abi.REASON_UNIFORMITY_LABEL_NOT_INDEXED, abi.REASON_NO_NODES_WITH_UNIFORMITY_LABEL, abi.REASON_GANG_FITS_NO_UNIFORMITY_VALUE,
                abi.REASON_FLOATING_RESOURCES} <= reasons


def job_priority_comparer(schedule, name):
    b, expected = order_cases.comparison_round(name)
    got, _ = assert_parity(schedule, b.input, name)
    order_cases.check_order(b, expected, got)
