"""Parity tests proper: the CUDA path (through the C ABI, host buffers in/out) against the CPU
oracle on the same inputs — bit-exact on every output array (job outcomes, nodes, priorities,
methods, reasons, final NodeDb allocatable vectors, per-queue accounting, fair-share doubles,
counters).  The bodies shared with the emulator module are in tests/round_cases.py.  Run on an
H100: pytest -m gpu."""
import numpy as np
import pytest

import gang_cases
import go_tables as gt
import oracle_lib
import order_cases
import round_cases as rc
import shape_cases
from armada_b200 import abi, synth
from armada_b200.scheduler import DeviceNodeDb, DeviceRound
from shape_cases import Case, compare_key  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

_dev = None


def device():
    global _dev
    if _dev is None:
        _dev = DeviceRound(0)
    return _dev


def cuda_round(inp):
    return device().schedule(inp)


def assert_parity(inp, label=""):
    return rc.assert_parity(cuda_round, inp, label)


@pytest.mark.parametrize("seed", range(24))
def test_random_rounds(seed):
    rc.random_rounds(cuda_round, seed)


@pytest.mark.parametrize("seed", range(100, 108))
def test_random_rounds_many_nodes(seed):
    # > 1 tile group (N > 4096) so every tree level is exercised
    rc.random_rounds_many_nodes(cuda_round, seed, n_nodes=5000 + 700 * (seed % 3), n_jobs=6000, n_running=3000)


@pytest.mark.parametrize("name,scale", [("C2", 0.02), ("C3", 0.004), ("C4", 0.006), ("C5", 0.004), ("C3", 0.05), ("C5", 0.03)])
def test_scaled_configs(name, scale):
    rc.scaled_config(cuda_round, name, scale)


@pytest.mark.parametrize("n_nodes", [7, 401, 5000])
def test_runs_of_known_unschedulable_jobs(n_nodes):
    rc.runs_of_known_unschedulable_jobs(cuda_round, n_nodes)


@pytest.mark.parametrize("seed,indexed", [(400, [synth.CPU, synth.MEM]), (401, [synth.CPU]), (402, [synth.MEM, synth.GPU]),
                                          (403, [synth.CPU, synth.MEM])])
def test_partly_indexed_resources(seed, indexed):
    rc.partly_indexed_resources(cuda_round, seed, indexed)


def test_batch_mode_covers_the_plain_iterations_and_is_deterministic():
    """Most of a C3-shaped round runs in batch mode (ArmadaRoundStats.phase_cycles[4] = loop
    iterations executed there); repeating the round gives bit-identical results (no timing
    dependence in the warp protocols)."""
    r = synth.scaled("C3", 0.08)
    inp = r.to_input()
    dev = device()
    dev.upload(inp)
    ref = None
    for _ in range(6):
        st = dev.run()
        got = dev.download()
        if ref is None:
            ref = got
        else:
            assert not got.diff(ref)
    assert int(st.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0.8 * int(st.loop_iterations)
    want = oracle_lib.round_schedule(inp)
    assert not ref.diff(want)


def test_c1_simulator_config():
    got, want = assert_parity(synth.config_c1().to_input(), "C1")
    assert got.out.num_result_scheduled == 1000


@pytest.mark.parametrize("name", sorted(rc.PQS.keys()))
def test_reference_pqs_tables_on_device(name):
    rc.reference_table(cuda_round, gt.run_pqs_case, rc.PQS[name])


@pytest.mark.parametrize("name", sorted(rc.QS.keys()))
def test_reference_queue_scheduler_tables_on_device(name):
    rc.reference_table(cuda_round, gt.run_queue_scheduler_case, rc.QS[name])


def test_unsupported_input_fails_loudly():
    """What the device cannot hold is refused with a status code, never computed wrongly: more queues
    than the shared-memory queue table has rows."""
    r = synth.random_round(1, n_queues=129)
    with pytest.raises(abi.ArmadaError) as ei:
        cuda_round(r.to_input())
    assert ei.value.status == abi.E_UNSUPPORTED


@pytest.mark.parametrize("seed", range(12))
def test_exact_mode_unaligned_rounds(seed):
    rc.exact_mode_unaligned_round(cuda_round, seed)


def test_exact_mode_many_nodes():
    r = synth.random_round(77, n_nodes=3000, n_queues=7, n_jobs=2500, n_running=1500, protected_fraction=0.5, unaligned=True)
    assert_parity(r.to_input(), r.name)


def test_exact_mode_resolution_rounding_blocks_a_feasible_node():
    rc.resolution_rounding_blocks_a_feasible_node(cuda_round)


@pytest.mark.parametrize("name", ["C2", "C3", "C4"])
def test_full_size_parity(name):
    """The BASELINE.json configurations at their stated size, bit-exact on every output array
    against the oracle (C3 is the benchmarked configuration; the oracle needs 1–3 s for it)."""
    r = {"C2": synth.config_c2, "C3": synth.config_c3, "C4": synth.config_c4}[name]()
    got, want = assert_parity(r.to_input(), f"{name} full size")
    assert got.out.num_result_scheduled == want.out.num_result_scheduled > 0


def test_c5_largest_oracle_scale_parity():
    """C5 (90 % utilisation, eviction round): the reference's fair-preemption walk is quadratic in
    the number of evicted jobs, so the oracle is run at the largest scale it finishes within about
    a minute (10k nodes); the full-size round is covered by bench.py's extra workloads."""
    r = synth.scaled("C5", 0.1)
    got, want = assert_parity(r.to_input(), "C5@0.1")
    assert got.out.num_result_preempted == want.out.num_result_preempted


def test_full_size_properties():
    """BASELINE-size C3 through size-independent properties: no oversubscription, every scheduled
    job fits its node, conservation of resources, idempotence of a second run."""
    r = synth.config_c3()
    inp = r.to_input()
    dev = device()
    dev.upload(inp)
    dev.run()
    a = dev.download()
    dev.run()
    b = dev.download()
    assert not a.diff(b), "armada_round_run is not idempotent"
    N = inp.num_nodes
    assert (a.node_alloc >= 0).all()
    sched = a.job_state == abi.JOB_SCHEDULED
    assert sched.sum() == a.out.num_result_scheduled > 0
    req = r.class_request[np.asarray(r.job_class).astype(np.int64)]
    used = np.zeros((synth.D, N), np.int64)
    np.add.at(used.T, a.job_node[sched].astype(np.int64), req[sched])
    assert (used + a.node_alloc[0] == r.node_allocatable).all()
    # gpu jobs only on gpu nodes
    gpu_jobs = sched & (req[:, synth.GPU] > 0)
    assert (np.asarray(r.node_static_class)[a.job_node[gpu_jobs].astype(np.int64)] == 1).all()
    # queue accounting equals the sum of scheduled requests
    qa = np.zeros_like(a.queue_allocated)
    np.add.at(qa, np.asarray(r.job_queue).astype(np.int64)[sched], req[sched])
    assert (qa == a.queue_allocated).all()


@pytest.mark.parametrize("seed,unaligned,n_nodes", [(0, False, 60), (1, True, 80), (2, True, 2500), (3, False, 5000)])
def test_dry_run_nodedb_matches_the_oracle(seed, unaligned, n_nodes):
    rc.dry_run_nodedb_matches_the_oracle(DeviceNodeDb, seed, unaligned, n_nodes, n_jobs=400, n_singles=120, n_gangs=30, max_gang=200)


def test_dry_run_nodedb_resolution_rounding():
    rc.dry_run_nodedb_resolution_rounding(DeviceNodeDb)


def test_more_classes_than_the_shared_memory_table_holds():
    rc.more_classes_than_the_shared_memory_table_holds(cuda_round, n_nodes=600, n_jobs=12000)


@pytest.mark.parametrize("seed", [2, 4, 10])
def test_snapshot_construction_on_the_device(seed):
    rc.snapshot_construction(cuda_round, seed)


def test_snapshot_construction_at_c5_scale():
    r = synth.scaled("C5", 0.05)
    inp = r.to_input()
    inp.queue_allocated_by_pc = None
    inp.queue_constrained_demand = None
    assert_parity(inp, "C5@0.05 with derived queue accounting")


def test_time_budget_aborts_the_round_and_leaves_the_snapshot_runnable():
    """The budget is measured on the device (%globaltimer)."""
    rc.time_budget(DeviceRound, synth.scaled("C3", 0.05).to_input(), budget_ns=1000)


@pytest.mark.parametrize("nodes,queues,jobs,seed", [(60, 4, 1500, 1), (250, 6, 5000, 3), (3000, 16, 40000, 5)])
def test_gangs_as_batch_items(nodes, queues, jobs, seed):
    """Simple gangs are items of the batch pipeline (placed member by member, all or nothing); the
    clusters fill up, so gangs also fail in the middle and are rolled back."""
    r = synth.config_c4(nodes, queues, jobs, seed=synth.SEED + seed)
    got, want = assert_parity(r.to_input(), f"C4 {nodes}x{jobs}")
    assert int(got.stats.placements) > int(got.stats.loop_iterations) - int(np.count_nonzero(np.asarray(want.job_state) == 4))


def test_rounds_of_different_handles_run_concurrently_and_stay_exact():
    """Four pools on one GPU at the same time (one handle and one host thread each, pools.PoolCycle):
    every result equals the oracle's, whatever the interleaving."""
    from armada_b200.pools import PoolCycle
    pools = [synth.random_round(900 + i, n_nodes=200 + 50 * i, n_queues=6, n_jobs=6000, n_running=0, gangs=i % 2 == 1, priorities=False).to_input()
             for i in range(4)]
    cyc = PoolCycle(pools, 0, 1, lambda: DeviceRound(0))
    try:
        for _ in range(3):
            out = cyc.schedule_cycle()
            for p, inp in enumerate(pools):
                assert not out[p].diff(oracle_lib.round_schedule(inp)), f"pool {p}"
    finally:
        cyc.close()


@pytest.mark.parametrize("seed", range(6))
def test_excluded_nodes_by_reason_kind(seed):
    rc.excluded_nodes_by_reason_kind(cuda_round, seed, unaligned=seed >= 4)


def test_excluded_nodes_at_c3_scale():
    r = synth.scaled("C3", 0.05)
    inp = r.to_input()
    inp.collect_excluded_nodes = 1
    got, _ = assert_parity(inp, "C3@0.05 with excluded-node kinds")
    assert rc.excluded_nodes_properties(inp, got) > 0


# ---- gang node uniformity + floating resources (gang_scheduler.go:143,154-223) ----------------------
@pytest.mark.parametrize("name", sorted(gang_cases.GANG.keys()))
def test_reference_gang_scheduler_table_on_device(name):
    rc.gang_scheduler_table(cuda_round, name)


@pytest.mark.parametrize("seed", range(10))
def test_uniformity_and_floating_rounds(seed):
    rc.uniformity_and_floating_round(cuda_round, seed)


@pytest.mark.parametrize("seed,unaligned,floating", [(40, False, False), (41, True, True), (42, False, True)])
def test_uniformity_rounds_at_scale(seed, unaligned, floating):
    b = gang_cases.uniformity_round(seed, n_nodes=1500, n_zones=12, n_queues=8, n_jobs=9000, floating=floating, unaligned=unaligned)
    got, want = assert_parity(b.input, f"uniformity round {seed} at scale")
    assert int(want.out.num_result_scheduled) > 1000


@pytest.mark.parametrize("name", sorted(order_cases.CASES))
def test_job_priority_comparer_on_device(name):
    rc.job_priority_comparer(cuda_round, name)


# ---- every resource count and key layout (tests/shape_cases.py), and the emulator's knob tests on the device ----
GPU_SHAPES = shape_cases.MATRIX + [
    # queue counts: the window width and the batch width switch with them (1 queue, more than 64, the maximum)
    Case(1, "k32", "batch", 200, n_nodes=300, n_queues=1, n_jobs=2500),
    Case(8, "k32", "batch", 201, n_nodes=300, n_queues=65, n_jobs=2500),
    Case(4, "k64", "batch", 202, n_nodes=300, n_queues=100, n_jobs=2500),
    Case(5, "k32", "batch", 203, n_nodes=300, n_queues=128, n_jobs=2500),
    Case(8, "run", "eviction", 204, n_nodes=300, n_queues=128, n_jobs=2500),
    # thousands of nodes: more than one tile group, hundreds of batches
    Case(8, "k32", "batch", 210, n_nodes=4097, n_queues=9, n_jobs=20000),
    Case(1, "k32", "batch", 211, n_nodes=4097, n_queues=9, n_jobs=20000),
    Case(8, "k64", "batch", 212, n_nodes=4500, n_queues=9, n_jobs=20000),
    Case(1, "k64", "batch", 213, n_nodes=3000, n_queues=9, n_jobs=20000),
    Case(8, "k32", "eviction", 214, n_nodes=3000, n_queues=9, n_jobs=6000),
    Case(1, "k32", "eviction", 215, n_nodes=5000, n_queues=9, n_jobs=6000),
]


@pytest.mark.parametrize("case", GPU_SHAPES, ids=lambda c: c.id)
def test_resource_counts_and_key_layouts(case, capfd):
    """k_schedule_pass<1|2|4|8> with each assignment-loop form (K32, K64, chain_run with unindexed resources or
    without guard bits, exact mode), field widths at the K32 / K64 boundaries, 1 to 5000 nodes, 1 to 128 queues,
    DRF multipliers 0 / 0.5 / 3 with a licence as the dominant resource: the layout the case was built for, and
    every output array equal to the oracle's."""
    shape_cases.check_case(case, device(), oracle_lib.round_schedule, capfd)


@pytest.mark.parametrize("case", [shape_cases.REFUSED, shape_cases.REFUSED_COARSENED, shape_cases.REFUSED_UNINDEXED], ids=lambda c: c.id)
def test_key_wider_than_63_bits_is_refused(case, capfd):
    with DeviceRound(0) as dev:
        shape_cases.check_case(case, dev, oracle_lib.round_schedule, capfd)


@pytest.mark.parametrize("case", [Case(8, "k32", "batch", 220, n_nodes=600, n_jobs=8000), Case(1, "k32", "batch", 221, n_nodes=600, n_jobs=8000)],
                         ids=lambda c: c.id)
def test_shape_rounds_are_deterministic(case):
    """A D = 8 and a D = 1 batch round repeated on one handle: bit-identical every time, and equal to the oracle."""
    inp = shape_cases.shape_round(case).to_input()
    with DeviceRound(0) as dev:
        dev.upload(inp)
        ref = None
        for _ in range(4):
            st = dev.run()
            got = dev.download()
            if ref is None:
                ref = got
            else:
                assert not got.diff(ref)
    assert int(st.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0
    assert not ref.diff(oracle_lib.round_schedule(inp))


@pytest.mark.parametrize("wq,seed", [(8, 500), (8, 501), (16, 502), (8, 503)])
def test_long_batch_pipelines(wq, seed, compare_key):
    shape_cases.long_batch_pipeline(lambda: DeviceRound(0), wq, seed)


@pytest.mark.parametrize("nodes,queues,jobs,wq,seed", [(60, 4, 1500, 0, 1), (120, 8, 3000, 8, 2), (250, 6, 5000, 16, 3), (40, 3, 900, 0, 4)])
def test_gangs_as_batch_items_with_knobs(nodes, queues, jobs, wq, seed, compare_key):
    """test_gangs_as_batch_items with small batches (ARMADA_BT_WQ) and the 64-bit compare keys (ARMADA_NO_K32)."""
    shape_cases.gangs_as_batch_items(lambda: DeviceRound(0), nodes, queues, jobs, wq, seed)


@pytest.mark.parametrize("seed", [0, 5])
def test_exact_mode_forced_on_aligned_rounds(seed):
    shape_cases.exact_mode_forced(lambda: DeviceRound(0), seed)
