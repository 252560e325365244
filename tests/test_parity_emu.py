"""Kernel-logic parity WITHOUT a GPU: the same CUDA source (armada_b200/csrc/*.cu|inc) compiled
by g++ against tools/simt_emu/cuda_emu.h (deterministic SIMT emulator, test tooling only) and
compared bit-for-bit with the CPU oracle.  The real parity tests are tests/test_parity_gpu.py
(pytest -m gpu, through the nvcc-built product library); this module exists so that control-flow /
data-structure bugs in the kernels are caught on a CPU-only box.  The bodies both modules run are in
tests/round_cases.py.  EMU_ORDER=reverse runs the lanes of every warp in the opposite order (catches
missing __syncwarp in either direction)."""
import os

import numpy as np

import pytest

import emu_lib
import gang_cases
import go_tables as gt
import oracle_lib
import order_cases
import round_cases as rc
import shape_cases
from armada_b200 import abi, synth
from armada_b200.scheduler import DeviceNodeDb
from shape_cases import compare_key  # noqa: F401  (fixture)

_dev = None


def emu_round(inp):
    global _dev
    if _dev is None:
        _dev = emu_lib.emu_round()
    return _dev.schedule(inp)


def emu_nodedb(inp):
    return DeviceNodeDb(inp, 0, lib=emu_lib.load())


def assert_parity(inp, label=""):
    return rc.assert_parity(emu_round, inp, label)


@pytest.fixture(params=["forward", "reverse"])
def lane_order(request):
    old = os.environ.get("EMU_ORDER")
    os.environ["EMU_ORDER"] = request.param
    yield request.param
    if old is None:
        os.environ.pop("EMU_ORDER", None)
    else:
        os.environ["EMU_ORDER"] = old


@pytest.mark.parametrize("seed", range(24))
def test_random_rounds(seed, lane_order):
    rc.random_rounds(emu_round, seed)


@pytest.mark.parametrize("seed", [100, 101])
def test_random_rounds_many_nodes(seed):
    rc.random_rounds_many_nodes(emu_round, seed, n_nodes=1500 + 700 * (seed % 3), n_jobs=2500, n_running=1200)


@pytest.mark.parametrize("n_queues", [40, 100, 128])
def test_many_queues(n_queues):
    """More queues than fit 64 batch items each (the batch windows shrink to 32 / the merge sort to
    a different power of two); priorities off so that most of the round runs in batch mode."""
    r = synth.random_round(300 + n_queues, n_nodes=300, n_queues=n_queues, n_jobs=2500, n_running=0, gangs=False, priorities=False)
    got, _ = assert_parity(r.to_input(), r.name)
    assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0


@pytest.mark.parametrize("name,scale", [("C2", 0.02), ("C3", 0.004), ("C4", 0.006), ("C5", 0.004)])
def test_scaled_configs(name, scale):
    rc.scaled_config(emu_round, name, scale)


@pytest.mark.parametrize("name", sorted(rc.PQS.keys()))
def test_reference_pqs_tables(name):
    rc.reference_table(emu_round, gt.run_pqs_case, rc.PQS[name])


@pytest.mark.parametrize("name", sorted(rc.QS.keys()))
def test_reference_queue_scheduler_tables(name):
    rc.reference_table(emu_round, gt.run_queue_scheduler_case, rc.QS[name])


@pytest.mark.parametrize("n_nodes", [7, 401])
def test_runs_of_known_unschedulable_jobs(n_nodes):
    rc.runs_of_known_unschedulable_jobs(emu_round, n_nodes)


@pytest.mark.parametrize("seed,indexed", [(400, [synth.CPU, synth.MEM]), (401, [synth.CPU]), (402, [synth.MEM, synth.GPU]),
                                          (403, [synth.CPU, synth.MEM])])
def test_partly_indexed_resources(seed, indexed, lane_order):
    rc.partly_indexed_resources(emu_round, seed, indexed)


@pytest.mark.parametrize("wq,seed", [(8, 500), (8, 501), (16, 502), (8, 503)])
def test_long_batch_pipelines(wq, seed, lane_order, compare_key):
    shape_cases.long_batch_pipeline(emu_lib.emu_round, wq, seed)


@pytest.mark.parametrize("nodes,queues,jobs,wq,seed", [(60, 4, 1500, 0, 1), (120, 8, 3000, 8, 2), (250, 6, 5000, 16, 3), (40, 3, 900, 0, 4)])
def test_gangs_as_batch_items(nodes, queues, jobs, wq, seed, lane_order, compare_key):
    shape_cases.gangs_as_batch_items(emu_lib.emu_round, nodes, queues, jobs, wq, seed)


@pytest.mark.parametrize("seed", range(10))
def test_exact_mode_unaligned_rounds(seed, lane_order):
    rc.exact_mode_unaligned_round(emu_round, seed)


def test_exact_mode_resolution_rounding_blocks_a_feasible_node():
    rc.resolution_rounding_blocks_a_feasible_node(emu_round)


@pytest.mark.parametrize("seed", [0, 5])
def test_exact_mode_forced_on_aligned_rounds(seed):
    shape_cases.exact_mode_forced(emu_lib.emu_round, seed)


def test_more_classes_than_the_shared_memory_table_holds():
    rc.more_classes_than_the_shared_memory_table_holds(emu_round)


def test_time_budget_aborts_the_round_and_leaves_the_snapshot_runnable():
    rc.time_budget(emu_lib.emu_round, synth.random_round(3, n_nodes=50, n_jobs=300, n_running=60).to_input(), budget_ns=1)


@pytest.mark.parametrize("seed,unaligned", [(0, False), (1, True), (2, True), (3, False)])
def test_dry_run_nodedb_matches_the_oracle(seed, unaligned):
    rc.dry_run_nodedb_matches_the_oracle(emu_nodedb, seed, unaligned, n_nodes=30 + 7 * seed, n_jobs=200, n_singles=40, n_gangs=12, max_gang=150)


def test_dry_run_nodedb_resolution_rounding():
    rc.dry_run_nodedb_resolution_rounding(emu_nodedb)


@pytest.mark.parametrize("seed", [2, 4, 10])
def test_snapshot_construction_on_the_device(seed):
    rc.snapshot_construction(emu_round, seed)


@pytest.mark.parametrize("seed", range(8))
def test_excluded_nodes_by_reason_kind(seed, lane_order):
    rc.excluded_nodes_by_reason_kind(emu_round, seed, unaligned=seed >= 6)


def test_excluded_nodes_on_the_reference_tables():
    """The same on the reference's QueueScheduler table (the test that states the property)."""
    seen = []

    def schedule(inp):
        inp.collect_excluded_nodes = 1
        got = rc.round_or_skip(emu_round, inp)  # (compares every array, job_excluded_nodes included, with the oracle)
        seen.append(rc.excluded_nodes_properties(inp, got))
        return got

    for name in sorted(rc.QS.keys()):
        try:
            gt.run_queue_scheduler_case(rc.QS[name], schedule)
        except gt.UnsupportedCase:
            continue
    assert sum(seen) > 0


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_excluded_nodes_static_and_resource_kinds(seed, lane_order):
    """Static classes finer than node types (a taint / label the node type index does not carry): nodes of a
    matching node type that the walk reaches and StaticJobRequirementsMet rejects count under
    ARMADA_EXCL_STATIC; with a resource that is not indexed, reached nodes can also fail on resources."""
    r = synth.random_round(740 + seed, n_nodes=60, n_queues=3, n_jobs=500, n_running=0, gangs=False, priorities=False)
    if seed == 2:
        r.indexed = [synth.CPU, synth.MEM]  # gpu is not in the index: a reached node can still lack gpus
    # half of the nodes of type 0 get a new static class that row 0 rejects (type_match still accepts their type)
    sc = np.asarray(r.node_static_class).astype(np.uint32).copy()
    typ = np.asarray(r.node_type).astype(np.uint32)
    new = r.num_static_classes
    pick = np.nonzero(typ == 0)[0][::2]
    sc[pick] = new
    sm = np.asarray(r.static_match).astype(np.uint32)
    rows = sm.shape[0]
    words = (new + 1 + 31) // 32
    sm2 = np.zeros((rows, words), np.uint32)
    for row in range(rows):
        for c in range(new):
            if (sm[row, c >> 5] >> (c & 31)) & 1:
                sm2[row, c >> 5] |= np.uint32(1 << (c & 31))
        if row != 0 and (sm[row, 0] & 1):  # the new class behaves like class 0, except for row 0
            sm2[row, new >> 5] |= np.uint32(1 << (new & 31))
    r.node_static_class, r.static_match, r.num_static_classes = sc, sm2, new + 1
    inp = r.to_input()
    inp.collect_excluded_nodes = 1
    _, want = assert_parity(inp, r.name)
    assert rc.excluded_nodes_properties(inp, want) > 0
    ex = np.asarray(want.job_excluded_nodes)
    assert ex[:, abi.EXCL_STATIC].sum() > 0


# ---- gang node uniformity + floating resources (gang_scheduler.go:143,154-223) ----------------------
@pytest.mark.parametrize("name", sorted(gang_cases.GANG.keys()))
def test_reference_gang_scheduler_table(name):
    rc.gang_scheduler_table(emu_round, name)


@pytest.mark.parametrize("seed", range(8))
def test_uniformity_and_floating_rounds(seed, lane_order):
    rc.uniformity_and_floating_round(emu_round, seed)


@pytest.mark.parametrize("seed", [20, 21, 22])
def test_uniformity_rounds_in_exact_mode(seed):
    assert_parity(gang_cases.uniformity_round(seed, unaligned=True).input, f"unaligned uniformity round {seed}")


def test_uniformity_rounds_without_floating_resources_keep_the_batch_pipeline():
    got, _ = assert_parity(gang_cases.uniformity_round(30, n_nodes=80, n_jobs=600, floating=False).input, "uniformity, no floating")


@pytest.mark.parametrize("name", sorted(order_cases.CASES))
def test_job_priority_comparer(name):
    rc.job_priority_comparer(emu_round, name)


def test_presorted_job_order_fast_path_equals_the_general_path(monkeypatch):
    """armada_round_upload ranks the jobs of a queue without building sort keys when every queue already arrives in
    SchedulingOrderCompare order (the BASELINE configs do); ARMADA_NO_PRESORTED forces the bucket sort."""
    for name, scale in (("C3", 0.004), ("C5", 0.004), ("C4", 0.006)):
        inp = synth.scaled(name, scale).to_input()
        fast, want = assert_parity(inp, f"{name} presorted")
        monkeypatch.setenv("ARMADA_NO_PRESORTED", "1")
        general, _ = assert_parity(inp, f"{name} general order path")
        monkeypatch.delenv("ARMADA_NO_PRESORTED")
        assert not fast.diff(general)


def test_job_order_over_several_host_slices():
    """70 000 jobs: the upload ranks them on 16 host threads.  (1) queues that arrive in order: the one-pass ranking,
    checked inside every slice and across the slices of a queue; (2) the same round with two jobs of one queue
    exchanged ACROSS a slice boundary (only the cross-slice check can see it) and (3) inside a slice: the bucket sort."""
    r = synth.scaled("C2", 0.7)
    assert len(r.job_queue) >= 65536
    assert_parity(r.to_input(), "presorted, 16 slices")
    per_slice = len(r.job_queue) // 16
    for name, lo, hi in (("across slices", per_slice - 40, per_slice + 40), ("inside a slice", 100, 180)):
        r = synth.scaled("C2", 0.7)
        q = r.job_queue[lo]
        a = next(j for j in range(lo, hi) if r.job_queue[j] == q and j < per_slice) if name == "across slices" else lo
        b = next(j for j in range(hi, lo, -1) if r.job_queue[j] == q and (j >= per_slice or name != "across slices"))
        assert a < b and r.job_queue[a] == r.job_queue[b]
        r.job_submit_time[a], r.job_submit_time[b] = r.job_submit_time[b], r.job_submit_time[a]
        got, want = assert_parity(r.to_input(), name)
        assert want.job_seq[b] < want.job_seq[a] or want.job_seq[a] == 0  # b now comes first in its queue


@pytest.mark.parametrize("seed", [50, 51, 52, 53])
def test_uniformity_rounds_with_large_and_running_gangs(seed):
    """Gangs of up to 40 members (more than one warp load of members per attempt) and running gangs with a uniformity
    label that are evicted and re-scheduled (pinned members inside the per-value attempts)."""
    b = gang_cases.uniformity_round(seed, n_nodes=60, n_zones=4, n_jobs=500, floating=(seed % 2 == 0), max_gang=40, running_gangs=6,
                                    protected_fraction=0.0 if seed >= 52 else 0.5)
    got, want = assert_parity(b.input, f"large / running uniformity gangs {seed}")
    if seed >= 52:
        assert int(want.stats.evicted_pass1) > 0  # the running gangs are evicted and go through the search pinned


def test_dry_run_nodedb_ignores_floating_resources_in_the_node_fit():
    """SubmitChecker's NodeDb with a floating resource in the factory: a job's floating request is no part of the node
    fit (KubernetesResourceRequirements) — oracle and device agree, and the job fits where its cpu / memory do."""
    class _R:  # what dry_run_case needs of a round
        def __init__(self, b):
            self.b, self.job_class = b, b.job_class

        def to_input(self):
            return self.b.input

    from armada_b200.model import RoundInputBuilder
    b0 = gang_cases.uniformity_round(3, n_nodes=12, n_jobs=80, floating=True)
    # (the SubmitChecker's NodeDb is the EMPTY cluster: no running jobs in the input)
    b = RoundInputBuilder(b0.cfg, b0.nodes, [j for j in b0.jobs if j.node is None], b0.queues)
    J = len(b.jobs)
    with_lic = [j for j in range(J) if "licences" in b.jobs[j].requests and b.jobs[j].node is None]
    assert with_lic
    gangs = [[j] for j in with_lic[:10]] + [[j] for j in range(J) if b.jobs[j].node is None][:10]
    oks = rc.dry_run_case(emu_nodedb, _R(b), gangs)
    assert all(oks[: len(with_lic[:10])])  # 1–16 cpu on 32-cpu nodes of an empty cluster: every one fits


# ---- every resource count and key layout (tests/shape_cases.py) ------------------------------------------
def _shape_params():
    """Every case once; the batch cases at D = 1 and D = 8 also with the lanes of every warp in reverse order."""
    out = []
    for c in shape_cases.MATRIX:
        orders = ("forward", "reverse") if c.kind == "batch" and c.D in (1, 8) else ("forward",)
        out += [pytest.param(c, o, id=f"{c.id}-{o}") for o in orders]
    return out


@pytest.mark.parametrize("case,order", _shape_params())
def test_resource_counts_and_key_layouts(case, order, capfd, monkeypatch):
    """k_schedule_pass<1|2|4|8> with each assignment-loop form (K32, K64, chain_run with unindexed resources or
    without guard bits, exact mode), field widths at the K32 / K64 boundaries, classes of exactly the largest
    node and larger than every node, index orders that differ from the resource order, 1–33 and 4097 nodes, DRF
    multipliers 0 / 0.5 / 3 with a licence as the dominant resource: the layout the case was built for, and
    every output array equal to the oracle's."""
    monkeypatch.setenv("EMU_ORDER", order)
    shape_cases.check_case(case, emu_lib.emu_round(), oracle_lib.round_schedule, capfd)


@pytest.mark.parametrize("case", [shape_cases.REFUSED, shape_cases.REFUSED_COARSENED, shape_cases.REFUSED_UNINDEXED], ids=lambda c: c.id)
def test_key_wider_than_63_bits_is_refused(case, capfd):
    """A best-fit key wider than 63 bits is refused with E_UNSUPPORTED and nothing is computed; the same nodes and
    jobs with the widest field coarsened, or not indexed, are scheduled bit-exactly."""
    shape_cases.check_case(case, emu_lib.emu_round(), oracle_lib.round_schedule, capfd)


def test_shape_matrix_is_covered(capfd):
    """The case generator reaches every (instantiation, assignment-loop form) pair it is meant to, and the refusal:
    an edit that quietly drops a path fails here."""
    dev = emu_lib.emu_round()
    reached = set()
    for c in shape_cases.MATRIX:
        inp = shape_cases.shape_round(c).to_input()
        capfd.readouterr()
        with shape_cases.knob("ARMADA_TIME_UPLOAD", 1):
            dev.upload(inp)
        form = shape_cases.form_of(shape_cases.layout_of(capfd.readouterr().err), inp)
        assert form == c.form, c.id
        reached.add((shape_cases.instantiation(c.D), form))
    assert reached == shape_cases.expected_pairs(), sorted(reached ^ shape_cases.expected_pairs())
    with pytest.raises(abi.ArmadaError) as ei:
        dev.upload(shape_cases.shape_round(shape_cases.REFUSED).to_input())
    assert ei.value.status == abi.E_UNSUPPORTED
    dev.close()
    print("reached:", ", ".join(f"<{i}> {f}" for i, f in sorted(reached)), "+ the 63-bit refusal")
