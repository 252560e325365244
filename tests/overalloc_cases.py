"""Rounds that start on over-allocated nodes: running jobs that need more than the node's allocatable, so its
AllocatableByPriority is negative on entry at every level those jobs hold, the evicted level (level 0) included.
The reference marks such nodes OVERALLOCATED (and UNSCHEDULABLE), scheduling_algo.go:905-920; a node whose gpu
count drops to 0 while gpu jobs run on it is the usual cause.  Shared by the emulator and GPU modules; every
case compares every output array with the oracle bit for bit and asserts what it was built to reach.

The generator places running jobs the way synth does (never over a node), then lowers the allocatable of some of
the busy nodes below what runs on them, never below 0 (negative allocatable is refused):
  resource     which resource goes negative (indexed, or left out of the index)
  steps        whole index-resolution steps over (the fast domain), or None: less than one step (exact mode)
  flags        node_flags of the over-allocated nodes (UNSCHEDULABLE / OVERALLOCATED)
Whether the running jobs are preemptible is the case's choice: non-preemptible ones keep the rows negative through
both passes, preemptible ones are evicted, re-bound and may be evicted again as oversubscribed."""
from __future__ import annotations

import numpy as np

import oracle_lib
import round_cases as rc
import shape_cases
from armada_b200 import abi, synth

MEM, CPU, GPU = synth.MEM, synth.CPU, synth.GPU
FLAGS = {"none": 0, "unschedulable": abi.NODE_UNSCHEDULABLE, "overallocated": abi.NODE_OVERALLOCATED,
         "both": abi.NODE_UNSCHEDULABLE | abi.NODE_OVERALLOCATED}


def resolution_of(r: synth.RawRound, d: int) -> int:
    """The index resolution of resource d (an unindexed resource: its smallest request step, 1000)."""
    idx = list(r.indexed) if r.indexed is not None else synth.INDEXED
    if d not in idx:
        return 1000
    res = list(r.resolution) if r.resolution is not None else [synth.RESOLUTION[synth.INDEXED.index(x)] for x in idx]
    return int(res[idx.index(d)])


def running_use(r: synth.RawRound) -> np.ndarray:
    """[D][N]: what the running jobs request on each node."""
    req = np.asarray(r.class_request)[np.asarray(r.job_class).astype(np.int64)]
    jn = np.asarray(r.job_node).astype(np.int64)
    used = np.zeros(np.asarray(r.node_total).shape, np.int64)
    run = jn != abi.NONE
    np.add.at(used.T, jn[run], req[run])
    return used


def level0_rows(r: synth.RawRound) -> np.ndarray:
    """[D][N]: the evicted level's rows on entry (allocatable minus every running job)."""
    return np.asarray(r.node_allocatable).astype(np.int64) - running_use(r)


def over_allocate(r: synth.RawRound, rng, resource: int, steps, frac=1 / 3, flags=0) -> np.ndarray:
    """Lowers `resource`'s allocatable below what runs on a share of the nodes that hold some of it; returns them."""
    used = running_use(r)
    res = resolution_of(r, resource)
    busy = np.nonzero(used[resource] > 0)[0]
    pick = np.sort(rng.choice(busy, max(1, int(len(busy) * frac)), replace=False))
    alloc = np.asarray(r.node_allocatable).astype(np.int64).copy()
    for n in pick:
        delta = steps * res if steps else int(rng.integers(1, res))
        alloc[resource, n] = max(0, used[resource, n] - delta)
    r.node_allocatable = alloc
    fl = np.zeros(alloc.shape[1], np.uint8)
    fl[pick] = flags
    r.node_flags = fl
    return pick


def split_priority_classes(r: synth.RawRound, running_pc: int, queued_pc: int = 0) -> None:
    """Running jobs move to their shape's class at `running_pc`, queued jobs to the one at `queued_pc` (classes are
    laid out priority class by priority class, as synth and shape_cases make them without away node types)."""
    n_shapes = len(r.class_request) // len(r.pcs)
    jc = np.asarray(r.job_class).astype(np.int64) % n_shapes
    running = np.asarray(r.job_node).astype(np.int64) != abi.NONE
    r.job_class = np.where(running, running_pc * n_shapes + jc, queued_pc * n_shapes + jc)
    r.job_scheduled_at_priority = np.where(running, r.pcs[running_pc][0], abi.NO_PRIORITY)


def _run(schedule, r, excl=False, derive=False, label=""):
    inp = r.to_input()
    inp.collect_excluded_nodes = int(excl)
    if derive:  # the library derives the queue accounting from the job arrays (k_snapshot_*)
        inp.queue_allocated_by_pc = None
        inp.queue_constrained_demand = None
    got, want = rc.assert_parity(schedule, inp, label or r.name)
    if excl:
        rc.excluded_nodes_properties(inp, want)
    return inp, got, want


def _failed_job_counts_resources(want) -> bool:
    """Some failed job counts a node it reached under ARMADA_EXCL_RESOURCES."""
    ex = np.asarray(want.job_excluded_nodes)
    return bool(ex[np.asarray(want.job_state) == abi.JOB_FAILED, abi.EXCL_RESOURCES].sum() > 0)


# ---- 1. fast domain, batch mode ------------------------------------------------------------------------------
def fast_batch_round(D: int, seed: int, n_nodes: int = 60) -> synth.RawRound:
    """shape_cases' eviction round at D resources with non-preemptible running jobs and queued jobs of one
    preemptible priority class: nothing is evicted, so the round runs the batch pipeline.  Over-allocated by one or
    two index-resolution steps of cpu on a third of the busy nodes."""
    r = shape_cases.shape_round(shape_cases.Case(D, "k32", "eviction", seed, n_nodes=n_nodes))
    split_priority_classes(r, running_pc=3)
    r.protected_fraction = 0.0
    over_allocate(r, np.random.default_rng(seed), 0, steps=1 + seed % 2)
    return r


def fast_domain_batch(dev, capfd, D, seed, excl=False, derive=False, n_nodes=60):
    """Negative level-0 rows on entry through the G0 sort (the "sorts last" marker), the SWAR frontier and the batch
    assignment loop (K32 or K64, whichever the compare_key knob leaves), and the level scans of the failing jobs."""
    r = fast_batch_round(D, seed, n_nodes)
    rows = level0_rows(r)
    assert (rows < 0).any(), "no node is over-allocated on entry"
    inp = r.to_input()
    inp.collect_excluded_nodes = int(excl)
    if derive:
        inp.queue_allocated_by_pc = None
        inp.queue_constrained_demand = None
    want = oracle_lib.round_schedule(inp)
    got, lay, form = shape_cases.schedule_with_layout(dev, inp, capfd)
    assert form in ("k32", "k64"), f"{r.name}: the library chose {form} ({lay})"
    bad = got.diff(want)
    assert not bad, f"{r.name}: device != oracle:\n  " + "\n  ".join(bad)
    assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0, "expected batch-mode iterations"
    # non-preemptible jobs hold the rows: still negative at level 0 when the round ends
    assert (np.asarray(want.node_alloc)[0] < 0).any()
    if excl:
        assert rc.excluded_nodes_properties(inp, want) > 0
    return form


# ---- 2. a negative resource that is not indexed ----------------------------------------------------------------
def unindexed_negative(schedule, seed, n_nodes=60, n_jobs=500):
    """gpu is left out of the index and over-allocated by whole gpus on gpu nodes: the keys do not see it, so the
    row-carrying assignment loop (chain_run) and the level scans must reject the node.  The reference rejects it for
    every job, a job that requests no gpu included: resourceRequirementsMet compares every resource of the request,
    and a zero request exceeds a negative allocatable (internaltypes/resource_list.go ExceedsAvailable)."""
    r = synth.random_round(seed, n_nodes=n_nodes, n_queues=4, n_jobs=n_jobs, n_running=n_nodes * 2, gangs=False)
    split_priority_classes(r, running_pc=3)
    # a third of the queued jobs: 16 cpu, 64Gi and no gpu, on gpu nodes only (a node selector), more than they hold
    r.static_match = r.type_match = synth._bitmap([[0], [0, 1], [1]], 2)
    r.class_request = np.concatenate([r.class_request, synth.rl(16, 64)[None, :]])
    r.class_pc = np.concatenate([r.class_pc, [0]])
    r.class_static_row = np.concatenate([r.class_static_row, [2]])
    r.class_away_row = np.concatenate([r.class_away_row, r.class_away_row[:1]])
    queued = np.asarray(r.job_node).astype(np.int64) == abi.NONE
    r.job_class = np.where(queued & (np.arange(len(r.job_class)) % 3 == 0), len(r.class_request) - 1, r.job_class)
    r.indexed = [CPU, MEM]
    neg = over_allocate(r, np.random.default_rng(seed), GPU, steps=1)
    assert (level0_rows(r)[GPU, neg] < 0).all()
    inp, got, want = _run(schedule, r, excl=True)
    # the nodes still have cpu and memory at level 0 that some failed job asked for …
    rows = level0_rows(r)
    st, jn = np.asarray(want.job_state), np.asarray(want.job_node)
    req = np.asarray(r.class_request)[np.asarray(r.job_class).astype(np.int64)]
    failed = np.nonzero(st == abi.JOB_FAILED)[0]
    tolerates = np.asarray(r.class_static_row)[np.asarray(r.job_class).astype(np.int64)] == 2
    fits_but_gpu = [j for j in failed if tolerates[j] and req[j, GPU] == 0 and any(
        (rows[[CPU, MEM], n] >= req[j, [CPU, MEM]]).all() for n in neg)]
    assert fits_but_gpu, "no failed job without gpus would fit an over-allocated node's cpu and memory"
    # … and still no new job lands there
    new = (np.asarray(r.job_node).astype(np.int64) == abi.NONE) & (st == abi.JOB_SCHEDULED)
    assert not np.isin(jn[new], neg).any()
    assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0
    assert _failed_job_counts_resources(want)


# ---- 3. exact mode, less than one step over ----------------------------------------------------------------------
def exact_less_than_a_step(schedule, seed, excl):
    """Exact mode (index resolutions cpu 100m / memory 100Mi / gpu 1) with gpu nodes over-allocated by less than one
    gpu: their gpu row lies in (-1000, 0), where the reference's truncating roundQuantityToResolution gives key 0 (the
    bucket of [0, 1000)) and the device's field is 0 (below it).  Classes that tolerate the gpu taint and request no
    gpu walk those nodes with a zero request on the gpu component.

    Why the nodes reached agree: every request is >= 0, so a negative row fails NodeTypeIterator.NextNode on both
    sides and is never yielded.  Failing there re-seeks to (the node's truncated quantities in front of the failing
    component, the request from it on).  The device's bound is always past the node; the reference's, with a zero
    request, is at or before the node's own key, and the reference then visits a key that is not greater than the one
    it left and fails the round ("iteration loop detected", nodeiteration.go:329-334).  The oracle instead walks the
    bucket again: it reaches the same nodes in the same order, but a node in that bucket that was yielded and
    rejected before is yielded and counted again.  So only the excluded-node counts can differ, and only when such a
    rejected node shares the bucket; test_exact_mode_rejected_node_counted_twice pins that case."""
    r = synth.random_round(seed, n_nodes=60, n_queues=4, n_jobs=400, n_running=150, gangs=False, unaligned=True)
    split_priority_classes(r, running_pc=3)
    neg = over_allocate(r, np.random.default_rng(seed), GPU, steps=None, frac=0.5)
    rows = level0_rows(r)
    assert ((rows[GPU, neg] < 0) & (rows[GPU, neg] > -1000)).all()
    req = np.asarray(r.class_request)
    walks = (np.asarray(r.class_static_row) == 1) & (req[:, GPU] == 0)
    assert walks[np.asarray(r.job_class).astype(np.int64)].any(), "no job walks the gpu nodes with a zero gpu request"
    _, got, want = _run(schedule, r, excl=excl)
    assert (np.asarray(want.node_alloc)[0][GPU, neg] < 0).any()


def two_node_round(neg_component: int, p_cpu: int) -> synth.RawRound:
    """Node 1 runs a non-preemptible 8.05-cpu job on 8 allocatable cpus: its cpu row is -50m (resolution 100m).
    Node 0 (smaller node index, a taint the queued job does not tolerate) has `p_cpu` millicores.  The queued job asks
    for no cpu and 4Gi; both nodes have 200Gi.  `neg_component`: where cpu sits in the index."""
    N = 2
    total = np.repeat(synth.rl(32, 200)[:, None], N, axis=1)
    alloc = total.copy()
    alloc[CPU, 1] = 8000
    alloc[CPU, 0] = p_cpu
    indexed = [CPU, MEM] if neg_component == 0 else [MEM, CPU]
    res = {CPU: 100, MEM: 100 * synth.MI}
    return synth.RawRound(
        node_total=total, node_allocatable=alloc, node_type=np.zeros(N), node_static_class=np.array([1, 0]), num_static_classes=2,
        class_request=np.stack([synth.rl(0, 4), synth.rl(8.05, 0)]), class_pc=np.array([0, 1]), class_static_row=np.zeros(2),
        static_match=synth._bitmap([[0]], 2), type_match=synth._bitmap([[0]], 1),
        job_class=np.array([0, 1]), job_queue=np.zeros(2), job_submit_time=np.arange(2), queue_weight=np.ones(1),
        job_node=np.array([abi.NONE, 1]), job_scheduled_at_priority=np.array([abi.NO_PRIORITY, 3]),
        pcs=((0, True), (3, False)), indexed=indexed, resolution=[res[d] for d in indexed], name=f"two-node-c{neg_component}")


def two_node_first_component(schedule):
    """With the negative row on the first index component the re-seek bound equals the request, so neither side
    re-seeks: the oracle passes the node over, the device never reaches it, and the job fails with the same counts."""
    for p_cpu in (50, 32000):
        r = two_node_round(0, p_cpu)
        _, got, want = _run(schedule, r, excl=True)
        assert np.asarray(want.job_state)[0] == abi.JOB_FAILED


def two_node_rejected_twice(schedule):
    """The negative row on the second component, node 0 in the same bucket ([0, 100m) cpu) and rejected by its taint:
    the oracle reaches node 0, then node 1, re-seeks back to node 0 and counts it twice (2 under STATIC); the device
    counts it once (1 under STATIC, 1 implicit).  The reference fails the round there."""
    _run(schedule, two_node_round(1, 50), excl=True)


# ---- 4. the re-bind of evicted jobs onto UNSCHEDULABLE | OVERALLOCATED nodes --------------------------------------
def rebind_round(seed, flags, protected_fraction, n_nodes=60, n_jobs=300):
    """Preemptible running jobs (priority classes 0-2; evicted by the first step) on nodes over-allocated by one or two
    cpus; the flags go on those nodes."""
    r = synth.random_round(seed, n_nodes=n_nodes, n_queues=4, n_jobs=n_jobs, n_running=n_nodes * 2, gangs=False,
                           protected_fraction=protected_fraction)
    running = np.asarray(r.job_node).astype(np.int64) != abi.NONE
    n_shapes = len(r.class_request) // len(r.pcs)
    jc = np.asarray(r.job_class).astype(np.int64)
    jc = np.where(running & (jc >= 3 * n_shapes), jc - 3 * n_shapes, jc)  # no non-preemptible running job
    r.job_class = jc
    r.job_scheduled_at_priority = np.where(running, np.asarray(r.class_pc)[jc], abi.NO_PRIORITY)
    over_allocate(r, np.random.default_rng(seed), CPU, steps=1 + seed % 2, frac=0.5, flags=FLAGS[flags])
    return r


def rebind_shortcut(schedule, seed, flags, protected_fraction, excl=False, derive=False, n_nodes=60, n_jobs=300):
    """An evicted job re-binds to its node without the dynamic check when the node is UNSCHEDULABLE and OVERALLOCATED
    (nodedb.go:774-783); with either flag alone, or none, it needs the resources like any job.  With both flags the
    oracle re-binds some job that it does not re-bind once the flags are cleared, and the device reports it
    RESCHEDULED; with fewer flags the round equals the unflagged one."""
    r = rebind_round(seed, flags, protected_fraction, n_nodes, n_jobs)
    assert (level0_rows(r) < 0).any()
    inp, got, want = _run(schedule, r, excl=excl, derive=derive)
    assert int(want.stats.evicted_pass1) > 0
    r.node_flags = np.zeros_like(r.node_flags)
    plain = r.to_input()
    plain.collect_excluded_nodes = int(excl)
    if derive:
        plain.queue_allocated_by_pc = None
        plain.queue_constrained_demand = None
    unflagged = oracle_lib.round_schedule(plain)
    if flags == "both":
        st = np.asarray(got.job_state)
        decided = (st == abi.JOB_RESCHEDULED) & (np.asarray(unflagged.job_state) != abi.JOB_RESCHEDULED)
        assert decided.any(), "the flags decided no re-bind"
    else:
        assert not want.diff(unflagged)
    return got, want


# ---- larger rounds and the C5 shape (GPU tier) -----------------------------------------------------------------
def c5_over_allocated(schedule, scale=0.02, share=0.05):
    """C5 (pre-filled nodes, eviction and oversubscription) with 5 % of the nodes over-allocated by a non-preemptible
    job: a cpu node's 28 cpus of running jobs get 8 cpus more in priority class 3, 4 cpus over its 32."""
    r = synth.scaled("C5", scale)
    rng = np.random.default_rng(5)
    jn = np.asarray(r.job_node).astype(np.int64)
    N = np.asarray(r.node_total).shape[1]
    cpu_nodes = np.nonzero(np.asarray(r.node_type) == 0)[0]
    pick = np.sort(rng.choice(cpu_nodes, max(1, int(N * share)), replace=False))
    shapes = len(synth.SHAPES)
    cr, cpc, crow, = np.asarray(r.class_request), np.asarray(r.class_pc), np.asarray(r.class_static_row)
    r.class_request = np.concatenate([cr, synth.rl(8, 64)[None, :]])  # class `shapes`: 8 cpu, non-preemptible
    r.class_pc = np.concatenate([cpc, [3]])
    r.class_static_row = np.concatenate([crow, [0]])
    r.pcs = tuple(synth.PCS)
    k = len(pick)
    r.job_class = np.concatenate([np.asarray(r.job_class), np.full(k, shapes)])
    r.job_queue = np.concatenate([np.asarray(r.job_queue), rng.integers(0, 32, k)])
    J = len(jn)
    r.job_submit_time = np.arange(J + k)
    r.job_node = np.concatenate([jn, pick])
    r.job_scheduled_at_priority = np.concatenate([np.asarray(r.job_scheduled_at_priority), np.full(k, 3)])
    r.job_active_run_timestamp = np.concatenate([np.asarray(r.job_active_run_timestamp), J + np.arange(k)])
    rows = level0_rows(r)
    assert (rows[CPU, pick] < 0).all()
    got, want = rc.assert_parity(schedule, r.to_input(), f"C5@{scale} over-allocated")
    assert int(want.stats.evicted_pass1) > 0
