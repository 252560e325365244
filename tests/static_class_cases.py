"""Rounds whose nodes fall into more than 32 and more than 256 static classes, shared by the emulator and GPU modules.

A node's static class is the set of taints and labels the job rows look at; a pool of many zones, instance types and
taints has many of them, and a row that selects on a per-node label (the hostname) makes one per node.  The kernels
read static classes in several ways that depend on their number S:
  S > 32     the batch assignment loop's shared class mask covers classes < 32 only: candidates of a class >= 32 are
             installed one at a time (install_general), and the duplicate-candidate check takes its wide form
  S > 256    a table slot's cached row of static_match (8 words) no longer holds the row: it is read from global memory
  any S      multi-word static_match rows in the exact-mode walks, the excluded-node counts, the dry-run NodeDb and the
             input validation.

`split_static_classes` gives every node a new class whose static_match bits, on every row (home, away and uniformity
rows alike), are those of its original class; node types, resources, jobs and rows stay.  The reference cannot tell
the two inputs apart, so every case checks
  (a) device == oracle on the split input, and
  (b) the oracle and the device on the split input == the oracle on the unsplit input, for every output array,
which does not trust the oracle's own multi-word static_match handling.

`placement` picks which classes the nodes get:
  interleaved  classes < 32 and >= 32 alternate along each key group of nodes (the order a window's G0 cursor lists
               them in), so that a batch install takes a prefix in bulk and hands the rest to install_general
  all_high     every node gets a class >= 32: every install goes through install_general
  boundary     classes 31, 32, 255 and 256 are all held by nodes
  per_node     one class per node (S = N)."""
from __future__ import annotations

import dataclasses

import numpy as np

import cluster_cases as cc
import explain_cases as ec
import gang_cases
import oracle_lib
import round_cases as rc
import shape_cases
from armada_b200 import abi, synth
from armada_b200.model import NODE_ID_LABEL, ClusterSnapshot, MatchExpression, RoundInputBuilder, _field, excluded_nodes_by_reason

BOUNDARY = (31, 32, 255, 256)


# ---- the transform ------------------------------------------------------------------------------------------
def expand_rows(static_match: np.ndarray, orig: np.ndarray) -> np.ndarray:
    """static_match [rows][ceil(K/32)] of the original classes -> [rows][ceil(S/32)] where class c has the bits of
    class orig[c]."""
    sm = np.asarray(static_match, np.uint32).reshape(len(static_match), -1)
    S = len(orig)
    bits = (sm[:, orig >> 5] >> (orig & 31).astype(np.uint32)) & 1
    w = (S + 31) // 32
    padded = np.zeros((len(sm), w * 32), np.uint8)
    padded[:, :S] = bits
    return np.packbits(padded.reshape(len(sm), w, 32), axis=2, bitorder="little").view("<u4").reshape(len(sm), w).astype(np.uint32)


def split_classes(node_class: np.ndarray, order_key: np.ndarray, K: int, S: int, placement: str, seed: int):
    """(new class per node [N], original class per new class [S]).  `order_key` [k][N]: lexicographic node order,
    last row first (the order the nodes of one original class are interleaved in)."""
    rng = np.random.default_rng(seed)
    old = np.asarray(node_class).astype(np.int64)
    N = len(old)
    if placement == "per_node":
        assert S == N, "per_node: one class per node"
        new = rng.permutation(N)
        orig = np.empty(S, np.int64)
        orig[new] = old
        return new.astype(np.uint32), orig
    assert S >= K
    orig = (np.arange(S) + int(rng.integers(K))) % K
    order = np.lexsort(np.vstack([order_key, old[None, :]]))
    # position of each node among the nodes of its original class, in that order
    pos = np.empty(N, np.int64)
    sorted_old = old[order]
    starts = np.searchsorted(sorted_old, sorted_old, side="left")
    pos[order] = np.arange(N) - starts
    if placement == "interleaved":
        high = pos % 2 == 1
    elif placement == "all_high":
        assert S >= 32 + K, "all_high needs a class >= 32 of every original class"
        high = np.ones(N, bool)
    elif placement == "boundary":
        assert S > max(BOUNDARY)
        high = rng.random(N) < 0.5
    else:
        raise ValueError(placement)
    new = np.empty(N, np.int64)
    cls = np.arange(S)
    for k in np.unique(old):
        for hi in (False, True):
            sel = order[(sorted_old == k) & (high[order] == hi)]
            if not len(sel):
                continue
            cand = cls[(orig == k) & ((cls >= 32) == hi)]
            if not len(cand):  # (S = 33: no class >= 32 of this original class)
                cand = cls[orig == k]
            new[sel] = cand[(np.arange(len(sel)) + int(rng.integers(len(cand)))) % len(cand)]
    if placement == "boundary":
        taken = np.zeros(N, bool)
        for t in BOUNDARY:
            n = int(np.nonzero((old == orig[t]) & ~taken)[0][0])
            new[n], taken[n] = t, True
        assert set(BOUNDARY) <= set(new.tolist())
    if placement == "all_high":
        assert (new >= 32).all()
    return new.astype(np.uint32), orig


def _order_key(node_index, allocatable) -> np.ndarray:
    """Nodes by allocatable (the best-fit key), then by their position in the index."""
    return np.vstack([np.asarray(node_index, np.int64)[None, :], np.asarray(allocatable, np.int64)[::-1]])


def split_static_classes(r: synth.RawRound, S_new: int, placement: str, seed: int):
    """(a copy of `r` with its nodes in S_new static classes of the same meaning, original class per new class)."""
    N = r.node_total.shape[1]
    index = r.node_index if r.node_index is not None else np.arange(N)
    new, orig = split_classes(r.node_static_class, _order_key(index, r.node_allocatable), r.num_static_classes, S_new, placement, seed)
    out = dataclasses.replace(r, node_static_class=new, static_match=expand_rows(r.static_match, orig), num_static_classes=S_new,
                              name=f"{r.name}/S{S_new}-{placement}", _keep=[])
    return out, orig


def split_input(inp: abi.RoundInput, S_new: int, placement: str, seed: int, cs: abi.ClusterState = None, attach=None):
    """split_static_classes on an input built elsewhere (RoundInputBuilder, cluster_cases), in place; `attach(**arrays)`
    points the input at the new arrays (default: abi.attach; a builder's `_attach` keeps its attributes in step).  With
    `cs`, each class's unschedulable variant becomes a class of the variant's original class, >= 32 where there is one.
    Returns the original class per new class."""
    N, D, K = inp.num_nodes, inp.num_resources, inp.num_static_classes
    sm = _field(inp, "static_match", inp.num_static_rows * ((K + 31) // 32)).reshape(inp.num_static_rows, -1)
    order = _order_key(_field(inp, "node_index", N), _field(inp, "node_allocatable", D * N).reshape(D, N))
    new, orig = split_classes(_field(inp, "node_static_class", N), order, K, S_new, placement, seed)
    (attach or (lambda **a: abi.attach(inp, inp._keepalive, **a)))(node_static_class=new, static_match=expand_rows(sm, orig))
    inp.num_static_classes = S_new
    if cs is not None:
        old_u = _field(cs, "static_class_unschedulable", K)
        last = {int(k): int(np.nonzero(orig == k)[0][-1]) for k in np.unique(orig)}
        u = np.array([abi.NONE if old_u[k] == abi.NONE else last[int(old_u[k])] for k in orig], np.uint32)
        abi.attach(cs, cs._keepalive, static_class_unschedulable=u)
    return orig


# ---- checks ------------------------------------------------------------------------------------------------
def check_same(label, got, want, base):
    """(a) device == oracle on the split input; (b) both == the oracle on the unsplit input, first-pass view included."""
    assert got.first_pass and want.first_pass and base.first_pass
    for who, a, b in (("device != oracle", got, want), ("oracle on the split input != unsplit", want, base),
                      ("device on the split input != oracle unsplit", got, base)):
        bad = a.diff(b)
        assert not bad, f"{label}: {who}:\n  " + "\n  ".join(bad)


def check_split(schedule, base: synth.RawRound, split: synth.RawRound, batch=False, prepare=None):
    """Both checks on one split round; `prepare(inp)` edits both inputs the same way.  Returns the device result."""
    base_inp, inp = base.to_input(), split.to_input()
    for i in (base_inp, inp):
        if prepare:
            prepare(i)
    base_res = oracle_lib.round_schedule(base_inp)
    got, want = rc.assert_parity(schedule, inp, split.name)
    check_same(split.name, got, want, base_res)
    if batch:
        assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0, f"{split.name}: expected batch-mode iterations"
    return got, want


def _twice(make, S, placement, seed):
    """(unsplit, split) of the round `make()` builds (built twice: a RawRound's input points into its own arrays)."""
    return make(), split_static_classes(make(), S, placement, seed)[0]


# ---- bodies: the batch pipeline -----------------------------------------------------------------------------
def batch_key_layout(dev, capfd, form, S, placement, seed, n_nodes, n_jobs):
    """The batch assignment loop with K32 or K64 compare keys, laid out the way tests/shape_cases.py lays them out."""
    case = shape_cases.Case(3, form, "batch", seed, n_nodes=n_nodes, n_jobs=n_jobs)
    base, split = _twice(lambda: shape_cases.shape_round(case), S or n_nodes, placement, seed)
    base_inp, inp = base.to_input(), split.to_input()
    want = oracle_lib.round_schedule(inp)
    got, lay, got_form = shape_cases.schedule_with_layout(dev, inp, capfd)
    assert got_form == form, f"{split.name}: built for {form}, the library chose {got_form} ({lay})"
    check_same(split.name, got, want, oracle_lib.round_schedule(base_inp))
    assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0, "expected batch-mode iterations"


def batch_chain_run(schedule, S, placement, seed, n_nodes, n_jobs, round_limit=False):
    """chain_run: not every resource is in the best-fit key (round_cases.partly_indexed_resources); with a round limit
    that trips inside a batch."""
    def make():
        r = synth.random_round(seed, n_nodes=n_nodes, n_queues=6, n_jobs=n_jobs, n_running=0, gangs=False, priorities=False,
                               round_limit=round_limit)
        r.indexed = [synth.CPU, synth.MEM]
        return r
    base, split = _twice(make, S, placement, seed)
    got, want = check_split(schedule, base, split, batch=True)
    if round_limit:
        assert want.out.num_result_scheduled < len(split.job_class)


def batch_gangs(schedule, S, placement, seed, n_nodes, n_queues, n_jobs, round_limit=None):
    """Simple gangs ordered by the batch pipeline as one item each (shape_cases.gangs_as_batch_items); `round_limit`: a
    cpu cap as a share of the pool, so that it trips in the middle of the pipeline."""
    def make():
        r = synth.config_c4(n_nodes, n_queues, n_jobs, seed=synth.SEED + seed)
        if round_limit is not None:
            lim = np.full(r.node_total.shape[0], synth.I64_MAX, np.int64)
            lim[synth.CPU] = int(r.node_allocatable[synth.CPU].sum() * round_limit)
            r.round_limit = lim
        return r
    base, split = _twice(make, S, placement, seed)
    got, want = check_split(schedule, base, split, batch=True)
    # gang members were placed in batch mode: more placements than iterations there
    assert int(got.stats.placements) > int(got.stats.loop_iterations) - int(np.count_nonzero(np.asarray(want.job_state) == abi.JOB_FAILED))
    if round_limit is not None:
        assert want.out.num_result_scheduled < len(split.job_class)


def scaled_per_node(schedule, name, scale):
    """A named config (synth.scaled) with a hostname-style static class per node."""
    base, split = _twice(lambda: synth.scaled(name, scale), synth.scaled(name, scale).node_total.shape[1], "per_node", 7)
    got, want = check_split(schedule, base, split, batch=True)
    assert got.out.num_result_scheduled == want.out.num_result_scheduled > 0


# ---- bodies: the general loop, exact mode, excluded nodes -----------------------------------------------------
def general_loop(schedule, S, placement, seed, unaligned=False, **sizes):
    """Running jobs, evictions and fair preemption, away jobs bound below their priority class (round_cases._seeded_round,
    or a round of `sizes` with protection and away jobs); `unaligned`: exact mode.  S = None: one class per node."""
    def make():
        if sizes:
            return synth.random_round(seed, protected_fraction=0.5, away=True, unaligned=unaligned, **sizes)
        return rc._seeded_round(seed, unaligned=unaligned)
    base, split = _twice(make, S or make().node_total.shape[1], placement, seed)
    got, want = check_split(schedule, base, split)
    assert (np.asarray(want.job_state) == abi.JOB_PREEMPTED).any()


def finer_than_types(r: synth.RawRound) -> synth.RawRound:
    """Half of the nodes of type 0 get a new static class that row 0 rejects (the node type still matches): the nodes
    a walk reaches and StaticJobRequirementsMet rejects count under ARMADA_EXCL_STATIC."""
    K = r.num_static_classes
    sc = np.asarray(r.node_static_class).astype(np.uint32).copy()
    sc[np.nonzero(np.asarray(r.node_type) == 0)[0][::2]] = K
    orig = np.append(np.arange(K), 0)
    sm = expand_rows(r.static_match, orig)
    sm[0, K >> 5] &= ~np.uint32(1 << (K & 31))
    return dataclasses.replace(r, node_static_class=sc, static_match=sm, num_static_classes=K + 1, _keep=[])


def excluded_nodes(schedule, S, placement, seed, n_nodes, n_jobs, disallowed=False):
    """collect_excluded_nodes: the per-kind counts are counts of nodes, the same however the nodes' classes are
    numbered.  `disallowed`: jobs that request gpus, which the pool disallows, count every node under
    ARMADA_EXCL_DISALLOWED."""
    def make():
        r = synth.random_round(760 + seed, n_nodes=n_nodes, n_queues=3, n_jobs=n_jobs, n_running=0 if disallowed else n_jobs // 5,
                               gangs=False, priorities=not disallowed)
        return r if disallowed else finer_than_types(r)

    def prepare(inp):
        inp.collect_excluded_nodes = 1
        if disallowed:
            inp.disallowed_resource_mask = 1 << synth.GPU

    base, split = _twice(make, S or n_nodes, placement, seed)
    got, want = check_split(schedule, base, split, prepare=prepare)
    ex = np.asarray(want.job_excluded_nodes)
    assert ex[:, abi.EXCL_DISALLOWED if disallowed else abi.EXCL_STATIC].sum() > 0


# ---- bodies: node-uniformity gangs through the builder ----------------------------------------------------------
def uniformity_per_node_classes(schedule, seed, **sizes):
    """gang_cases.uniformity_round with one queued job whose node affinity looks at the node-id label (Exists: every
    node passes): the builder derives one static class per node.  Unsplit, the same job's affinity asks for a label
    no node carries not to exist (DoesNotExist: every node passes), which adds no class."""
    def build(expr):
        b0 = gang_cases.uniformity_round(seed, **sizes)
        jobs = list(b0.jobs)
        j = next(i for i, x in enumerate(jobs) if x.node is None and x.gang_id is None)
        jobs[j] = dataclasses.replace(jobs[j], affinity=((expr,),))
        return RoundInputBuilder(b0.cfg, b0.nodes, jobs, b0.queues)
    base = build(MatchExpression("no-such-label", "DoesNotExist"))
    split = build(MatchExpression(NODE_ID_LABEL, "Exists"))
    N = split.input.num_nodes
    assert split.input.num_static_classes == N > 32 and base.input.num_static_classes < 32
    got, want = rc.assert_parity(schedule, split.input, f"uniformity {seed}, a class per node")
    check_same(f"uniformity {seed}", got, want, oracle_lib.round_schedule(base.input))


# ---- bodies: the dry-run NodeDb -----------------------------------------------------------------------------
def dry_run(make_nodedb, S, placement, seed, n_nodes, n_jobs, n_singles, n_gangs, max_gang, unaligned=False):
    """armada_nodedb_schedule_many / select_nodes on the split input against the oracle's NodeDb
    (round_cases.dry_run_case), and the oracle's verdicts and nodes against the unsplit input's."""
    def make():
        return synth.random_round(seed, n_nodes=n_nodes, n_jobs=n_jobs, n_running=0, gangs=False, unaligned=unaligned)
    base, split = _twice(make, S or n_nodes, placement, seed)
    rng = np.random.default_rng(seed)
    jc = np.asarray(split.job_class)
    J = len(jc)
    gangs = [[int(j)] for j in rng.choice(J, n_singles, replace=False)]
    for _ in range(n_gangs):
        same = np.nonzero(jc == jc[int(rng.integers(0, J))])[0]
        gangs.append(list(dict.fromkeys(int(same[i % len(same)]) for i in range(int(rng.integers(2, max_gang))))))
    assert any(rc.dry_run_case(make_nodedb, split, gangs))  # (a)
    odb, odb0 = oracle_lib.OracleNodeDb(split.to_input()), oracle_lib.OracleNodeDb(base.to_input())
    try:
        for g in gangs:
            (ok, nodes), (ok0, nodes0) = odb.dry_run(g), odb0.dry_run(g)
            assert ok == ok0 and (np.asarray(nodes) == np.asarray(nodes0)).all(), g
    finally:
        odb.close()
        odb0.close()


def explain(lib, S, placement, seed, **sizes):
    """armada_nodedb_explain on the split input against the oracle-backed reference of explain_cases.py; its records,
    with each static class mapped back to the original one, render to the unsplit input's NumExcludedNodesByReason."""
    base = ec.Case(seed, **sizes)
    want, _ = ec.check_case(base, lib)
    split = ec.Case(seed, **sizes)
    b = split.b
    orig = split_input(b.input, S or b.input.num_nodes, placement, seed, attach=b._attach)
    b.static_specs = [base.b.static_specs[int(k)] for k in orig]  # the taints and labels of each new class
    got, failed = ec.check_case(split, lib)  # (a)
    assert failed > 0
    static = 0
    for g, ((ok, node, placed, away, recs), (ok0, node0, placed0, away0, recs0)) in enumerate(zip(got, want)):
        assert (ok, placed, away) == (ok0, placed0, away0) and (node == node0).all(), g
        if not ok and len(split.groups[g]) == 1:
            cls = split.classes[g][0]
            static += sum(int(r.count) for r in recs if r.kind == abi.EXCL_STATIC)
            mapped = [abi.ExcludedReason(kind=r.kind, sub=int(orig[r.sub]) if r.kind == abi.EXCL_STATIC else r.sub, quantity=r.quantity,
                                         count=r.count) for r in recs]
            assert excluded_nodes_by_reason(base.b, cls, mapped) == excluded_nodes_by_reason(base.b, cls, recs0), g
    assert static > 0, "no node rejected on its static class"


# ---- bodies: the cluster upload -----------------------------------------------------------------------------
def cluster_upload(dev, capfd, S, placement, seed, **case_kw):
    """armada_round_upload_cluster with cordoned and over-allocated nodes whose unschedulable variants are classes >= 32:
    cluster_cases.check_inputs on the split input (a), and the round against the oracle on the unsplit input's derived
    node set (b)."""
    def oracle(inp, cs):
        cl = ClusterSnapshot(inp, cs)
        return cl.in_caller_nodes(oracle_lib.round_schedule(cl.input), inp)

    case = cc.Case(seed, **case_kw)
    base = oracle(*cc.build(case))
    inp, cs = cc.build(case)
    split_input(inp, S or inp.num_nodes, placement, seed, cs)
    u = _field(cs, "static_class_unschedulable", inp.num_static_classes)
    assert (u[u != abi.NONE] >= 32).all() and (u != abi.NONE).any()
    label = f"{case.name}/S{inp.num_static_classes}-{placement}"
    cc.check_inputs(dev, inp, cs, label, capfd, case.unaligned)
    check_same(label, cc.run_cluster(dev, inp, cs)[0], oracle(inp, cs), base)
