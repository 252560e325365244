"""Rounds of every resource count the schedule pass accepts (D = 1…8) and every best-fit key layout it chooses
between, built from a seed; shared by the emulator and GPU parity modules.

`k_schedule_pass<D>` is instantiated for D = 1, 2, 3, 4 and 8 (5–8 resources run `<8>` with run-time `d < D`
guards), and the batch assignment loop has three forms picked at upload from the key layout
(armada_host.inc, "the best-fit key packs into 64 bits"):
  k32        every resource indexed, guard bits kept, fields (without guards) <= 26 bits and with guards <= 31
  k64        every resource indexed, guard bits kept, wider fields                      (chain_swar<false>)
  unguarded  every resource indexed, the key fits 63 bits only without guard bits        (chain_run)
  run        not every resource indexed                                                  (chain_run)
  exact      quantities that are not multiples of their index resolution (no batch loop; literal walks)
A round whose key does not fit 63 bits at all is refused with E_UNSUPPORTED.

Resources are a prefix of (cpu, memory, gpu) followed by extras: ephemeral-storage and single-seat licences. Every
quantity is a whole number of quanta of its resource; a layout widens a field by k bits by refining the index
resolution (the quantities stay) or, where the quantum has no factor 2**k, by measuring the resource in 2**-k
quanta at resolution 1.  The extras are scarce (one licence seat per node), so jobs fail on them.

The library reports the layout it chose on the "smem layout" line it prints under ARMADA_TIME_UPLOAD;
`layout_of` reads it, and every case asserts the form it was built for."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np
import pytest

from armada_b200 import abi, synth

GI = synth.GI
# resources 0–7: cpu [milli], memory [bytes], gpu [milli], ephemeral-storage [bytes], licence-a … licence-d [seats]
QUANTUM = [1000, 16 * GI, 1000, 64 * GI, 1, 1, 1, 1]
# node capacity in quanta for the three node kinds: small cpu node, cpu node, gpu node (tainted)
NODE_Q = np.array([[16, 32, 64], [8, 16, 64], [0, 0, 4], [1, 2, 3], [1, 1, 1], [1, 1, 1], [1, 1, 1], [1, 1, 1]], np.int64)
PCS = synth.PCS
FORMS = ("k32", "k64", "unguarded", "run", "exact")


def instantiation(D: int) -> int:
    """The k_schedule_pass<D> template argument a round with D resources runs."""
    return D if D <= 4 else 8


def bits_for(v: int) -> int:
    return int(v).bit_length()


@dataclass(frozen=True)
class Case:
    D: int
    form: str                       # one of FORMS, or "refused" (key wider than 63 bits)
    kind: str                       # "batch" | "eviction"
    seed: int
    n_nodes: int = 60
    n_queues: int = 5
    n_jobs: int = 0                 # 0: sized from the node count
    fields: int = 0                 # total width of the resource fields (0: whatever the form needs)
    order: Optional[Tuple[int, ...]] = None   # indexed resources in index order (default: resource order)
    edges: bool = False             # + a class of exactly the largest node, + a class larger than every node
    tag: str = ""

    @property
    def id(self) -> str:
        parts = [f"D{self.D}", self.form, self.kind, f"s{self.seed}"]
        if self.n_nodes != 60:
            parts.append(f"n{self.n_nodes}")
        if self.n_queues != 5:
            parts.append(f"q{self.n_queues}")
        if self.fields:
            parts.append(f"f{self.fields}")
        if self.order is not None:
            parts.append("o" + "".join(map(str, self.order)))
        if self.tag:
            parts.append(self.tag)
        return "-".join(parts)


def _node_kinds(N: int, rng) -> np.ndarray:
    """0 small cpu node, 1 cpu node, 2 gpu node (one in four, spread over the id order)."""
    kind = np.where(rng.random(N) < 0.3, 0, 1).astype(np.int64)
    n_gpu = N // 4
    if n_gpu:
        kind[np.floor(np.arange(n_gpu) * (N / n_gpu)).astype(np.int64)] = 2
    return kind


def _plan(case: Case, maxq: np.ndarray, indexed: Sequence[int], N: int):
    """Per resource: (value of one quantum, index resolution) so that the key has the form the case asks for."""
    D = case.D
    unit = [QUANTUM[d] for d in range(D)]
    res = [QUANTUM[d] for d in range(D)]
    base = {d: max(1, bits_for(int(maxq[d]))) for d in indexed}
    nb = bits_for(N - 1 if N > 1 else 1)
    R = len(indexed)
    F = sum(base.values())
    if case.fields:
        target = case.fields
    elif case.form == "k64":
        target = max(F + 10, 27)                  # memory at 1 MiB resolution, or a cpu field as wide
    elif case.form == "unguarded":
        target = 63 - nb - (R - 1) // 2           # fits 63 bits, but not with one guard bit per field
    elif case.form == "refused":
        target = 64 - nb + 2
    else:
        target = F
    extra = target - F
    assert extra >= 0, (case.id, F, target)
    # memory takes the extra bits first (finer resolution), then cpu
    for d in ([1, 0] if 1 in indexed else [0] + [d for d in indexed if d != 0]):
        if extra <= 0 or d not in indexed:
            continue
        k = min(extra, 34 if d == 1 else 46)
        if QUANTUM[d] % (1 << k) == 0:
            res[d] = QUANTUM[d] >> k
        else:
            unit[d], res[d] = 1 << k, 1
        extra -= k
    assert extra == 0, case.id
    return unit, res


def shape_round(case: Case) -> synth.RawRound:
    D, seed, N, Q = case.D, case.seed, case.n_nodes, case.n_queues
    rng = np.random.default_rng(10_000 + seed)
    batch = case.kind == "batch"
    kind = _node_kinds(N, rng)
    capq = NODE_Q[:D, :][:, kind].copy()                 # [D][N] quanta
    # classes: (cpu, memory, gpu, storage, licences…) in quanta; gpu classes tolerate the gpu taint
    shapes, rows = [], []
    n_shapes = 9
    for s in range(n_shapes):
        gpu = s % 4 == 3
        q = np.array([rng.choice([1, 2, 4, 8, 16]), rng.choice([1, 2, 4, 8]), 1 if gpu else 0, int(rng.random() < 0.4)]
                     + [int(rng.random() < 0.35) for _ in range(4)], np.int64)[:D]
        shapes.append(q)
        rows.append(1 if gpu or s % 5 == 0 else 0)
    if case.edges:
        big = capq[0].max()
        shapes.append(np.concatenate([[big], np.ones(D - 1, np.int64)])[:D])      # exactly the largest node's cpu
        rows.append(1)
        shapes.append(np.concatenate([[2 * NODE_Q[0].max()], np.zeros(D - 1, np.int64)])[:D])  # larger than every node
        rows.append(1)
    npc = 1 if batch else len(PCS)
    pcs = list(PCS[:npc])
    pc_away = None
    cls_q, cls_pc, cls_row, away_rows = [], [], [], []
    for pc in range(npc):
        for q, rw in zip(shapes, rows):
            cls_q.append(q)
            cls_pc.append(pc)
            cls_row.append(rw)
            away_rows.append([abi.NONE] * abi.MAX_AWAY)
    away = not batch and seed % 2 == 1
    if away:  # home priority 30000, away 29000 on the gpu nodes
        pcs.append((30000, True))
        pc_away = {len(pcs) - 1: [29000]}
        for q, rw in zip(shapes[:5], rows[:5]):
            cls_q.append(q)
            cls_pc.append(len(pcs) - 1)
            cls_row.append(rw)
            away_rows.append([1] + [abi.NONE] * (abi.MAX_AWAY - 1))
    cls_q = np.stack(cls_q)
    Cn = len(cls_q)

    if case.order is not None:
        indexed = list(case.order)
    elif case.form == "run":  # the extras (D = 2: memory) are not indexed
        indexed = [0] if D == 2 else list(range(min(D, 3)))
    else:
        indexed = list(range(D))
    unit, res = _plan(case, capq.max(axis=1), indexed, N)
    unit = np.array(unit, np.int64)

    n_jobs = case.n_jobs or min(20_000, max(40, 25 * N))
    n_running = 0 if batch else max(4, n_jobs // 4)
    J = n_jobs + n_running
    job_class = rng.integers(0, Cn, J)
    job_queue = rng.integers(0, Q, J)
    job_node = np.full(J, abi.NONE, np.int64)
    sap = np.full(J, abi.NO_PRIORITY, np.int64)
    art = np.zeros(J, np.int64)
    # running jobs: placed greedily, never over any of the D resources of a node
    free = capq.copy()
    placed = 0
    for j in range(n_jobs, J):
        c = job_class[j]
        ok_kind = (kind != 2) | (cls_row[c] == 1) | (away_rows[c][0] != abi.NONE)
        cand = np.nonzero((free >= cls_q[c][:, None]).all(axis=0) & ok_kind)[0]
        if len(cand) == 0:
            continue
        n = int(cand[rng.integers(0, len(cand))])
        free[:, n] -= cls_q[c]
        job_node[j] = n
        pc = cls_pc[c]
        sap[j] = pcs[pc][0] if rng.random() < 0.8 else abi.NO_PRIORITY
        if away and pc == len(pcs) - 1 and kind[n] == 2:
            sap[j] = 29000
        art[j] = placed
        placed += 1
    gang = np.full(J, abi.NONE, np.int64)
    cards = []
    if batch and seed % 2 == 1:  # simple gangs: contiguous members of one class in one queue
        j = 0
        while j < n_jobs - 8:
            if rng.random() < 0.04:
                s = int(rng.integers(2, 6))
                gang[j:j + s] = len(cards)
                cards.append(s)
                job_class[j:j + s] = job_class[j]
                job_queue[j:j + s] = job_queue[j]
                j += s
            else:
                j += 1

    total = capq * unit[:, None]
    req = cls_q * unit[None, :]
    if case.form == "exact":
        # quantities off the index resolution: cpu nodes a little short of whole cores, 250m requests
        total[0] -= rng.integers(0, 4, N) * 30
        req[::3, 0] += 250
    drf = np.array([1.0, 0.0, 0.5, 3.0])[rng.integers(0, 4, D)]
    if D >= 5:
        drf[4] = 3.0   # licence-a is the dominant resource of the queues that hold seats: lanes 4–7 of the DRF cost
    limit = qlimit = None
    if not batch and seed % 3 == 2:
        limit = (total.sum(axis=1) * 0.3).astype(np.int64)
    if not batch and seed % 3 == 1:
        qlimit = np.full((Q, len(pcs), D), synth.I64_MAX, np.int64)
        qlimit[:, :, seed % D] = int(total[seed % D].sum() * 0.2)
    static_match = synth._bitmap([[0], [0, 1]], 2)
    typ = (kind == 2).astype(np.uint32)
    return synth.RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=typ, node_static_class=typ,
        num_node_types=2, num_static_classes=2,
        class_request=req, class_pc=np.array(cls_pc), class_static_row=np.array(cls_row),
        class_away_row=np.array(away_rows, np.uint32), static_match=static_match, type_match=static_match.copy(),
        job_class=job_class, job_queue=job_queue, job_submit_time=rng.permutation(J), job_node=job_node,
        job_scheduled_at_priority=sap, job_active_run_timestamp=art, job_queue_priority=rng.integers(0, 3, J),
        job_gang=gang if cards else None, gang_cardinality=np.array(cards, np.uint32) if cards else None,
        queue_weight=np.array([1.0, 0.5, 0.25, 2.0])[np.arange(Q) % 4], pcs=tuple(pcs), pc_away=pc_away,
        priorities=tuple(synth.PRIORITIES), protected_fraction=0.0 if batch else 0.5,
        round_limit=limit, queue_limit=qlimit, indexed=indexed, resolution=[res[d] for d in indexed],
        drf_multipliers=drf, name=case.id)


# ---- the layout the library chose ----------------------------------------------------------------------
_LAYOUT = re.compile(r"smem layout: .* exact (\d+) swar_ok (\d+) k32_ok (\d+) key_total_bits (\d+) node_bits (\d+) bt_wq (\d+)")


def layout_of(err: str) -> dict:
    """The fields of the last "smem layout" line in a captured stderr."""
    m = _LAYOUT.findall(err)
    assert m, "no layout line on stderr (ARMADA_TIME_UPLOAD)"
    keys = ("exact", "swar_ok", "k32_ok", "key_total_bits", "node_bits", "bt_wq")
    return dict(zip(keys, map(int, m[-1])))


def form_of(layout: dict, inp) -> str:
    if layout["exact"]:
        return "exact"
    if layout["swar_ok"]:
        return "k32" if layout["k32_ok"] else "k64"
    return "run" if inp.num_indexed < inp.num_resources else "unguarded"


def schedule_with_layout(dev, inp, capfd):
    """dev.schedule(inp) with the upload's layout line switched on; returns (result, layout, form).  A refused
    upload raises as usual."""
    capfd.readouterr()
    try:
        with knob("ARMADA_TIME_UPLOAD", 1):
            got = dev.schedule(inp)
    finally:
        err = capfd.readouterr().err
    lay = layout_of(err)
    return got, lay, form_of(lay, inp)


def check_case(case: Case, dev, oracle_round, capfd):
    """One case through `dev` against the oracle: the form it was built for, then every output array."""
    r = shape_round(case)
    inp = r.to_input()
    if case.form == "run" and case.kind == "batch":
        inp.collect_excluded_nodes = 1
    if case.form == "refused":
        with pytest.raises(abi.ArmadaError) as ei:
            dev.schedule(inp)
        assert ei.value.status == abi.E_UNSUPPORTED and "63 bits" in str(ei.value)
        with pytest.raises(abi.ArmadaError):   # nothing was uploaded, so nothing runs
            dev.run()
        return None, None
    want = oracle_round(inp)
    got, lay, form = schedule_with_layout(dev, inp, capfd)
    assert form == case.form, f"{case.id}: built for {case.form}, the library chose {form} ({lay})"
    if case.fields:
        assert lay["key_total_bits"] - lay["node_bits"] == case.fields + (inp.num_indexed if lay["swar_ok"] else 0)
    bad = got.diff(want)
    assert not bad, f"{case.id}: device != oracle:\n  " + "\n  ".join(bad)
    if case.kind == "batch" and case.form != "exact" and case.n_nodes >= 32:  # (1–2 nodes may fill up before a batch)
        assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0, "expected batch-mode iterations"
    if case.form == "run" and case.kind == "batch":
        ex = np.asarray(want.job_excluded_nodes)
        assert ex[:, abi.EXCL_RESOURCES].sum() > 0, "the unindexed extras never rejected a reached node"
    return got, want


# ---- the case matrix -------------------------------------------------------------------------------------
def _matrix():
    cases = []
    s = 0
    for D in (1, 2, 4, 5, 6, 7, 8):
        forms = ["k32", "k64", "run", "exact"]
        if D == 8:
            forms.append("unguarded")
        for form in forms:
            for kind in ("batch", "eviction"):
                s += 1
                if D == 1 and form == "run":   # one resource: chain_run only when the key drops its guard bit
                    cases.append(Case(1, "unguarded", kind, s, n_nodes=4097, n_jobs=1500))
                else:
                    cases.append(Case(D, form, kind, s))
    # field edges: K32 needs the fields within 26 bits and, with one guard bit each, within 31.  D = 8 with 26-bit
    # fields once ran K32 on a 32-bit word that lost its top fields (wrong nodes); it must run K64
    for D, f, form in ((3, 26, "k32"), (3, 27, "k64"), (5, 26, "k32"), (5, 27, "k64"), (8, 23, "k32"), (8, 24, "k64"), (8, 26, "k64")):
        s += 1
        cases.append(Case(D, form, "batch", s, fields=f, edges=True))
    cases.append(Case(3, "k32", "batch", 80, order=(2, 0, 1), edges=True))
    cases.append(Case(3, "k64", "eviction", 81, order=(1, 2, 0)))
    cases.append(Case(8, "k32", "batch", 82, order=(7, 3, 1, 5, 0, 2, 6, 4), edges=True))
    cases.append(Case(8, "k64", "batch", 83, order=(1, 0, 2, 3, 4, 5, 6, 7), edges=True))
    cases.append(Case(3, "unguarded", "batch", 84))
    cases.append(Case(3, "unguarded", "eviction", 85))
    # node counts: node_bits boundaries and the warp width
    for D in (1, 8):
        for n in (1, 2, 32, 33):
            s += 1
            cases.append(Case(D, "k32", "batch", s, n_nodes=n))
    return cases


MATRIX = _matrix()
# a key wider than 63 bits is refused; the same nodes and jobs with the widest field coarsened or unindexed run
REFUSED = Case(8, "refused", "batch", 90)
REFUSED_COARSENED = Case(8, "k64", "batch", 90, fields=40, tag="coarsened")
REFUSED_UNINDEXED = Case(8, "run", "batch", 90, order=(0, 2, 3, 4, 5, 6, 7), tag="unindexed")


def expected_pairs():
    """(instantiation, form) pairs the matrix must reach."""
    want = {(i, f) for i in (1, 2, 4, 8) for f in ("k32", "k64", "exact")}
    want |= {(1, "unguarded"), (2, "run"), (4, "run"), (8, "run"), (3, "unguarded"), (8, "unguarded")}
    want |= {(3, "k32"), (3, "k64")}  # (the field-edge and index-order cases at D = 3)
    return want


# ---- test knobs read by the library at upload (shared by the emulator and GPU modules) -----------------
@pytest.fixture(params=["k32", "k64"])
def compare_key(request):
    """The assignment loop compares 32-bit compact keys when the resource fields fit 26 bits
    (ARMADA_NO_K32 forces the general 64-bit form)."""
    if request.param == "k64":
        os.environ["ARMADA_NO_K32"] = "1"
    yield request.param
    os.environ.pop("ARMADA_NO_K32", None)


class knob:
    """Sets a library environment knob for the duration of a `with` block (None or "": leave it unset)."""

    def __init__(self, name: str, value):
        self.name, self.value = name, value

    def __enter__(self):
        if self.value not in (None, "", 0):
            os.environ[self.name] = str(self.value)
        return self

    def __exit__(self, *exc):
        os.environ.pop(self.name, None)


# ---- bodies of the knob tests (ARMADA_BT_WQ, ARMADA_NO_K32, ARMADA_FORCE_EXACT), run on either library ----
def long_batch_pipeline(make_dev, wq, seed):
    """Small batches (ARMADA_BT_WQ: items per queue per batch) make one pipeline run span many batches: batch k+1
    is produced from the speculative queue state while batch k is assigned, jobs that find no node cut a batch
    short (the batch built behind it is dropped), runs of known-unschedulable jobs sit between committed items."""
    import oracle_lib
    with knob("ARMADA_BT_WQ", wq):
        dev = make_dev()
        if seed == 503:
            r = synth.unfeasible_runs_round(7)
        else:
            r = synth.random_round(seed, n_nodes=24 + 10 * (seed % 3), n_queues=5 + seed % 4, n_jobs=1400, n_running=0, gangs=seed == 502,
                                   priorities=False, round_limit=seed == 501)
        inp = r.to_input()
        want = oracle_lib.round_schedule(inp)
        got = dev.schedule(inp)
        bad = got.diff(want)
        assert not bad, f"{r.name}: device != oracle:\n  " + "\n  ".join(bad)
        if seed != 503:
            assert int(got.stats.batch_cycles[abi.BATCH_COUNT]) >= {500: 8, 501: 2, 502: 3}[seed], "expected several batches per pipeline run"
        dev.close()


def gangs_as_batch_items(make_dev, nodes, queues, jobs, wq, seed):
    """Simple gangs (complete, one class, contiguous in their queue — what the C4 generator makes) are ordered by
    the batch pipeline as ONE item and placed member by member by the assignment loop, all or nothing: the
    clusters fill up, so gangs fail in the middle (roll-back of the table, of the touched bits and of the window a
    refill replaced) and the general loop fails them the reference's way."""
    import oracle_lib
    with knob("ARMADA_BT_WQ", wq):
        dev = make_dev()
        r = synth.config_c4(nodes, queues, jobs, seed=synth.SEED + seed)
        inp = r.to_input()
        want = oracle_lib.round_schedule(inp)
        got = dev.schedule(inp)
        bad = got.diff(want)
        assert not bad, f"C4 {nodes}x{jobs}: device != oracle:\n  " + "\n  ".join(bad)
        # gang members were placed in batch mode: more placements than iterations there
        assert int(got.stats.placements) > int(got.stats.loop_iterations) - int(np.count_nonzero(np.asarray(want.job_state) == 4))
        assert int(got.stats.phase_cycles[abi.PHASE_BATCH_ITERATIONS]) > 0
        dev.close()


def exact_mode_forced(make_dev, seed):
    """ARMADA_FORCE_EXACT: the literal walk on inputs the fast path also accepts gives the same round."""
    import oracle_lib
    with knob("ARMADA_FORCE_EXACT", 1):
        dev = make_dev()
        r = synth.random_round(seed, away=(seed % 4 == 1), n_nodes=60, n_jobs=350, n_running=90, protected_fraction=0.5 if seed else 0.0)
        inp = r.to_input()
        assert not dev.schedule(inp).diff(oracle_lib.round_schedule(inp))
        dev.close()
