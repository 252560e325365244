"""Rounds uploaded as the cluster reports them (armada_round_upload_cluster): cordoned nodes with and without jobs,
jobs of other pools on a share of the nodes (some overfilling a node, some making its rows unaligned), round and
per-queue caps as fractions, floating resources, pod limits.  Shared by the emulator and GPU modules.

Every case checks, bit for bit:
  (a) armada_round_upload_cluster on the raw inputs, run and downloaded,
  (b) armada_round_upload on the inputs model.ClusterSnapshot derives, in the caller's node numbering,
  (c) the oracle on those derived inputs,
and armada_round_download_snapshot against model.ClusterSnapshot.  (b) and (c) test the round on the derived node set;
the derivation itself is checked against a restatement written on the specs instead (model.populate_node_db, through
the RoundInputBuilder: tests/cluster_specs.py) and against the reference's TestPopulateNodeDb table."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import Optional

import numpy as np

import oracle_lib
from armada_b200 import abi, synth
from armada_b200.model import ClusterSnapshot, RoundResult

CPU, MEM, GPU = synth.CPU, synth.MEM, synth.GPU
INF = float("inf")


@dataclass
class Case:
    seed: int
    n_nodes: int = 60
    n_jobs: int = 400
    n_running: int = 160
    cordon: float = 0.15          # share of the nodes reported cordoned (about half of them run jobs of this pool)
    other: float = 0.2            # share of the nodes running jobs of other pools
    overfill: float = 0.3         # share of those whose other-pool jobs overfill them
    unaligned: bool = False       # other-pool requests that are not multiples of the index resolution (exact mode)
    limits: bool = False          # round cap and per-queue caps as fractions
    floating: bool = False        # one floating resource after the node resources
    pods: Optional[int] = None    # RespectNodePodLimits with this many pods per node
    derive_queues: bool = True    # the queue accounting derived on the device too (NULL arrays)

    @property
    def name(self) -> str:
        return "-".join(f"{k}={v}" for k, v in vars(self).items())


def build(case: Case):
    """(inp, cs) of one case; the arrays they point into live on the structs."""
    return to_cluster(synth.random_round(case.seed, n_nodes=case.n_nodes, n_jobs=case.n_jobs, n_running=case.n_running), case)


def c3_round(share_running: float = 0.25) -> synth.RawRound:
    """C3 at full size with a quarter of its jobs of the two small cpu shapes running, up to 8 per cpu node."""
    r = synth.config_c3()
    cls = np.asarray(r.job_class).astype(np.int64)
    cpu_nodes = np.nonzero(np.asarray(r.node_type) == 0)[0]
    small = np.nonzero(cls < 2)[0]
    run = small[: min(int(len(cls) * share_running), 8 * len(cpu_nodes))]
    jn = np.full(len(cls), abi.NONE, np.int64)
    jn[run] = cpu_nodes[np.arange(len(run)) % len(cpu_nodes)]
    r.job_node = jn
    r.job_scheduled_at_priority = np.where(jn != abi.NONE, 0, abi.NO_PRIORITY)
    r.job_active_run_timestamp = np.arange(len(cls))
    return r


def to_cluster(r: synth.RawRound, case: Case):
    """`r` as the cluster reports it, per `case` (its size fields are not read)."""
    rng = np.random.default_rng(case.seed)
    if case.pods is not None:
        r = synth.with_pod_limits(r, case.pods)
    D, N = r.node_total.shape
    fdim = None
    if case.floating:  # a resource no node holds: in the accounting and DRF, never in a node fit
        fdim = D
        r.indexed = list(r.indexed) if r.indexed is not None else list(synth.INDEXED)
        r.node_total = np.vstack([r.node_total, np.zeros((1, N), np.int64)])
        r.node_allocatable = np.vstack([r.node_allocatable, np.zeros((1, N), np.int64)])
        col = rng.integers(0, 3, len(r.class_request))[:, None] * 1000
        r.class_request = np.hstack([np.asarray(r.class_request, np.int64), col])
        if r.drf_multipliers is not None:
            r.drf_multipliers = list(r.drf_multipliers) + [1.0]
        D += 1
    # cordoned as reported: the node carries the unschedulable taint (static classes 2, 3 = 0, 1 with it; no row
    # tolerates it)
    kind = np.asarray(r.node_static_class).astype(np.int64)
    jn = np.asarray(r.job_node).astype(np.int64)
    if (np.bincount(jn[jn != abi.NONE], minlength=N) > 0).all():  # every node busy: the jobs of one go back to the queue
        gang = np.asarray(r.job_gang).astype(np.int64) if r.job_gang is not None else np.full(len(jn), abi.NONE)
        n = int(next(n for n in range(N) if (gang[jn == n] == abi.NONE).all()))
        back = jn == n
        jn[back] = abi.NONE
        r.job_node = jn
        r.job_scheduled_at_priority = np.where(back, abi.NO_PRIORITY, r.job_scheduled_at_priority)
        r.job_queue = np.where(back & (np.asarray(r.job_queue).astype(np.int64) == abi.NONE), 0, r.job_queue)
    busy = np.zeros(N, bool)
    busy[jn[jn != abi.NONE]] = True
    cordoned = rng.random(N) < case.cordon
    cordoned[np.nonzero(busy)[0][:1]] = True   # at least one cordoned node with jobs …
    cordoned[np.nonzero(~busy)[0][:1]] = True  # … and one without
    r.node_flags = np.where(cordoned, abi.NODE_UNSCHEDULABLE, 0).astype(np.uint8)
    r.node_static_class = np.where(cordoned, kind + 2, kind).astype(np.uint32)
    r.num_static_classes = 4
    inp = r.to_input()
    Q, PC = inp.num_queues, inp.num_priority_classes
    # jobs of other pools
    used = np.zeros((D, N), np.int64)
    req = np.asarray(r.class_request, np.int64)[np.asarray(r.job_class).astype(np.int64)]
    np.add.at(used.T, jn[jn != abi.NONE], req[jn != abi.NONE])
    alloc = np.asarray(r.node_allocatable, np.int64)
    on, oreq = [], []
    for n in np.nonzero(rng.random(N) < case.other)[0]:
        for _ in range(int(rng.integers(1, 4))):
            q = np.zeros(D, np.int64)
            q[CPU] = int(rng.choice([250, 1000, 2000])) if case.unaligned else int(rng.choice([1000, 2000]))
            q[MEM] = int(rng.choice([1, 4])) * synth.GI + (int(rng.integers(1, 100)) * synth.MI if case.unaligned else 0)
            if case.pods is not None:
                q[synth.D] = 1  # (pods sit right after cpu, memory and gpu)
            if rng.random() < case.overfill:
                q[CPU] = max(q[CPU], int(alloc[CPU, n] - used[CPU, n]) + 1000)
            used[:, n] += q
            on.append(n)
            oreq.append(q)
    K = len(on)
    cs = abi.ClusterState()
    cs.abi_version = abi.ABI_VERSION
    cs.num_other_pool_jobs = K
    keep = []
    abi.attach(cs, keep, other_pool_job_node=np.asarray(on or [0]), other_pool_job_request=np.asarray(oreq or [np.zeros(D)]),
               static_class_unschedulable=[2, 3, abi.NONE, abi.NONE])
    for d in range(abi.MAX_RESOURCES):
        cs.max_fraction_to_schedule[d] = INF
    if case.limits:
        cs.has_round_limit = 1
        cs.max_fraction_to_schedule[CPU] = 0.3
        cs.max_fraction_to_schedule[MEM] = 0.45
        qf = np.full((Q, PC, D), INF)
        qf[:, :, CPU] = rng.choice([0.1, 0.25, 1.0], (Q, PC))
        qf[0, :, MEM] = 0.2
        abi.attach(cs, keep, queue_limit_fraction=qf)
        abi.attach(inp, inp._keepalive, queue_has_limit=np.ones((Q, PC)))
    cs._keepalive = keep
    if fdim is not None:
        inp.floating_resource_mask = 1 << fdim
        inp.floating_limits_configured = 1
        inp.floating_limit[fdim] = 40_000
    if case.derive_queues:
        inp.queue_allocated_by_pc = None
        inp.queue_constrained_demand = None
    # what the case was built to reach
    assert (cordoned & busy).any() and (cordoned & ~busy).any()
    return inp, cs


def run_cluster(dev, inp, cs, capfd=None):
    """(result, exact): the round uploaded with armada_round_upload_cluster; with `capfd`, also whether the upload
    chose exact mode (from its layout line), else None."""
    exact = None
    if capfd is not None:
        capfd.readouterr()
        os.environ["ARMADA_TIME_UPLOAD"] = "1"
    try:
        dev.upload_cluster(inp, cs)
    finally:
        if capfd is not None:
            del os.environ["ARMADA_TIME_UPLOAD"]
            exact = bool(int(re.findall(r"smem layout: .* exact (\d)", capfd.readouterr().err)[-1]))
    res = RoundResult(inp)
    res.stats = dev.run()
    return dev.download(res), exact


def check(dev, case: Case, capfd) -> ClusterSnapshot:
    """`capfd`: the round must run in exact mode exactly when the case makes rows unaligned."""
    return check_inputs(dev, *build(case), case.name, capfd, case.unaligned)


def check_inputs(dev, inp, cs, name: str, capfd=None, want_exact=None) -> ClusterSnapshot:
    cl = ClusterSnapshot(inp, cs)
    got_a, exact = run_cluster(dev, inp, cs, capfd)
    if want_exact is not None:
        assert exact == want_exact, f"{name}: exact mode {exact}, the case was built for {want_exact}"
    snap = dev.download_snapshot()
    for k, v in cl.snapshot.items():
        assert np.array_equal(snap[k], v), f"{name}: download_snapshot {k} != model"
    got_b = cl.in_caller_nodes(dev.schedule(cl.input), inp)
    want = cl.in_caller_nodes(oracle_lib.round_schedule(cl.input), inp)
    for label, got in (("upload_cluster", got_a), ("upload of the derived input", got_b)):
        bad = got.diff(want)
        assert not bad, f"{name}: {label} != oracle:\n  " + "\n  ".join(bad)
    state = cl.snapshot["node_state"]
    assert (state & abi.NODE_DROPPED).any(), "no node dropped"
    assert (state & abi.NODE_OVERALLOCATED).any(), "no node over-allocated"
    assert len(cl.kept) < inp.num_nodes
    return cl
