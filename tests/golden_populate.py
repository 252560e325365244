"""The reference's TestPopulateNodeDb table (tests/golden/populate_node_db.json) as rounds uploaded with
armada_round_upload_cluster: one Test32CpuNode, cordoned or not, running N1Cpu4GiJobs of priority class 0.  The
library refuses a round without nodes, so every case has a second, empty and schedulable node; the table's
expectations are about the first.  Checked on the oracle (the derived round against the table), then the device
against the model and the oracle."""
from __future__ import annotations

import numpy as np

import oracle_lib
from armada_b200 import abi, synth
from armada_b200.model import ClusterSnapshot, RoundResult


def build(tc, node, job):
    n_jobs = tc["jobs"]
    J = n_jobs + 1  # + one queued job
    total = np.stack([synth.rl(node["cpu"], node["memory_gi"])] * 2, axis=1)
    r = synth.RawRound(
        node_total=total, node_allocatable=total.copy(), node_type=np.zeros(2), node_static_class=np.array([1 if tc["cordoned"] else 0, 0]),
        num_node_types=1, num_static_classes=2, node_flags=np.array([abi.NODE_UNSCHEDULABLE if tc["cordoned"] else 0, 0]),
        class_request=synth.rl(job["cpu"], job["memory_gi"])[None, :], class_pc=np.zeros(1), class_static_row=np.zeros(1),
        static_match=synth._bitmap([[0]], 2), type_match=synth._bitmap([[0]], 1),
        job_class=np.zeros(J), job_queue=np.zeros(J), job_submit_time=np.arange(J),
        job_node=np.array([0] * n_jobs + [abi.NONE]), job_scheduled_at_priority=np.array([0] * n_jobs + [abi.NO_PRIORITY]),
        job_active_run_timestamp=np.arange(J), queue_weight=np.ones(1), name=tc["name"])
    inp = r.to_input()
    cs = abi.ClusterState()
    cs.abi_version = abi.ABI_VERSION
    keep = []
    abi.attach(cs, keep, static_class_unschedulable=[1, abi.NONE])
    for d in range(abi.MAX_RESOURCES):
        cs.max_fraction_to_schedule[d] = float("inf")
    cs._keepalive = keep
    inp.queue_allocated_by_pc = None
    inp.queue_constrained_demand = None
    return inp, cs


def expect(cl: ClusterSnapshot, tc) -> None:
    state = int(cl.snapshot["node_state"][0])
    assert bool(state & abi.NODE_DROPPED) == (not tc["added"])
    if tc["added"]:
        assert bool(state & abi.NODE_UNSCHEDULABLE) == tc["unschedulable"]
        assert bool(state & abi.NODE_OVERALLOCATED) == tc["over_allocated"]
        jn = np.ctypeslib.as_array(cl.input.job_node, (cl.input.num_jobs,))
        assert (jn[: tc["jobs"]] == 0).all()  # every job is bound to the node (AllocatedByJobId)
        assert int(cl.snapshot["node_static_class"][0]) == (1 if tc["unschedulable"] else 0)


def check(dev, tc, golden) -> None:
    inp, cs = build(tc, golden["node"], golden["job"])
    cl = ClusterSnapshot(inp, cs)
    expect(cl, tc)
    want = cl.in_caller_nodes(oracle_lib.round_schedule(cl.input), inp)
    dev.upload_cluster(inp, cs)
    snap = dev.download_snapshot()
    for k, v in cl.snapshot.items():
        assert np.array_equal(snap[k], v), f"{tc['name']}: download_snapshot {k} != model"
    got = RoundResult(inp)
    got.stats = dev.run()
    bad = dev.download(got).diff(want)
    assert not bad, f"{tc['name']}: device != oracle:\n  " + "\n  ".join(bad)
