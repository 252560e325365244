"""Pools built from specs (NodeSpec / JobSpec / QueueSpec) for armada_round_upload_cluster: the RoundInputBuilder's
cluster path (other_pool_jobs given) against model.populate_node_db fed to the builder's explicit path.  The two routes
share no derivation code: the cluster path derives the node set on the device from the flattened pool as reported,
the explicit path restates populateNodeDb on the specs and flattens its result.

The pool: 12 Test32CpuNodes and 4 tainted Test8GpuNodes; nodes 0-3 cordoned, 0 and 1 running jobs of the pool, 2 running
only an other-pool job (dropped all the same), 3 empty (dropped); node 5 overfilled by another pool (over-allocated),
node 6 carrying a small other-pool job (its allocatable shrinks); an other-pool job on a node outside the pool (skipped).
Knobs: `unaligned` (an other-pool job of 1500m cpu: the rows leave the index resolution, exact mode), `limits` (round and
per-queue caps as fractions), `floating` (a floating resource with a pool total), `pods` (RespectNodePodLimits)."""
from __future__ import annotations

import os
import re
from dataclasses import replace

import numpy as np

import fixtures as fx_mod
import oracle_lib
from armada_b200 import abi
from armada_b200.model import (ClusterSnapshot, FloatingResource, QueueSpec, RoundInputBuilder, RoundResult, apply_respect_node_pod_limits,
                               populate_node_db, result_in_caller_nodes)

PC0, PC1 = fx_mod.PriorityClass0, fx_mod.PriorityClass1


def scenario(seed: int, unaligned=False, limits=False, floating=False, pods=False):
    rng = np.random.default_rng(seed)
    fx = fx_mod.Fixtures()
    cfg = fx_mod.test_scheduling_config()
    if limits:
        cfg.maximum_resource_fraction_to_schedule = {"cpu": 0.4, "memory": 0.7}
        cfg.priority_classes[PC0] = replace(cfg.priority_classes[PC0], maximum_resource_fraction_per_queue={"cpu": 0.3})
    extra = {}
    if floating:
        cfg.floating_resources = [FloatingResource("storage-connections", "1", "20")]
        extra = {"storage-connections": "1"}
    if pods:
        cfg.respect_node_pod_limits = True
        apply_respect_node_pod_limits(cfg)
    nodes = fx.n_cpu32(12) + [fx.gpu8_tainted() for _ in range(4)]
    if pods:
        for n in nodes:
            n.total = {**n.total, "pods": "10"}
    for i in range(4):
        nodes[i].unschedulable = True
    jobs = []
    running_on = [0, 1, 4, 5, 5, 6, 7, 8, 12]
    for k, i in enumerate(running_on):
        req = {"cpu": "8", "memory": "32Gi", **extra} if i == 5 else {"cpu": "1", "memory": "4Gi"}
        tol = (fx_mod.Toleration("gpu", "", "true"),) if i >= 12 else ()
        jobs.append(fx.job("A" if k % 2 else "B", PC0, req, tol, node=nodes[i].id, scheduled_at_priority=0))
    for _ in range(60):
        q = "A" if rng.random() < 0.6 else "B"
        shape = [{"cpu": "1", "memory": "4Gi"}, {"cpu": "4", "memory": "16Gi", **extra}, {"cpu": "16", "memory": "128Gi"}][int(rng.integers(0, 3))]
        jobs.append(fx.job(q, PC0 if rng.random() < 0.7 else PC1, shape))
    other = [fx.job("elsewhere", PC0, {"cpu": "2", "memory": "8Gi"}, node=nodes[2].id),
             fx.job("elsewhere", PC0, {"cpu": "20", "memory": "8Gi"}, node=nodes[5].id),
             fx.job("elsewhere", PC0, {"cpu": "2", "memory": "8Gi"}, node=nodes[6].id),
             fx.job("elsewhere", PC0, {"cpu": "1500m" if unaligned else "2", "memory": "1Gi"}, node=nodes[7].id),
             fx.job("elsewhere", PC0, {"cpu": "4", "memory": "8Gi"}, node="node-not-in-this-pool")]
    queues = [QueueSpec("A"), QueueSpec("B", priority_factor=2.0, resource_limits_by_pc={PC0: {"cpu": 0.2}} if limits else {})]
    return cfg, nodes, jobs, other, queues


def _derive_queues(inp):
    inp.queue_allocated_by_pc = None  # the queue accounting from the job arrays, on the device, on both routes
    inp.queue_constrained_demand = None


def check(dev, capfd, seed: int, **knobs):
    cfg, nodes, jobs, other, queues = scenario(seed, **knobs)
    bc = RoundInputBuilder(cfg, nodes, jobs, queues, other_pool_jobs=other)
    kept, total, constraints = populate_node_db(cfg, nodes, jobs, other, queues)
    bx = RoundInputBuilder(cfg, kept, jobs, queues, total_resources=total)
    _derive_queues(bc.input)
    _derive_queues(bx.input)
    kept_idx = [bc.node_pos[n.id] for n in kept]
    ids = [n.id for n in kept]
    assert [n.id for n in nodes if n.id not in ids] == [nodes[2].id, nodes[3].id]  # cordoned without a job of the pool
    assert [n.id for n in kept if n.over_allocated] == [nodes[5].id]
    # (a) the cluster path on the device
    capfd.readouterr()
    os.environ["ARMADA_TIME_UPLOAD"] = "1"
    try:
        dev.upload_cluster(bc.input, bc.cluster_state)
    finally:
        del os.environ["ARMADA_TIME_UPLOAD"]
    exact = int(re.findall(r"smem layout: .* exact (\d)", capfd.readouterr().err)[-1])
    want_exact = int(knobs.get("unaligned", False))
    assert exact == want_exact, f"exact mode {exact}, the case was built for {want_exact}"
    snap = dev.download_snapshot()
    got_a = RoundResult(bc.input)
    got_a.stats = dev.run()
    dev.download(got_a)
    # the snapshot against the spec-level restatement and the array-level one
    assert np.array_equal(snap["total_resources"], total)
    assert np.array_equal(snap["max_resources_to_schedule"], constraints["max_resources_to_schedule"])
    for q, qs in enumerate(bc.queues):
        for pc, name in enumerate(bc.pc_names):
            assert np.array_equal(snap["queue_limit"][q, pc], constraints["queue_limit"][qs.name][name])
    state = snap["node_state"]
    assert [i for i in range(len(nodes)) if not state[i] & abi.NODE_DROPPED] == kept_idx
    assert [bool(state[i] & abi.NODE_OVERALLOCATED) for i in kept_idx] == [n.over_allocated for n in kept]
    assert [bool(state[i] & abi.NODE_UNSCHEDULABLE) for i in kept_idx] == [n.unschedulable for n in kept]
    assert np.array_equal(snap["node_allocatable"][:, kept_idx], np.ctypeslib.as_array(bx.input.node_allocatable, (bx.factory.D, len(kept))))
    cl = ClusterSnapshot(bc.input, bc.cluster_state)
    for k, v in cl.snapshot.items():
        assert np.array_equal(snap[k], v), f"download_snapshot {k} != ClusterSnapshot"
    # (b) the explicit path on the device, (c) the oracle on it
    got_b = result_in_caller_nodes(dev.schedule(bx.input), kept_idx, bc.input)
    want = result_in_caller_nodes(oracle_lib.round_schedule(bx.input), kept_idx, bc.input)
    for label, got in (("upload_cluster", got_a), ("upload of populate_node_db's pool", got_b)):
        bad = got.diff(want)
        assert not bad, f"seed {seed} {knobs}: {label} != oracle:\n  " + "\n  ".join(bad)
    assert got_a.out.num_result_scheduled > 0
