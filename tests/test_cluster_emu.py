"""armada_round_upload_cluster through the emulated kernels: the derived node set, total and caps against the Python
restatement, the round against armada_round_upload on the derived inputs and against the oracle; the refusals of a
malformed ArmadaClusterState; the reference's TestPopulateNodeDb table."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import cluster_cases as cc
import cluster_specs
import emu_lib
import golden_populate
from armada_b200 import abi
from armada_b200.scheduler import DeviceRound

_dev = None


def dev() -> DeviceRound:
    global _dev
    if _dev is None:
        _dev = emu_lib.emu_round()
    return _dev


CASES = [
    cc.Case(1),
    cc.Case(2, limits=True),
    cc.Case(3, unaligned=True),
    cc.Case(4, floating=True, limits=True),
    cc.Case(5, pods=6),
    cc.Case(6, cordon=0.3, other=0.4, derive_queues=False),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_cluster_round(case, capfd):
    cc.check(dev(), case, capfd)


def _malformed():
    """(name, edit of (inp, cs)) for every field the library validates."""
    def node(inp, cs):
        cs.other_pool_job_node[0] = inp.num_nodes

    def request(inp, cs):
        cs.other_pool_job_request[1] = -1

    def unsched(inp, cs):
        cs.static_class_unschedulable[0] = inp.num_static_classes

    def round_nan(inp, cs):
        cs.max_fraction_to_schedule[0] = float("nan")

    def queue_nan(inp, cs):
        qf = np.full((inp.num_queues, inp.num_priority_classes, inp.num_resources), cc.INF)
        qf[1, 0, 2] = float("nan")
        abi.attach(cs, cs._keepalive, queue_limit_fraction=qf)

    def version(inp, cs):
        cs.abi_version = abi.ABI_VERSION + 1

    def null_unsched(inp, cs):
        cs.static_class_unschedulable = None

    def null_jobs(inp, cs):
        cs.other_pool_job_node = None

    return [("other_pool_job_node", node), ("other_pool_job_request", request), ("static_class_unschedulable", unsched),
            ("max_fraction_to_schedule", round_nan), ("queue_limit_fraction", queue_nan), ("abi_version", version),
            ("null static_class_unschedulable", null_unsched), ("null other_pool_job_node", null_jobs)]


@pytest.mark.parametrize("name,edit", _malformed(), ids=[m[0] for m in _malformed()])
def test_malformed_cluster_state_is_refused(name, edit):
    inp, cs = cc.build(cc.Case(7, limits=True))
    edit(inp, cs)
    with DeviceRound(0, lib=emu_lib.load()) as d:
        with pytest.raises(abi.ArmadaError) as e:
            d.upload_cluster(inp, cs)
        assert e.value.status == abi.E_INVALID
        # nothing was computed: no snapshot, no round
        assert d.lib.armada_round_download_snapshot(d.h, None, None, None, None, None, None) == abi.E_STATE
        assert d.lib.armada_round_run(d.h, C.byref(abi.RoundStats())) == abi.E_STATE


def test_snapshot_needs_upload_cluster():
    """After a plain upload there is no derived snapshot to download."""
    inp, cs = cc.build(cc.Case(8))
    with DeviceRound(0, lib=emu_lib.load()) as d:
        d.upload_cluster(inp, cs)
        d.download_snapshot()
        from armada_b200.model import ClusterSnapshot
        d.upload(ClusterSnapshot(inp, cs).input)
        with pytest.raises(abi.ArmadaError) as e:
            d.download_snapshot()
        assert e.value.status == abi.E_STATE


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "populate_node_db.json")


with open(GOLDEN) as _f:
    TABLE = json.load(_f)


@pytest.mark.parametrize("tc", TABLE["cases"], ids=lambda tc: tc["name"])
def test_populate_node_db_table(tc):
    golden_populate.check(dev(), tc, TABLE)


SPEC_KNOBS = [{}, {"unaligned": True}, {"limits": True}, {"floating": True, "limits": True}, {"pods": True}]


@pytest.mark.parametrize("knobs", SPEC_KNOBS, ids=lambda k: "-".join(k) or "plain")
def test_builder_cluster_path_against_populate_node_db(knobs, capfd):
    cluster_specs.check(dev(), capfd, 3, **knobs)


def test_cluster_state_size_matches_the_library():
    assert emu_lib.load().armada_abi_sizeof(3) == C.sizeof(abi.ClusterState)
