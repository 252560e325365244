"""armada_round_upload_cluster on the GPU: the emulator's cases, the same with thousands of nodes, and C3 at full size
(100 000 nodes, 1M jobs) with a few percent of its nodes cordoned and a fifth running jobs of other pools, some of
them over-allocated.  Each against armada_round_upload on the derived inputs, the oracle and the Python restatement."""
import json

import numpy as np
import pytest

import cluster_cases as cc
import cluster_specs
import golden_populate
from armada_b200.scheduler import DeviceRound
from test_cluster_emu import CASES, GOLDEN, SPEC_KNOBS

pytestmark = pytest.mark.gpu

_dev = None


def dev() -> DeviceRound:
    global _dev
    if _dev is None:
        _dev = DeviceRound(0)
    return _dev


BIG = [cc.Case(11, n_nodes=3000, n_jobs=20000, n_running=9000),
       cc.Case(12, n_nodes=4000, n_jobs=20000, n_running=12000, unaligned=True, limits=True),
       cc.Case(13, n_nodes=3000, n_jobs=15000, n_running=9000, floating=True, pods=8, limits=True)]


@pytest.mark.parametrize("case", CASES + BIG, ids=lambda c: c.name)
def test_cluster_round(case, capfd):
    cc.check(dev(), case, capfd)


with open(GOLDEN) as _f:
    TABLE = json.load(_f)


@pytest.mark.parametrize("tc", TABLE["cases"], ids=lambda tc: tc["name"])
def test_populate_node_db_table(tc):
    golden_populate.check(dev(), tc, TABLE)


def test_c3_cluster(capfd):
    r = cc.c3_round()
    inp, cs = cc.to_cluster(r, cc.Case(20, cordon=0.03, other=0.2, overfill=0.2, limits=True))
    cl = cc.check_inputs(dev(), inp, cs, "C3 cluster", capfd, want_exact=False)
    state = cl.snapshot["node_state"]
    assert 1000 <= len(cl.kept) < inp.num_nodes and int((state & 2 != 0).sum()) > 100


@pytest.mark.parametrize("knobs", SPEC_KNOBS, ids=lambda k: "-".join(k) or "plain")
def test_builder_cluster_path_against_populate_node_db(knobs, capfd):
    cluster_specs.check(dev(), capfd, 3, **knobs)


def test_cluster_state_size_matches_the_library():
    import ctypes as C
    from armada_b200 import abi
    assert abi.load_product().armada_abi_sizeof(3) == C.sizeof(abi.ClusterState)
