"""More than 32 and more than 256 node static classes under the SIMT emulator (no GPU): each case splits the static
classes of a round into S classes of the same meaning and checks the device against the oracle on the split input and
both against the oracle on the unsplit input (tests/static_class_cases.py).  The batch cases run with the lanes of
every warp in both orders."""
import os

import pytest

import emu_lib
import static_class_cases as scc
from armada_b200.scheduler import DeviceNodeDb

_dev = None


def dev():
    global _dev
    if _dev is None:
        _dev = emu_lib.emu_round()
    return _dev


def emu_round(inp):
    return dev().schedule(inp)


def emu_nodedb(inp):
    return DeviceNodeDb(inp, 0, lib=emu_lib.load())


@pytest.fixture(params=["forward", "reverse"])
def lane_order(request):
    old = os.environ.get("EMU_ORDER")
    os.environ["EMU_ORDER"] = request.param
    yield request.param
    if old is None:
        os.environ.pop("EMU_ORDER", None)
    else:
        os.environ["EMU_ORDER"] = old


# S = None: one class per node
@pytest.mark.parametrize("form,S,placement,seed", [("k32", 33, "interleaved", 1), ("k64", 64, "all_high", 2), ("k32", 257, "boundary", 3),
                                                   ("k64", None, "per_node", 4)])
def test_batch_key_layouts(form, S, placement, seed, lane_order, capfd):
    scc.batch_key_layout(dev(), capfd, form, S, placement, seed, n_nodes=300, n_jobs=2500)


@pytest.mark.parametrize("S,placement,seed,round_limit", [(40, "interleaved", 400, False), (256, "all_high", 401, True),
                                                          (120, "per_node", 402, True)])
def test_batch_chain_run(S, placement, seed, round_limit, lane_order):
    scc.batch_chain_run(emu_round, S, placement, seed, n_nodes=120, n_jobs=900, round_limit=round_limit)


@pytest.mark.parametrize("S,placement,seed,round_limit", [(96, "interleaved", 1, None), (257, "boundary", 2, 0.5), (33, "interleaved", 3, 0.7)])
def test_batch_gangs(S, placement, seed, round_limit, lane_order):
    scc.batch_gangs(emu_round, S, placement, seed, n_nodes=120, n_queues=8, n_jobs=2500, round_limit=round_limit)


@pytest.mark.parametrize("S,placement,seed", [(32, "interleaved", 2), (257, "boundary", 5), (None, "per_node", 8), (64, "all_high", 11)])
def test_general_loop(S, placement, seed):
    scc.general_loop(emu_round, S, placement, seed)


@pytest.mark.parametrize("S,placement,seed", [(33, "interleaved", 2), (None, "per_node", 5), (257, "boundary", 8)])
def test_exact_mode(S, placement, seed):
    scc.general_loop(emu_round, S, placement, seed, unaligned=True)


@pytest.mark.parametrize("S,placement,seed", [(64, "all_high", 0), (None, "per_node", 1)])
def test_excluded_nodes_by_kind(S, placement, seed):
    scc.excluded_nodes(emu_round, S, placement, seed, n_nodes=80, n_jobs=600)


def test_disallowed_class_with_excluded_nodes():
    scc.excluded_nodes(emu_round, 40, "interleaved", 2, n_nodes=60, n_jobs=300, disallowed=True)


@pytest.mark.parametrize("seed", [1, 2])
def test_uniformity_gangs_with_a_class_per_node(seed):
    scc.uniformity_per_node_classes(emu_round, seed, n_nodes=60, n_jobs=400)


@pytest.mark.parametrize("S,placement,seed,unaligned", [(257, "boundary", 0, False), (None, "per_node", 1, True)])
def test_dry_run_nodedb(S, placement, seed, unaligned):
    scc.dry_run(emu_nodedb, S, placement, seed, n_nodes=300, n_jobs=300, n_singles=40, n_gangs=12, max_gang=150, unaligned=unaligned)


@pytest.mark.parametrize("S,placement,seed", [(64, "all_high", 1), (None, "per_node", 2)])
def test_explain(S, placement, seed):
    scc.explain(emu_lib.load(), S, placement, seed, n_nodes=60)


@pytest.mark.parametrize("S,placement,seed,kw", [(40, "interleaved", 1, {}), (257, "boundary", 3, {"unaligned": True})])
def test_cluster_upload(S, placement, seed, kw, capfd):
    scc.cluster_upload(dev(), capfd, S, placement, seed, n_nodes=80, **kw)
