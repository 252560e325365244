"""More than 32 and more than 256 node static classes on the GPU: the bodies of tests/static_class_cases.py at 2 000 to
20 000 nodes, and batch-mode rounds with one static class per node, as a hostname selector makes them: C3 at a fifth of
its size and at full size (100 000 nodes and classes).  Each against the oracle on the split input and on the unsplit
input.  Run on an H100: pytest -m gpu."""
import pytest

import static_class_cases as scc
from armada_b200.scheduler import DeviceNodeDb, DeviceRound

pytestmark = pytest.mark.gpu

_dev = None


def dev():
    global _dev
    if _dev is None:
        _dev = DeviceRound(0)
    return _dev


def cuda_round(inp):
    return dev().schedule(inp)


def cuda_nodedb(inp):
    return DeviceNodeDb(inp, 0)


# S = None: one class per node
@pytest.mark.parametrize("form,S,placement,seed,n_nodes", [("k32", 33, "interleaved", 11, 2000), ("k64", 64, "all_high", 12, 5000),
                                                           ("k32", 257, "boundary", 13, 5000), ("k64", None, "per_node", 14, 20000)])
def test_batch_key_layouts(form, S, placement, seed, n_nodes, capfd):
    scc.batch_key_layout(dev(), capfd, form, S, placement, seed, n_nodes=n_nodes, n_jobs=20000)


@pytest.mark.parametrize("S,placement,seed,round_limit", [(40, "interleaved", 410, False), (256, "all_high", 411, True),
                                                          (None, "per_node", 412, True)])
def test_batch_chain_run(S, placement, seed, round_limit):
    scc.batch_chain_run(cuda_round, S or 3000, placement, seed, n_nodes=3000, n_jobs=20000, round_limit=round_limit)


@pytest.mark.parametrize("S,placement,seed,round_limit", [(96, "interleaved", 11, None), (257, "boundary", 12, 0.5), (4000, "per_node", 13, 0.7)])
def test_batch_gangs(S, placement, seed, round_limit):
    scc.batch_gangs(cuda_round, S, placement, seed, n_nodes=4000, n_queues=32, n_jobs=40000, round_limit=round_limit)


@pytest.mark.parametrize("scale", [0.2, 1.0])
def test_c3_with_a_class_per_node(scale):
    scc.scaled_per_node(cuda_round, "C3", scale)


@pytest.mark.parametrize("S,placement,seed", [(32, "interleaved", 102), (257, "boundary", 103), (None, "per_node", 104), (64, "all_high", 105)])
def test_general_loop(S, placement, seed):
    scc.general_loop(cuda_round, S, placement, seed, n_nodes=3000, n_jobs=6000, n_running=3000)


@pytest.mark.parametrize("S,placement,seed", [(33, "interleaved", 106), (None, "per_node", 107), (257, "boundary", 108)])
def test_exact_mode(S, placement, seed):
    scc.general_loop(cuda_round, S, placement, seed, unaligned=True, n_nodes=2000, n_jobs=5000, n_running=2000)


@pytest.mark.parametrize("S,placement,seed", [(64, "all_high", 10), (None, "per_node", 11)])
def test_excluded_nodes_by_kind(S, placement, seed):
    scc.excluded_nodes(cuda_round, S, placement, seed, n_nodes=2000, n_jobs=6000)


def test_disallowed_class_with_excluded_nodes():
    scc.excluded_nodes(cuda_round, 300, "boundary", 12, n_nodes=2000, n_jobs=4000, disallowed=True)


def test_uniformity_gangs_with_a_class_per_node():
    scc.uniformity_per_node_classes(cuda_round, 5, n_nodes=2000, n_zones=8, n_jobs=6000)


@pytest.mark.parametrize("S,placement,seed,unaligned", [(257, "boundary", 10, False), (None, "per_node", 11, True)])
def test_dry_run_nodedb(S, placement, seed, unaligned):
    scc.dry_run(cuda_nodedb, S, placement, seed, n_nodes=5000, n_jobs=2000, n_singles=200, n_gangs=40, max_gang=600, unaligned=unaligned)


@pytest.mark.parametrize("S,placement,seed", [(64, "all_high", 11), (None, "per_node", 12)])
def test_explain(S, placement, seed):
    scc.explain(None, S, placement, seed, n_nodes=2000, n_gangs=60)


@pytest.mark.parametrize("S,placement,seed,kw", [(40, "interleaved", 21, {}), (300, "boundary", 22, {"unaligned": True, "limits": True})])
def test_cluster_upload(S, placement, seed, kw, capfd):
    scc.cluster_upload(dev(), capfd, S, placement, seed, n_nodes=3000, n_jobs=20000, n_running=9000, **kw)
