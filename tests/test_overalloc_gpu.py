"""Rounds that start on over-allocated nodes (overalloc_cases) on the GPU, bit for bit against the oracle: the
emulator's cases, the same with 3 000-5 000 nodes, and C5 with 5 % of its nodes over-allocated."""
import pytest

import overalloc_cases as oc
from armada_b200.scheduler import DeviceRound
from shape_cases import compare_key  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

_dev = None


def gpu_round(inp):
    global _dev
    if _dev is None:
        _dev = DeviceRound(0)
    return _dev.schedule(inp)


@pytest.mark.parametrize("D,seed,excl,derive,n_nodes", [(1, 6, False, False, 60), (3, 6, True, False, 60), (8, 12, False, False, 60),
                                                        (3, 12, False, True, 60), (8, 6, True, False, 60), (3, 12, False, False, 4000),
                                                        (8, 12, False, False, 3000)])
def test_fast_domain_batch_mode(D, seed, excl, derive, n_nodes, compare_key, capfd):
    with DeviceRound(0) as dev:
        assert oc.fast_domain_batch(dev, capfd, D, seed, excl=excl, derive=derive, n_nodes=n_nodes) == compare_key


@pytest.mark.parametrize("seed,n_nodes,n_jobs", [(1, 60, 500), (2, 60, 500), (4, 3000, 20000)])
def test_unindexed_negative_resource(seed, n_nodes, n_jobs):
    oc.unindexed_negative(gpu_round, seed, n_nodes=n_nodes, n_jobs=n_jobs)


@pytest.mark.parametrize("seed,excl", [(1, False), (2, True), (3, True)])
def test_exact_mode_less_than_one_step_over(seed, excl):
    oc.exact_less_than_a_step(gpu_round, seed, excl)


def test_exact_mode_negative_first_index_component():
    oc.two_node_first_component(gpu_round)


@pytest.mark.xfail(strict=True, reason="the oracle yields a rejected node twice after a re-seek the reference fails as an "
                                       "iteration loop; the device counts it once")
def test_exact_mode_rejected_node_counted_twice():
    oc.two_node_rejected_twice(gpu_round)


@pytest.mark.parametrize("flags", sorted(oc.FLAGS))
@pytest.mark.parametrize("seed,protected_fraction", [(1, 0.0), (2, 0.5)])
def test_rebind_onto_over_allocated_nodes(seed, protected_fraction, flags):
    oc.rebind_shortcut(gpu_round, seed, flags, protected_fraction)


@pytest.mark.parametrize("excl,derive", [(True, False), (False, True)])
def test_rebind_with_excluded_nodes_and_snapshot_construction(excl, derive):
    oc.rebind_shortcut(gpu_round, 3, "both", 0.5, excl=excl, derive=derive)


@pytest.mark.parametrize("protected_fraction", [0.0, 0.5])
def test_rebind_onto_over_allocated_nodes_many_nodes(protected_fraction):
    oc.rebind_shortcut(gpu_round, 7, "both", protected_fraction, n_nodes=5000, n_jobs=8000)


def test_c5_with_over_allocated_nodes():
    oc.c5_over_allocated(gpu_round)
