"""RespectNodePodLimits without a GPU: the config rule, the round input, the reference's tables on the oracle, and the
shared bodies of tests/pod_limit_cases.py through the emulated kernel, bit for bit against the oracle."""
import numpy as np
import pytest

import emu_lib
import fixtures as fx
import pod_limit_cases as pl
from armada_b200.model import PODS, ResourceType, RoundInputBuilder, QueueSpec, apply_respect_node_pod_limits

_dev = None


def emu_dev():
    global _dev
    if _dev is None:
        _dev = emu_lib.emu_round()
    return _dev


def emu_round(inp):
    return emu_dev().schedule(inp)


# ---- apply_respect_node_pod_limits (ApplyRespectNodePodLimits / ensurePodsResourceType) ----------------------
def test_knob_off_changes_nothing():
    cfg = fx.test_scheduling_config()
    supported, indexed = list(cfg.supported_resource_types), list(cfg.indexed_resources)
    assert apply_respect_node_pod_limits(cfg) is False
    assert list(cfg.supported_resource_types) == supported and list(cfg.indexed_resources) == indexed
    assert cfg.job_requests({"cpu": "1"}) == {"cpu": "1"}


def test_knob_on_appends_pods_to_both_lists():
    cfg = fx.test_scheduling_config(respect_node_pod_limits=True)
    supported, indexed = list(cfg.supported_resource_types), list(cfg.indexed_resources)
    assert apply_respect_node_pod_limits(cfg) is True
    assert list(cfg.supported_resource_types) == supported + [ResourceType(PODS, "1")]
    assert list(cfg.indexed_resources) == indexed + [ResourceType(PODS, "1")]
    f = cfg.factory()
    assert f.names[-1] == PODS and f.scales[-1] == 0


def test_existing_pods_entry_is_normalised_in_place():
    cfg = fx.test_scheduling_config(respect_node_pod_limits=True)
    cfg.supported_resource_types = [ResourceType(PODS, "10")] + list(cfg.supported_resource_types)
    cfg.indexed_resources = list(cfg.indexed_resources[:1]) + [ResourceType(PODS, "10")] + list(cfg.indexed_resources[1:])
    assert apply_respect_node_pod_limits(cfg)
    assert cfg.supported_resource_types[0] == ResourceType(PODS, "1") and len(cfg.supported_resource_types) == 4
    assert cfg.indexed_resources[1] == ResourceType(PODS, "1") and len(cfg.indexed_resources) == 4


def test_apply_is_idempotent():
    cfg = fx.test_scheduling_config(respect_node_pod_limits=True)
    assert apply_respect_node_pod_limits(cfg)
    once = (list(cfg.supported_resource_types), list(cfg.indexed_resources))
    assert apply_respect_node_pod_limits(cfg)
    assert (list(cfg.supported_resource_types), list(cfg.indexed_resources)) == once


def test_every_job_of_a_built_input_asks_for_one_pod():
    """Queued and running jobs, whatever they request themselves; a node's pods come from its totals and allocatable,
    and a node that reports none has 0; the round's totals and the queues' demand count pods like any resource."""
    cfg = pl.pod_limits_config()
    F = fx.Fixtures()
    nodes = [F.node({"cpu": "32", "memory": "256Gi", PODS: "110"}), F.node({"cpu": "32", "memory": "256Gi"})]
    nodes[0].allocatable = {"cpu": "31", "memory": "250Gi", PODS: "100"}
    jobs = F.n_1cpu_4gi("A", fx.PriorityClass0, 3) + [F.job("A", fx.PriorityClass0, {"cpu": "2", PODS: "7"})]
    jobs[0].node = nodes[0].id
    b = RoundInputBuilder(cfg, nodes, jobs, [QueueSpec("A")])
    pods = b.factory.index[PODS]
    assert (b.class_request[b.job_class[: len(jobs)], pods] == 1).all()
    assert b.node_total[pods].tolist() == [110, 0] and b.node_allocatable[pods].tolist() == [100, 0]
    assert b.total_resources[pods] == 100
    assert [b.input.indexed_resource[i] for i in range(b.input.num_indexed)][-1] == pods
    assert b.input.indexed_resolution[b.input.num_indexed - 1] == 1
    assert b.input.drf_multipliers[pods] == 0.0  # pods are not among the DRF resources
    off = RoundInputBuilder(fx.test_scheduling_config(), nodes, jobs, [QueueSpec("A")])
    assert PODS not in off.factory.index and off.input.num_resources == b.input.num_resources - 1


# ---- the reference's tables ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(pl.TABLE))
def test_respect_node_pod_limits_table_on_the_oracle(name):
    pl.table_on_the_oracle(pl.respect_node_pod_limits_round(name))


def test_non_preemptible_over_pack_on_the_oracle():
    pl.table_on_the_oracle(pl.non_preemptible_over_pack_round())


@pytest.mark.parametrize("name", sorted(pl.TABLE))
def test_respect_node_pod_limits_table(name):
    pl.table_against_the_oracle(emu_round, pl.respect_node_pod_limits_round(name))


def test_non_preemptible_over_pack():
    pl.table_against_the_oracle(emu_round, pl.non_preemptible_over_pack_round())


def test_binding_eviction_unbinding_releases_the_pod_slot():
    pl.releases_pod_slot()


# ---- seeded rounds ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", pl.CASES, ids=lambda c: c.id)
def test_seeded_rounds(case, capfd):
    pl.seeded_round(emu_dev(), case, capfd)


def test_c3_with_pods_scaled():
    inp = pl.c3_with_pods(0.004).to_input()
    got, want = emu_round(inp), pl.oracle_lib.round_schedule(inp)
    assert not got.diff(want)
    assert np.asarray(want.job_state).any()


# ---- SubmitChecker and simulator --------------------------------------------------------------------------
def test_submit_checker_refuses_on_pods():
    pl.submit_checker_refuses_on_pods(emu_lib.load())


def test_simulator_pod_cap_binds(tmp_path):
    pl.simulator_pod_cap_binds(tmp_path, emu_round)


def test_simulator_knob_off(tmp_path):
    pl.simulator_knob_off(tmp_path, pl.oracle_lib.round_schedule)
