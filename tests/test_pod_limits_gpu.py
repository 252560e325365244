"""RespectNodePodLimits on the GPU (tests/pod_limit_cases.py), bit for bit against the oracle: the reference's tables,
seeded rounds in every assignment-loop form a pods field gives (also with thousands of nodes), C3 at full size with
110 pods per node, the SubmitChecker and the simulator."""
import pytest

import oracle_lib
import pod_limit_cases as pl
from armada_b200 import simulator as sim
from armada_b200.scheduler import DeviceRound

pytestmark = pytest.mark.gpu

_dev = None


def device():
    global _dev
    if _dev is None:
        _dev = DeviceRound(0)
    return _dev


def cuda_round(inp):
    return device().schedule(inp)


@pytest.mark.parametrize("name", sorted(pl.TABLE))
def test_respect_node_pod_limits_table(name):
    pl.table_against_the_oracle(cuda_round, pl.respect_node_pod_limits_round(name))


def test_non_preemptible_over_pack():
    pl.table_against_the_oracle(cuda_round, pl.non_preemptible_over_pack_round())


@pytest.mark.parametrize("case", pl.CASES + [pl.PodCase(c.form, c.kind, c.caps, c.seed + 100, n_nodes=3000) for c in pl.CASES],
                         ids=lambda c: c.id)
def test_seeded_rounds(case, capfd):
    pl.seeded_round(device(), case, capfd)


def test_c3_with_110_pods_per_node(capfd):
    """C3 at full size with the knob on: the pods field (7 bits) takes the key's fields past the 32-bit compare keys."""
    inp = pl.c3_with_pods().to_input()
    want = oracle_lib.round_schedule(inp)
    got, lay, form = pl.shape_cases.schedule_with_layout(device(), inp, capfd)
    assert form == "k64", lay
    bad = got.diff(want)
    assert not bad, "device != oracle:\n  " + "\n  ".join(bad)


def test_submit_checker_refuses_on_pods():
    pl.submit_checker_refuses_on_pods(None)


def test_simulator_pod_cap_binds(tmp_path):
    pl.simulator_pod_cap_binds(tmp_path, sim.device_engine(0))
