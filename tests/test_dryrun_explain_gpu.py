"""armada_nodedb_explain on the H100: the emulator's matrix, a 100 000-node cluster with a few thousand
checks, and run-to-run determinism — every output bit-exact against the oracle-backed reference."""
import pytest

import explain_cases as ec
from armada_b200.scheduler import DeviceNodeDb

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("config", sorted(ec.CONFIGS))
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_explain_matches_the_oracle_gpu(config, seed):
    case = ec.Case(seed, cfg_over=ec.CONFIGS[config], allocatable_extra=seed == 3)
    _, failed_single = ec.check_case(case, None)
    assert failed_single > 0


def test_explain_reaches_every_record_kind_gpu():
    ec.check_case(ec.held_back_gpus_case(), None)


@pytest.fixture(scope="module")
def big_case():
    return ec.Case(11, n_nodes=100_000, n_gangs=3000, indexed_only=True, allocatable_extra=True)


def test_explain_100k_nodes_matches_the_oracle(big_case):
    got, failed_single = ec.check_case(big_case, None, capacity=1 << 16, round_kinds=False)
    assert failed_single > 100 and sum(not g[0] for g in got) > 500


def test_explain_is_deterministic(big_case):
    db = DeviceNodeDb(big_case.b.input)
    try:
        runs = [db.explain(big_case.classes, capacity=1 << 16) for _ in range(2)]
    finally:
        db.close()
    def flat(r):
        return [(ok, node.tobytes(), placed, away, bytes(memoryview(bytearray(b"".join(bytes(x) for x in recs)))))
                for ok, node, placed, away, recs in r]
    assert flat(runs[0]) == flat(runs[1])
