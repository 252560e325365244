"""Jobs failed inside the batch pipeline (pipeline_fail_cases) on the GPU, bit for bit against the oracle."""
import pytest

import pipeline_fail_cases as pf
from armada_b200.scheduler import DeviceRound

pytestmark = pytest.mark.gpu

_dev = None


@pytest.mark.parametrize("name", sorted(pf.CASES))
def test_pipeline_fail(name, capfd, monkeypatch):
    global _dev
    monkeypatch.setenv("ARMADA_PRINT_STATS", "1")
    if _dev is None:
        _dev = DeviceRound(0)
    pf.run_case(_dev.schedule, name, capfd)
