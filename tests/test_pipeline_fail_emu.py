"""Jobs failed inside the batch pipeline (pipeline_fail_cases) through the emulated kernel, bit for bit against the
oracle, with the lanes of every warp run in both orders."""
import os

import pytest

import emu_lib
import pipeline_fail_cases as pf

_dev = None


@pytest.fixture(params=["forward", "reverse"])
def lane_order(request):
    old = os.environ.get("EMU_ORDER")
    os.environ["EMU_ORDER"] = request.param
    yield request.param
    if old is None:
        os.environ.pop("EMU_ORDER", None)
    else:
        os.environ["EMU_ORDER"] = old


@pytest.mark.parametrize("name", sorted(pf.CASES))
def test_pipeline_fail(name, lane_order, capfd, monkeypatch):
    global _dev
    monkeypatch.setenv("ARMADA_PRINT_STATS", "1")
    if _dev is None:
        _dev = emu_lib.emu_round()
    pf.run_case(_dev.schedule, name, capfd)
