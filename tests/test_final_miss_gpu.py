"""Final level-0 misses (final_miss_cases) on the GPU, bit for bit against the oracle."""
import pytest

import final_miss_cases as fm
import oracle_lib
from armada_b200.scheduler import DeviceRound

pytestmark = pytest.mark.gpu

_dev = None


@pytest.mark.parametrize("name", sorted(fm.CASES))
def test_final_miss(name, capfd, monkeypatch):
    global _dev
    monkeypatch.setenv("ARMADA_PRINT_STATS", "1")
    if _dev is None:
        _dev = DeviceRound(0)
    make, skips, scans = fm.CASES[name]
    inp = make()
    capfd.readouterr()
    got = _dev.schedule(inp)
    err = capfd.readouterr().err
    want = oracle_lib.round_schedule(inp)
    bad = got.diff(want)
    assert not bad, f"{name}: CUDA != oracle:\n  " + "\n  ".join(bad)
    assert got.out.num_result_scheduled < inp.num_jobs
    fm.check_stats(err, skips, scans, name)
    fm.check_round(name, got)
