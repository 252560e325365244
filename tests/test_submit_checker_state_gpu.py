"""SubmitChecker across checks and its time budgets on the GPU; the bodies are in submit_checker_state_cases.py."""
import pytest

import submit_checker_state_cases as ss

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_checks_with_kept_dbs_match_a_fresh_checker_gpu(seed, monkeypatch):
    ss.check_state_sequence(seed, None, monkeypatch)


@pytest.mark.parametrize("name", sorted(ss.TIME_LIMIT_CASES))
def test_submit_checker_time_limits_gpu(name):
    ss.replay_time_limit(name)


def test_pinned_job_then_more_checks_gpu(monkeypatch):
    ss.check_pinned_job_then_more_checks(None, monkeypatch)


def test_refused_append_rolls_back_gpu(monkeypatch):
    ss.check_refused_append_rolls_back(None, monkeypatch)
