"""SubmitChecker across checks and its time budgets under the SIMT emulator (no GPU); the bodies are in
submit_checker_state_cases.py."""
import pytest

import emu_lib
import submit_checker_state_cases as ss


@pytest.mark.parametrize("seed", [1, 2])
def test_checks_with_kept_dbs_match_a_fresh_checker(seed, monkeypatch):
    ss.check_state_sequence(seed, emu_lib.load(), monkeypatch)


@pytest.mark.parametrize("name", sorted(ss.TIME_LIMIT_CASES))
def test_submit_checker_time_limits(name):
    ss.replay_time_limit(name, emu_lib.load())


def test_pinned_job_then_more_checks(monkeypatch):
    ss.check_pinned_job_then_more_checks(emu_lib.load(), monkeypatch)


def test_refused_append_rolls_back(monkeypatch):
    ss.check_refused_append_rolls_back(emu_lib.load(), monkeypatch)
