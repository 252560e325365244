"""TestSubmitChecker (submitcheck_test.go:28-429) through SubmitChecker over the dry-run NodeDb, the
kernel stepped by the SIMT emulator; and the `reason` text getSchedulingResult assembles."""
import pytest

import emu_lib
import submit_checker_cases as sc


@pytest.mark.parametrize("name", sorted(sc.CASES))
def test_submit_checker(name):
    sc.replay(name, emu_lib.load())


def test_reason_of_a_job_that_fits_nowhere():
    got = sc.replay("No jobs schedulable due to resources", emu_lib.load())
    # pool cpu, its one executor: the pod scheduling context (submitcheck.go:398-407); no other pool has executors
    assert got["largeJob1"].reason == ("executor-0:\n"
                                       "Node:                       none\n"
                                       "Number of nodes in cluster: 1\n"
                                       "Excluded nodes:\n"
                                       " 1: insufficient resources available\n"
                                       "\n---\n")
    got = sc.replay("No jobs schedulable due to selector", emu_lib.load())
    assert " 1: node does not match pod NodeSelector: label foo not set\n" in got["smallJob1"].reason


def test_reason_of_a_gang_and_of_the_pre_checks():
    got = sc.replay("Individual jobs fit but gang doesn't", emu_lib.load())
    assert got["largeGangJob[0]"].reason == "executor-0: 2 out of 4 pods schedulable\n"  # :409-414
    got = sc.replay("One job exceeds total floating resources", emu_lib.load())
    reason = got["smallJob1"].reason
    assert reason.startswith("pool cpu:\njob/gang requests floating resources (test-floating-resource=11) but not enough floating "
                             "resource test-floating-resource in pool cpu\n\n---\n")  # :319-326
    assert "pool cpu2:\njob/gang requests floating resources (test-floating-resource=11) but floating resources not configured for pool cpu2\n" in reason
    got = sc.replay("One job exceeds queue fraction limit", emu_lib.load())
    # the cpu limit is 2 cpu × 0.0001 = 0 and ResourceList.String() leaves zero entries out; no limit is MaxInt64
    assert got["smallJob1"].reason == ("pool cpu:\njob/gang requests resources (memory=4294967296,cpu=1) which exceeds the total limit of "
                                       "(memory=9223372036854775807,nvidia.com/gpu=9223372036854775807m,test-floating-resource=9223372036854775807) "
                                       "for its queue/priority class\n\n---\n")  # :329-337
