"""Rounds in which single jobs fail inside the batch pipeline.  When a class's level-0 miss is final
(final_miss_cases: no evicted job alive, no job bound below its priority, no away node types, no
excluded-node counts), the assignment loop fails the class's first job that fits no node itself: the
batch is cut behind it and the run goes on with a batch built afresh.  A queue head of that class that
was peeked before the failure becomes an item of its own that fails without a node.

Each case names whether jobs fail in the pipeline (bt_fails of the ARMADA_PRINT_STATS line) and how many
pipeline runs the round has.  Small batches (ARMADA_BT_WQ) make many short batches, so the failing
records land at many places of a batch (first, last, second of a pair, inside a run's first, quarter-size
batch); the place each one takes is not asserted."""
from __future__ import annotations

import contextlib
import os
import re

import numpy as np

import final_miss_cases as fm
from armada_b200 import abi

STATS_RE = re.compile(r"armada stats: .*failed_iters=(\d+) .*bt_fails=(\d+)")


def _small_batches(seed, **kw):
    return fm._full(seed, **kw).to_input()


def _round_limit(seed):
    # a limit of 80 % of the cluster: the cluster fills before the limit trips, under the limit's one-at-a-time loop
    r = fm._full(seed, round_limit=True)
    r.round_limit = (np.asarray(r.node_total).sum(axis=1) * 0.8).astype(np.int64)
    return r.to_input()


# name -> (builds the round input, ARMADA_BT_WQ or None, jobs fail in the pipeline, pipeline runs)
CASES = {
    "one_class_fills": (fm.CASES["one_class_fills"][0], None, True, 1),
    "many_queues": (fm.CASES["many_queues"][0], None, True, 1),
    "few_nodes": (fm.CASES["few_nodes"][0], None, True, 1),
    "tight_fit": (fm.CASES["tight_fit"][0], None, True, 1),
    "small_batches_a": (lambda: _small_batches(41), 8, True, 1),
    "small_batches_b": (lambda: _small_batches(42, n_queues=3, n_jobs=600), 8, True, 1),
    "small_batches_c": (lambda: _small_batches(43, n_queues=20, n_jobs=1500), 16, True, 1),
    "round_limit": (lambda: _round_limit(44), 8, True, 2),
    # the shortcut must not fire: every job that fails goes through the general loop
    "evicted_alive": (fm.CASES["evicted_alive"][0], None, False, None),
    "collect_excluded_nodes": (fm.CASES["collect_excluded_nodes"][0], None, False, None),
    fm.URGENCY: (fm.CASES[fm.URGENCY][0], None, False, None),
    # single jobs fail in the pipeline; the gangs still fail in the general loop
    "gangs": (fm.CASES["gangs"][0], None, True, None),
}


@contextlib.contextmanager
def batch_items(wq):
    """ARMADA_BT_WQ (read when a round is uploaded) while the case runs."""
    old = os.environ.get("ARMADA_BT_WQ")
    if wq is not None:
        os.environ["ARMADA_BT_WQ"] = str(wq)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop("ARMADA_BT_WQ", None)
        else:
            os.environ["ARMADA_BT_WQ"] = old


def run_case(schedule, name, capfd) -> None:
    """One case on `schedule` (an emulated or CUDA DeviceRound's schedule), bit for bit against the oracle."""
    import oracle_lib
    make, wq, in_pipeline, runs = CASES[name]
    inp = make()
    capfd.readouterr()
    with batch_items(wq):
        got = schedule(inp)
    err = capfd.readouterr().err
    want = oracle_lib.round_schedule(inp)
    bad = got.diff(want)
    assert not bad, f"{name}: device != oracle:\n  " + "\n  ".join(bad)
    m = STATS_RE.findall(err)
    assert m, f"{name}: no stats line"
    failed, bt_fails = (int(v) for v in m[-1])
    assert (bt_fails > 0) == in_pipeline, f"{name}: {bt_fails} jobs failed in the pipeline"
    n_runs = int(got.stats.batch_debug[abi.DEBUG_PIPELINE_RUNS])
    if runs is not None:
        assert n_runs == runs, f"{name}: {n_runs} pipeline runs"
    if name in ("many_queues", "small_batches_c"):
        # more failures than classes that failed: heads peeked before their class failed failed as batch items
        reason = np.asarray(want.job_reason_first_pass)
        failed_cls = np.ctypeslib.as_array(inp.job_class, shape=(inp.num_jobs,))[reason == abi.REASON_JOB_DOES_NOT_FIT]
        assert bt_fails == failed and bt_fails > len(np.unique(failed_cls)), f"{name}: {bt_fails} of {failed} failures"
    if name == "gangs":
        assert failed > bt_fails, f"{name}: no gang failed in the general loop"
    fm.check_round(name, got)
