"""Rounds that fill their cluster while queued single jobs keep arriving, for the "a level-0 miss is
final" shortcut of the general loop: when no evicted job is alive, no job can be bound below the
failing job's priority, the job is a single job without away node types and no excluded-node counts
are collected, its priority level holds the same rows as level 0, so the gate probe there is skipped.

Each case names whether gate probes at the job's own level are skipped and whether some run.  Both
are read from the gate_skips / gate_scans counts of the ARMADA_PRINT_STATS line."""
from __future__ import annotations

import re

import numpy as np

from armada_b200 import abi, synth

STATS_RE = re.compile(r"armada stats: .*failed_iters=(\d+) .*gate_scans=(\d+) gate_skips=(\d+)")


def _full(seed, **kw):
    # far more work than the nodes hold: the round ends with every class failing, at any point of a batch
    args = dict(n_nodes=30, n_queues=8, n_jobs=1400, n_running=0, gangs=False, priorities=False)
    args.update(kw)
    return synth.random_round(seed, **args)


def _collect_excl(r):
    inp = r.to_input()
    inp.collect_excluded_nodes = 1
    return inp


# A round whose running jobs survive the eviction step (no queue is above its protected share) while
# queued jobs of higher priority classes fail at level 0: they must reach the gate and preempt by
# urgency; only the jobs of the lowest priority class may skip it.
URGENCY = "running_lower_priority"

# name -> (builds the round input, some gate probes skipped, some gate probes run)
CASES = {
    "one_class_fills": (lambda: _full(11).to_input(), True, False),
    "many_queues": (lambda: _full(12, n_queues=40, n_jobs=2000).to_input(), True, False),
    "few_nodes": (lambda: _full(13, n_nodes=6, n_queues=3, n_jobs=300).to_input(), True, False),
    "tight_fit": (lambda: _full(14, n_nodes=50, n_jobs=1100).to_input(), True, False),
    # the shortcut must not fire
    URGENCY: (lambda: _full(21, n_running=100, priorities=True, protected_fraction=1e6).to_input(), True, True),
    "evicted_alive": (lambda: _full(22, n_running=150, protected_fraction=0.5).to_input(), False, True),
    "away_node_types": (lambda: _full(23, away=True).to_input(), True, True),  # (classes without away types skip)
    "collect_excluded_nodes": (lambda: _collect_excl(_full(24)), False, True),
    "gangs": (lambda: _full(31, gangs=True).to_input(), True, True),  # (the gangs' members reach the gate; single jobs skip it)
}


def check_stats(err: str, skips: bool, scans: bool, label: str) -> None:
    m = STATS_RE.findall(err)
    assert m, f"{label}: no stats line"
    failed, n_scans, n_skips = (int(v) for v in m[-1])
    assert failed > 0, f"{label}: no job failed in the general loop"
    assert (n_skips > 0) == skips, f"{label}: {n_skips} gate probes skipped"
    assert (n_scans > 0) == scans, f"{label}: {n_scans} gate probes run"


def check_round(name: str, got) -> None:
    """What makes a case test what it is named for."""
    if name == URGENCY:
        assert got.stats.evicted_pass1 == 0  # (the first pass has no evicted job: the priority clause decides)
        assert int((np.asarray(got.job_method) == abi.METHOD_URGENCY).sum()) > 0
    if name == "evicted_alive":
        assert got.stats.evicted_pass1 > 0
