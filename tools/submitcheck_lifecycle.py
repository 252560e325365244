"""Milliseconds per SubmitChecker check with NodeDbs kept alive across checks against rebuilding them for every
check, on the 100 000-node cluster of tools/submitcheck_rate.py (one executor, one pool).  The workload is a
sequence of small checks, each a few hundred gangs drawn from the same 3 000, so that most scheduling keys
repeat from one check to the next.  Each mode runs the sequence once, timed by the host clock around each
`check` (which returns after the device finished); the results of the two modes are compared check by check.
`--hostname-labels` gives every node a label of its own (kubernetes.io/hostname, as real nodes carry), which
no job looks at.  Prints one JSON line.

    python tools/submitcheck_lifecycle.py [--checks K] [--gangs G] [--hostname-labels]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import explain_cases as ec  # noqa: E402
import fixtures as fx  # noqa: E402
from armada_b200.model import QueueSpec  # noqa: E402
from armada_b200.submitcheck import Executor, PoolConfig, SubmitChecker  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--checks", type=int, default=8)
    ap.add_argument("--gangs", type=int, default=300)
    ap.add_argument("--nodes", type=int, default=100_000)
    ap.add_argument("--hostname-labels", action="store_true")
    args = ap.parse_args()
    case = ec.Case(11, n_nodes=args.nodes, n_gangs=3000, indexed_only=True, allocatable_extra=True)
    if args.hostname_labels:
        for n in case.nodes:
            n.labels[fx.TestHostnameLabel] = n.id
    rng = random.Random(5)
    checks = [[case.jobs[j] for g in rng.sample(case.groups, args.gangs) for j in g] for _ in range(args.checks)]
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    setup = (case.cfg, [PoolConfig("cpu")], [Executor("executor-0", [("cpu", n) for n in case.nodes])], [QueueSpec("A", 1.0)])

    def summary(results):
        return {jid: (r.is_schedulable, tuple(r.pools), r.reason) for jid, r in results.items()}

    # rebuilt: a new checker (its dbs built and uploaded) for every check, as before the dbs were kept
    rebuilt_ms, rebuilt_out = [], []
    for jobs in checks:
        t = time.perf_counter()
        with SubmitChecker(*setup) as checker:
            rebuilt_out.append(summary(checker.check(jobs)))
        rebuilt_ms.append((time.perf_counter() - t) * 1e3)
    # kept: the dbs built once (timed apart), every check appends its new keys and reuses the result cache
    t = time.perf_counter()
    kept = SubmitChecker(*setup)
    setup_ms = (time.perf_counter() - t) * 1e3
    kept_ms, same = [], True
    with kept:
        for jobs, want in zip(checks, rebuilt_out):
            t = time.perf_counter()
            got = summary(kept.check(jobs))
            kept_ms.append((time.perf_counter() - t) * 1e3)
            same = same and got == want
    out = {"gpu": gpu, "nodes": len(case.nodes), "hostname_labels": args.hostname_labels, "checks": args.checks, "gangs_per_check": args.gangs,
           "jobs_per_check": [len(c) for c in checks], "results_equal": same,
           "rebuilt_ms_per_check": [round(v, 1) for v in rebuilt_ms], "kept_setup_ms": round(setup_ms, 1),
           "kept_ms_per_check": [round(v, 1) for v in kept_ms],
           "rebuilt_mean_ms": round(sum(rebuilt_ms) / len(rebuilt_ms), 1), "kept_mean_ms": round(sum(kept_ms) / len(kept_ms), 1)}
    print(json.dumps(out))
    if not same:
        sys.exit(1)


if __name__ == "__main__":
    main()
