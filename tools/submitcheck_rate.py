"""Dry-run checks per second on one GPU: `armada_nodedb_schedule_many` against `armada_nodedb_explain` on a
100 000-node cluster with 3 000 submitted jobs and gangs of mixed classes, many of which fit nowhere (the
cluster of tests/test_dryrun_explain_gpu.py).  Each call is one launch and returns after the device
finished; the time is the host clock around the call.  Prints one JSON line.

    python tools/submitcheck_rate.py [--repeats N]   (the median of N timed calls; N = 1 by default)
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import explain_cases as ec  # noqa: E402
from armada_b200.scheduler import DeviceNodeDb  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=1)
    args = ap.parse_args()
    case = ec.Case(11, n_nodes=100_000, n_gangs=3000, indexed_only=True, allocatable_extra=True)
    gangs = case.classes
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    db = DeviceNodeDb(case.b.input)
    try:
        res = db.explain(gangs, capacity=1 << 16)  # warm-up; sizes the record buffer
        cap = max(1, sum(len(g[4]) for g in res))
        db.schedule_many(gangs)
        times = {"schedule_many": [], "explain": []}
        for _ in range(args.repeats):
            t = time.perf_counter()
            db.schedule_many(gangs)
            times["schedule_many"].append(time.perf_counter() - t)
            t = time.perf_counter()
            db.explain(gangs, capacity=cap)
            times["explain"].append(time.perf_counter() - t)
    finally:
        db.close()
    out = {"gpu": gpu, "nodes": case.b.input.num_nodes, "gangs": len(gangs), "jobs": sum(len(g) for g in gangs),
           "failed_gangs": sum(not g[0] for g in res), "records": cap}
    for k, v in times.items():
        out[f"{k}_s"] = sorted(v)
        out[f"{k}_checks_per_s"] = round(len(gangs) / sorted(v)[len(v) // 2], 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
