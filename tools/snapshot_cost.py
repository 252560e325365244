"""What deriving the pool's NodeDb snapshot on the device costs a C3-shaped round.

Times, alternating, over --reps repetitions on the same inputs:
  cluster   armada_round_upload_cluster on the pool as reported (per-node usage, state, total and caps on the
            device, one D x N copy back, then the upload)
  explicit  model.ClusterSnapshot (the Python derivation) + armada_round_upload on what it derives
  upload    armada_round_upload alone on the derived inputs (what a caller that derives the snapshot itself pays
            on top of its own derivation)
Each call ends in a device synchronise, so host clock times are call times.  The round is C3 with a quarter of
its jobs running, 3 % of the nodes cordoned and a fifth running jobs of other pools.  Prints one JSON line with
the GPU's name, power limit and SM clock; with ARMADA_TIME_UPLOAD=1 the library also prints its stage laps
(`cluster: derive` is the new device stages with their copies) on stderr.

    python tools/snapshot_cost.py [--reps 5]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import cluster_cases as cc  # noqa: E402
from armada_b200.model import ClusterSnapshot  # noqa: E402
from armada_b200.scheduler import DeviceRound  # noqa: E402


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    inp, cs = cc.to_cluster(cc.c3_round(), cc.Case(20, cordon=0.03, other=0.2, overfill=0.2, limits=True))
    times = {"cluster": [], "explicit": [], "upload": []}
    with DeviceRound(0) as dev:
        for rep in range(args.reps + 1):  # the first repetition warms up
            t0 = time.perf_counter()
            dev.upload_cluster(inp, cs)
            t1 = time.perf_counter()
            cl = ClusterSnapshot(inp, cs)
            t2 = time.perf_counter()
            dev.upload(cl.input)
            t3 = time.perf_counter()
            if rep:
                times["cluster"].append((t1 - t0) * 1e3)
                times["explicit"].append((t3 - t1) * 1e3)
                times["upload"].append((t3 - t2) * 1e3)
    out = {"config": "C3 cluster", "nodes": int(inp.num_nodes), "kept_nodes": int(len(cl.kept)), "jobs": int(inp.num_jobs),
           "other_pool_jobs": int(cs.num_other_pool_jobs), "gpu": gpu_info()}
    for k, v in times.items():
        out[f"{k}_ms_median"] = round(float(np.median(v)), 2)
        out[f"{k}_ms_min"] = round(float(np.min(v)), 2)
        out[f"{k}_ms_max"] = round(float(np.max(v)), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
