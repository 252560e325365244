"""Device time of one round per named config (dev tooling; needs a GPU):
    python tools/time_configs.py C2 C3 C4 C5@0.1 ...   ->  one JSON line per config"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from armada_b200 import abi, synth  # noqa: E402
from armada_b200.scheduler import DeviceRound  # noqa: E402


def make(name):
    if "@" in name:
        base, sc = name.split("@")
        return synth.scaled(base, float(sc))
    return {"C1": synth.config_c1, "C2": synth.config_c2, "C3": synth.config_c3, "C4": synth.config_c4, "C5": synth.config_c5}[name]()


with DeviceRound(0) as dev:
    for name in sys.argv[1:] or ["C2", "C3", "C4"]:
        r = make(name)
        dev.upload(r.to_input())
        best = None
        for _ in range(3):
            st = dev.run()
            if best is None or st.device_ms < best.device_ms:
                best = st
        it = max(1, int(best.phase_cycles[abi.PHASE_BATCH_ITERATIONS]))
        print(json.dumps({"config": name, "device_ms": round(best.device_ms, 3), "pass_ms": round(best.schedule_pass_ms, 3),
                          "placements": int(best.placements), "iterations": int(best.loop_iterations),
                          "batched": int(best.phase_cycles[abi.PHASE_BATCH_ITERATIONS]), "batches": int(best.batch_cycles[abi.BATCH_COUNT]),
                          "placements_per_s": round(best.placements / (best.device_ms / 1e3)),
                          "batch_cycles_per_iter": [round(int(best.batch_cycles[i]) / it, 1) for i in range(6)],
                          "chain_busy_wait_per_iter": [round(int(best.batch_debug[i]) / it, 1) for i in range(2)], "runs_cut": [int(best.batch_debug[abi.DEBUG_PIPELINE_RUNS]), int(best.batch_debug[abi.DEBUG_BATCHES_CUT])],
                          "slow_steps": int(best.batch_debug[abi.DEBUG_SLOW_STEPS]), "cycles_per_slow_step": round(int(best.batch_debug[abi.DEBUG_SLOW_CYCLES]) / max(1, int(best.batch_debug[abi.DEBUG_SLOW_STEPS]))),
                          "refills": int(best.batch_debug[abi.DEBUG_REFILLS]), "cycles_per_refill": round(int(best.batch_debug[abi.DEBUG_REFILL_CYCLES]) / max(1, int(best.batch_debug[abi.DEBUG_REFILLS]))),
                          "fair_scans": int(best.fair_preemption_scans), "ev1": int(best.evicted_pass1), "ev2": int(best.evicted_pass2),
                          "probes": int(best.probes), "rescans": int(best.tree_rescans),
                          "phase_mcycles": [round(int(best.phase_cycles[i]) / 1e6, 1) for i in range(8)]}), flush=True)
