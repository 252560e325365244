#!/usr/bin/env python3
"""Extract the reference's TestPreemptingQueueScheduler_RespectNodePodLimits table into
tests/golden/respect_node_pod_limits.json, with the parser of extract_go_tables.py and in its format:

    python tests/golden/extract_pod_limit_table.py

Fields of a case: incumbentPriorityClass, challengerCount, challengerIsGang, nodePodCapacity,
extraNodePodCapacities, incumbentCount, expectedPreemptions, expectedNewlyScheduled.  tests/pod_limit_cases.py
restates the test's driver.  Nothing but DATA (inputs + expected answers) is extracted."""
from __future__ import annotations

import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from extract_go_tables import OUT, REF, extract  # noqa: E402

REL = "scheduling/preempting_queue_scheduler_test.go"


def main():
    if not os.path.isdir(REF):
        print(f"{REF} not present; nothing to do (the fixture is committed)", file=sys.stderr)
        return 0
    cases = extract(os.path.join(REF, REL), r"func TestPreemptingQueueScheduler_RespectNodePodLimits\(", r"tests := map\[string\]struct \{")
    out = os.path.join(OUT, "respect_node_pod_limits.json")
    with open(out, "w") as f:
        json.dump({"source": f"internal/scheduler/{REL}", "cases": cases}, f, separators=(",", ":"), sort_keys=False)
    print(f"respect_node_pod_limits: {len(cases)} cases -> {out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
