#!/usr/bin/env python3
"""Extract the reference's TestPopulateNodeDb table into tests/golden/populate_node_db.json with the parser of
extract_go_tables.py:

    python tests/golden/extract_populate_node_db.py

The table's cases are one Test32CpuNode, cordoned (`.WithSchedulable(false)`) or not, and N1Cpu4GiJobs of
PriorityClass0 on it; each parsed case is reduced to those facts and the expected outcome (a missing Expect* field is
false, as in Go).  Any other shape is refused, so a change of the table shows here.  Nothing but DATA is extracted."""
from __future__ import annotations

import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from extract_go_tables import OUT, REF, extract  # noqa: E402

REL = "scheduling/scheduling_algo_test.go"
NODE = {"call": "testfixtures.Test32CpuNode", "args": [{"id": "testfixtures.TestPriorities"}]}


def reduce_case(name, ast):
    f = {k["id"]: v for k, v in ast["elems"]}
    jobs = f["Jobs"]
    if jobs == {"lit": "[]*jobdb.Job", "elems": []}:
        n = 0
    else:
        assert jobs["call"] == "testfixtures.N1Cpu4GiJobs" and jobs["args"][1] == {"id": "testfixtures.PriorityClass0"}, jobs
        n = int(jobs["args"][2])
    node = f["Node"]
    cordoned = node != NODE
    if cordoned:
        assert node == {"callexpr": {"sel": NODE, "name": "WithSchedulable"}, "args": [False]}, node
    return {"name": name, "cordoned": cordoned, "jobs": n, "added": bool(f.get("ExpectNodeAdded", False)),
            "unschedulable": bool(f.get("ExpectNodeUnschedulable", False)), "over_allocated": bool(f.get("ExpectNodeOverAllocated", False))}


def main():
    if not os.path.isdir(REF):
        print(f"{REF} not present; nothing to do (the fixture is committed)", file=sys.stderr)
        return 0
    cases = extract(os.path.join(REF, REL), r"func TestPopulateNodeDb\(", r"tests := map\[string\]struct \{")
    out = os.path.join(OUT, "populate_node_db.json")
    with open(out, "w") as fh:
        json.dump({"source": f"internal/scheduler/{REL}", "node": {"cpu": 32, "memory_gi": 256},
                   "job": {"cpu": 1, "memory_gi": 4, "priority_class": "priority-0"},
                   "cases": [reduce_case(k, v) for k, v in cases.items()]}, fh, indent=1)
        fh.write("\n")
    print(f"populate_node_db: {len(cases)} cases -> {out}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
