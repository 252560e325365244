"""The reference's exclusion reason strings as the host renders them (model.py): hand-derived vectors,
each with the rule it follows."""
import pytest

from armada_b200.model import (MatchExpression, Taint, insufficient_resources_reason, missing_label_reason, node_selector_string,
                               pod_scheduling_context_string, quantity_string, unmatched_label_reason, untolerated_taint_reason)


@pytest.mark.parametrize("value,scale,want", [
    (0, -3, "0"),                    # IsZero → "0"
    (1, -3, "1m"),                   # 1e-3: exponent already a multiple of 3
    (100, -3, "100m"),               # 1e-1 → exponent −1 ⇒ ×100, e−3
    (1500, -3, "1500m"),             # 15e-1 → ×100, e−3
    (7500, -3, "7500m"),
    (-1500, -3, "-1500m"),           # the sign stays on the integer
    (2000, -3, "2"),                 # trailing zeros move into the exponent: 2e0
    (16000, -3, "16"),
    (120, 0, "120"),                 # 12e1 → exponent 1 ⇒ ×10, e0
    (10000, 0, "10k"),               # 1e4 → ×10, e3 → "k"
    (1000000000, 0, "1G"),           # 1e9
    (4294967296, 0, "4294967296"),   # 4Gi: no trailing zero, DecimalSI prints the integer
    (137438953472, 0, "137438953472"),
])
def test_quantity_string(value, scale, want):
    assert quantity_string(value, scale) == want


def test_reason_strings():
    assert untolerated_taint_reason(Taint("gpu", "true", "NoSchedule")) == "taint gpu=true:NoSchedule not tolerated"
    assert missing_label_reason("zone") == "node does not match pod NodeSelector: label zone not set"
    assert unmatched_label_reason("zone", "a", "b") == "node does not match pod NodeSelector: required label zone = a, but node has b"
    assert insufficient_resources_reason("cpu", "4", "2") == "pod requires 4 cpu, but only 2 is available"
    assert node_selector_string(((MatchExpression("cluster", "In", ("c1", "c2")),),)) == (
        "&NodeSelector{NodeSelectorTerms:[]NodeSelectorTerm{NodeSelectorTerm{MatchExpressions:[]NodeSelectorRequirement{"
        "NodeSelectorRequirement{Key:cluster,Operator:In,Values:[c1 c2],},},MatchFields:[]NodeSelectorRequirement{},},},}")


def test_pod_scheduling_context_string():
    # tabwriter: "Node:" and "Number of nodes in cluster:" share a column 28 wide; the count column is as
    # wide as its widest cell ("10:") plus one; the empty first cell of a count line pads to one space
    got = pod_scheduling_context_string(13, {"taint gpu=true:NoSchedule not tolerated": 3, "insufficient resources available": 10})
    assert got == ("Node:                       none\n"
                   "Number of nodes in cluster: 13\n"
                   "Excluded nodes:\n"
                   " 10: insufficient resources available\n"
                   " 3:  taint gpu=true:NoSchedule not tolerated\n")
    assert pod_scheduling_context_string(0, {}) == ("Node:                       none\n"
                                                    "Number of nodes in cluster: 0\n"
                                                    "Excluded nodes:             none\n")
