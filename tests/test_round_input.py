"""The arrays behind a RoundInput (CPU only): the library trusts every pointer of ArmadaRoundInput to reach an array
of the field's element type, laid out contiguously and as long as include/armada_b200.h says the field is.  Checked
for the inputs RoundInputBuilder and synth.RawRound make."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import explain_cases
import fixtures as fx
import gang_cases
from armada_b200 import abi, synth
from armada_b200.model import QueueSpec, RoundInputBuilder

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "armada_b200.h")
C_TYPES = {"uint8_t": np.uint8, "int32_t": np.int32, "uint32_t": np.uint32, "int64_t": np.int64, "uint64_t": np.uint64,
           "double": np.float64}


def header_pointer_fields():
    """ArmadaRoundInput's pointer fields as the header declares them: name -> (element type, the dimensions of the
    field's comment, e.g. ["D", "N"] for `[D][N]`)."""
    text = open(HEADER).read()
    end = text.index("} ArmadaRoundInput;")
    body = text[text.rindex("typedef struct {", 0, end):end]
    fields = {}
    for ctype, name, dims in re.findall(r"const (\w+)\* (\w+);\s*/\*\s*((?:\[[^\]]*\])+)", body):
        fields[name] = (np.dtype(C_TYPES[ctype]), re.findall(r"\[([^\]]*)\]", dims))
    return fields


FIELDS = header_pointer_fields()


def test_header_declares_every_pointer_field():
    pointers = [name for name, t in abi.RoundInput._fields_ if hasattr(t, "contents")]
    assert sorted(FIELDS) == sorted(pointers)


def kept_arrays(inp):
    """The array each non-NULL pointer field points at, after checking it against the header."""
    kept = {a.ctypes.data: a for a in inp._keepalive}
    arrays = {}
    for name in FIELDS:
        addr = C.cast(getattr(inp, name), C.c_void_p).value
        if addr is not None:
            assert addr in kept, f"{name} points outside the arrays the input keeps alive"
            arrays[name] = kept[addr]
    sizes = {"N": inp.num_nodes, "D": inp.num_resources, "C": inp.num_classes, "rows": inp.num_static_rows,
             "S": inp.num_static_classes, "T": inp.num_node_types, "J": inp.num_jobs, "G": inp.num_gangs,
             "Q": inp.num_queues, "PC": inp.num_priority_classes, "L": inp.num_uniformity_labels,
             "ARMADA_MAX_AWAY": abi.MAX_AWAY, "ceil": math.ceil}
    if "uniformity_value_start" in arrays:
        sizes["V"] = int(arrays["uniformity_value_start"][inp.num_uniformity_labels])
    if "queued_start" in arrays:
        sizes["queued"] = int(arrays["queued_start"][inp.num_queues])
    for name, a in arrays.items():
        dtype, dims = FIELDS[name]
        assert a.dtype == dtype, f"{name}: {a.dtype}, the header says {dtype}"
        assert a.flags.c_contiguous, name
        need = math.prod(eval(d.replace("#", ""), {"__builtins__": {}}, sizes) for d in dims)
        assert a.size >= need, f"{name}: {a.size} elements, the library reads {'x'.join(dims)} = {need}"
    return arrays


def _with_queued_order():
    b = gang_cases.uniformity_round(3)
    order = {q.name: [j.id for j in reversed(b.jobs) if j.queue == q.name and j.node is None] for q in b.queues}
    return RoundInputBuilder(b.cfg, b.nodes, b.jobs, b.queues, queued_order=order)


BUILDERS = {
    "gang table NodeUniformityLabel": lambda: gang_cases.gang_case_round("NodeUniformityLabel")[0],
    "uniformity and floating round": lambda: gang_cases.uniformity_round(0),
    "explain case": lambda: explain_cases.Case(0).b,
    "queued order": _with_queued_order,
    "no nodes or jobs": lambda: RoundInputBuilder(fx.test_scheduling_config(), [], [], [QueueSpec("A")]),
}

RAW_ROUNDS = {
    "random round": lambda: synth.random_round(0),
    "random round with away types and queue limits": lambda: synth.random_round(1, away=True, queue_limits=True),
    "C1": synth.config_c1,
}


@pytest.mark.parametrize("name", BUILDERS)
def test_builder_input(name):
    b = BUILDERS[name]()
    arrays = kept_arrays(b.input)
    for field in FIELDS:  # what the builder calls `field` is what the library reads there (None: NULL)
        assert getattr(b, field) is arrays.get(field), field
    for former, field in RoundInputBuilder.FORMER_NAMES.items():
        assert getattr(b, former) is arrays[field], former


@pytest.mark.parametrize("name", RAW_ROUNDS)
def test_raw_round_input(name):
    r = RAW_ROUNDS[name]()
    inp = r.to_input()
    kept_arrays(inp)
    assert r.h2d_bytes() == sum(a.nbytes for a in inp._keepalive)
