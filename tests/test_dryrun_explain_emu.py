"""armada_nodedb_explain under the SIMT emulator (no GPU): every output against the oracle-backed
reference of explain_cases.py, and against schedule_many on the same db."""
import numpy as np
import pytest

import emu_lib
import explain_cases as ec
from armada_b200 import abi
from armada_b200.model import excluded_nodes_by_reason
from armada_b200.scheduler import DeviceNodeDb


@pytest.mark.parametrize("config", sorted(ec.CONFIGS))
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_explain_matches_the_oracle(config, seed):
    case = ec.Case(seed, cfg_over=ec.CONFIGS[config], allocatable_extra=seed == 3)
    got, failed_single = ec.check_case(case, emu_lib.load())
    assert failed_single > 0


def test_explain_reaches_every_record_kind():
    case = ec.held_back_gpus_case()
    got, failed_single = ec.check_case(case, emu_lib.load())
    assert failed_single == 2 and got[2][0]
    kinds = {int(r.kind) for g in got for r in g[4]}
    assert kinds == {abi.EXCL_RESOURCES, abi.EXCL_STATIC_TOTAL}  # (the seeded matrix reaches the other kinds)
    strings = excluded_nodes_by_reason(case.b, case.classes[1][0], got[1][4])
    # nodes 0, 4 and 8 have 6 gpus in total, nodes 1, 7 and 10 six allocatable: one string
    assert strings["pod requires 7500m nvidia.com/gpu, but only 6 is available"] == 6
    assert strings["pod requires 7500m nvidia.com/gpu, but only 0 is available"] == 3


def test_gangs_fail_at_first_middle_and_last_member():
    # two 32-cpu nodes: gangs of 16-cpu members fail at the member that finds no room left
    import fixtures as fx
    f = fx.Fixtures()
    cfg = fx.test_scheduling_config()
    nodes = [f.cpu32(), f.cpu32()]
    gangs = [
        fx.with_gang([f.job("A", fx.PriorityClass1, {"cpu": "40", "memory": "1Gi"}) for _ in range(2)], "first"),
        fx.with_gang([f.job("A", fx.PriorityClass1, {"cpu": "16", "memory": "1Gi"}) for _ in range(6)], "middle"),
        fx.with_gang([f.job("A", fx.PriorityClass1, {"cpu": "16", "memory": "1Gi"}) for _ in range(4)] +
                     [f.job("A", fx.PriorityClass1, {"cpu": "17", "memory": "1Gi"})], "last"),
    ]
    jobs = [j for g in gangs for j in g]
    case = ec.case_from(cfg, nodes, jobs, [[0, 1], list(range(2, 8)), list(range(8, 13))])
    got, _ = ec.check_case(case, emu_lib.load())
    assert [g[2] for g in got] == [0, 4, 4] and not any(g[0] for g in got)


def test_too_small_record_buffer_reports_the_size_and_writes_nothing():
    import ctypes as C
    case = ec.Case(5, n_nodes=20, n_gangs=12)
    lib = emu_lib.load()
    db = DeviceNodeDb(case.b.input, lib=lib)
    try:
        full = db.explain(case.classes, capacity=4096)
        total = sum(len(g[4]) for g in full)
        assert total > 1
        G = len(case.classes)
        start = np.zeros(G + 1, np.uint32)
        start[1:] = np.cumsum([len(g) for g in case.classes])
        members = np.asarray([c for g in case.classes for c in g], np.uint32)
        ok, node = np.zeros(G, np.uint8), np.zeros(int(start[-1]), np.uint32)
        placed, away, rstart = np.zeros(G, np.uint32), np.zeros(G, np.uint8), np.zeros(G + 1, np.uint32)
        sentinel = abi.ExcludedReason(kind=77, sub=77, quantity=77, count=77)
        recs = (abi.ExcludedReason * (total + 1))(*([sentinel] * (total + 1)))
        needed = C.c_uint32(0)
        st = lib.armada_nodedb_explain(db.h, G, start.ctypes.data_as(abi.u32p), members.ctypes.data_as(abi.u32p), ok.ctypes.data_as(abi.u8p),
                                       node.ctypes.data_as(abi.u32p), placed.ctypes.data_as(abi.u32p), away.ctypes.data_as(abi.u8p),
                                       rstart.ctypes.data_as(abi.u32p), recs, total - 1, C.byref(needed))
        assert st == abi.OK and needed.value == total and int(rstart[-1]) == total
        assert all(r.kind == 77 and r.count == 77 for r in recs)  # nothing written
        assert [bool(x) for x in ok] == [g[0] for g in full] and [int(x) for x in placed] == [g[2] for g in full]
        # the Python wrapper grows the buffer once and gets the same records
        again = db.explain(case.classes, capacity=1)
        assert [ec.records_tuples(g[4]) for g in again] == [ec.records_tuples(g[4]) for g in full]
    finally:
        db.close()


def test_gang_of_more_than_256_members_is_unsupported():
    case = ec.Case(6, n_nodes=4, n_gangs=1, gang_sizes=(1,))
    db = DeviceNodeDb(case.b.input, lib=emu_lib.load())
    try:
        with pytest.raises(abi.ArmadaError) as e:
            db.explain([case.classes[0] * 257])
        assert e.value.status == abi.E_UNSUPPORTED
    finally:
        db.close()
