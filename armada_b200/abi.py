"""ctypes mirror of include/armada_b200.h (the C ABI shared by the CUDA product library and
the CPU oracle).  Field order and types must match the header exactly; tests/test_abi.py
cross-checks sizeof() against the compiled libraries.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

ABI_VERSION = 2
MAX_RESOURCES = 8
EXCLUDED_KINDS = 5  # ARMADA_EXCL_*: node type, static, resources (reached), implicit, disallowed
EXCL_NODE_TYPE, EXCL_STATIC, EXCL_RESOURCES, EXCL_IMPLICIT, EXCL_DISALLOWED = range(5)
EXCL_STATIC_TOTAL = 5  # ExcludedReason.kind only: counted as EXCL_RESOURCES in the round's histogram
MAX_PRIORITIES = 16
MAX_PRIORITY_CLASSES = 32
MAX_AWAY = 4
NONE = 0xFFFFFFFF
NO_PRIORITY = -(2**31)

# status codes
OK, E_INVALID, E_UNSUPPORTED, E_CUDA, E_NO_DEVICE, E_INTERNAL, E_STATE, E_DEADLINE = range(8)
# job states
JOB_NONE, JOB_SCHEDULED, JOB_PREEMPTED, JOB_RESCHEDULED, JOB_FAILED, JOB_SCHEDULED_AND_EVICTED = range(6)
# scheduling methods
METHOD_NONE, METHOD_RESCHEDULED, METHOD_NO_PREEMPTION, METHOD_FAIRSHARE, METHOD_URGENCY, METHOD_AWAY = range(6)
# reasons
(REASON_NONE, REASON_MAX_RESOURCES_SCHEDULED, REASON_MAX_RESOURCES_PER_QUEUE, REASON_GLOBAL_RATE_LIMIT,
 REASON_QUEUE_RATE_LIMIT, REASON_QUEUE_CORDONED, REASON_GLOBAL_RATE_LIMIT_GANG, REASON_QUEUE_RATE_LIMIT_GANG,
 REASON_GANG_EXCEEDS_GLOBAL_BURST, REASON_GANG_EXCEEDS_QUEUE_BURST, REASON_GANG_DOES_NOT_FIT,
 REASON_JOB_DOES_NOT_FIT, REASON_NO_REMAINING_CANDIDATES, REASON_UNIFORMITY_LABEL_NOT_INDEXED,
 REASON_NO_NODES_WITH_UNIFORMITY_LABEL, REASON_GANG_FITS_NO_UNIFORMITY_VALUE, REASON_FLOATING_RESOURCES) = range(17)
LABEL_NOT_INDEXED = 0xFFFFFFFE

NODE_UNSCHEDULABLE = 1
NODE_OVERALLOCATED = 2
NODE_DROPPED = 4  # armada_round_download_snapshot only: the node is not in the NodeDb

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
i32p = C.POINTER(C.c_int32)
u64p = C.POINTER(C.c_uint64)
i64p = C.POINTER(C.c_int64)
f64p = C.POINTER(C.c_double)


class PriorityClass(C.Structure):
    _fields_ = [
        ("priority", C.c_int32),
        ("preemptible", C.c_uint8),
        ("_pad", C.c_uint8 * 3),
        ("num_away", C.c_uint32),
        ("away_priority", C.c_int32 * MAX_AWAY),
        ("away_well_known", C.c_uint32 * MAX_AWAY),
    ]


class RoundInput(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("num_resources", C.c_uint32),
        ("num_indexed", C.c_uint32),
        ("indexed_resource", C.c_uint32 * MAX_RESOURCES),
        ("indexed_resolution", C.c_int64 * MAX_RESOURCES),
        ("num_priorities", C.c_uint32),
        ("priorities", C.c_int32 * MAX_PRIORITIES),
        ("num_priority_classes", C.c_uint32),
        ("priority_classes", PriorityClass * MAX_PRIORITY_CLASSES),
        ("total_resources", C.c_int64 * MAX_RESOURCES),
        ("drf_multipliers", C.c_double * MAX_RESOURCES),
        ("has_round_limit", C.c_uint8),
        ("protect_uncapped_adjusted_fair_share", C.c_uint8),
        ("prefer_large_job_ordering", C.c_uint8),
        ("disable_home_scheduling", C.c_uint8),
        ("disable_away_scheduling", C.c_uint8),
        ("disable_gang_away_scheduling", C.c_uint8),
        ("global_limiter_is_inf", C.c_uint8),
        ("collect_excluded_nodes", C.c_uint8),
        ("max_resources_to_schedule", C.c_int64 * MAX_RESOURCES),
        ("protected_fraction_of_fair_share", C.c_double),
        ("max_queue_lookback", C.c_uint32),
        ("disallowed_resource_mask", C.c_uint32),
        ("global_limiter_tokens", C.c_double),
        ("global_limiter_burst", C.c_int64),
        ("num_nodes", C.c_uint32),
        ("num_node_types", C.c_uint32),
        ("num_static_classes", C.c_uint32),
        ("node_index", u64p),
        ("node_id_rank", u32p),
        ("node_type", u32p),
        ("node_static_class", u32p),
        ("node_flags", u8p),
        ("node_total", i64p),
        ("node_allocatable", i64p),
        ("num_classes", C.c_uint32),
        ("num_static_rows", C.c_uint32),
        ("class_request", i64p),
        ("class_pc", u32p),
        ("class_static_row", u32p),
        ("class_away_row", u32p),
        ("class_key_valid", u8p),
        ("static_match", u32p),
        ("type_match", u32p),
        ("num_jobs", C.c_uint32),
        ("num_gangs", C.c_uint32),
        ("job_class", u32p),
        ("job_queue", u32p),
        ("job_queue_priority", u32p),
        ("job_submit_time", i64p),
        ("job_id_rank", u32p),
        ("job_gang", u32p),
        ("job_node", u32p),
        ("job_scheduled_at_priority", i32p),
        ("job_active_run_timestamp", i64p),
        ("gang_cardinality", u32p),
        ("num_queues", C.c_uint32),
        ("queue_weight", f64p),
        ("queue_cordoned", u8p),
        ("queue_allocated_by_pc", i64p),
        ("queue_demand", i64p),
        ("queue_constrained_demand", i64p),
        ("queue_short_job_penalty", i64p),
        ("queue_has_limit", u8p),
        ("queue_limit", i64p),
        ("queue_limiter_tokens", f64p),
        ("queue_limiter_burst", i64p),
        ("queue_limiter_is_inf", u8p),
        ("queued_start", u32p),
        ("queued_order", u32p),
        # ABI 2: gang node uniformity, floating resources
        ("gang_uniformity_label", u32p),
        ("num_uniformity_labels", C.c_uint32),
        ("_pad_uniformity", C.c_uint32),
        ("uniformity_value_start", u32p),
        ("class_uniformity_row", u32p),
        ("floating_resource_mask", C.c_uint32),
        ("floating_limits_configured", C.c_uint8),
        ("_pad_floating", C.c_uint8 * 3),
        ("floating_limit", C.c_int64 * MAX_RESOURCES),
    ]


class ClusterState(C.Structure):
    """ArmadaClusterState: the pool as reported, for armada_round_upload_cluster."""
    _fields_ = [
        ("abi_version", C.c_uint32),
        ("num_other_pool_jobs", C.c_uint32),
        ("other_pool_job_node", u32p),
        ("other_pool_job_request", i64p),
        ("static_class_unschedulable", u32p),
        ("has_round_limit", C.c_uint8),
        ("_pad", C.c_uint8 * 7),
        ("max_fraction_to_schedule", C.c_double * MAX_RESOURCES),
        ("queue_limit_fraction", f64p),
    ]


class RoundOutput(C.Structure):
    _fields_ = [
        ("job_state", u8p),
        ("job_node", u32p),
        ("job_scheduled_at_priority", i32p),
        ("job_preempted_at_priority", i32p),
        ("job_method", u8p),
        ("job_reason", u8p),
        ("job_seq", u32p),
        ("node_alloc", i64p),
        ("queue_allocated", i64p),
        ("queue_allocated_by_pc", i64p),
        ("queue_fair_share", f64p),
        ("scheduled_resources", i64p),
        ("evicted_resources", i64p),
        ("job_excluded_nodes", u32p),
        ("job_seq_first_pass", u32p),
        ("job_reason_first_pass", u8p),
        ("num_scheduled_jobs", C.c_uint32),
        ("num_scheduled_gangs", C.c_uint32),
        ("num_evicted_jobs", C.c_int32),
        ("termination_reason", C.c_uint32),
        ("num_result_scheduled", C.c_uint32),
        ("num_result_preempted", C.c_uint32),
    ]


class RoundStats(C.Structure):
    _fields_ = [
        ("loop_iterations", C.c_uint64),
        ("probes", C.c_uint64),
        ("placements", C.c_uint64),
        ("evicted_pass1", C.c_uint64),
        ("evicted_pass2", C.c_uint64),
        ("fair_preemption_scans", C.c_uint64),
        ("tree_rescans", C.c_uint64),
        ("gpu_launches", C.c_uint64),
        ("device_ms", C.c_double),
        ("schedule_pass_ms", C.c_double),
        ("phase_cycles", C.c_uint64 * 8),
        ("batch_cycles", C.c_uint64 * 8),
        ("batch_debug", C.c_uint64 * 8),
    ]


# Elements of the RoundStats arrays read by name (their meanings: include/armada_b200.h)
PHASE_BATCH_ITERATIONS = 4  # phase_cycles: loop iterations run in batch mode (a count, not cycles)
BATCH_COUNT = 6             # batch_cycles: batches (a count, not cycles)
DEBUG_PIPELINE_RUNS = 2     # batch_debug: pipeline runs
DEBUG_BATCHES_CUT = 3       # batch_debug: batches cut short
DEBUG_SLOW_STEPS = 4        # batch_debug: slow steps of the assignment loop, then their cycles
DEBUG_SLOW_CYCLES = 5
DEBUG_REFILLS = 6           # batch_debug: candidate refills from the sorted index, then their cycles
DEBUG_REFILL_CYCLES = 7


class ExcludedReason(C.Structure):
    _fields_ = [
        ("kind", C.c_uint32),
        ("sub", C.c_uint32),
        ("quantity", C.c_int64),
        ("count", C.c_uint32),
        ("_pad", C.c_uint32),
    ]


def field_dtype(struct_type, name: str) -> np.dtype:
    """The element type of pointer field `name` of a structure above, as a numpy dtype."""
    return np.dtype(dict(struct_type._fields_)[name]._type_)


def attach(struct, keep: list, **arrays) -> dict:
    """Point the pointer fields of `struct` named by the keywords at their arrays.  Each array is first made
    C-contiguous with its field's element type (declared once, in `_fields_`), so the library never reads
    bytes as the wrong type; it is appended to `keep`, because the struct holds only raw pointers.  Returns
    the arrays the fields point into, by field name."""
    fields, out = dict(type(struct)._fields_), {}
    for name, a in arrays.items():
        a = np.ascontiguousarray(a, dtype=np.dtype(fields[name]._type_))
        keep.append(a)
        setattr(struct, name, a.ctypes.data_as(fields[name]))
        out[name] = a
    return out


REPO_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT_LIB_PATH = os.path.join(REPO_ROOT, "armada_b200", "libarmada_b200.so")

_product = None


class ArmadaError(RuntimeError):
    def __init__(self, status: int, message: str):
        super().__init__(f"armada status {status}: {message}")
        self.status = status


def declare_prototypes(lib: C.CDLL) -> None:
    """argtypes/restype of every entry point of include/armada_b200.h."""
    vp = C.c_void_p
    lib.armada_round_create.argtypes = [C.c_int32, C.POINTER(vp)]
    lib.armada_round_create.restype = C.c_int32
    lib.armada_round_upload.argtypes = [vp, C.POINTER(RoundInput)]
    lib.armada_round_upload.restype = C.c_int32
    lib.armada_round_upload_cluster.argtypes = [vp, C.POINTER(RoundInput), C.POINTER(ClusterState)]
    lib.armada_round_upload_cluster.restype = C.c_int32
    lib.armada_round_download_snapshot.argtypes = [vp, u8p, i64p, u32p, i64p, i64p, i64p]
    lib.armada_round_download_snapshot.restype = C.c_int32
    lib.armada_round_run.argtypes = [vp, C.POINTER(RoundStats)]
    lib.armada_round_run.restype = C.c_int32
    lib.armada_round_run_deadline.argtypes = [vp, C.POINTER(RoundStats), C.c_uint64]
    lib.armada_round_run_deadline.restype = C.c_int32
    lib.armada_round_download.argtypes = [vp, C.POINTER(RoundOutput)]
    lib.armada_round_download.restype = C.c_int32
    lib.armada_round_destroy.argtypes = [vp]
    lib.armada_round_destroy.restype = C.c_int32
    lib.armada_round_schedule.argtypes = [vp, C.POINTER(RoundInput), C.POINTER(RoundOutput), C.POINTER(RoundStats)]
    lib.armada_round_schedule.restype = C.c_int32
    lib.armada_nodedb_create.argtypes = [C.c_int32, C.POINTER(RoundInput), C.POINTER(vp)]
    lib.armada_nodedb_create.restype = C.c_int32
    lib.armada_nodedb_schedule_many.argtypes = [vp, C.c_uint32, u32p, u32p, u8p, u32p]
    lib.armada_nodedb_schedule_many.restype = C.c_int32
    lib.armada_nodedb_explain.argtypes = [vp, C.c_uint32, u32p, u32p, u8p, u32p, u32p, u8p, u32p, C.POINTER(ExcludedReason), C.c_uint32, u32p]
    lib.armada_nodedb_explain.restype = C.c_int32
    lib.armada_nodedb_select_nodes.argtypes = [vp, C.c_uint32, u32p, u32p]
    lib.armada_nodedb_select_nodes.restype = C.c_int32
    lib.armada_nodedb_add_classes.argtypes = [vp, C.c_uint32, i64p, u32p, u32p, u32p, u8p, C.c_uint32, u32p, u32p, u32p]
    lib.armada_nodedb_add_classes.restype = C.c_int32
    lib.armada_nodedb_destroy.argtypes = [vp]
    lib.armada_nodedb_destroy.restype = C.c_int32
    lib.armada_strerror.argtypes = [C.c_int32]
    lib.armada_strerror.restype = C.c_char_p
    lib.armada_last_error.argtypes = []
    lib.armada_last_error.restype = C.c_char_p
    lib.armada_abi_version.argtypes = []
    lib.armada_abi_version.restype = C.c_uint32
    lib.armada_abi_sizeof.argtypes = [C.c_uint32]
    lib.armada_abi_sizeof.restype = C.c_uint32


def load_product() -> C.CDLL:
    """Load libarmada_b200.so (the CUDA product).  Fails loudly: there is no CPU fallback."""
    global _product
    if _product is not None:
        return _product
    if not os.path.exists(PRODUCT_LIB_PATH):
        raise ArmadaError(E_NO_DEVICE, f"{PRODUCT_LIB_PATH} not built; run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(PRODUCT_LIB_PATH)
    declare_prototypes(lib)
    _product = lib
    return lib


PRODUCT_SYMBOLS = [
    "armada_round_create",
    "armada_round_upload",
    "armada_round_upload_cluster",
    "armada_round_download_snapshot",
    "armada_round_run",
    "armada_round_run_deadline",
    "armada_round_download",
    "armada_round_destroy",
    "armada_round_schedule",
    "armada_nodedb_create",
    "armada_nodedb_schedule_many",
    "armada_nodedb_explain",
    "armada_nodedb_select_nodes",
    "armada_nodedb_add_classes",
    "armada_nodedb_destroy",
    "armada_strerror",
    "armada_last_error",
    "armada_abi_version",
    "armada_abi_sizeof",
]
