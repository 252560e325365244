// armada_dev.h — device-side data layout of one scheduling round (sm_90a).
//
// HBM layout (all SoA, resource-major so a warp reads consecutive nodes):
//   alloc      [PL][D][N] int64   Node.AllocatableByPriority (internaltypes/node.go:57).  Nodes are
//                                 stored in NODE-ID ORDER (device index == id rank) and indexed
//                                 resources are held in units of their index resolution, so the
//                                 best-fit key of nodedb/encoding.go:37-58 is a pure bit-pack.
//   total      [D][N]  int64      Node.totalResources (same units)
//   node_sclass[N]     u32        static class (taints/labels) id → column of static_match
//   jobs       SoA over J         class / queue / gang / order rank / run binding
//   per-job round state           bound node, evicted flag, scheduled-at priority, qctx set
//                                 membership, pod scheduling result
//   g0         [N]     u64        nodes sorted by their packed level-0 best-fit key (rebuilt before
//                                 every schedule pass that has queued jobs)
// The persistent round kernel keeps per-queue DRF state and the heads of the best-fit index
// (32-entry sorted windows per job class) in shared memory (see armada_pass.inc).
#pragma once
#include <stdint.h>
#ifndef ARMADA_EMU
#include <vector_types.h>
#endif

#include "armada_b200.h"

#define ARMADA_DEV_MAX_QUEUES 128
#define ARMADA_DEV_MAX_SLOTS 22  // best-fit index slots: 2 per owning index warp (11 owners; batch mode keeps both in registers)
#define ARMADA_DEV_VARIANTS (1 + ARMADA_MAX_AWAY)  // home + away node types per class

// Slots of the schedule pass's counters (SmemHdr::stat, summed into DevPtrs::stats over the passes of a round;
// k_reset zeroes them; the host reads them into ArmadaRoundStats and the ARMADA_PRINT_STATS lines).  Cycles are SM
// clock cycles.  Index warp 0 writes the batch_cycles slots but STAT_BT_CONTROL, and STAT_BT_CUT; the index warps add
// STAT_RESCANS atomically; the control warp writes the others.
enum StatSlot {
  STAT_ITERS = 0,          // loop iterations (the general loop's and the batched ones)
  STAT_PROBES = 1,         // SelectNode index walks
  STAT_PLACEMENTS = 2,     // successful binds
  STAT_FAIR = 3,           // fair-preemption scans
  STAT_RESCANS = 4,        // ArmadaRoundStats::tree_rescans: windows refilled from scratch
  STAT_KERNEL = 5,         // control-warp cycles: the whole kernel
  STAT_STARTUP = 6,        // … before the loop
  STAT_RUNS = 7,           // … in pipeline runs (Ctl::run_batch)
  // ArmadaRoundStats::phase_cycles: control-warp cycles in the general loop
  STAT_PROF = 8,
  STAT_PROF_PQ_TOP = 8,    // queue arg-min
  STAT_PROF_GANG = 9,      // gang bookkeeping and constraints (the whole gang_schedule)
  STAT_PROF_SELECT = 10,   // node selection
  STAT_PROF_BIND = 11,     // node row update
  STAT_BATCH_ITERS = 12,   // loop iterations run in batch mode (a count)
  STAT_PROF_RESULT = 13,   // result algebra
  STAT_PROF_ADVANCE = 14,  // iterator advance (it_peek)
  STAT_PROF_CLEAR = 15,    // cost update (candidate_clear)
  // ArmadaRoundStats::batch_cycles: index-warp cycles of the batch pipeline
  STAT_BT_CYC = 16,
  STAT_BT_BUILD = 16,      // item build
  STAT_BT_HORIZON = 17,    // horizon
  STAT_BT_RANK = 18,       // merge ranks and speculative advance
  STAT_BT_WAIT = 19,       // waiting for the assignment loop
  STAT_BT_COMMIT = 20,     // apply and commit
  STAT_BT_CONTROL = 21,    // control warp: bookkeeping after a pipeline run
  STAT_BT_BATCHES = 22,    // batches (a count)
  STAT_BT_EPILOGUE = 23,   // pipeline epilogue
  // ArmadaRoundStats::batch_debug: the assignment loop
  STAT_BT_DBG = 24,
  STAT_CHAIN_BUSY = 24,    // cycles busy
  STAT_CHAIN_WAIT = 25,    // cycles waiting for records
  STAT_PIPELINE_RUNS = 26, // pipeline runs
  STAT_BT_CUT = 27,        // batches cut short
  STAT_SLOW_STEPS = 28,    // slow steps (ensure_groups; chain_swar only)
  STAT_SLOW_CYCLES = 29,   // … their cycles
  STAT_REFILLS = 30,       // candidate refills from the G0 cursor (chain_swar only)
  STAT_REFILL_CYCLES = 31, // … their cycles
  // control-warp timeline (ARMADA_PRINT_STATS)
  STAT_TL_PRECREATE = 32,         // creating windows up front
  STAT_TL_FIRST_BATCH_WAIT = 33,  // waiting for the first batch of a run
  STAT_TL_AFTER_CHAIN_WAIT = 34,  // waiting for the index warps after the assignment loop
  STAT_TL_FAILED_ITERS = 35,      // loop iterations that failed (STAT_BT_FAILS of them in the batch pipeline)
  STAT_TL_FAILED_CYCLES = 36,     // … the cycles of those in the general loop
  STAT_TL_FAIR_QUERY = 37,        // fair-preemption queries
  STAT_TL_LEVEL_SCAN = 38,        // level scans
  STAT_TL_EVICTED_REBIND = 39,    // re-binds of evicted single jobs
  // general-loop timeline (ARMADA_PRINT_STATS)
  STAT_GL_WAIT_INDEX = 40,     // waiting for the index warps (wait_consumed)
  STAT_GL_RING_FULL = 41,      // message ring full (post)
  STAT_GL_SELECT_QUEUED = 42,  // node selection of queued jobs
  STAT_GL_BIND_QUEUED = 43,    // their binds
  STAT_GL_FAIR_VICTIMS = 44,   // victims of fair preemption
  STAT_GL_PROLOGUE = 45,       // iteration prologue (members, accounting, constraints)
  STAT_GL_SELECT_COUNT = 46,   // node selections of queued jobs (a count)
  // fast domain, after a level-0 miss: gate probes at the job's own level
  STAT_GATE_RUN = 47,      // … that ran
  STAT_GATE_SKIPPED = 48,  // … skipped (final miss)
  STAT_BT_FAILS = 49,      // jobs the batch pipeline failed (their level-0 miss final, Ctl::level0_miss_final)
  STAT_COUNT = 50,
};

// Slots of DevPtrs::s_counts: the round's sctx counts, carried from kernel to kernel (k_reset sets them; the schedule
// pass loads them in its prologue and stores them back in its epilogue).
enum CountSlot {
  CNT_SCHED_JOBS = 0,     // numScheduledJobs
  CNT_SCHED_GANGS = 1,    // numScheduledGangs
  CNT_EVICTED_JOBS = 2,   // numEvictedJobs
  CNT_TERMINATION = 3,    // termination reason of the first pass
  CNT_GLOBAL_TOKENS = 4,  // global rate-limiter tokens (double bits)
  CNT_ERROR = 5,          // error code of the passes (0 = none; an error of the first pass survives the second)
  CNT_COUNT = 8,
};
#define ARMADA_DEV_E_DEADLINE 100  // CNT_ERROR: a pass ran out of its time budget (PassArgs::budget_ns)

struct DevCfg {  // small POD, lives in global memory, hot parts copied to smem
  int32_t D, R, PL, PC, Q, C, T, S, rows;
  uint32_t N, J, G;
  int32_t indexed_resource[ARMADA_MAX_RESOURCES];
  int64_t res_scale[ARMADA_MAX_RESOURCES];  // per FACTORY resource: index resolution or 1
  int32_t key_shift[ARMADA_MAX_RESOURCES];  // per indexed resource i: bit position in the packed key
  int32_t res_key_shift[ARMADA_MAX_RESOURCES];  // per FACTORY resource d: bit position, or -1 if not indexed
  int32_t res_key_width[ARMADA_MAX_RESOURCES];  // per FACTORY resource d: field width (0 if not indexed)
  int32_t node_bits;                        // low bits of the key hold the node (id-rank) index
  int32_t key_total_bits;                   // bits used by the packed key (< 64)
  int32_t key_width[ARMADA_MAX_RESOURCES];  // per indexed resource i: field width in bits
  unsigned long long key_guard;             // one always-zero bit above every field (0 = no guard bits)
  int32_t swar_ok;                          // guard bits present and every resource is indexed
  int32_t cls_global;                       // the job-class table is in global memory (more than 256 classes)
  int32_t exact;                            // exact mode (see armada_host.inc "domain"): raw units everywhere, probes are literal
                                            // ordered walks over per-level rounded keys (Ctl::scan_probe_exact), no sorted index / batches
  int64_t index_res[ARMADA_MAX_RESOURCES];  // exact mode: index resolution of the i-th indexed resource (raw units)
  int32_t collect_excl;                     // keep NumExcludedNodesByReason of the jobs that fail (DevPtrs.excl)
  int32_t k32_ok;                           // … and the resource fields fit 26 bits without guard bits, 31 with them (32-bit compare keys)
  int32_t min_bind_prio;                    // lowest priority a job of a preemptible class can be bound at this round, evicted jobs
                                            // aside: running jobs' scheduled-at priorities, the classes' priority classes and away priorities
  int32_t priorities[ARMADA_MAX_PRIORITIES];
  ArmadaPriorityClass pcs[ARMADA_MAX_PRIORITY_CLASSES];
  int64_t total_resources[ARMADA_MAX_RESOURCES];
  double drf_mult[ARMADA_MAX_RESOURCES];
  int64_t max_to_schedule[ARMADA_MAX_RESOURCES];
  uint8_t has_round_limit, protect_uncapped, prefer_large, disable_home, disable_away, disable_gang_away,
      global_inf, _pad;
  double protected_fraction;
  uint32_t max_lookback, disallowed_mask;
  double global_tokens;
  int64_t global_burst;
  int32_t max_slots, sw, tw;
  // shared-memory layout of k_schedule_pass (byte offsets from the dynamic smem base)
  int32_t win_w;       // stream-window records per queue (power of two, <= 32)
  uint32_t off_cls, off_win, off_touched, off_slot, off_skey, off_srow, off_ssc, off_sgpos, off_hb_key, off_hb_row, off_hb_sc,
      off_ring, off_bt_k0, off_bt_k1, off_bt_id;
  int32_t bt_wq;  // batch mode: items per queue per batch (0 = batch mode off)
  int32_t bt_np;  // Q * bt_wq rounded up to a power of two (sort size)
  // gang node uniformity / floating resources (gang_scheduler.go:143,154-223)
  uint32_t uni_V;            // value slots over all uniformity labels (0 = no gang carries one)
  uint32_t floating_mask;    // bit d: resource d is floating (never part of the node fit)
  int32_t floating_configured;
  int64_t floating_limit[ARMADA_MAX_RESOURCES];
};

// one step of a gang's node transaction, undone by txn.Abort (Ctl::txn_abort in armada_pass.inc) in reverse order
enum UndoKind : uint32_t {
  UNDO_BIND = 1,        // bindJobToNodeInPlace of a job onto `node`
  UNDO_REBIND_EVICTED,  // the same for an evicted jctx re-bound to its own node
  UNDO_UNBIND_VICTIM,   // unbindJobFromNodeInPlace of a fair-preemption victim evicted from `node`
  UNDO_DROP_EVICTED,    // deleteEvictedJobSchedulingContextIfExistsWithTxn (node unused)
};
struct UndoRec {
  uint32_t kind, job, node;
  uint32_t arg;  // bind and re-bind: the priority bound at (int32_t); unbind and drop: the jctx's evicted index
  uint32_t cls;
};
static_assert(sizeof(UndoRec) == 20, "five words per undo record");

struct DevPtrs {
  // ---- immutable snapshot (uploaded once per round input) ----
  const int64_t* node_total;       // [D][N]
  const int64_t* node_allocatable; // [D][N]
  const uint32_t* node_sclass;     // [N]
  const uint8_t* node_flags;       // [N]
  const int64_t* class_req_raw;    // [C][D] factory units (queue / DRF accounting)
  const int64_t* class_req_node;   // [C][D] node units (indexed resources ÷ resolution)
  const uint32_t* class_pc;        // [C]
  const uint32_t* class_row;       // [C][VARIANTS] static row per variant (ARMADA_NONE = absent)
  const uint8_t* class_key_valid;  // [C]
  const double* class_cost;        // [C] DRF UnweightedCostFromAllocation(request)
  const uint4* q_rec;              // [#queued] stream records aligned with queued_order
  uint4* ev_rec;                   // [J] stream records aligned with evq_jobs (per pass)
  const uint32_t* static_match;    // [rows][sw]
  unsigned char* cls_glob;         // [C] ClassRec table when it does not fit shared memory (DevCfg.cls_global)
  const uint32_t* type_match;      // exact mode: [rows][tw] NodeTypeJobRequirementsMet
  const uint32_t* node_type;       // exact mode: [N] dense node type
  const uint32_t* node_xrank;      // exact mode: [N] rank of the node in (node type, NodeFactory index) order
  const uint32_t* node_of_xrank;   // exact mode: [N] inverse of node_xrank
  unsigned long long* xkey;        // exact mode: [PL][N] rounded best-fit key of every node at every level
  const uint32_t* job_class;       // [J]
  const uint32_t* job_queue;       // [J]
  const uint32_t* job_gang;        // [J]
  const uint32_t* job_node0;       // [J] run binding at round start (device node index)
  const int32_t* job_sap0;         // [J] run's scheduled-at priority or ARMADA_NO_PRIORITY
  const uint32_t* job_rank;        // [J] rank under SchedulingOrderCompare (unique)
  const uint32_t* gang_card;       // [G] declared cardinality
  const uint32_t* gang_count;      // [G] active members in this input
  const uint32_t* gang_off;        // [G+1] CSR offsets into gang_buf
  const uint32_t* queued_start;    // [Q+1]
  const uint32_t* queued_order;    // [#queued]
  const double* queue_weight;      // [Q]
  const uint8_t* queue_cordoned;   // [Q]
  const int64_t* queue_alloc_pc0;  // [Q][PC][D]
  const int64_t* queue_cdemand;    // [Q][D]
  const int64_t* queue_penalty;    // [Q][D]
  const uint8_t* queue_has_limit;  // [Q][PC]
  const int64_t* queue_limit;      // [Q][PC][D]
  const double* queue_tokens0;     // [Q]
  const int64_t* queue_burst;      // [Q]
  const uint8_t* queue_inf;        // [Q]
  // ---- mutable round state ----
  int64_t* alloc;                  // [PL][D][N]
  uint32_t* bound_node;            // [J]
  uint8_t* evicted_on_node;        // [J] Node.EvictedJobRunIds
  int32_t* sched_prio;             // [J] scheduledAtPriorityByJobId (ARMADA_NO_PRIORITY = absent)
  uint8_t* q_successful;           // [J] qctx.SuccessfulJobSchedulingContexts
  uint8_t* q_unsuccessful;         // [J]
  uint8_t* q_rescheduled;          // [J]
  uint8_t* q_evicted;              // [J] qctx.EvictedJobsById
  uint8_t* q_reason;               // [J]
  uint8_t* jc_evicted;             // [J] job is carried by an evicted jctx this pass
  uint32_t* jc_card;               // [J] jctx.CurrentGangCardinality
  uint32_t* assigned_node;         // [J] jctx.AssignedNode of the evicted jctx
  uint8_t* in_preempted;           // [J] preemptedJobsById
  uint8_t* in_scheduled;           // [J] scheduledJobsById
  uint8_t* in_sae;                 // [J] scheduledAndEvictedJobsById
  uint8_t* ev_mark;                // [J] evicted by the evictor currently running
  uint8_t* gang_ev;                // [G] gang has >=1 evicted member (current evictor)
  uint8_t* has_pctx;               // [J]
  uint32_t* res_node;              // [J] pctx.NodeId
  int32_t* res_sched_at;           // [J]
  int32_t* res_preempted_at;       // [J]
  uint8_t* res_method;             // [J]
  uint32_t* res_seq;               // [J] loop iteration of the job's last gang attempt
  // the first schedule pass as it ended (copies taken between the passes: the inputs of QueueStats)
  uint32_t* fp_seq;                // [J] res_seq
  uint8_t* fp_flags;               // [4][J] q_successful, q_rescheduled, q_unsuccessful, q_reason
  uint32_t* gang_fill;             // [G] members gathered so far by the gang iterator
  uint32_t* gang_buf;              // [sum gang_count] members in arrival order
  int32_t* ev_index_of_job;        // [J] "evictedJobs" table: index or -1
  uint32_t* ev_job_by_index;       // [J]
  uint8_t* ev_alive;               // [J]
  uint32_t* evq_start;             // [Q+1] evicted jobs per queue (sorted) for the current pass
  uint32_t* evq_jobs;              // [J]
  uint64_t* sort_keys;             // [J] scratch
  uint64_t* sort_keys2;            // [J]
  uint32_t* sort_vals;             // [J]
  uint32_t* sort_vals2;            // [J]
  uint32_t* counters;              // [16] misc device counters (evicted count, …)
  uint8_t* unfeasible;             // [C] UnfeasibleSchedulingKeys: reason or 0
  unsigned long long* g0;          // [N] nodes sorted by packed level-0 key (best-fit order)
  unsigned long long* g0_tmp;      // [N] radix-sort ping-pong buffer
  uint32_t* g0_sc;                 // [N] static class of the node at every G0 position (aliases g0_tmp after the sort)
  // batch mode scratch, [Q * bt_wq] each
  uint32_t* bt_job;
  uint32_t* bt_cls;
  uint32_t* bt_pos;                // stream position of the item
  uint32_t* bt_rank;               // merged position
  uint2* bt_seq;                   // merged sequence: {job, class}
  int64_t* bt_asum;                // [2][Q][MAX_RESOURCES] requests of every queue's items below the horizon, per batch buffer
  uint32_t* bt_card;               // [2][Q * bt_wq] members of the item (1 = single job, > 1 = a simple gang)
  uint4* bt_item;                  // [2][Q * bt_wq] merged order: {queue, stream position of the item's last job, members, 0}
  uint32_t* bt_gnode;              // [2][Q * bt_wq][64] merged order: the nodes of a gang item's members
  uint32_t* gang_bak;              // the window a gang's candidates come from, as it was when the gang started (32 entries)
  const uint32_t* gang_uni_label;  // [G] uniformity label of the gang (ARMADA_NONE, ARMADA_LABEL_NOT_INDEXED)
  const uint32_t* uni_start;       // [L+1] value slots of label l
  const uint32_t* class_uni_row;   // [C][uni_V][ARMADA_DEV_VARIANTS] static rows with the slot's node selector added
  const uint8_t* gang_simple;      // [G] every member queued, complete, one class, contiguous in its queue (batchable)
  uint32_t* excl;                  // [J][ARMADA_EXCLUDED_KINDS] NumExcludedNodesByReason by kind of the failed single jobs (collect_excl)
  const uint32_t* row_type_excl;   // [rows] nodes of the node types the row does not match (NodeTypesMatchingJob)
  UndoRec* undo_log;               // [3 * J + 16] txn undo records
  // fair preemption scratch
  uint32_t* fp_head;               // [N] most recent visited evicted index on the node
  uint32_t* fp_next;               // [J] chain by evicted index
  uint32_t* nl_start;              // [N+1] node n's evicted jobs = nl_item[nl_start[n] .. nl_start[n+1]) (built after the indices are assigned)
  uint2* nl_item;                  // [E] {evicted index | alive << 31, job class}, per node by descending index
  uint32_t* nl_pos;                // [E] position of evicted index i in nl_item (NONE: the job sits on no node)
  uint32_t* nver;                  // [N] changes of the node's rows / evicted jobs so far (trigger caches)
  uint32_t* fc_ver;                // [8][N] pairs {nver the cached trigger was computed at, cached fair-preemption trigger index (-1 none)}
  uint32_t* bver;                  // [ceil(N/256)] changes of any node of the 256-node block (sum of its nver)
  uint32_t* fc_bver;               // [8][ceil(N/256)] bver the block's cached maximum was computed at
  unsigned long long* fc_bmax;     // [8][ceil(N/256)] largest (trigger + 1) << 32 | node of the block, 0 = none
  // ---- queue / sctx state persisted between kernels ----
  int64_t* q_alloc;                // [Q][D]
  int64_t* q_alloc_pc;             // [Q][PC][D]
  double* q_fair;                  // [Q][3]
  double* q_tokens;                // [Q]
  int64_t* s_scheduled;            // [D]
  int64_t* s_evicted;              // [D]
  int64_t* s_counts;               // [CNT_COUNT] (CountSlot)
  uint32_t* dbg_host;              // [64] host-mapped: written by the device watchdog before it traps
  unsigned long long* stats;       // [STAT_COUNT] counters of the round's schedule passes (StatSlot)
};
