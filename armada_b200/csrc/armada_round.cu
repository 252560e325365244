// armada_round.cu — hand-written CUDA (sm_90a) for Armada's scheduling round.
//
// Reference path being replaced (relative to internal/scheduler/ of armadaproject/armada):
//   scheduling/preempting_queue_scheduler.go:84-285   PreemptingQueueScheduler.Schedule
//   scheduling/queue_scheduler.go:91-272,315-383,495-674  QueueScheduler loop, gang iterator, cost PQ
//   scheduling/gang_scheduler.go:100-254              GangScheduler
//   nodedb/nodedb.go:386-512,605-1098                 ScheduleMany / SelectNode cascade / bind / evict / unbind
//   nodedb/nodeiteration.go:74-382 + encoding.go      best-fit ordered walk
//   scheduling/eviction.go:132-273                    evictors
//   scheduling/context/{scheduling,queue}.go          per-round accounting, fair shares
//   scheduling/fairness/fairness.go:99-105            DRF cost
//
// H100 mapping (see DESIGN.md):
//   * data-parallel phases (bind running jobs, both evictors, gang completion, accounting,
//     result algebra) are grid-wide kernels over the job SoA with int64 atomics on the node SoA;
//   * evicted jobs are ranked per queue with an LSD radix sort on (queue, order-rank) keys;
//   * the inherently sequential QueueScheduler loop runs in ONE persistent CTA of 16 warps
//     (armada_pass.inc, DESIGN §5.1–5.2): warp 15 is the control warp (DRF arg-min over queues,
//     gang iterator, constraints, bind); the 15 index warps keep the best-fit index — all nodes
//     radix-sorted by their packed (resources…, node-id) key in HBM, plus a 32-entry sorted window
//     of the smallest feasible keys per (job class × node-type variant) in shared memory.
//     A probe reads a window head; a bind posts the node's new row to the index warps.
//   Tensor cores are not used: this is integer compare/select work.
#ifdef ARMADA_EMU
#include "cuda_emu.h"  // tools/simt_emu: deterministic CPU SIMT emulator (dev/test tooling only)
#else
#include <cuda_runtime.h>
#define ARMADA_LAUNCH(kern, grid, block, smem, stream, ...) kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define ARMADA_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#define ARMADA_NAMED_BARRIER(id, count) asm volatile("bar.sync %0, %1;" ::"n"(id), "n"(count) : "memory")
static __device__ __forceinline__ void armada_emu_yield() {}
#define ARMADA_NOINLINE __noinline__
#define ARMADA_EMU_MARK(id) ((void)0)
#define ARMADA_PREFETCH_L1(p) asm volatile("prefetch.global.L1 [%0];" ::"l"(p))
#endif

#include <algorithm>
#include <atomic>
#include <memory>
#include <condition_variable>
#include <mutex>
#include <chrono>
#include <thread>
#include <type_traits>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <numeric>
#include <string>
#include <vector>

#include "armada_dev.h"

#define NONE ARMADA_NONE
#define NOPRIO ARMADA_NO_PRIORITY
#define KEY_INF 0xFFFFFFFFFFFFFFFFull
#define FULL 0xFFFFFFFFu

namespace {

thread_local std::string g_last_error;

// =====================================================================================
// device helpers
// =====================================================================================
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }
__device__ __forceinline__ int warp_id() { return threadIdx.x >> 5; }

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long k) {
  unsigned hi = (unsigned)(k >> 32);
  unsigned mhi = __reduce_min_sync(FULL, hi);
  unsigned lo = (hi == mhi) ? (unsigned)k : 0xFFFFFFFFu;
  unsigned mlo = __reduce_min_sync(FULL, lo);
  return ((unsigned long long)mhi << 32) | mlo;
}

__device__ __forceinline__ void atomic_add_i64(int64_t* p, int64_t v) {
  atomicAdd((unsigned long long*)p, (unsigned long long)v);
}

// priorityCutoffFor (nodedb.go:1031-1036): preemptible ⇒ scheduled priority, else every level.
__device__ __forceinline__ int32_t cutoff_for(const DevCfg& c, uint32_t pc, int32_t scheduled_priority) {
  return c.pcs[pc].preemptible ? scheduled_priority : INT32_MAX;
}

// =====================================================================================
// grid-wide kernels (data-parallel phases)
// =====================================================================================

// newAllocatableByPriorityAndResourceType (nodedb.go:1185-1191) + per-job state reset.
__global__ void k_reset(DevCfg c, DevPtrs P) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t stride = (size_t)gridDim.x * blockDim.x;
  size_t DN = (size_t)c.D * c.N;
  for (size_t k = i; k < (size_t)c.PL * DN; k += stride) P.alloc[k] = P.node_allocatable[k % DN];
  for (size_t j = i; j < c.J; j += stride) {
    P.bound_node[j] = NONE;
    P.evicted_on_node[j] = 0;
    P.sched_prio[j] = NOPRIO;
    P.q_successful[j] = P.q_unsuccessful[j] = P.q_rescheduled[j] = P.q_evicted[j] = P.q_reason[j] = 0;
    P.jc_evicted[j] = 0;
    uint32_t g = P.job_gang[j];
    P.jc_card[j] = g == NONE ? 1u : P.gang_card[g];
    P.assigned_node[j] = NONE;
    P.in_preempted[j] = P.in_scheduled[j] = P.in_sae[j] = P.ev_mark[j] = 0;
    P.has_pctx[j] = 0;
    P.res_node[j] = NONE;
    P.res_sched_at[j] = NOPRIO;
    P.res_preempted_at[j] = NOPRIO;
    P.res_method[j] = 0;
    P.res_seq[j] = 0;
    P.ev_index_of_job[j] = -1;
    P.ev_alive[j] = 0;
  }
  for (size_t g = i; g < c.G; g += stride) {
    P.gang_fill[g] = 0;
    P.gang_ev[g] = 0;
  }
  for (size_t k = i; k < (size_t)c.C; k += stride) P.unfeasible[k] = 0;
  if (i < 16) P.counters[i] = 0;
  if (i < STAT_COUNT) P.stats[i] = 0;
}

// CreateAndInsertWithJobDbJobsWithTxn (nodedb.go:43-60): bind every running job at its
// scheduled-at priority.  Integer atomics commute, so the result is order independent.
__global__ void k_bind_running(DevCfg c, DevPtrs P) {
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= c.J) return;
  uint32_t n = P.job_node0[j];
  if (n == NONE) return;
  uint32_t cls = P.job_class[j];
  uint32_t pc = P.class_pc[cls];
  int32_t pr = P.job_sap0[j];
  if (pr == NOPRIO) pr = c.pcs[pc].priority;
  int32_t cut = cutoff_for(c, pc, pr);
  for (int p = 0; p < c.PL; ++p) {
    if (c.priorities[p] > cut) continue;
    for (int d = 0; d < c.D; ++d) {
      int64_t r = P.class_req_node[(size_t)cls * c.D + d];
      if (r) atomic_add_i64(&P.alloc[((size_t)p * c.D + d) * c.N + n], -r);
    }
  }
  P.bound_node[j] = n;
  P.sched_prio[j] = pr;
}

// DominantResourceFairness.UnweightedCostFromAllocation (fairness/fairness.go:103-105).
__device__ double drf_cost_seq(const DevCfg& c, const int64_t* a) {
  double result = -INFINITY;
  for (int d = 0; d < c.D; ++d) {
    double frac = 0.0;
    if (c.total_resources[d] != 0) frac = __ddiv_rn((double)a[d], (double)c.total_resources[d]);
    double v = __dmul_rn(frac, c.drf_mult[d]);
    if (v > result) result = v;
  }
  if (result != result) return result;
  return result > 0.0 ? result : 0.0;
}

// AddQueueSchedulingContext + UpdateFairShares (context/scheduling.go:104-156,252-332).  Q is
// small; one thread restates the iterative water-filling exactly (same op order ⇒ same doubles).
__global__ void k_queue_init(DevCfg c, DevPtrs P) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const int Q = c.Q, D = c.D;
  double weight_sum = 0.0;
  for (int q = 0; q < Q; ++q) {
    for (int d = 0; d < D; ++d) {
      int64_t s = 0;
      for (int pc = 0; pc < c.PC; ++pc) {
        int64_t v = P.queue_alloc_pc0[((size_t)q * c.PC + pc) * D + d];
        P.q_alloc_pc[((size_t)q * c.PC + pc) * D + d] = v;
        s += v;
      }
      P.q_alloc[(size_t)q * D + d] = s;
    }
    P.q_tokens[q] = P.queue_tokens0[q];
    weight_sum += P.queue_weight[q];
  }
  for (int d = 0; d < D; ++d) P.s_scheduled[d] = P.s_evicted[d] = 0;
  for (int k = 0; k < CNT_COUNT; ++k) P.s_counts[k] = 0;
  P.s_counts[CNT_GLOBAL_TOKENS] = __double_as_longlong(c.global_tokens);
  bool total_all_zero = true;
  for (int d = 0; d < D; ++d)
    if (c.total_resources[d] != 0) total_all_zero = false;
  // scratch in q_fair: [q][0]=fair, [1]=capped, [2]=uncapped ; cds/spare/achieved in registers per pass
  // Q <= ARMADA_DEV_MAX_QUEUES, keep small local arrays
  double cds[ARMADA_DEV_MAX_QUEUES], spare[ARMADA_DEV_MAX_QUEUES];
  bool achieved[ARMADA_DEV_MAX_QUEUES];
  for (int q = 0; q < Q; ++q) {
    double v = 1.0;
    if (!total_all_zero) v = drf_cost_seq(c, P.queue_cdemand + (size_t)q * D);
    cds[q] = v;
    spare[q] = 0.0;
    achieved[q] = false;
    P.q_fair[q * 3 + 0] = __ddiv_rn(P.queue_weight[q], weight_sum);
    P.q_fair[q * 3 + 1] = 0.0;
    P.q_fair[q * 3 + 2] = 0.0;
  }
  double unallocated = 1.0;
  for (int it = 0; it < 10 && unallocated > 0.01; ++it) {
    double total_weight = 0.0;
    for (int q = 0; q < Q; ++q)
      if (!achieved[q]) total_weight += P.queue_weight[q];
    for (int q = 0; q < Q; ++q) {
      double tw = total_weight;
      if (achieved[q]) tw += P.queue_weight[q];
      double share = __dmul_rn(__ddiv_rn(P.queue_weight[q], tw), __dsub_rn(unallocated, spare[q]));
      P.q_fair[q * 3 + 2] = __dadd_rn(P.q_fair[q * 3 + 2], share);
    }
    if (total_weight <= 0.0) break;
    for (int q = 0; q < Q; ++q)
      if (!achieved[q])
        P.q_fair[q * 3 + 1] = __dadd_rn(P.q_fair[q * 3 + 1], __dmul_rn(__ddiv_rn(P.queue_weight[q], total_weight), unallocated));
    unallocated = 0.0;
    for (int q = 0; q < Q; ++q) {
      double sp = __dsub_rn(P.q_fair[q * 3 + 1], cds[q]);
      if (sp > 0) {
        P.q_fair[q * 3 + 1] = cds[q];
        achieved[q] = true;
        spare[q] = sp;
        unallocated = __dadd_rn(unallocated, sp);
      } else {
        spare[q] = 0;
      }
    }
  }
}

// evictJobFromNodeInPlace (nodedb.go:974-1003) applied with atomics: markAllocatable at the
// job's cutoff, markAllocated at EvictedPriority ⇒ levels 1.. (p>=0, p<=cutoff) += req.
__device__ void evict_alloc(const DevCfg& c, const DevPtrs& P, uint32_t j, uint32_t n) {
  uint32_t cls = P.job_class[j];
  int32_t cut = cutoff_for(c, P.class_pc[cls], P.sched_prio[j]);
  for (int p = 1; p < c.PL; ++p) {  // level 0 (EvictedPriority) nets to zero
    if (c.priorities[p] > cut) continue;
    for (int d = 0; d < c.D; ++d) {
      int64_t r = P.class_req_node[(size_t)cls * c.D + d];
      if (r) atomic_add_i64(&P.alloc[((size_t)p * c.D + d) * c.N + n], r);
    }
  }
}

// NodeEvictor + balancing job filter (eviction.go:85-103, preempting_queue_scheduler.go:99-134).
// The filter only depends on per-queue constants (queue allocation is read BEFORE any eviction is
// applied to the scheduling context), so it is evaluated once per queue into evict_queue[].
__global__ void k_evict_queue_flags(DevCfg c, DevPtrs P, uint8_t* evict_queue) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= c.Q) return;
  double actual = drf_cost_seq(c, P.q_alloc + (size_t)q * c.D);
  double dc = P.q_fair[q * 3 + 1], fs = P.q_fair[q * 3 + 0];
  double fair = (dc != dc || fs != fs) ? NAN : fmax(dc, fs);  // math.Max
  if (c.protect_uncapped) fair = P.q_fair[q * 3 + 2];
  double fraction = __ddiv_rn(actual, fair);
  evict_queue[q] = !(fraction <= c.protected_fraction);
}

__global__ void k_evict_balance(DevCfg c, DevPtrs P, const uint8_t* evict_queue) {
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= c.J) return;
  uint32_t n = P.bound_node[j];
  if (n == NONE || P.evicted_on_node[j]) return;
  uint32_t q = P.job_queue[j];
  if (q == NONE) return;                                        // invalid_queue
  if (!c.pcs[P.class_pc[P.job_class[j]]].preemptible) return;   // job_not_preemptible
  if (!evict_queue[q]) return;                                  // below_protected_fair_share
  P.ev_mark[j] = 1;
  P.evicted_on_node[j] = 1;
  evict_alloc(c, P, j, n);
  uint32_t g = P.job_gang[j];
  if (g != NONE) P.gang_ev[g] = 1;
}

// NewOversubscribedEvictor (eviction.go:132-184): a node is processed iff some p >= 0 has a
// negative allocatable; a job is evicted iff preemptible and its scheduled-at level is one.
// oversub_mask[n] is computed first (k_oversub_mask) because evicting changes alloc.
__global__ void k_oversub_mask(DevCfg c, DevPtrs P, uint32_t* mask) {
  size_t n = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (n >= c.N) return;
  uint32_t m = 0;
  for (int p = 1; p < c.PL; ++p)
    for (int d = 0; d < c.D; ++d)
      if (P.alloc[((size_t)p * c.D + d) * c.N + n] < 0) m |= 1u << p;
  mask[n] = m;
}

__global__ void k_evict_oversub(DevCfg c, DevPtrs P, const uint32_t* mask) {
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= c.J) return;
  uint32_t n = P.bound_node[j];
  if (n == NONE || P.evicted_on_node[j]) return;
  if (P.job_queue[j] == NONE) return;
  if (!c.pcs[P.class_pc[P.job_class[j]]].preemptible) return;
  int32_t pr = P.sched_prio[j];
  if (pr == NOPRIO) return;
  uint32_t m = mask[n];
  if (!m) return;
  int lvl = -1;
  for (int p = 0; p < c.PL; ++p)
    if (c.priorities[p] == pr) lvl = p;
  if (lvl < 0 || !((m >> lvl) & 1u)) return;
  P.ev_mark[j] = 1;
  P.evicted_on_node[j] = 1;
  evict_alloc(c, P, j, n);
  uint32_t g = P.job_gang[j];
  if (g != NONE) P.gang_ev[g] = 1;
}

// evictGangs (preempting_queue_scheduler.go:353-420): every bound, not yet evicted member of a
// gang with an evicted member is evicted too (its own node is in gangNodeIds by construction).
__global__ void k_evict_gangs(DevCfg c, DevPtrs P) {
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= c.J) return;
  uint32_t g = P.job_gang[j];
  if (g == NONE || !P.gang_ev[g]) return;
  uint32_t n = P.bound_node[j];
  if (n == NONE || P.evicted_on_node[j]) return;
  if (P.sched_prio[j] == NOPRIO) return;
  P.ev_mark[j] = 1;
  P.evicted_on_node[j] = 1;
  evict_alloc(c, P, j, n);
}

// sctx.EvictJob for every evicted job (context/scheduling.go:470-491, queue.go:296-331),
// setEvictedGangCardinality (:458-479), result-set algebra of :141-194, and emission of the
// (queue, order-rank) sort key for InMemoryJobRepository.sortQueue (jobiteration.go:72-95).
__global__ void k_evict_account(DevCfg c, DevPtrs P, int pass) {
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= c.J) return;
  if (!P.ev_mark[j]) return;
  P.ev_mark[j] = 0;
  uint32_t q = P.job_queue[j];
  uint32_t cls = P.job_class[j];
  uint32_t pc = P.class_pc[cls];
  bool sched = P.q_successful[j], resched = P.q_rescheduled[j];
  if (sched || resched) {
    P.q_successful[j] = 0;
    P.q_rescheduled[j] = 0;
  } else {
    P.q_evicted[j] = 1;
  }
  for (int d = 0; d < c.D; ++d) {
    int64_t r = P.class_req_raw[(size_t)cls * c.D + d];
    if (!r) continue;
    atomic_add_i64(&P.q_alloc[(size_t)q * c.D + d], -r);
    atomic_add_i64(&P.q_alloc_pc[((size_t)q * c.PC + pc) * c.D + d], -r);
    if (sched) atomic_add_i64(&P.s_scheduled[d], -r);
    else atomic_add_i64(&P.s_evicted[d], r);
  }
  if (sched) atomic_add_i64(&P.s_counts[CNT_SCHED_JOBS], -1);
  else atomic_add_i64(&P.s_counts[CNT_EVICTED_JOBS], 1);
  // jctx for re-scheduling (eviction.go:241-256)
  P.jc_evicted[j] = 1;
  P.assigned_node[j] = P.bound_node[j];
  uint32_t g = P.job_gang[j];
  P.jc_card[j] = g == NONE ? 1u : P.gang_count[g];
  P.has_pctx[j] = 0;
  if (pass == 1) {
    P.in_preempted[j] = 1;
  } else {
    if (P.in_scheduled[j]) {
      P.in_scheduled[j] = 0;
      P.in_sae[j] = 1;
    } else {
      P.in_preempted[j] = 1;
    }
  }
  uint32_t slot = atomicAdd(&P.counters[0], 1u);
  P.sort_keys[slot] = ((unsigned long long)q << 32) | P.job_rank[j];
  P.sort_vals[slot] = (uint32_t)j;
}

__global__ void k_clear_gang_ev(DevCfg c, DevPtrs P) {
  size_t g = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (g < c.G) P.gang_ev[g] = 0;
}

// ---- LSD radix sort of (u64 key, u32 value) pairs, 8 bits per pass --------------------------
// Ranks eviction candidates per queue: key = queue << 32 | SchedulingOrderCompare rank.
#define RS_THREADS 256
#define RS_ITEMS 16
__global__ void k_rs_hist(const unsigned long long* keys, uint32_t n, int shift, uint32_t* hist /*[256][blocks]*/) {
  __shared__ uint32_t h[256];
  h[threadIdx.x] = 0;
  __syncthreads();
  size_t base = (size_t)blockIdx.x * RS_THREADS * RS_ITEMS;
  for (int i = 0; i < RS_ITEMS; ++i) {
    size_t k = base + (size_t)i * RS_THREADS + threadIdx.x;
    if (k < n) atomicAdd(&h[(keys[k] >> shift) & 255], 1u);
  }
  __syncthreads();
  hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}
// exclusive scan over the digit-major histogram (single block; length = 256 * blocks)
__global__ void k_rs_scan(uint32_t* hist, uint32_t len) {
  __shared__ uint32_t carry;
  __shared__ uint32_t tmp[1024];
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < len; base += 1024) {
    uint32_t i = base + threadIdx.x;
    uint32_t v = i < len ? hist[i] : 0;
    tmp[threadIdx.x] = v;
    __syncthreads();
    for (int off = 1; off < 1024; off <<= 1) {
      uint32_t t = threadIdx.x >= (unsigned)off ? tmp[threadIdx.x - off] : 0;
      __syncthreads();
      tmp[threadIdx.x] += t;
      __syncthreads();
    }
    uint32_t incl = tmp[threadIdx.x];
    if (i < len) hist[i] = carry + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry += incl;
    __syncthreads();
  }
}
__global__ void k_rs_scatter(const unsigned long long* keys, const uint32_t* vals, unsigned long long* keys_out,
                             uint32_t* vals_out, uint32_t n, int shift, const uint32_t* hist) {
  // stable within a block: one thread per digit value walks the block's items in order
  __shared__ unsigned long long sk[RS_THREADS * RS_ITEMS];
  __shared__ uint32_t sv[RS_THREADS * RS_ITEMS];
  size_t base = (size_t)blockIdx.x * RS_THREADS * RS_ITEMS;
  uint32_t cnt = 0;
  for (int i = 0; i < RS_ITEMS; ++i) {
    size_t k = base + (size_t)i * RS_THREADS + threadIdx.x;
    uint32_t li = i * RS_THREADS + threadIdx.x;
    if (k < n) {
      sk[li] = keys[k];
      sv[li] = vals[k];
    }
  }
  __syncthreads();
  uint32_t m = n - base < (size_t)RS_THREADS * RS_ITEMS ? (uint32_t)(n - base) : RS_THREADS * RS_ITEMS;
  uint32_t off = hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x];
  for (uint32_t li = 0; li < m; ++li) {
    if (((sk[li] >> shift) & 255) == threadIdx.x) {
      keys_out[off + cnt] = sk[li];
      vals_out[off + cnt] = sv[li];
      ++cnt;
    }
  }
}

// Packed level-0 key of every node (the input of the G0 sort).  A node with a negative row can
// fit nothing until it changes (and then it is "touched"): it sorts last.
__global__ void k_g0_keys(DevCfg c, DevPtrs P) {
  size_t n = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (n >= c.N) return;
  unsigned long long key = n;
  bool neg = false;
  for (int i = 0; i < c.R; ++i) {
    int64_t v = P.alloc[(size_t)c.indexed_resource[i] * c.N + n];
    neg = neg || v < 0;
    key |= (unsigned long long)v << c.key_shift[i];
  }
  unsigned long long marker = 1ull << c.key_total_bits;
  P.g0[n] = neg ? (marker | n) : key;
}

// Exact mode: the rounded best-fit key of one node at one level (nodedb/encoding.go:37-58):
// field i = floor(allocatable_i / resolution_i) + 1, 0 for a negative row (every negative value sorts
// before every non-negative one and is below every request), low bits = the node's rank in
// (node type, NodeFactory index) order.  Go's roundQuantityToResolution truncates, which for the
// non-negative values that matter is the floor.
__device__ __forceinline__ unsigned long long xfield_of(int64_t v, int64_t res) {
  if (v < 0) return 0ull;
  long long q = (long long)((double)v / (double)res);  // estimate, corrected below
  while (q * res > v) --q;
  while ((q + 1) * res <= v) ++q;
  return (unsigned long long)q + 1ull;
}
__global__ void k_xkeys(DevCfg c, DevPtrs P) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= (size_t)c.PL * c.N) return;
  const size_t p = i / c.N, n = i - p * c.N;
  unsigned long long key = P.node_xrank[n];
  for (int k = 0; k < c.R; ++k)
    key |= xfield_of(P.alloc[(p * c.D + c.indexed_resource[k]) * c.N + n], c.index_res[k]) << c.key_shift[k];
  P.xkey[i] = key;
}

// Snapshot construction on the device (calculateJobSchedulingInfo + constructSchedulingContext,
// scheduling_algo.go:522-632,664-676) when the caller leaves the queue accounting to the library:
// segmented sums over the job SoA — allocation per (queue, priority class) over the running jobs,
// demand over every job (running jobs only for a cordoned queue) — then the demand capped at the
// per-queue per-class limit (constraints.go:187-197) and summed over the classes.
__global__ void k_snapshot_jobs(DevCfg c, DevPtrs P, int64_t* alloc_pc, int64_t* demand_pc, int want_alloc) {
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= c.J) return;
  const uint32_t q = P.job_queue[j];
  if (q == NONE) return;
  const uint32_t cls = P.job_class[j];
  const uint32_t pc = P.class_pc[cls];
  const bool running = P.job_node0[j] != NONE;
  const bool cordoned = P.queue_cordoned[q] != 0;
  for (int d = 0; d < c.D; ++d) {
    const int64_t r = P.class_req_raw[(size_t)cls * c.D + d];
    if (!r) continue;
    if (running && want_alloc) atomic_add_i64(&alloc_pc[((size_t)q * c.PC + pc) * c.D + d], r);
    if (running || !cordoned) atomic_add_i64(&demand_pc[((size_t)q * c.PC + pc) * c.D + d], r);
  }
}
__global__ void k_snapshot_queues(DevCfg c, DevPtrs P, const int64_t* demand_pc, int64_t* cdemand) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= c.Q * c.D) return;
  const int q = i / c.D, d = i - q * c.D;
  int64_t sum = 0;
  for (int pc = 0; pc < c.PC; ++pc) {
    int64_t v = demand_pc[((size_t)q * c.PC + pc) * c.D + d];
    if (P.queue_has_limit[(size_t)q * c.PC + pc]) {
      const int64_t lim = P.queue_limit[((size_t)q * c.PC + pc) * c.D + d];
      if (lim < v) v = lim;
    }
    sum += v;
  }
  cdemand[i] = sum;
}

// static class of the node at every G0 position
__global__ void k_g0_sc(DevCfg c, DevPtrs P) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= c.N) return;
  P.g0_sc[i] = P.node_sclass[(uint32_t)(P.g0[i] & ((1ull << c.node_bits) - 1ull))];
}

// evq_start[q] = first position in the sorted evicted list whose queue is >= q.
__global__ void k_evq_bounds(DevCfg c, DevPtrs P, const unsigned long long* keys, uint32_t n) {
  int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q > c.Q) return;
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    uint32_t mid = (lo + hi) >> 1;
    if ((uint32_t)(keys[mid] >> 32) < (uint32_t)q) lo = mid + 1;
    else hi = mid;
  }
  P.evq_start[q] = lo;
}
__global__ void k_copy_u32(uint32_t* dst, const uint32_t* src, uint32_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
}


// Stream records for the evicted list of the current pass, aligned with evq_jobs (sorted):
// {job, class | flags, assigned node, scheduled-at priority}.  Prefetched by the schedule pass.
__global__ void k_build_ev_records(DevCfg c, DevPtrs P, uint32_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t j = P.evq_jobs[i];
  uint32_t f = P.job_class[j] | 0x80000000u;
  if (P.job_gang[j] != NONE) f |= 0x40000000u;
  if (P.q_evicted[j]) f |= 0x20000000u;
  P.ev_rec[i] = make_uint4(j, f, P.assigned_node[j], (uint32_t)P.sched_prio[j]);
}

// =====================================================================================
// persistent schedule-pass kernel (one CTA)
// =====================================================================================
#include "armada_pass.inc"


// unbindJobs(preempted ∪ scheduledAndEvicted) (preempting_queue_scheduler.go:256, :766-789) and
// the per-job outcome.
__global__ void k_finalize(DevCfg c, DevPtrs P, uint8_t* out_state, uint32_t* out_node, int32_t* out_sched_at,
                           int32_t* out_preempted_at, uint8_t* out_method, uint8_t* out_reason) {
  size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (j >= c.J) return;
  uint8_t st = ARMADA_JOB_NONE;
  uint32_t node = NONE;
  bool pre = P.in_preempted[j], sae = P.in_sae[j];
  if (pre || sae) {
    uint32_t n = P.assigned_node[j];
    if (P.bound_node[j] == n && n != NONE) {  // unbindJobFromNodeInPlace
      uint32_t cls = P.job_class[j];
      bool is_ev = P.evicted_on_node[j];
      int32_t cut = cutoff_for(c, P.class_pc[cls], P.sched_prio[j]);
      for (int p = 0; p < c.PL; ++p) {
        bool hit = is_ev ? (p == 0) : (c.priorities[p] <= cut);
        if (!hit) continue;
        for (int d = 0; d < c.D; ++d) {
          int64_t r = P.class_req_node[(size_t)cls * c.D + d];
          if (r) atomic_add_i64(&P.alloc[((size_t)p * c.D + d) * c.N + n], r);
        }
      }
      P.bound_node[j] = NONE;
      P.evicted_on_node[j] = 0;
    }
  }
  if (pre) {
    st = ARMADA_JOB_PREEMPTED;
    node = P.assigned_node[j];
  } else if (P.in_scheduled[j]) {
    st = ARMADA_JOB_SCHEDULED;
    node = P.res_node[j];
  } else if (sae) {
    st = ARMADA_JOB_SCHEDULED_AND_EVICTED;
    node = P.assigned_node[j];
  } else if (P.q_rescheduled[j]) {
    st = ARMADA_JOB_RESCHEDULED;
    node = P.res_node[j];
  } else if (P.q_unsuccessful[j]) {
    st = ARMADA_JOB_FAILED;
  }
  bool has = P.has_pctx[j] && st != ARMADA_JOB_NONE && st != ARMADA_JOB_FAILED;
  out_state[j] = st;
  out_node[j] = node;
  out_sched_at[j] = has ? P.res_sched_at[j] : NOPRIO;
  out_preempted_at[j] = has ? P.res_preempted_at[j] : NOPRIO;
  out_method[j] = has ? P.res_method[j] : 0;
  out_reason[j] = P.q_unsuccessful[j] ? P.q_reason[j] : 0;
}

}  // namespace

#include "armada_dryrun.inc"
#include "armada_snapshot.inc"
#include "armada_host.inc"
