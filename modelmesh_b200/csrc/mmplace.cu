// mmplace.cu — libmmplace: the sm_90a CUDA implementation behind include/mmplace.h.
//
// Data layout in HBM (DESIGN.md §4), per snapshot epoch (double-buffered, flipped atomically at commit):
//   excl      [n_models][row_words] u32   model x instance exclusion bitmap (loaded ∪ failed, MR:69,73), bit = RANK of
//                                         the instance under PLACEMENT_ORDER; row stride is a multiple of 128 B
//   excl_ranks [n_models] int4            the ranks of a model's <= 4 inline edges (-1: none), r[0] = -2: overflow ids,
//                                         read the row (unsharded fleets)
//   zero_row  [row_words]           u32   all zero, one per fleet: the row of every MMP_DF_REQUEST_MODEL decision (unsharded fleets)
//   cand/pref [n_slots][row_words]  u32   per type-constraint slot: allowed ∧ active / preferred instances (TCM:242-251)
//   candx     [n_slots][row_words]  u32   cand minus likely-replaced replicaset members (MM:4769-4770)
//   full      [row_words]           u32   isFull instances (MM:4640)
//   rows      [n_ranks] RankRow 32 B      per-rank instance columns the walk reads (lru, remaining, count, rpm, idx)
//   csum/lsum [row_words]                 per-32-rank min/max of count / lruTime (threshold searches skip whole words)
//   rank_of   [max_instances] i32, models [n_models] mmp_model_row 24 B, type_slot [n_type_ids] u16
//   nzw/nz_n  [n_slots][row_words] u16    compressed word lists: the row words that hold any candidate of the slot (walks beyond the window)
//   front     [n_models][16] u32          instance-sharded fleets: the first row words, replicated on every shard
// Kernels (DESIGN.md §5, §7):
//   k_place_direct<4, 5>     the scoring kernel (default): one decision per lane, the row rebuilt from the model's excl_ranks,
//                            longer walks through the word lists; optional slot-sorted batches (k_slot_keys + cub radix sort)
//   k_slot_summary, k_place_split, k_place_walk<4, 5>, k_place_ovf   large batches in two passes (launch_split): per-slot
//                            summaries answer the decisions clear of their slot's reach, k_place_direct's body walks the rest
//   k_place_lanes            round 1's streaming kernel (whole rows through TMA landing stages): MMP_KERNEL=lanes and the
//                            collective instance-shard path
//   k_place_small            tiny batches as a stream launch / replayed CUDA graph;  k_place_server: the resident B = 1 server
//   k_place_dealt, k_dealt_wait   instance shards over peer memory;  k_shard_*: the kernels around the NCCL all-reduce
//   k_place<...>             cooperative tiles: traced calls / very wide rows
//   The one-decision-per-lane kernels share their steps through one helper each: no_decision / no_ctx (an absent lane),
//   load_decision_stream (the streamed record load), redo_declined (the warp redo of what the lane routine declined; not
//   k_place_dealt, which assembles the row in shared memory), WinTabs (the window tables in shared memory) and slot_key.
//   k_build_bitmap*, k_sparse_slots + commit_kernels.cuh (device-path commit), scan_kernels.cuh (k_stats, k_reaper_flag,
//   k_lru_events), churn_kernels.cuh (the closed loop), registry_kernels.cuh (k_scale_eval, k_registry_prune)
#include <cuda_runtime.h>
#include <unistd.h>
#include <dlfcn.h>
#include <nccl.h>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "host_state.hpp"

using namespace mmp;

static thread_local std::string g_err;

#define CK(call)                                                                                         \
  do {                                                                                                   \
    cudaError_t e_ = (call);                                                                             \
    if (e_ != cudaSuccess) {                                                                             \
      g_err = std::string(#call) + ": " + cudaGetErrorString(e_);                                        \
      return MMP_E_CUDA;                                                                                 \
    }                                                                                                    \
  } while (0)

// ---------------------------------------------------------------------------------------------------------------
// kernels
// ---------------------------------------------------------------------------------------------------------------
// One thread per model scatters its (<= 4) inline edges into its own bitmap row: no atomics needed.
// (instance-sharded: a stored row holds row words [word_lo, word_hi) at a stride of `stride` words)
// ranks (optional, SnapshotView::excl_ranks): the rank of every bit set here, -1 for an edge that sets none.
__global__ void k_build_bitmap(uint32_t *__restrict__ excl, const int4 *__restrict__ edge_inl,
                               const int32_t *__restrict__ rank_of, int n_models, int stride, int word_lo, int word_hi,
                               int4 *__restrict__ ranks) {
  int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  int4 e = edge_inl[m];
  uint32_t *row = excl + (size_t)m * stride;
  int es[4] = {e.x, e.y, e.z, e.w};
  int rs[4] = {-1, -1, -1, -1};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    if (es[i] >= 0) {
      int r = rank_of[es[i]];
      if (r >= 0 && (r >> 5) >= word_lo && (r >> 5) < word_hi) { row[(r >> 5) - word_lo] |= 1u << (r & 31); rs[i] = r; }
    }
  }
  if (ranks) ranks[m] = make_int4(rs[0], rs[1], rs[2], rs[3]);
}
// (launched after k_build_bitmap: a model with overflow edges gets the EXCL_RANKS_OVF marker in its rank entry)
__global__ void k_build_bitmap_ovf(uint32_t *__restrict__ excl, const OvfEdge *__restrict__ ovf, int n_ovf,
                                   const int32_t *__restrict__ rank_of, int stride, int word_lo, int word_hi, int4 *__restrict__ ranks) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_ovf) return;
  const int m = ovf[i].model, r = rank_of[ovf[i].inst];
  if (r >= 0 && (r >> 5) >= word_lo && (r >> 5) < word_hi)
    atomicOr(&excl[(size_t)m * stride + ((r >> 5) - word_lo)], 1u << (r & 31));
  if (ranks) ranks[m].x = EXCL_RANKS_OVF;
}

// ---- TMA 1-D bulk copy + mbarrier helpers (cp.async.bulk: SASS UBLKCP) ----
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

// The scoring kernel (TMA-staged).  One warp per decision; every warp owns a ring of K exclusion-row buffers in shared
// memory that one elected lane keeps filled ahead with cp.async.bulk (a row is one contiguous, 128-byte-aligned run of
// row_words*4 bytes), so K-1 rows per warp are in flight from HBM while the current decision is resolved out of the
// K-th by window scans (mmp::decide_ctx: 32 words of the row at a time, one per lane).  Decisions are taken in
// batches of 32: lane j prepares the context of decision j (its dependent gathers: decision -> model row,
// rank_of[self] -> rows[self]) one batch ahead into a double-buffered shared-memory table, so those latencies overlap
// across lanes and with the previous batch.
// The warp-wide redo of a decision its tile could not resolve inside its window: the 32-word fast path first, then the
// general routine.  Kept out of line so the kernel's tile loop stays small.
__device__ __noinline__ void decide_warp(const SnapshotView s, const DecisionCtx &c, const uint32_t *erow, const int32_t *extra,
                                         int64_t now, uint64_t seed, uint64_t decision_id, int32_t *target, int32_t *n_candidates,
                                         int32_t *first_rank = nullptr, int32_t *flags = nullptr) {
  Coop32 co;
  DecideOut o;
  o.first_rank = -1; o.flags = 0;
  const bool whole_rows = s.word_lo == 0 && s.word_hi == s.row_words;  // decide_fast reads rows by absolute word index
  if (!whole_rows || !decide_fast<false>(s, c, erow, now, seed, decision_id, co, o)) decide_ctx(s, c, erow, extra, now, seed, decision_id, co, o, nullptr);
  *target = o.target; *n_candidates = o.n_candidates;
  if (first_rank) { *first_rank = o.first_rank; *flags = o.flags; }
}

// ---- what the one-decision-per-lane kernels share: the record of a lane without a decision, the context of a lane whose
// decision is absent, the streamed record load and the warp redo of what the lane routine declined ----
__device__ __forceinline__ mmp_decision_in no_decision() {
  mmp_decision_in d;
  d.model = -1; d.self = -1; d.last_used = 0; d.flags = 0; d.fresh = -1; d.extra_off = 0; d.extra_n = 0;
  return d;
}
__device__ __forceinline__ DecisionCtx no_ctx() {
  DecisionCtx c;
  c.slot = -2; c.self_rank = -1; c.self_bits = 0; c.self_count = 0;
  return c;
}
// decision record i, read once as a stream: no L1 allocation (the lane routine's tables are what should stay there)
__device__ __forceinline__ mmp_decision_in load_decision_stream(const mmp_decision_in *in, int i) {
  const int4 *dp = reinterpret_cast<const int4 *>(in + i);
  int4 v[2];
#pragma unroll
  for (int h = 0; h < 2; h++)
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v[h].x), "=r"(v[h].y), "=r"(v[h].z), "=r"(v[h].w) : "l"(dp + h));
  mmp_decision_in d;
  d.model = v[0].x; d.self = v[0].y; d.last_used = (int64_t)(((uint64_t)(uint32_t)v[0].w << 32) | (uint32_t)v[0].z);
  d.flags = (uint32_t)v[1].x; d.fresh = v[1].y; d.extra_off = v[1].z; d.extra_n = v[1].w;
  return d;
}
// The lanes of `pending` declined their decisions: the whole warp redoes them one at a time with decide_warp, reading
// the row of lane l's row_id (excl_row_id) from global memory, with lane l's context c staged in *ctx_s.  The answer
// lands in lane l's o: target, n_candidates, first_rank and flags.
__device__ __forceinline__ void redo_declined(uint32_t pending, int lane, const DecisionCtx &c, int32_t row_id, uint64_t my_id, DecisionCtx *ctx_s,
                                              const SnapshotView &s, const int32_t *extra, int64_t now, uint64_t seed, DecideOut &o) {
  while (pending) {
    const int l = __ffs((int)pending) - 1;
    pending &= pending - 1;
    if (lane == l) *ctx_s = c;
    const int32_t rl = __shfl_sync(0xffffffffu, row_id, l);
    const uint64_t idl = __shfl_sync(0xffffffffu, my_id, l);
    __syncwarp();
    int32_t t2, c2, f2, g2;
    decide_warp(s, *ctx_s, excl_row(s, rl), extra, now, seed, idl, &t2, &c2, &f2, &g2);
    if (lane == l) { o.target = t2; o.n_candidates = c2; o.first_rank = f2; o.flags = g2; }
    __syncwarp();
  }
}

struct RingLayout {
  uint32_t row_bytes, k;
  size_t per_warp;
  __host__ __device__ RingLayout(int row_words, int k_) : row_bytes((uint32_t)row_words * 4u), k((uint32_t)k_) {
    per_warp = ((size_t)k * row_bytes + 32 * sizeof(DecisionCtx) + (size_t)k * 8 + 127) / 128 * 128;
  }
};

template <int WARPS, int K, int MINB, int T, bool TRACE>
__global__ void __launch_bounds__(WARPS * 32, MINB) k_place(const SnapshotView s, const mmp_decision_in *__restrict__ in, int n,
                                                     const FreshRow *__restrict__ fresh, int n_fresh,
                                                     const int32_t *__restrict__ extra, mmp_decision_out *__restrict__ out,
                                                     mmp_decision_trace *__restrict__ tr, uint32_t *__restrict__ cand,
                                                     int64_t now, uint64_t seed, uint64_t id_base) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int RW = s.excl_stride;  // words per stored row
  const bool whole_rows = s.word_lo == 0 && s.word_hi == s.row_words;  // decide_fast needs whole rows (not instance-sharded)
  const RingLayout lay(RW, K);
  const uint32_t row_bytes = lay.row_bytes;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned char *base = smem_raw + (size_t)wib * lay.per_warp;
  uint32_t *rows_s = reinterpret_cast<uint32_t *>(base);
  DecisionCtx *ctx_s = reinterpret_cast<DecisionCtx *>(base + (size_t)K * row_bytes);  // [32]
  uint64_t *bars = reinterpret_cast<uint64_t *>(base + (size_t)K * row_bytes + 32 * sizeof(DecisionCtx));
  if (lane == 0) {
    for (int k = 0; k < K; k++) mbar_init(&bars[k], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const int nb = (n + 31) >> 5;
  const int gw = blockIdx.x * WARPS + wib, nw = gridDim.x * WARPS;
  Coop32 co;
  CoopTile<T> cot;
  constexpr int G = 32 / T;  // decisions resolved per step by the tiles of one warp
  uint32_t use = 0;  // ring position of the next row to consume (warp-uniform)
  auto prep = [&](int batch, DecisionCtx *dst) {  // lane j stages the context of decision j of `batch`
    const int i = batch * 32 + lane;
    DecisionCtx cn;
    cn.slot = -2;  // absent
    cn.d.model = 0; cn.d.flags = 0;
    if (batch < nb && i < n) {
      const int4 *dp = reinterpret_cast<const int4 *>(in + i);
      int4 a = __ldg(dp), b = __ldg(dp + 1);
      mmp_decision_in d;
      d.model = a.x; d.self = a.y; d.last_used = (int64_t)(((uint64_t)(uint32_t)a.w << 32) | (uint32_t)a.z);
      d.flags = (uint32_t)b.x; d.fresh = b.y; d.extra_off = b.z; d.extra_n = b.w;
      prepare_ctx(s, d, fresh, n_fresh, extra, cn);
    }
    dst[lane] = cn;
  };
  auto issue = [&](int row_id, uint32_t pos) {  // lane 0 only; row_id from excl_row_id
    const uint32_t sl = pos % (uint32_t)K;
    mbar_expect_tx(&bars[sl], row_bytes);
    bulk_g2s(rows_s + (size_t)sl * RW, excl_row(s, row_id), row_bytes, &bars[sl]);
  };
  int b = gw;
  prep(b, ctx_s);
  __syncwarp();
  if (b < nb) {
    const int count = min(32, n - b * 32);
    if (lane == 0)
      for (int t = 0; t < K && t < count; t++) issue(excl_row_id(s, ctx_s[t].d.model, ctx_s[t].d.flags), (uint32_t)t);
  }
  while (b < nb) {
    const int bn = b + nw;
    const DecisionCtx *cc = ctx_s;
    // the next batch's contexts are staged when this batch is done (one buffer); only its row ids are fetched now,
    // because the ring must start loading its first rows K positions before the batch boundary
    int next_model = -1;
    {
      const int i = bn * 32 + lane;
      if (bn < nb && i < n) next_model = excl_row_id(s, __ldg(&in[i].model), __ldg(&in[i].flags));
    }
    const int count = min(32, n - b * 32);
    mmp_decision_out mine{MMP_TARGET_NONE, 0};
    int nm_next[K];  // model indices of the next batch's first K decisions (held by every lane, used by lane 0)
#pragma unroll
    for (int t = 0; t < K; t++) nm_next[t] = -2;
    bool nm_loaded = false;
    int jbase = 0;
    auto refill = [&](int jdone) {  // lane 0: the row of decision jdone has been consumed; fetch the one K positions ahead
      const int t = jdone + K;
      int nm = 0;
      bool have = false;
      if (t < count) { nm = excl_row_id(s, cc[t].d.model, cc[t].d.flags); have = true; }
      else if (t - count < K && nm_next[t - count] != -1) { nm = nm_next[t - count]; have = true; }
      if (have) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        issue(nm, use + (uint32_t)(jdone - jbase) + (uint32_t)K);
      }
    };
    if constexpr (!TRACE) {
      // ---- G decisions per warp step: each T-lane tile resolves one out of a T-word window (CoopTile<T>); whatever a
      // tile cannot resolve inside its window is redone warp-wide by the general routine ----
      const int tile = lane / T;
      for (int jp = 0; jp < count; jp += G) {
        jbase = jp;
        if (!nm_loaded && jp + G - 1 + K >= count) {
#pragma unroll
          for (int t = 0; t < K; t++) nm_next[t] = __shfl_sync(0xffffffffu, next_model, t);
          nm_loaded = true;
        }
        const int j = jp + tile;
        const bool valid = j < count;
        const uint32_t myuse = use + (uint32_t)tile;
        const uint32_t slot = myuse % (uint32_t)K, parity = (myuse / (uint32_t)K) & 1u;
        if (valid) { while (!mbar_try_wait(&bars[slot], parity)) {} }
        DecideOut o;
        o.target = MMP_TARGET_NONE; o.n_candidates = 0;
        bool resolved = false;
        if (valid && whole_rows) resolved = decide_fast<false>(s, cc[j], rows_s + (size_t)slot * RW, now, seed, pick_id(cc[j].d, id_base + (uint64_t)(b * 32 + j)), cot, o);
        __syncwarp();
        {
          const uint32_t pending = __ballot_sync(0xffffffffu, valid && !resolved);
#pragma unroll 1
          for (int h = 0; h < G; h++) {
            if (pending & (1u << (h * T))) {
              const int jj = jp + h;
              const uint32_t sl2 = (use + (uint32_t)h) % (uint32_t)K;
              int32_t t2, c2;
              decide_warp(s, cc[jj], rows_s + (size_t)sl2 * RW, extra, now, seed, pick_id(cc[jj].d, id_base + (uint64_t)(b * 32 + jj)), &t2, &c2);
              if (tile == h) { o.target = t2; o.n_candidates = c2; }
            }
          }
        }
#pragma unroll
        for (int h = 0; h < G; h++) {
          const int th = __shfl_sync(0xffffffffu, o.target, h * T), ch = __shfl_sync(0xffffffffu, o.n_candidates, h * T);
          if (lane == jp + h) { mine.target = th; mine.n_candidates = ch; }
        }
        __syncwarp();
        const int nstep = min(G, count - jp);
        if (lane == 0)
          for (int h = 0; h < nstep; h++) refill(jp + h);
        use += (uint32_t)nstep;
      }
    } else {
      for (int j = 0; j < count; j++) {
        jbase = j;
        if (!nm_loaded && j + K >= count) {
#pragma unroll
          for (int t = 0; t < K; t++) nm_next[t] = __shfl_sync(0xffffffffu, next_model, t);
          nm_loaded = true;
        }
        const uint32_t slot = use % (uint32_t)K, parity = (use / (uint32_t)K) & 1u;
        while (!mbar_try_wait(&bars[slot], parity)) {}
        const uint32_t *erow = rows_s + (size_t)slot * RW;
        const int gi = b * 32 + j;
        DecideOut o;
        if (cand || !whole_rows || !decide_fast<true>(s, cc[j], erow, now, seed, pick_id(cc[j].d, id_base + (uint64_t)gi), co, o))
          decide_ctx(s, cc[j], erow, extra, now, seed, pick_id(cc[j].d, id_base + (uint64_t)gi), co, o, cand ? cand + (size_t)gi * 2 * s.row_words : nullptr);
        if (lane == j) { mine.target = o.target; mine.n_candidates = o.n_candidates; }
        if (tr && lane == 0) {
          mmp_decision_trace t;
          t.best = o.best; t.n_remaining = o.n_remaining; t.pick_index = o.pick_index; t.flags = o.flags;
          t.cut_rank = o.cut_rank; t.best_rank = o.best_rank; t.reserved[0] = t.reserved[1] = 0;
          tr[gi] = t;
        }
        __syncwarp();
        if (lane == 0) refill(j);
        use++;
      }
    }
    if (lane < count) out[b * 32 + lane] = mine;
    b = bn;
    __syncwarp();
    prep(b, ctx_s);
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// k_place_lanes — the production scoring kernel: ONE DECISION PER LANE.
//
// One persistent block per SM.  Shared memory holds NS "landing stages" of 32 exclusion rows each (TMA bulk-copy
// destinations, one mbarrier per stage) that the block's warps share, and a small private window buffer per warp.
// A warp's step over a batch of 32 decisions:
//   1. batches are dealt round-robin to the grid's warps; the batch's 32 decision records were requested a step ahead;
//   2. take a landing stage (FIFO tickets); every lane issues the cp.async.bulk of its model's bitmap row into it
//      (32 arrivals + 32 x row bytes of transaction count on the stage's mbarrier);
//   3. finish the decision context (type slot, the caller's row, self's mask bits) while the rows stream in; its
//      first gathers (model row from HBM, rank_of[self]) were issued a step ahead -- a warp stalls in order;
//   4. when the stage has landed, copy the first WIN words of its row and the word holding self's bit out of the stage
//      and RELEASE the stage, so the next 41 KB of rows is in flight while this warp is still computing;
//   5. resolve the 32 decisions in lockstep from the window buffer (mmp::decide_stream) and write the 8-byte results.
// PLACEMENT_ORDER puts best and the shortlist at the front of the rank order, so the window answers almost every
// decision; what it cannot (long walks on adversarial fleets, uncommon paths) is redone by the whole warp with the
// cooperative general routine reading the row from global memory (it was just streamed: L2).
// The stages keep ~NS x 41 KB per SM in flight from HBM independently of how many warps are computing, and the
// per-decision instruction cost is ~85 warp instructions instead of ~450 for a cooperative tile (ncu, C3 sweep).
// ---------------------------------------------------------------------------------------------------------------
static constexpr int SHARD_FRONT_WORDS = 16;  // instance-sharded fleets: row words replicated on every shard (512 ranks: where almost every walk ends)
static constexpr int LANE_WIN = MMP_LANE_WIN;  // row words copied out of the landing stage per decision: the first LANE_WIN words of the
                                               // stored row (384 ranks); later steps go through the compressed word list and read the row from L2
static constexpr int LANE_STRIDE = LANE_WIN + 1;  // words per lane in the window buffer (odd: bank-conflict free)
static constexpr int SPLIT_MIN_BATCH = 1 << 18;  // k_place_direct batches from this size take the two-pass path (launch_split)
static constexpr int LANE_BUDGET = 192;  // walk steps a lane may spend before handing its decision to the whole warp
static constexpr int LANE_SLOTS = 64;    // type-constraint mask slots whose window words are kept in shared memory
static constexpr int LANE_WARPS = 12;    // warps per block of k_place_lanes
static constexpr int LANE_STAGES = 4;    // landing stages per SM at most: a fifth takes the shared-memory carve-out from 196 to
                                         // 228 KB and leaves too little L1 for the lane tables to stay resident
// The window part of the lane tables in shared memory (k_place_lanes, k_place_server): the masks of the first LANE_SLOTS
// slots and full / csum / count_col / rows over the first LANE_WIN words of this process's rows, zero past their end.
struct WinTabs {
  uint32_t cx[LANE_SLOTS * LANE_WIN], p[LANE_SLOTS * LANE_WIN], full[LANE_WIN];
  WordSumI csum[LANE_WIN];
  __align__(16) int32_t count[LANE_WIN * 32];
  __align__(16) RankRow rows[LANE_WIN * 32];
  // thread tid of nthreads copies its share of the tables (the caller synchronises).  N: the type of the stride, blockDim.x
  // or a constant int, as each kernel steps its loops (it decides how far the compiler unrolls them)
  template <class N>
  __device__ __forceinline__ void fill(const SnapshotView &s, int tid, N nthreads) {
    const int WS = s.word_lo;
    const uint32_t win_words = (uint32_t)min(LANE_WIN, s.word_hi - s.word_lo);
    const int nsl = min(s.n_slots, LANE_SLOTS);
    const uint32_t *gcx = s.any_rs ? s.candx : s.cand;
    for (int i = tid; i < nsl * LANE_WIN; i += nthreads) {
      const int sl = i / LANE_WIN, w = i - sl * LANE_WIN;
      const bool in = (uint32_t)w < win_words;
      cx[i] = in ? gcx[(size_t)sl * s.row_words + WS + w] : 0u;
      p[i] = in ? s.pref[(size_t)sl * s.row_words + WS + w] : 0u;
    }
    for (int w = tid; w < LANE_WIN; w += nthreads) {
      const bool in = (uint32_t)w < win_words;
      full[w] = in ? s.full[WS + w] : 0u;
      csum[w] = in ? s.csum[WS + w] : WordSumI{0, 0};
    }
    for (int i = tid; i < LANE_WIN * 32; i += nthreads) {
      const int r = WS * 32 + i;
      const bool in = (uint32_t)(i >> 5) < win_words && r < s.n_ranks;
      count[i] = in ? s.count_col[r] : 0;
      RankRow z; z.lru = 0; z.rem = 0; z.count = 0; z.rpm = 0; z.idx = -1; z.flags = 0;
      rows[i] = in ? s.rows[r] : z;
    }
  }
  // T (the slot's global tables) with its window part pointed here: indexed by absolute row word / rank, so biased by the
  // window's first word
  __device__ __forceinline__ LaneTables view(const LaneTables &T, int slot, int word_lo) const {
    LaneTables Tw = T;
    if (slot < LANE_SLOTS) { Tw.cx = cx + slot * LANE_WIN - word_lo; Tw.p = p + slot * LANE_WIN - word_lo; }
    Tw.full = full - word_lo; Tw.csum = csum - word_lo; Tw.count_col = count - word_lo * 32; Tw.rows = rows - word_lo * 32;
    return Tw;
  }
};
struct LaneLayout {
  uint32_t row_bytes, stride, stage_bytes, ns, warps;
  uint32_t off_bar, off_busy, off_uses, off_warp, per_warp;
  uint32_t off_tabs;  // the WinTabs
  size_t total;
  __host__ __device__ LaneLayout(int row_words, int ns_, int warps_, bool front) {
    row_bytes = (uint32_t)row_words * 4u; stride = row_bytes + 16u;  // + 16: lanes copying their windows out spread over the banks
    stage_bytes = (32u * stride + 127u) / 128u * 128u;
    ns = (uint32_t)ns_; warps = (uint32_t)warps_;
    off_bar = ns * stage_bytes; off_busy = off_bar + ns * 8u; off_uses = off_busy + ns * 4u;
    off_warp = (off_uses + ns * 4u + 127u) / 128u * 128u;
    per_warp = 32u * (LANE_STRIDE + MMP_CHUNK_WORDS) * 4u + (uint32_t)((sizeof(DecisionCtx) + 15) / 16 * 16);
    off_tabs = (off_warp + warps * per_warp + 15u) / 16u * 16u;
    total = front ? (size_t)off_tabs + sizeof(WinTabs) : (size_t)off_tabs;
  }
};

__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__global__ void __launch_bounds__(LANE_WARPS * 32, 1) k_place_lanes(const SnapshotView s, const mmp_decision_in *__restrict__ in, int n,
                                                                    const FreshRow *__restrict__ fresh, int n_fresh,
                                                                    const int32_t *__restrict__ extra, mmp_decision_out *__restrict__ out,
                                                                    int64_t now, uint64_t seed, uint64_t id_base, int ns,
                                                                    int emit_keys, int shard_rank, const int32_t *__restrict__ orig_id, int budget) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int RW = s.excl_stride;  // words per stored row (the whole row unless the fleet is instance-sharded)
  const LaneLayout lay(RW, ns, LANE_WARPS, true);
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + lay.off_bar);
  int *ticket = reinterpret_cast<int *>(smem_raw + lay.off_busy);               // next stage ticket of this block
  uint32_t *released = reinterpret_cast<uint32_t *>(smem_raw + lay.off_uses);  // [ns] completed uses per stage
  uint32_t *win = reinterpret_cast<uint32_t *>(smem_raw + lay.off_warp + (size_t)wib * lay.per_warp);  // [32][LANE_STRIDE]
  uint32_t *chunk = win + 32 * LANE_STRIDE;                                                             // [32][MMP_CHUNK_WORDS]
  DecisionCtx *ctx_one = reinterpret_cast<DecisionCtx *>(chunk + 32 * MMP_CHUNK_WORDS);
  if (threadIdx.x == 0) {
    for (int k = 0; k < ns; k++) { mbar_init(&bars[k], 32); released[k] = 0; }
    *ticket = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  const int nb = (n + 31) >> 5;
  // ---- the window part of the lane tables in shared memory (with the SM's shared memory given to the landing stages the
  // L1 is too small to keep them resident: every in-window gather would be an L2 round trip) ----
  WinTabs *tabs = reinterpret_cast<WinTabs *>(smem_raw + lay.off_tabs);
  const uint32_t win_words = (uint32_t)min(LANE_WIN, s.word_hi - s.word_lo);
  const bool front = nb >= 64;  // tiny launches read the snapshot directly
  if (front) tabs->fill(s, threadIdx.x, blockDim.x);
  __syncthreads();
  // batches of 32 decisions are dealt round-robin to the grid's warps (consecutive batches to the warps of one block)
  const int gw = blockIdx.x * LANE_WARPS + wib, nw = gridDim.x * LANE_WARPS;
  auto load_dec = [&](int b, mmp_decision_in &d) -> bool {
    const int i = b * 32 + lane;
    if (b >= nb || i >= n) return false;
    d = load_decision_stream(in, i);
    return true;
  };
  // Software pipeline per warp (every load is issued at least one phase before its first use, because a warp stalls in
  // order): batch k+2 is claimed and its records requested while batch k is resolved; the first context gathers of batch
  // k+1 (model row from HBM, rank_of[self]) are issued right after batch k's stage has been handed on; what depends on
  // them (type slot, the caller's row, self's mask bits) is gathered while batch k+1's rows are in flight.
  int b = gw;
  mmp_decision_in d;
  bool valid = load_dec(b, d);
  CtxA ca;
  prepare_ctx_a(s, d, ca);
  int bn = b + nw;
  mmp_decision_in dn;
  bool valid_n = load_dec(bn, dn);
  while (b < nb) {
    // ---- acquire a landing stage and send the 32 rows on their way ----
    int st = 0;
    uint32_t parity = 0;
    if (lane == 0) {
      // stages are handed out in ticket order (a FIFO ring): ticket q uses stage q % ns for the (q / ns)-th time and may
      // start when that stage's previous use has been released.  The wait is a plain poll of a shared-memory counter:
      // a hand-over costs tens of cycles (a sleeping poll left the stages idle two thirds of the time).
      const uint32_t q = (uint32_t)atomicAdd(ticket, 1);
      st = (int)(q % (uint32_t)ns);
      const uint32_t u = q / (uint32_t)ns;
      volatile uint32_t *rel = released + st;
      while (*rel < u) {}
      __threadfence_block();
      parity = u & 1u;
    }
    st = __shfl_sync(0xffffffffu, st, 0);
    parity = __shfl_sync(0xffffffffu, parity, 0);
    unsigned char *stage = smem_raw + (size_t)st * lay.stage_bytes;
    const uint32_t *my_row = reinterpret_cast<const uint32_t *>(stage + (size_t)lane * lay.stride);
    // row of this decision: its model's, or row i of a gathered row set (orig_id != nullptr: the instance-shard gather pass)
    const int m = orig_id ? (valid ? b * 32 + lane : 0) : (valid ? excl_row_id(s, d.model, d.flags) : 0);
    DecisionCtx c = no_ctx();
    bool skip = false;  // instance-sharded, not the first shard: an entry in a lower shard wins, the row is not even read
    if (s.word_lo > 0) {
      if (valid) { prepare_ctx_b(s, d, ca, fresh, n_fresh, extra, c); skip = shard_cannot_win(s, c, ca.mr.reserved); }
    }
    if (valid && !skip) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // the previous owner's reads precede this async write
      mbar_expect_tx(&bars[st], lay.row_bytes);
      bulk_g2s(const_cast<uint32_t *>(my_row), excl_row(s, m), lay.row_bytes, &bars[st]);
    } else mbar_arrive(&bars[st]);
    // ---- the rest of this batch's context while its rows are in flight ----
    if (s.word_lo == 0 && valid) prepare_ctx_b(s, d, ca, fresh, n_fresh, extra, c);
    while (!mbar_try_wait(&bars[st], parity)) {}
    // ---- copy the window out and hand the stage on ----
    uint32_t self_eword = 0;
    {
      uint32_t *w = win + lane * LANE_STRIDE;
      if (!skip) {
#pragma unroll
        for (int j = 0; j < LANE_WIN / 4; j++) {
          if ((uint32_t)(j * 4) < win_words) {  // (stored rows are a multiple of 4 words: a 16-byte read stays inside the row)
            const uint4 q = *reinterpret_cast<const uint4 *>(my_row + j * 4);
            w[j * 4] = q.x; w[j * 4 + 1] = q.y; w[j * 4 + 2] = q.z; w[j * 4 + 3] = q.w;
          }
        }
      }
      const int sw = c.self_rank >> 5;
      if (!skip && c.self_rank >= 0 && sw >= s.word_lo && sw < s.word_hi) self_eword = my_row[sw - s.word_lo];
    }
    __syncwarp();
    if (lane == 0) { __threadfence_block(); atomicAdd(const_cast<uint32_t *>(released + st), 1u); }
    // ---- requests for the batches behind this one ----
    CtxA cn;
    cn.ok = 0; cn.self_rank = -1;
    if (valid_n) prepare_ctx_a(s, dn, cn);
    const int bnn = bn + nw;
    mmp_decision_in dnn;
    const bool valid_nn = load_dec(bnn, dnn);
    // ---- one decision per lane, the 32 lanes in lockstep ----
    DecideOut o;
    const uint64_t my_id = pick_id(d, id_base + (uint64_t)(orig_id ? (valid ? orig_id[b * 32 + lane] : 0) : b * 32 + lane));
    const int slot = c.slot >= 0 ? ctx_slot(c) : 0;
    const LaneTables T = lane_tables_global(s, slot);
    const LaneTables Tw = front ? tabs->view(T, slot, s.word_lo) : T;
    const bool handled = decide_stream(s, Tw, T, c, valid && !skip, win + lane * LANE_STRIDE, win_words, RowPtr{excl_row(s, m), (uint32_t)s.word_lo},
                                       self_eword, now, seed, my_id, WarpVote(), o, budget, chunk + lane * MMP_CHUNK_WORDS);
    // ---- what the lane routine declined: the whole warp redoes it, reading the row from global memory (L2) ----
    redo_declined(__ballot_sync(0xffffffffu, valid && !skip && !handled), lane, c, m, my_id, ctx_one, s, extra, now, seed, o);
    if (valid) {
      if (emit_keys) {  // instance-sharded: one min-loc key per decision instead of the result (same 8 bytes)
        uint64_t key = ~(uint64_t)0;
        if (!skip) key = shard_key(o, shard_rank);
        reinterpret_cast<uint64_t *>(out)[b * 32 + lane] = key;
      } else out[b * 32 + lane] = mmp_decision_out{o.target, o.n_candidates};
    }
    b = bn; d = dn; valid = valid_n; ca = cn;
    bn = bnn; dn = dnn; valid_n = valid_nn;
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// k_place_small -- the latency path (B = 1 .. a few hundred decisions: one getNext on a request thread).  No landing
// stages: a lane reads its decision's row words straight from global memory in chunks of 8 (decide_stream with an empty
// window), so a single decision costs a handful of dependent L2 reads instead of a whole pipeline step of
// k_place_lanes.  hdr (optional, pinned mapped memory): {now, seed, n} read by the kernel, so that a captured CUDA graph can
// be replayed for every call without touching its node parameters.
// ---------------------------------------------------------------------------------------------------------------
struct SmallHdr { long long now; unsigned long long seed, id_base; int n, n_fresh, n_extra, stop; unsigned long long seq; unsigned long long pad[2]; };
static_assert(sizeof(SmallHdr) == 64, "header is one 64-byte line");
// one block of 32 threads resolves decisions [blk * 32, blk * 32 + 32) of a small batch
__device__ __forceinline__ void place_small_block(const SnapshotView &s, const mmp_decision_in *in, int n, const FreshRow *fresh, int n_fresh,
                                                  const int32_t *extra, mmp_decision_out *out, int64_t now, uint64_t seed, uint64_t id_base,
                                                  int budget, int blk, DecisionCtx *ctx_one) {
  const int lane = threadIdx.x;
  const int i = blk * 32 + lane;
  const bool valid = i < n;
  mmp_decision_in d = no_decision();
  if (valid) d = in[i];
  DecisionCtx c = no_ctx();
  if (valid) prepare_ctx(s, d, fresh, n_fresh, extra, c);
  const int m = excl_row_id(s, d.model, d.flags);
  const uint32_t *row = excl_row(s, m);
  const LaneTables T = lane_tables_global(s, c.slot >= 0 ? ctx_slot(c) : 0);
  uint32_t self_eword = 0;
  if (valid && c.self_rank >= 0) self_eword = __ldg(row + (c.self_rank >> 5));
  DecideOut o;
  const uint64_t my_id = pick_id(d, id_base + (uint64_t)i);
  __shared__ uint32_t chunk_b[32 * MMP_CHUNK_WORDS];  // (callers are one-warp blocks)
  const bool handled = decide_stream<TabGlob>(s, T, T, c, valid, nullptr, 0u, RowPtr{row, (uint32_t)s.word_lo}, self_eword,
                                              now, seed, my_id, WarpVote(), o, budget, chunk_b + lane * MMP_CHUNK_WORDS);
  redo_declined(__ballot_sync(0xffffffffu, valid && !handled), lane, c, m, my_id, ctx_one, s, extra, now, seed, o);
  if (valid) out[i] = mmp_decision_out{o.target, o.n_candidates};
}
__global__ void __launch_bounds__(32) k_place_small(const SnapshotView s_arg, const mmp_decision_in *__restrict__ in, int n_arg,
                                                    const FreshRow *__restrict__ fresh, int n_fresh_arg, const int32_t *__restrict__ extra,
                                                    mmp_decision_out *__restrict__ out, int64_t now_arg, uint64_t seed_arg, uint64_t id_base_arg,
                                                    const volatile SmallHdr *hdr, int budget) {
  __shared__ DecisionCtx ctx_one;
  SnapshotView s = s_arg;
  if (hdr) s.n_extra = hdr->n_extra;
  place_small_block(s, in, hdr ? hdr->n : n_arg, fresh, hdr ? hdr->n_fresh : n_fresh_arg, extra, out, hdr ? hdr->now : now_arg,
                    hdr ? hdr->seed : seed_arg, hdr ? hdr->id_base : id_base_arg, budget, blockIdx.x, &ctx_one);
}

// ---------------------------------------------------------------------------------------------------------------
// k_place_direct -- one decision per lane WITHOUT landing stages and without reading the bitmap: a lane loads its
// model's 16-byte entry of excl_ranks (the ranks of its <= 4 inline edges) and rebuilds from it, in registers, the first
// MMP_LANE_WIN words of its exclusion row into its warp's window buffer, self's row word, and whatever word a walk needs
// beyond the window (RowRanks in decide_stream's second loop).  A plain decision reads 80 B, all of it sequential in a
// sweep: 32 B record, 24 B model row, 16 B ranks, 8 B result -- instead of scattered sectors of its 1 280-byte row.
// A model with overflow ids (more than 4: rare) is marked in its entry and resolved from its row by the warp
// (decide_warp).  Without the 41 KB stages an SM holds 16-32 warps instead of 12.  One warp per batch of 32 decisions,
// no per-warp software pipeline: the other resident warps hide the gathers.
// ---------------------------------------------------------------------------------------------------------------
// how many type slots have fewer than `few` candidates among the first `win` row words (one thread per slot)
__global__ void k_sparse_slots(const uint32_t *__restrict__ cx, int row_words, int n_slots, int word_lo, int win, int few, int *__restrict__ out) {
  const int sl = blockIdx.x * blockDim.x + threadIdx.x;
  if (sl >= n_slots) return;
  int c = 0;
  for (int w = word_lo; w < word_lo + win && w < row_words; w++) c += __popc(cx[(size_t)sl * row_words + w]);
  if (c < few) atomicAdd(out, 1);
}
// type slot of every decision of a batch (the sort key of the slot-ordered launch) and the identity permutation
__global__ void k_slot_keys(const SnapshotView s, const mmp_decision_in *__restrict__ in, int n, uint16_t *__restrict__ keys, int32_t *__restrict__ idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const mmp_decision_in d = in[i];
  uint32_t k = 0xffffu;
  if (request_model(d) ? (d.model >= 0 && d.model < 65535) : (d.model >= 0 && d.model < s.n_models))
    k = slot_key(s, request_model(d) ? d.model : s.models[d.model].type_id);
  keys[i] = (uint16_t)k;
  idx[i] = i;
}
template <int WARPS>
__device__ __forceinline__ void place_direct(const SnapshotView &s, const mmp_decision_in *__restrict__ in, int n,
                                             const FreshRow *__restrict__ fresh, int n_fresh, const int32_t *__restrict__ extra,
                                             mmp_decision_out *__restrict__ out, int64_t now, uint64_t seed, uint64_t id_base, int budget,
                                             const int32_t *__restrict__ perm) {
  __shared__ uint32_t win_s[WARPS][32 * LANE_STRIDE];
  __shared__ uint32_t chunk_s[WARPS][32 * MMP_CHUNK_WORDS];
  __shared__ DecisionCtx ctx_w[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j_ = (blockIdx.x * WARPS + warp) * 32 + lane;
  const bool valid = j_ < n;
  // perm (optional): the batch in type-slot order -- decisions of one slot walk the same masks, so the 32 lanes of a warp
  // finish their walks together instead of waiting for the longest (fleets with sparse candidate sets: C5)
  const int i = valid ? (perm ? perm[j_] : j_) : 0;
  mmp_decision_in d = no_decision();
  if (valid) d = load_decision_stream(in, i);
  const int m = excl_row_id(s, d.model, d.flags);
  // the model's excluded ranks go out first: they depend on the record only (a request-model decision has none: its
  // model's instances are among its extras)
  RowRanks row;
  row.r[0] = row.r[1] = row.r[2] = row.r[3] = -1;
  if (valid && m != ZERO_ROW) row = load_ranks(s.excl_ranks + (size_t)m * 4);
  DecisionCtx c = no_ctx();
  if (valid) prepare_ctx(s, d, fresh, n_fresh, extra, c);
  // a model with overflow ids is resolved from its bitmap row by the warp (decide_warp)
  const bool ovf = valid && row.overflow();
  const uint32_t win_words = (uint32_t)min(LANE_WIN, s.word_hi - s.word_lo);
  const uint32_t self_eword = c.self_rank >= 0 ? row.word((uint32_t)c.self_rank >> 5) : 0u;
  // the window's words go to the warp's window buffer (one shared-memory load per window step: rebuilding each word from
  // the ranks at every step measured slower), its tables are the snapshot's own (global memory: the read-only path)
  uint32_t *w = win_s[warp] + lane * LANE_STRIDE;
#pragma unroll
  for (int j = 0; j < LANE_WIN; j++) w[j] = 0u;
#pragma unroll
  for (int j = 0; j < 4; j++) {  // (a negative rank is no word of the window)
    const uint32_t wi = (uint32_t)row.r[j] >> 5;
    if (wi < (uint32_t)LANE_WIN) w[wi] |= 1u << (row.r[j] & 31);
  }
  __syncwarp();
  const LaneTables T = lane_tables_global(s, c.slot >= 0 ? ctx_slot(c) : 0);
  DecideOut o;
  const uint64_t my_id = pick_id(d, id_base + (uint64_t)i);
  const bool handled = decide_stream<TabGlob>(s, T, T, c, valid && !ovf, w, win_words, row, self_eword, now, seed, my_id, WarpVote(), o, budget,
                                              chunk_s[warp] + lane * MMP_CHUNK_WORDS);
  redo_declined(__ballot_sync(0xffffffffu, valid && (ovf || !handled)), lane, c, m, my_id, &ctx_w[warp], s, extra, now, seed, o);
  if (valid) out[i] = mmp_decision_out{o.target, o.n_candidates};
}
template <int WARPS, int MINB>
__global__ void __launch_bounds__(WARPS * 32, MINB) k_place_direct(const SnapshotView s, const mmp_decision_in *__restrict__ in, int n,
                                                                  const FreshRow *__restrict__ fresh, int n_fresh,
                                                                  const int32_t *__restrict__ extra, mmp_decision_out *__restrict__ out,
                                                                  int64_t now, uint64_t seed, uint64_t id_base, int budget,
                                                                  const int32_t *__restrict__ perm) {
  place_direct<WARPS>(s, in, n, fresh, n_fresh, extra, out, now, seed, id_base, budget, perm);
}
// k_place_direct over the first *n_live positions of perm, a worklist whose length is on the device (the grid is sized
// for n: blocks past the length leave at once)
template <int WARPS, int MINB>
__global__ void __launch_bounds__(WARPS * 32, MINB) k_place_walk(const SnapshotView s, const mmp_decision_in *__restrict__ in, int n,
                                                                const FreshRow *__restrict__ fresh, int n_fresh,
                                                                const int32_t *__restrict__ extra, mmp_decision_out *__restrict__ out,
                                                                int64_t now, uint64_t seed, uint64_t id_base, int budget,
                                                                const int32_t *__restrict__ perm, const int32_t *__restrict__ n_live) {
  n = min(n, __ldg(n_live));
  if ((int)(blockIdx.x * WARPS * 32) >= n) return;
  place_direct<WARPS>(s, in, n, fresh, n_fresh, extra, out, now, seed, id_base, budget, perm);
}

// ---- the two-pass path of a large batch (launch_place, DESIGN.md §5.2) ----
// one lane per (type slot, c_self): the slot summaries of this call's view (slot_summary); also zeroes the worklist counters
__global__ void __launch_bounds__(128) k_slot_summary(const SnapshotView s, int64_t now, SlotSummary *__restrict__ sums,
                                                      int32_t *__restrict__ members, int32_t *__restrict__ counts) {
  __shared__ uint32_t win_s[4][32 * LANE_STRIDE];
  __shared__ uint32_t chunk_s[4][32 * MMP_CHUNK_WORDS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = blockIdx.x * 128 + threadIdx.x, sl = t >> 1, cs = t & 1;
  if (t < 2) counts[t] = 0;
  const bool active = sl < s.n_slots;
  uint32_t *w = win_s[warp] + lane * LANE_STRIDE;
#pragma unroll
  for (int j = 0; j < LANE_WIN; j++) w[j] = 0u;
  __syncwarp();
  const int slot = active ? sl : 0;
  const uint32_t win_words = (uint32_t)min(LANE_WIN, s.word_hi - s.word_lo);
  const LaneTables T = lane_tables_global(s, slot);
  slot_summary(s, T, slot, active, cs, w, win_words, now, WarpVote(), chunk_s[warp] + lane * MMP_CHUNK_WORDS, sums[slot],
               members + ((size_t)slot * 2 + cs) * SPLIT_CAP);
}
// appends v to list (length in *count) for the lanes where p holds: one atomic per warp
__device__ __forceinline__ void warp_append(bool p, int32_t v, int32_t *list, int32_t *count) {
  const uint32_t m = __ballot_sync(0xffffffffu, p);
  if (!m) return;
  const int lane = threadIdx.x & 31, leader = __ffs((int)m) - 1;
  int base = 0;
  if (lane == leader) base = atomicAdd(count, __popc(m));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (p) list[base + __popc(m & ((1u << lane) - 1u))] = v;
}
// one thread per decision: answered from its slot's summary (split_answer), or put on a worklist -- a model with overflow
// ids on ovf_list (k_place_ovf), everything else on walk_list (k_place_direct).  keys / key_idx (sparse snapshots): the
// slot-order sort of the batch, the walked decisions' keys below everyone else's.
__global__ void __launch_bounds__(256) k_place_split(const SnapshotView s, const mmp_decision_in *__restrict__ in, int n,
                                                     const FreshRow *__restrict__ fresh, int n_fresh, mmp_decision_out *__restrict__ out,
                                                     int64_t now, uint64_t seed, uint64_t id_base, const SlotSummary *__restrict__ sums,
                                                     const int32_t *__restrict__ members, int32_t *__restrict__ walk_list,
                                                     int32_t *__restrict__ ovf_list, int32_t *__restrict__ counts, uint16_t *__restrict__ keys,
                                                     int32_t *__restrict__ key_idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool valid = i < n;
  mmp_decision_in d = no_decision();
  if (valid) d = load_decision_stream(in, i);
  const int m = excl_row_id(s, d.model, d.flags);
  RowRanks row;  // (read as k_place_direct reads it: its overflow mark routes the decision the same way)
  row.r[0] = row.r[1] = row.r[2] = row.r[3] = -1;
  if (valid && m != ZERO_ROW) row = load_ranks(s.excl_ranks + (size_t)m * 4);
  CtxA a;
  a.ok = 0; a.self_rank = -1; a.mr.type_id = 0;
  if (valid) prepare_ctx_a(s, d, a);
  mmp_decision_out r;
  const bool fast = valid && split_answer(s, d, a, row, fresh, n_fresh, sums, members, now, seed, pick_id(d, id_base + (uint64_t)i), r);
  if (fast) out[i] = r;
  const bool ovf = valid && !fast && row.overflow();
  const bool walk = valid && !fast && !ovf;
  warp_append(walk, i, walk_list, counts);
  warp_append(ovf, i, ovf_list, counts + 1);
  if (keys && valid) {
    uint32_t k = 0xffffu;
    if (walk) k = a.ok ? slot_key(s, a.mr.type_id) : 0xfffeu;
    keys[i] = (uint16_t)k;
    key_idx[i] = i;
  }
}
// the decisions of ovf_list (length *count), one warp each, resolved as k_place_direct's warp redo resolves them
__global__ void __launch_bounds__(128) k_place_ovf(const SnapshotView s, const mmp_decision_in *__restrict__ in, const int32_t *__restrict__ list,
                                                   const int32_t *__restrict__ count, const FreshRow *__restrict__ fresh, int n_fresh,
                                                   const int32_t *__restrict__ extra, mmp_decision_out *__restrict__ out, int64_t now,
                                                   uint64_t seed, uint64_t id_base) {
  __shared__ DecisionCtx ctx_w[4];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = __ldg(count);
  for (int k = blockIdx.x * 4 + warp; k < n; k += gridDim.x * 4) {
    const int i = list[k];
    const mmp_decision_in d = in[i];
    if (lane == 0) prepare_ctx(s, d, fresh, n_fresh, extra, ctx_w[warp]);
    __syncwarp();
    int32_t t, c;
    decide_warp(s, ctx_w[warp], excl_row(s, excl_row_id(s, d.model, d.flags)), extra, now, seed, pick_id(d, id_base + (uint64_t)i), &t, &c);
    if (lane == 0) out[i] = mmp_decision_out{t, c};
    __syncwarp();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// k_place_server -- the B = 1 path without a launch per call.  One warp stays resident for a BOUNDED time (life_ns, or
// idle_ns without a request), polling the sequence word of a request header in pinned mapped host memory; a request (up to
// 32 decisions, laid out like the graph path's buffer) is resolved with the same routine as k_place_small and answered by
// a release store of the sequence number into the response line.  The host posts a request with one store and spins on
// the response: two PCIe round trips instead of launch + synchronise.  Bounded lifetime: anything that waits for the
// device to drain (cudaFree inside a commit) waits at most life_ns, and a crashed host leaves no kernel behind.
// ---------------------------------------------------------------------------------------------------------------
// request line 0 (one 64-byte line = one PCIe read per poll): everything a single decision without side tables needs.
// seq: low 56 bits = request counter, top 8 bits = kind (1: one decision, its fresh row and up to SRV_INLINE_EXTRA extra
// excludes -- if any -- in line 1; 2: a batch of up to 32 laid out like the graph path's buffer, sizes in line 1; 0xff: leave)
static constexpr int SRV_INLINE_EXTRA = 4;  // a request-thread getNext carries its model's copies and failures (< 5 and < 3 at a cache miss)
struct SrvLine0 { unsigned long long seq; long long now; unsigned long long seed, id_base; mmp_decision_in d; };
struct SrvLine1 { int n, n_fresh, n_extra, pad; FreshRow fr; int32_t extra[SRV_INLINE_EXTRA]; unsigned long long pad2; };
struct ServerResp { unsigned long long done_seq; int alive, served; mmp_decision_out out0; unsigned long long pad[5]; };
static_assert(sizeof(SrvLine0) == 64 && sizeof(SrvLine1) == 64 && sizeof(ServerResp) == 64, "one line each");
__global__ void __launch_bounds__(32) k_place_server(const SnapshotView s_arg, volatile SrvLine0 *l0, volatile SrvLine1 *l1, volatile ServerResp *resp,
                                                     const mmp_decision_in *in_tab, const FreshRow *fresh_tab, const int32_t *extra,
                                                     mmp_decision_out *out_tab, unsigned long long life_ns, unsigned long long idle_ns, int budget) {
  __shared__ DecisionCtx ctx_one;
  __shared__ __align__(16) uint32_t line_s[16];
  __shared__ __align__(16) uint32_t line1_s[16];  // kind 1's line 1: fresh row and inline extras (extra[] of the decision)
  __shared__ FreshRow fresh_s;
  __shared__ uint32_t win_s[32 * LANE_STRIDE];
  __shared__ uint32_t chunk_v[32 * MMP_CHUNK_WORDS];
  // the window part of the lane tables, as in k_place_lanes: the in-window steps of a decision read shared memory only
  __shared__ WinTabs tabs;
  const int lane = threadIdx.x;
  const uint32_t win_words = (uint32_t)min(LANE_WIN, s_arg.word_hi - s_arg.word_lo);
  tabs.fill(s_arg, lane, 32);
  __syncwarp();
  unsigned long long t0, t_last, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  t_last = t0;
  unsigned long long last = resp->done_seq;
  int served = 0;
  for (;;) {
    // one poll = one 64-byte read of line 0 (lanes 0..15, four bytes each)
    uint32_t v = 0;
    if (lane < 16) v = reinterpret_cast<volatile uint32_t *>(l0)[lane];
    const unsigned long long seq = (unsigned long long)__shfl_sync(0xffffffffu, v, 0) | ((unsigned long long)__shfl_sync(0xffffffffu, v, 1) << 32);
    if (seq == last) {
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
      if (t - t0 > life_ns || t - t_last > idle_ns) break;
      continue;
    }
    const unsigned kind = (unsigned)(seq >> 56);
    if (kind == 0xffu) break;
    if (lane < 16) line_s[lane] = v;
    __syncwarp();
    const long long now = (long long)((unsigned long long)line_s[2] | ((unsigned long long)line_s[3] << 32));
    const unsigned long long seed = (unsigned long long)line_s[4] | ((unsigned long long)line_s[5] << 32);
    const unsigned long long id_base = (unsigned long long)line_s[6] | ((unsigned long long)line_s[7] << 32);
    SnapshotView s = s_arg;
    if (kind == 1u) {
      // ---- one decision: record from the line, window straight from the row, tables from shared memory ----
      const bool valid = lane == 0;
      mmp_decision_in d = no_decision();
      if (valid) d = *reinterpret_cast<const mmp_decision_in *>(line_s + 8);
      int n_fresh = 0;
      s.n_extra = 0;
      // the decision's extra[] is line 1's inline part (extra_off = 0, at most SRV_INLINE_EXTRA entries: place_server)
      const int32_t *extra1 = reinterpret_cast<const int32_t *>(line1_s + offsetof(SrvLine1, extra) / 4);
      if (__shfl_sync(0xffffffffu, d.fresh, 0) >= 0 || __shfl_sync(0xffffffffu, d.extra_n, 0) > 0) {  // side tables: a second read, one line
        if (lane < 16) line1_s[lane] = reinterpret_cast<volatile uint32_t *>(l1)[lane];
        __syncwarp();
        n_fresh = (int)line1_s[offsetof(SrvLine1, n_fresh) / 4];
        s.n_extra = (int)line1_s[offsetof(SrvLine1, n_extra) / 4];
        if (lane == 0) fresh_s = *reinterpret_cast<const FreshRow *>(line1_s + offsetof(SrvLine1, fr) / 4);
        __syncwarp();
      }
      const int m = excl_row_id(s, d.model, d.flags);
      const uint32_t *row = excl_row(s, m);
      uint4 q[LANE_WIN / 4];
#pragma unroll
      for (int j = 0; j < LANE_WIN / 4; j++) {
        q[j] = make_uint4(0u, 0u, 0u, 0u);
        if (valid && (uint32_t)(j * 4) < win_words) q[j] = __ldg(reinterpret_cast<const uint4 *>(row) + j);
      }
      DecisionCtx c = no_ctx();
      if (valid) prepare_ctx(s, d, &fresh_s, min(n_fresh, 1), extra1, c);
      uint32_t self_eword = 0;
      if (valid && c.self_rank >= 0) self_eword = __ldg(row + (c.self_rank >> 5) - s.word_lo);
      uint32_t *w = win_s + lane * LANE_STRIDE;
#pragma unroll
      for (int j = 0; j < LANE_WIN / 4; j++) { w[j * 4] = q[j].x; w[j * 4 + 1] = q[j].y; w[j * 4 + 2] = q[j].z; w[j * 4 + 3] = q[j].w; }
      __syncwarp();
      const int slot = c.slot >= 0 ? ctx_slot(c) : 0;
      const LaneTables T = lane_tables_global(s, slot);
      const LaneTables Tw = tabs.view(T, slot, s.word_lo);
      DecideOut o;
      const uint64_t my_id = pick_id(d, id_base);
      const bool handled = decide_stream(s, Tw, T, c, valid, w, win_words, RowPtr{row, (uint32_t)s.word_lo}, self_eword, now, seed, my_id, WarpVote(), o, budget,
                                         chunk_v + lane * MMP_CHUNK_WORDS);
      // pending: lane 0, the only lane with a decision, if it declined
      redo_declined(__shfl_sync(0xffffffffu, (uint32_t)!handled, 0), lane, c, m, my_id, &ctx_one, s, extra1, now, seed, o);
      if (lane == 0) { resp->out0.target = o.target; resp->out0.n_candidates = o.n_candidates; }
    } else {
      // ---- a batch of up to 32 through the mapped tables (sizes in line 1) ----
      int n = 0, n_fresh = 0, n_extra = 0;
      if (lane == 0) { n = l1->n; n_fresh = l1->n_fresh; n_extra = l1->n_extra; }
      n = __shfl_sync(0xffffffffu, n, 0); n_fresh = __shfl_sync(0xffffffffu, n_fresh, 0); n_extra = __shfl_sync(0xffffffffu, n_extra, 0);
      s.n_extra = n_extra;
      place_small_block(s, in_tab, n, fresh_tab, n_fresh, extra, out_tab, now, seed, id_base, budget, 0, &ctx_one);
    }
    __threadfence_system();
    __syncwarp();
    if (lane == 0) asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&resp->done_seq), "l"(seq) : "memory");
    last = seq;
    served++;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_last));
    if (t_last - t0 > life_ns) break;  // (a busy server leaves too: the host restarts it with its next request)
  }
  if (lane == 0) {
    resp->served = served;
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(&resp->alive), "r"(0) : "memory");
  }
}

// ---------------------------------------------------------------------------------------------------------------
// instance-sharded placement with peer access (SURVEY.md §8e) -- k_place_dealt.  The decisions of a batch are DEALT to the
// shards by warp batch (batch wb goes to shard wb % G), so G GPUs each decide 1/G of the batch instead of all of it.  A
// decision is resolved completely by the shard it was dealt to: the first SHARD_FRONT_WORDS words of its exclusion row are
// replicated on every shard (DeviceSnapshot::front: where almost every walk ends), the words beyond come from the column
// block of the shard that owns them -- this GPU's HBM or a peer's, through its NVLink-mapped pointer (RowDealt).  The
// result (8 bytes) is stored into the result buffer of EVERY shard (peer stores over NVLink), so all shards end with the
// whole batch's answers.  No collective call, no host synchronisation between the shards: k_dealt_wait, the next kernel on
// the stream, raises this shard's flag in every peer's flag array (release, system scope) and spins until all G flags of
// the step have arrived (bounded by a timeout: a missing peer ends in an error, not a hang).
// ---------------------------------------------------------------------------------------------------------------
static constexpr int MAX_SHARDS = 16;
struct DealtPeers {
  const uint32_t *blocks[MAX_SHARDS];   // column block of every shard for the current epoch (own block: local pointer)
  mmp_decision_out *out[MAX_SHARDS];    // result buffer of every shard for this step's parity
  unsigned long long *flags[MAX_SHARDS];  // flag array of every shard: [G] arrival counters
};
template <int WARPS, int MINB>
__global__ void __launch_bounds__(WARPS * 32, MINB) k_place_dealt(const SnapshotView s, const uint32_t *__restrict__ front, int front_words,
                                                            const uint16_t *__restrict__ nzw_full, const int32_t *__restrict__ nz_n_full,
                                                            const __grid_constant__ DealtPeers P, int G, int me, const mmp_decision_in *__restrict__ in, int n,
                                                            const FreshRow *__restrict__ fresh, int n_fresh, const int32_t *__restrict__ extra,
                                                            int64_t now, uint64_t seed, uint64_t id_base, int budget, unsigned long long step,
                                                            unsigned int *__restrict__ done, unsigned long long *__restrict__ remote_words) {
  extern __shared__ __align__(16) unsigned char dealt_smem[];
  __shared__ DecisionCtx ctx_w[WARPS];
  __shared__ uint32_t win_d[WARPS][32 * LANE_STRIDE];
  __shared__ uint32_t chunk_d[WARPS][32 * MMP_CHUNK_WORDS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int RW = s.row_words;
  uint32_t *row_s = reinterpret_cast<uint32_t *>(dealt_smem) + (size_t)warp * RW;  // whole row of a decision redone by the warp
  const long long wb = ((long long)blockIdx.x * WARPS + warp) * G + me;             // this warp's batch of 32 decisions
  const long long i = wb * 32 + lane;
  const bool valid = i < n;
  mmp_decision_in d = no_decision();
  if (valid) d = in[i];
  DecisionCtx c = no_ctx();
  if (valid) prepare_ctx(s, d, fresh, n_fresh, extra, c);
  const int m = (valid && d.model >= 0 && d.model < s.n_models) ? d.model : 0;
  LaneTables T = lane_tables_global(s, c.slot >= 0 ? ctx_slot(c) : 0);
  {
    const int slot = c.slot >= 0 ? ctx_slot(c) : 0;
    T.nzw = nzw_full + (size_t)slot * RW; T.nz_n = nz_count(nz_n_full[slot]); T.nz_skip = nz_skipped(nz_n_full[slot]);
  }
  RowDealt row{front, P.blocks, (uint32_t)front_words, (uint32_t)s.excl_stride, (uint32_t)s.excl_stride, (uint64_t)m, (uint32_t)me, 0u};
  uint32_t self_eword = 0;
  if (valid && c.self_rank >= 0) self_eword = row.word((uint32_t)(c.self_rank >> 5));
  // the window: the first MMP_LANE_WIN words of the row, from the replicated front (local memory on every shard)
  const uint32_t win_words = (uint32_t)min(min(LANE_WIN, front_words), RW);
  uint32_t *w = win_d[warp] + lane * LANE_STRIDE;
  if ((front_words & 3) == 0) {  // (front rows are 16-byte aligned then: three vector loads)
#pragma unroll
    for (int j = 0; j < LANE_WIN / 4; j++) {
      uint4 q = make_uint4(0u, 0u, 0u, 0u);
      if (valid && (uint32_t)(j * 4) < win_words) q = __ldg(reinterpret_cast<const uint4 *>(front + (size_t)m * front_words) + j);
      w[j * 4] = q.x; w[j * 4 + 1] = q.y; w[j * 4 + 2] = q.z; w[j * 4 + 3] = q.w;
    }
  } else {
#pragma unroll
    for (int j = 0; j < LANE_WIN; j++) w[j] = (valid && (uint32_t)j < win_words) ? __ldg(front + (size_t)m * front_words + j) : 0u;
  }
  __syncwarp();
  if (win_words < (uint32_t)LANE_WIN) T.nz_skip = 0;  // (a front shorter than the window: no window at all)
  DecideOut o;
  o.target = MMP_TARGET_NONE; o.n_candidates = 0;
  const uint64_t my_id = pick_id(d, id_base + (uint64_t)i);
  const bool handled = decide_stream<TabGlob>(s, T, T, c, valid, w, win_words < (uint32_t)LANE_WIN ? 0u : win_words, row, self_eword, now, seed, my_id,
                                              WarpVote(), o, budget, chunk_d[warp] + lane * MMP_CHUNK_WORDS);
  // (redo_declined, but the row is assembled in shared memory: passing that step to the helper as a callable costs this
  // kernel 8 B more stack and spills)
  uint32_t pending = __ballot_sync(0xffffffffu, valid && !handled);
  while (pending) {  // the cooperative general routine over the whole row, assembled in shared memory
    const int l = __ffs((int)pending) - 1;
    pending &= pending - 1;
    if (lane == l) ctx_w[warp] = c;
    const int ml = __shfl_sync(0xffffffffu, m, l);
    const uint64_t idl = __shfl_sync(0xffffffffu, my_id, l);
    RowDealt rl = row;
    rl.model = (uint64_t)ml; rl.remote = 0;
    for (int w = lane; w < RW; w += 32) row_s[w] = rl.word((uint32_t)w);
    row.remote += rl.remote;
    __syncwarp();
    int32_t t2, c2, f2, g2;
    decide_warp(s, ctx_w[warp], row_s, extra, now, seed, idl, &t2, &c2, &f2, &g2);
    if (lane == l) { o.target = t2; o.n_candidates = c2; }
    __syncwarp();
  }
  if (valid) {
    const mmp_decision_out r{o.target, o.n_candidates};
    for (int g = 0; g < G; g++) P.out[g][i] = r;  // 256 contiguous bytes per warp and shard
  }
  uint32_t rem = row.remote;
  for (int of = 16; of > 0; of >>= 1) rem += __shfl_xor_sync(0xffffffffu, rem, of);
  if (lane == 0 && rem) atomicAdd(remote_words, (unsigned long long)rem);
  // (arrival is signalled by k_dealt_wait, the next kernel on this stream: a kernel boundary orders this kernel's stores --
  // peer stores included -- before it, which spares every block a system-scope fence over NVLink)
}
// one warp, launched behind k_place_dealt on the same stream: lane g raises this shard's flag in shard g's flag array
// (release, system scope: ordered after everything the dealt kernel stored) and then waits for shard g's arrival at `step`;
// err[0] = 1 after `timeout_ns`
__global__ void k_dealt_wait(const __grid_constant__ DealtPeers P, int G, int me, unsigned long long step, unsigned long long timeout_ns, int *err) {
  const int g = threadIdx.x;
  if (g >= G) return;
  __threadfence_system();
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(P.flags[g] + me), "l"(step) : "memory");
  const unsigned long long *flags = P.flags[me];
  unsigned long long t0, t1, v;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  for (;;) {
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flags + g) : "memory");
    if (v >= step) break;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
    if (t1 - t0 > timeout_ns) { atomicExch(err, 1); break; }
    __nanosleep(200);
  }
}
// ---------------------------------------------------------------------------------------------------------------
// instance-sharded combine (SURVEY.md §8e): kernels around the one collective
// ---------------------------------------------------------------------------------------------------------------
// keys -> results in place (both 8 bytes per decision) + a flag per decision whose winning shard left it open
__global__ void k_shard_decode(uint64_t *__restrict__ keys_out, int n, uint8_t *__restrict__ open_flag, int *__restrict__ n_open) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint64_t k = keys_out[i];
  int32_t t, c;
  shard_key_decode(k, t, c);
  const bool open = shard_key_open(k);
  open_flag[i] = open ? 1 : 0;
  if (open) atomicAdd(n_open, 1);  // only a count: the ordered list is built (cub::DeviceSelect) when there is anything to list
  reinterpret_cast<mmp_decision_out *>(keys_out)[i] = mmp_decision_out{open ? MMP_TARGET_NONE : t, open ? 0 : c};
}
// this shard's block of the exclusion row of every open decision, and the decision records themselves, compacted
__global__ void k_shard_pack(const SnapshotView s, const mmp_decision_in *__restrict__ in, const int32_t *__restrict__ open_idx,
                             int n_open, uint32_t *__restrict__ blocks, mmp_decision_in *__restrict__ in_open) {
  const int stride = s.excl_stride;
  const size_t total = (size_t)n_open * stride;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(t / stride), w = (int)(t - (size_t)j * stride);
    const mmp_decision_in d = in[open_idx[j]];
    const int m = (d.model >= 0 && d.model < s.n_models) ? d.model : 0;
    blocks[t] = s.excl[(size_t)m * stride + w];
    if (w == 0) in_open[j] = d;
  }
}
// gathered[g][j][stride] -> rows[j][row_words]
__global__ void k_shard_assemble(const uint32_t *__restrict__ gathered, int n_open, int stride, int shards, int row_words,
                                 uint32_t *__restrict__ rows) {
  const size_t total = (size_t)n_open * row_words;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(t / row_words), w = (int)(t - (size_t)j * row_words);
    const int g = w / stride;
    rows[t] = g < shards ? gathered[((size_t)g * n_open + j) * stride + (w - g * stride)] : 0u;
  }
}
__global__ void k_shard_scatter(const mmp_decision_out *__restrict__ res, const int32_t *__restrict__ open_idx, int n_open,
                                mmp_decision_out *__restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_open) out[open_idx[j]] = res[j];
}

// Registry sweep: decision i = place model first_model + i for instance self[i] (self[0] when self_stride == 0), lastUsed
// from the model row, favourSelf from a bit vector -- the records the scoring kernel reads, built on the device
__global__ void k_expand_sweep(mmp_decision_in *__restrict__ out, int n, int first_model, const int32_t *__restrict__ self,
                               int self_stride, const uint32_t *__restrict__ favour_bits) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  mmp_decision_in d;
  d.model = first_model + i;
  d.self = self[(size_t)i * self_stride];
  d.last_used = 0;
  d.flags = MMP_DF_MODEL_LAST_USED | ((favour_bits && ((favour_bits[i >> 5] >> (i & 31)) & 1u)) ? MMP_DF_FAVOUR_SELF : 0u);
  d.fresh = -1; d.extra_off = 0; d.extra_n = 0;
  out[i] = d;
}

// NCCL is bound at run time (dlopen): a single-GPU deployment needs no NCCL at all, and inside a process that already
// carries a copy (PyTorch's) the same one is used.
struct NcclApi {
  void *lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
static NcclApi &nccl_api() {
  static NcclApi a = [] {
    NcclApi x;
    for (const char *name : {"libnccl.so.2", "libnccl.so"}) {
      x.lib = dlopen(name, RTLD_NOW | RTLD_GLOBAL);
      if (x.lib) break;
    }
    if (!x.lib) return x;
    x.GetUniqueId = (decltype(x.GetUniqueId))dlsym(x.lib, "ncclGetUniqueId");
    x.CommInitRank = (decltype(x.CommInitRank))dlsym(x.lib, "ncclCommInitRank");
    x.CommDestroy = (decltype(x.CommDestroy))dlsym(x.lib, "ncclCommDestroy");
    x.AllReduce = (decltype(x.AllReduce))dlsym(x.lib, "ncclAllReduce");
    x.AllGather = (decltype(x.AllGather))dlsym(x.lib, "ncclAllGather");
    x.GetErrorString = (decltype(x.GetErrorString))dlsym(x.lib, "ncclGetErrorString");
    x.ok = x.GetUniqueId && x.CommInitRank && x.CommDestroy && x.AllReduce && x.AllGather && x.GetErrorString;
    return x;
  }();
  return a;
}
#define NK(call)                                                                                         \
  do {                                                                                                   \
    ncclResult_t r_ = (call);                                                                            \
    if (r_ != ncclSuccess) {                                                                             \
      g_err = std::string(#call) + ": " + nccl_api().GetErrorString(r_);                                 \
      return MMP_E_NCCL;                                                                                 \
    }                                                                                                    \
  } while (0)

// ---------------------------------------------------------------------------------------------------------------
// device-side containers
// ---------------------------------------------------------------------------------------------------------------
// Every CUDA resource a fleet holds is owned by one of these: it is freed when its owner goes out of scope, so a struct
// that holds them needs no cleanup list.  A device buffer that grows on demand (ensure); the memory is its own.
struct DevBuf {
  void *p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(DevBuf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
  DevBuf &operator=(DevBuf &&o) noexcept {
    if (this != &o) { release(); p = std::exchange(o.p, nullptr); cap = std::exchange(o.cap, 0); }
    return *this;
  }
  ~DevBuf() { release(); }
  cudaError_t ensure(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    release();
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e == cudaSuccess) cap = want;
    return e;
  }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
  template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

// A runtime handle and the call that frees it.  It converts to the raw handle, so it is passed as one; put() frees the
// handle held and hands the runtime's create call the slot for a new one.
template <class T, cudaError_t (*Free)(T)>
class Owned {
 public:
  Owned() = default;
  Owned(Owned &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
  Owned &operator=(Owned &&o) noexcept { if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); } return *this; }
  ~Owned() { reset(); }
  void reset() { if (h_) Free(h_); h_ = nullptr; }
  T *put() { reset(); return &h_; }
  T get() const { return h_; }
  operator T() const { return h_; }

 private:
  T h_ = nullptr;
};
inline cudaError_t free_host(unsigned char *p) { return cudaFreeHost(p); }
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using Graph = Owned<cudaGraph_t, cudaGraphDestroy>;
using GraphExec = Owned<cudaGraphExec_t, cudaGraphExecDestroy>;
using PinnedBuf = Owned<unsigned char *, free_host>;        // cudaHostAlloc
using IpcMapping = Owned<void *, cudaIpcCloseMemHandle>;   // cudaIpcOpenMemHandle

#include "commit_kernels.cuh"

struct DeviceSnapshot {
  DevBuf excl, excl_ranks, cand, candx, pref, has_pref, type_slot, full, rows, rank_of, csum, lsum, models;
  DevBuf cap_col, lthreads_col, linprog_col, part_of_rank, count_col, cand_before, nzw, nz_n;
  DevBuf front, nzw_full, nz_n_full;  // instance-sharded fleets: replicated first words of every row; word lists over the whole row
  SnapshotView view{};
  HostSnapshot host;  // kept for introspection and the small host-side parts of stats / reaper
  DevBuf sparse_dev;
  bool sparse_slots = false;  // most type slots have few candidates inside a decision's window: long walks (k_place_direct sorts big batches by slot)
  bool host_stale = false;  // built on the device: the rank-space vectors of `host` are downloaded on first use (host_mirror)
  int32_t n_models = 0;
};

struct PlaceCtx {
  Stream stream;
  static constexpr int NPIPE = 3;
  Stream pipe[NPIPE];  // H2D / kernel / D2H of consecutive chunks overlap across these
  Event e0, e1, ready;
  DevBuf d_in, d_out, d_fresh, d_extra, d_trace, d_cand;
  // slot sort of a batch (k_slot_keys + cub radix sort -> perm): set 0 for single launches, 1 + pipe for the chunks of a pipelined call
  static constexpr int NSORT = 4;
  DevBuf d_skey[NSORT], d_skey2[NSORT], d_sidx[NSORT], d_sidx2[NSORT], d_stmp[NSORT];
  // the two-pass path (same scratch sets): slot summaries, their shortlist members, the two worklists and their lengths
  DevBuf d_sums[NSORT], d_members[NSORT], d_walk[NSORT], d_ovf[NSORT], d_counts[NSORT];
  DevBuf d_open_flag, d_open_idx, d_n_open, d_cub, d_blocks, d_gathered, d_rows, d_in_open, d_out_open;  // instance-shard combine
  std::vector<FreshRow> fresh_host;
  // pinned, device-mapped scratch for tiny batches: the kernel reads the decisions and writes the results straight
  // through PCIe, so a B = 1 call is one launch + one synchronise (no copy calls)
  PinnedBuf mapped;
  static constexpr size_t MAPPED_BYTES = 16384;
  // the B = 1 path as a captured CUDA graph (one k_place_small node; now / seed / n travel through the mapped header)
  Graph graph;
  GraphExec graph_exec;  // (declared after the graph it was instantiated from: destroyed before it)
  int32_t graph_epoch = -1;
  // a call-wide exclude set (mmp_place_batch_excluding): its ids and the per-slot tables derived from the snapshot's
  // (k_exclude_slots, k_slot_lists) that the call's view points at
  DevBuf d_xids, d_xcand, d_xcandx, d_xpref, d_xnzw, d_xnz_n, d_xbefore;
};

// The scoring kernel of untraced batches (MMP_KERNEL = direct | lanes | tile; launch_place): k_place_direct (rows rebuilt
// from excl_ranks), k_place_lanes (whole rows through TMA landing stages) or the cooperative tile kernel k_place.
enum class PlaceKernel { direct, lanes, tile };

struct mmp_fleet {
  HostState hs;
  int device = 0;
  int sm_count = 132;           // (H100 SXM; replaced by the device's own count in mmp_fleet_create)
  std::mutex ingest_mu;         // single-writer ingest, but do not corrupt state if violated
  std::shared_mutex snap_mu;    // readers: place/stats; writer: the epoch flip in commit
  DeviceSnapshot snaps[2];
  int cur = 0;
  int32_t epoch = 0;
  Stream commit_stream;
  DevBuf d_flush;
  DevBuf zero_row;              // one all-zero exclusion row (SnapshotView::zero_row), unsharded fleets: allocated at the first commit
  ChurnState churn;             // the closed loop (churn_kernels.cuh)
  int64_t structural_epoch = 0; // bumped by every structural commit
  LiveState live;               // device-resident tables every non-structural commit works from (commit_kernels.cuh)
  std::mutex mirror_mu;         // host_mirror(): lazy download of a device-built snapshot's rank-space vectors
  int commit_host_only = 0;     // MMP_COMMIT=host: every commit takes the structural (host) path (A/B and cross-check)
  bool device_ahead = false;    // the closed loop (churn_kernels.cuh) changed the registry on the device: host tables are behind
  float t_stats_ms = 0, t_reaper_ms = 0, t_lru_ms = 0, t_prune_ms = 0;  // CUDA-event time of the device part of the last mmp_stats / mmp_reaper_select / mmp_lru_apply
  float t_lru_read_ms = 0;      // ... and of the last mmp_lru_read (its count + scan part plus its emit part)
  int32_t last_commit_path = 0; // 1 structural (host), 2 device
  double last_commit_ms = 0;
  ncclComm_t comm = nullptr;    // instance-shard communicator (mmp_shard_connect)
  // peer-access path of the instance-sharded layout (mmp_shard_ipc_export / _import, k_place_dealt)
  struct Peers {
    bool ready = false;
    int32_t max_batch = 0;
    DevBuf arena, done, err;                // arena (exported): 4 KB of arrival counters + statistics, then 2 x max_batch results (step parity)
    static constexpr size_t IPC_MIN_BYTES = (size_t)8 << 20;  // exported buffers get allocation blocks of their own (an IPC handle names a block)
    mmp_decision_out *out_buf() const { return reinterpret_cast<mmp_decision_out *>(arena.as<unsigned char>() + 4096); }
    unsigned long long *flag_buf() const { return arena.as<unsigned long long>(); }
    void *peer_base[MAX_SHARDS][4] = {};    // every peer's buffers as mapped here: excl of snapshot 0 / 1, out, flags
    IpcMapping opened[MAX_SHARDS][3];       // ... and the allocation blocks opened for them (a peer in this process: none)
    uint64_t step = 0;
    int64_t batches = 0, result_bytes = 0;
    Event ev[3];                            // around k_place_dealt and k_dealt_wait of the last step
    float t_kernel_ms = 0, t_wait_ms = 0;
    int off = 0;                            // MMP_SHARD_PEERS=0 keeps the collective path although peers were imported
  } peers;
  std::mutex comm_mu;           // collectives of one communicator are issued by one thread at a time
  std::atomic<int64_t> open_decisions{0};  // decisions that needed the row-gather pass so far
  std::atomic<uint64_t> id_base{0};        // decision i of a batch hashes as id_base + i (mmp_fleet_set_id_base)
  std::mutex ctx_mu;
  std::vector<std::unique_ptr<PlaceCtx>> ctx_free;
  std::atomic<int64_t> launches{0};
  int one_mode = 3;             // MMP_ONE = lanes | small | graph | server: how tiny batches are launched (0: launch_place, 1: k_place_small
                                // as a stream launch, 2: k_place_small as a replayed CUDA graph, 3: a request to the resident k_place_server)
  // the resident B = 1 server (one_mode 3, k_place_server)
  struct Server {
    std::mutex mu;                 // one request at a time; a caller that finds it taken uses the graph path
    PinnedBuf mapped;
    Stream stream;
    int32_t epoch = -1;
    bool running = false;
    uint64_t seq = 0;
    int64_t launches = 0, requests = 0;
    int64_t life_us = 2000, idle_us = 300;
  } srv;
  int sort_slots = 2;           // MMP_SORT_SLOTS = 0 never | 1 always | 2 (default) when the snapshot's candidate sets are sparse: k_place_direct
                                // resolves a large batch in type-slot order
  PlaceKernel kernel = PlaceKernel::direct;  // MMP_KERNEL, mmp_tune("direct"): which kernel resolves untraced unsharded batches
  int lane_budget = LANE_BUDGET;  // MMP_LANE_BUDGET: walk steps per lane before a decision is handed to the whole warp
  int split = 2;                // mmp_tune("split"): 0 never | 1 always | 2 (default) from SPLIT_MIN_BATCH decisions on snapshots whose
                                // candidate sets are not sparse: k_place_direct batches go through the two-pass path (launch_split)
  // LRU store (plug point 3)
  DevBuf lru_ts, lru_seq, lru_weight, lru_model, lru_cap, lru_wsize, lru_count, lru_seqctr, lru_loadts, lru_pin;
  int32_t lru_n = 0, lru_slots = 0;
  bool lru_loop = false;        // the store was set up by mmp_churn_init: its load times are registrations (mmp_lru_read reports them)
};

static int32_t set_device(mmp_fleet *f) {
  CK(cudaSetDevice(f->device));
  return MMP_OK;
}

template <class T>
static cudaError_t upload_vec(DevBuf &b, const std::vector<T> &v, cudaStream_t st) {
  size_t bytes = v.size() * sizeof(T);
  cudaError_t e = b.ensure(bytes ? bytes : 16);
  if (e != cudaSuccess) return e;
  if (bytes) e = cudaMemcpyAsync(b.p, v.data(), bytes, cudaMemcpyHostToDevice, st);
  return e;
}

static PlaceCtx *acquire_ctx(mmp_fleet *f) {
  {
    std::lock_guard<std::mutex> g(f->ctx_mu);
    if (!f->ctx_free.empty()) {
      PlaceCtx *c = f->ctx_free.back().release();
      f->ctx_free.pop_back();
      return c;
    }
  }
  auto c = std::make_unique<PlaceCtx>();
  bool ok = cudaStreamCreateWithFlags(c->stream.put(), cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreate(c->e0.put()) == cudaSuccess && cudaEventCreate(c->e1.put()) == cudaSuccess &&
            cudaEventCreateWithFlags(c->ready.put(), cudaEventDisableTiming) == cudaSuccess &&
            cudaHostAlloc((void **)c->mapped.put(), PlaceCtx::MAPPED_BYTES, cudaHostAllocMapped) == cudaSuccess;
  for (int i = 0; ok && i < PlaceCtx::NPIPE; i++) ok = cudaStreamCreateWithFlags(c->pipe[i].put(), cudaStreamNonBlocking) == cudaSuccess;
  return ok ? c.release() : nullptr;
}
// A PlaceCtx leased from the fleet's pool for the length of one call; it goes back to the pool when the lease goes out of
// scope.  A lease is empty when a new context could not be created.
class CtxLease {
 public:
  explicit CtxLease(mmp_fleet *f) : f_(f), c_(acquire_ctx(f)) {}
  ~CtxLease() {
    if (!c_) return;
    std::lock_guard<std::mutex> g(f_->ctx_mu);
    f_->ctx_free.emplace_back(c_);
  }
  CtxLease(const CtxLease &) = delete;
  CtxLease &operator=(const CtxLease &) = delete;
  explicit operator bool() const { return c_ != nullptr; }
  PlaceCtx *operator->() const { return c_; }
  PlaceCtx *get() const { return c_; }

 private:
  mmp_fleet *f_;
  PlaceCtx *c_;
};

// ---------------------------------------------------------------------------------------------------------------
// kernel dispatch on the row width
// ---------------------------------------------------------------------------------------------------------------
struct PlaceArgs {
  SnapshotView s;
  const mmp_decision_in *in;
  int n;
  const FreshRow *fresh;
  int n_fresh;
  const int32_t *extra;
  mmp_decision_out *out;
  mmp_decision_trace *tr;
  uint32_t *cand;
  int64_t now;
  uint64_t seed, id_base;
  int emit_keys = 0;            // instance-sharded: write shard keys (uint64) into `out` instead of results
  const int32_t *orig_id = nullptr;  // gather pass: decision i reads row i of s.excl and hashes with id orig_id[i]
  struct PlaceCtx *ctx = nullptr;    // scratch for the slot sort (the call's own context)
  int sort_slot = 0;                 // ... which of its scratch sets (chunks in flight on different streams use different ones)
};

// ring depth (a power of two) / warps per block by row size: rows up to 2 KiB (16k instances) K=4 x 8 warps, up to 4 KiB K=2 x 8, beyond K=2 x 4
template <int WARPS, int K, int MINB, int T, bool TRACE>
static cudaError_t launch_place_t(mmp_fleet *f, const PlaceArgs &a, cudaStream_t st) {
  static std::atomic<bool> attr_set[64];  // function attributes are per device
  const RingLayout lay(a.s.excl_stride, K);
  const size_t smem = lay.per_warp * WARPS;
  auto kern = k_place<WARPS, K, MINB, T, TRACE>;
  if (!attr_set[f->device & 63].load()) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    if (e != cudaSuccess) return e;
    attr_set[f->device & 63] = true;
  }
  int bps = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&bps, kern, WARPS * 32, smem);
  if (e != cudaSuccess) return e;
  if (bps < 1) bps = 1;
  int want = (a.n + 32 * WARPS - 1) / (32 * WARPS);
  int grid = std::min(want, f->sm_count * bps);
  if (grid < 1) grid = 1;
  kern<<<grid, WARPS * 32, smem, st>>>(a.s, a.in, a.n, a.fresh, a.n_fresh, a.extra, a.out, a.tr, a.cand, a.now, a.seed, a.id_base);
  f->launches++;
  return cudaGetLastError();
}

// landing stages of k_place_lanes for a stored row width: as many 32-row stages as fit beside the warps' window buffers, at
// most LANE_STAGES; false when not even two fit (rows wider than about 580 words)
static bool lanes_geometry(int row_words, int &ns) {
  for (ns = LANE_STAGES; ns >= 2; ns--)
    if (LaneLayout(row_words, ns, LANE_WARPS, true).total <= (size_t)227 * 1024) return true;
  return false;
}

static cudaError_t launch_place_lanes(mmp_fleet *f, const PlaceArgs &a, cudaStream_t st, int ns) {
  static std::atomic<bool> attr_set[64];  // function attributes are per device
  const LaneLayout lay(a.s.excl_stride, ns, LANE_WARPS, true);  // (instance-sharded rows are short: well under half an SM's shared memory)
  if (!attr_set[f->device & 63].load()) {
    cudaError_t e = cudaFuncSetAttribute(k_place_lanes, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_set[f->device & 63] = true;
  }
  const int nb = (a.n + 31) / 32;
  const int grid = std::max(1, std::min((nb + LANE_WARPS - 1) / LANE_WARPS, f->sm_count));
  k_place_lanes<<<grid, LANE_WARPS * 32, lay.total, st>>>(a.s, a.in, a.n, a.fresh, a.n_fresh, a.extra, a.out, a.now, a.seed, a.id_base, ns,
                                                          a.emit_keys, f->hs.cfg.shard_rank, a.orig_id, f->lane_budget);
  f->launches++;
  return cudaGetLastError();
}

// k_place_direct's slot order (sparse snapshots, MMP_SORT_SLOTS): keys in ctx scratch set a.sort_slot, then a 16-bit radix
// sort of the positions by key (a few tens of microseconds per million decisions)
static bool sorts_slots(const mmp_fleet *f) { return f->sort_slots == 1 || (f->sort_slots == 2 && f->snaps[f->cur].sparse_slots); }
static int sort_set(const PlaceArgs &a) { return a.sort_slot >= 0 && a.sort_slot < PlaceCtx::NSORT ? a.sort_slot : 0; }
static cudaError_t slot_key_buffers(const PlaceArgs &a) {
  PlaceCtx *c = a.ctx;
  const int ss = sort_set(a);
  cudaError_t e;
  if ((e = c->d_skey[ss].ensure((size_t)a.n * 2)) != cudaSuccess || (e = c->d_skey2[ss].ensure((size_t)a.n * 2)) != cudaSuccess ||
      (e = c->d_sidx[ss].ensure((size_t)a.n * 4)) != cudaSuccess || (e = c->d_sidx2[ss].ensure((size_t)a.n * 4)) != cudaSuccess) return e;
  return cudaSuccess;
}
static cudaError_t slot_keys(mmp_fleet *f, const PlaceArgs &a, cudaStream_t st) {
  cudaError_t e;
  if ((e = slot_key_buffers(a)) != cudaSuccess) return e;
  PlaceCtx *c = a.ctx;
  const int ss = sort_set(a);
  k_slot_keys<<<(a.n + 255) / 256, 256, 0, st>>>(a.s, a.in, a.n, c->d_skey[ss].as<uint16_t>(), c->d_sidx[ss].as<int32_t>());
  f->launches++;
  return cudaSuccess;
}
static cudaError_t sort_slot_keys(mmp_fleet *f, const PlaceArgs &a, cudaStream_t st, const int32_t **perm) {
  PlaceCtx *c = a.ctx;
  const int ss = sort_set(a);
  size_t tmp = 0;
  cudaError_t e;
  if ((e = cub::DeviceRadixSort::SortPairs(nullptr, tmp, c->d_skey[ss].as<uint16_t>(), c->d_skey2[ss].as<uint16_t>(), c->d_sidx[ss].as<int32_t>(), c->d_sidx2[ss].as<int32_t>(), a.n, 0, 16, st)) != cudaSuccess) return e;
  if ((e = c->d_stmp[ss].ensure(tmp + 16)) != cudaSuccess) return e;
  if ((e = cub::DeviceRadixSort::SortPairs(c->d_stmp[ss].p, tmp, c->d_skey[ss].as<uint16_t>(), c->d_skey2[ss].as<uint16_t>(), c->d_sidx[ss].as<int32_t>(), c->d_sidx2[ss].as<int32_t>(), a.n, 0, 16, st)) != cudaSuccess) return e;
  *perm = c->d_sidx2[ss].as<int32_t>();
  f->launches++;
  return cudaSuccess;
}

// The two-pass path of a k_place_direct batch (DESIGN.md §5.2): the slot summaries of the call's view (k_slot_summary), one
// streaming pass that answers every decision lying clear of its slot's reach and lists the others (k_place_split), then
// k_place_direct over the walk list -- in slot order on sparse snapshots -- and k_place_ovf over the models with overflow
// ids.  The lists' lengths stay on the device: both launches are sized for the whole batch and stop at the length.
static cudaError_t launch_split(mmp_fleet *f, const PlaceArgs &a, cudaStream_t st) {
  PlaceCtx *c = a.ctx;
  const int ss = sort_set(a);
  const int n_slots = std::max(a.s.n_slots, 1);
  const bool sorted = sorts_slots(f);
  cudaError_t e;
  if ((e = c->d_sums[ss].ensure((size_t)n_slots * sizeof(SlotSummary))) != cudaSuccess ||
      (e = c->d_members[ss].ensure((size_t)n_slots * 2 * SPLIT_CAP * 4)) != cudaSuccess ||
      (e = c->d_walk[ss].ensure((size_t)a.n * 4)) != cudaSuccess || (e = c->d_ovf[ss].ensure((size_t)a.n * 4)) != cudaSuccess ||
      (e = c->d_counts[ss].ensure(16)) != cudaSuccess) return e;
  if (sorted && (e = slot_key_buffers(a)) != cudaSuccess) return e;
  int32_t *counts = c->d_counts[ss].as<int32_t>();
  k_slot_summary<<<(2 * n_slots + 127) / 128, 128, 0, st>>>(a.s, a.now, c->d_sums[ss].as<SlotSummary>(), c->d_members[ss].as<int32_t>(), counts);
  k_place_split<<<(a.n + 255) / 256, 256, 0, st>>>(a.s, a.in, a.n, a.fresh, a.n_fresh, a.out, a.now, a.seed, a.id_base,
                                                   c->d_sums[ss].as<SlotSummary>(), c->d_members[ss].as<int32_t>(), c->d_walk[ss].as<int32_t>(),
                                                   c->d_ovf[ss].as<int32_t>(), counts, sorted ? c->d_skey[ss].as<uint16_t>() : nullptr,
                                                   sorted ? c->d_sidx[ss].as<int32_t>() : nullptr);
  f->launches += 2;
  const int32_t *perm = c->d_walk[ss].as<int32_t>();
  if (sorted && (e = sort_slot_keys(f, a, st, &perm)) != cudaSuccess) return e;
  k_place_walk<4, 5><<<(a.n + 127) / 128, 128, 0, st>>>(a.s, a.in, a.n, a.fresh, a.n_fresh, a.extra, a.out, a.now, a.seed, a.id_base,
                                                       f->lane_budget, perm, counts);
  k_place_ovf<<<std::max(1, std::min((a.n + 3) / 4, f->sm_count * 4)), 128, 0, st>>>(a.s, a.in, c->d_ovf[ss].as<int32_t>(), counts + 1, a.fresh, a.n_fresh,
                                                                                   a.extra, a.out, a.now, a.seed, a.id_base);
  f->launches += 2;
  return cudaGetLastError();
}

static cudaError_t launch_place(mmp_fleet *f, const PlaceArgs &a, cudaStream_t st) {
  const int rw = a.s.row_words;
  int ns = 0;
  // traced calls (parity tests): the single-decision-per-warp tile kernel, kept apart so that the untraced kernels'
  // instruction footprint stays small
  if (a.tr || a.cand)
    return rw <= 512 ? launch_place_t<4, 4, 4, 32, true>(f, a, st) : rw <= 1024 ? launch_place_t<4, 4, 3, 32, true>(f, a, st) : launch_place_t<4, 2, 2, 32, true>(f, a, st);
  // the instance-shard key pass and gather pass: only k_place_lanes writes shard keys and reads rows by batch position
  // (place_sharded has checked that the rows fit its landing stages)
  if (a.emit_keys || a.orig_id) return lanes_geometry(a.s.excl_stride, ns) ? launch_place_lanes(f, a, st, ns) : cudaErrorInvalidValue;
  // the direct kernel: rows rebuilt from the snapshot's excl_ranks (whole-row fleets), no landing stages
  if (f->kernel == PlaceKernel::direct && a.s.word_lo == 0 && a.s.word_hi == a.s.row_words && a.s.excl_ranks) {
    if (a.ctx && a.s.n_slots > 0 && (f->split == 1 || (f->split == 2 && a.n >= SPLIT_MIN_BATCH && !f->snaps[f->cur].sparse_slots)))
      return launch_split(f, a, st);
    const int32_t *perm = nullptr;  // k_place_direct: position j of the launch resolves decision perm[j]
    if (a.ctx && a.n >= 8192 && sorts_slots(f)) {
      cudaError_t e;
      if ((e = slot_keys(f, a, st)) != cudaSuccess || (e = sort_slot_keys(f, a, st, &perm)) != cudaSuccess) return e;
    }
    k_place_direct<4, 5><<<(a.n + 127) / 128, 128, 0, st>>>(a.s, a.in, a.n, a.fresh, a.n_fresh, a.extra, a.out, a.now, a.seed, a.id_base,
                                                           f->lane_budget, perm);
    f->launches++;
    return cudaGetLastError();
  }
  // one decision per lane with the rows through landing stages (any row width of which at least two stages fit)
  if (f->kernel != PlaceKernel::tile && lanes_geometry(a.s.excl_stride, ns)) return launch_place_lanes(f, a, st, ns);
  // the cooperative tile kernel by row width: rows <= 2 KiB (16k instances) 7 blocks x 4 warps per SM, then <= 4 KiB, then wider
  if (rw <= 512) return launch_place_t<4, 4, 7, 16, false>(f, a, st);
  if (rw <= 1024) return launch_place_t<4, 4, 3, 16, false>(f, a, st);
  return launch_place_t<4, 2, 2, 16, false>(f, a, st);
}

// the peer-access path of place_sharded: one k_place_dealt over this shard's deal of the batch, the arrival wait, the
// results from this shard's result buffer into d_out.  Every shard is given the same batch in the same call sequence.
static int32_t place_dealt(mmp_fleet *f, PlaceCtx *c, const DeviceSnapshot &ds, const mmp_decision_in *d_in, int32_t n,
                           const FreshRow *d_fresh, int32_t n_fresh, const int32_t *d_extra, int32_t n_extra, mmp_decision_out *d_out,
                           int64_t now_ms, uint64_t seed, cudaStream_t st) {
  mmp_fleet::Peers &pr = f->peers;
  const int G = f->hs.cfg.shard_count, me = f->hs.cfg.shard_rank;
  if (n > pr.max_batch) { g_err = "batch larger than the max_batch given to mmp_shard_ipc_export"; return MMP_E_ARG; }
  std::lock_guard<std::mutex> g(f->comm_mu);  // one dealt step at a time per fleet: the steps are numbered
  SnapshotView vw = ds.view;
  vw.n_extra = n_extra;
  vw.word_lo = 0; vw.word_hi = vw.row_words;  // a dealt decision walks the whole rank range (excl_stride stays the block stride)
  const int cur = (int)(&ds - f->snaps);
  const uint64_t step = ++pr.step;
  DealtPeers P;
  for (int q = 0; q < MAX_SHARDS; q++) { P.blocks[q] = nullptr; P.out[q] = nullptr; P.flags[q] = nullptr; }
  for (int q = 0; q < G; q++) {
    P.blocks[q] = q == me ? ds.excl.as<uint32_t>() : reinterpret_cast<const uint32_t *>(pr.peer_base[q][cur]);
    mmp_decision_out *ob = q == me ? pr.out_buf() : reinterpret_cast<mmp_decision_out *>((unsigned char *)pr.peer_base[q][2] + 4096);
    P.out[q] = ob + (size_t)(step & 1) * pr.max_batch;
    P.flags[q] = q == me ? pr.flag_buf() : reinterpret_cast<unsigned long long *>(pr.peer_base[q][2]);
  }
  constexpr int WARPS = 4;
  const long long n_wb = ((long long)n + 31) / 32;                     // warp batches of the whole batch
  const long long mine = n_wb > me ? (n_wb - me + G - 1) / G : 0;      // ... dealt to this shard
  const int blocks = (int)std::max<long long>(1, (mine + WARPS - 1) / WARPS);  // (an empty deal still arrives)
  const size_t smem = (size_t)WARPS * vw.row_words * 4;
  auto kern = k_place_dealt<WARPS, 6>;  // 6 resident blocks per SM: 24 warps, some spills
  if (smem > 48 * 1024) CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  unsigned long long *stats = pr.flag_buf() + MAX_SHARDS;
  if (!pr.ev[0]) for (int k = 0; k < 3; k++) CK(cudaEventCreate(pr.ev[k].put()));
  CK(cudaEventRecord(pr.ev[0], st));
  kern<<<blocks, WARPS * 32, smem, st>>>(vw, ds.front.as<uint32_t>(), std::min(SHARD_FRONT_WORDS, vw.row_words), ds.nzw_full.as<uint16_t>(),
                                                       ds.nz_n_full.as<int32_t>(), P, G, me, d_in, n, d_fresh, n_fresh, d_extra, now_ms, seed,
                                                       f->id_base.load(), f->lane_budget, step, pr.done.as<unsigned int>(), stats);
  CK(cudaGetLastError());
  CK(cudaEventRecord(pr.ev[1], st));
  k_dealt_wait<<<1, 32, 0, st>>>(P, G, me, step, 4000000000ull, pr.err.as<int>());
  CK(cudaGetLastError());
  CK(cudaEventRecord(pr.ev[2], st));
  CK(cudaMemcpyAsync(d_out, pr.out_buf() + (size_t)(step & 1) * pr.max_batch, (size_t)n * sizeof(mmp_decision_out),
                     cudaMemcpyDeviceToDevice, st));
  int err = 0;
  CK(cudaMemcpyAsync(&err, pr.err.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  f->launches += 2;
  cudaEventElapsedTime(&pr.t_kernel_ms, pr.ev[0], pr.ev[1]);
  cudaEventElapsedTime(&pr.t_wait_ms, pr.ev[1], pr.ev[2]);
  pr.batches++;
  {
    const long long nb = n / 32, full = nb > me ? (nb - me + G - 1) / G : 0;
    pr.result_bytes += (full * 32 + ((nb % G) == me ? n % 32 : 0)) * 8 * (G - 1);
  }
  if (err) { pr.ready = false; g_err = "instance shards: a peer did not arrive at the step within 4 s (peer path disabled)"; return MMP_E_STATE; }
  return MMP_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// instance-sharded placement: every shard resolves the whole batch over its own rank range, ONE all-reduce(min) of the
// 64-bit keys gives every rank the answer of the shard that holds the first entry under PLACEMENT_ORDER (min-loc), and
// the (rare) decisions whose walk left the winning shard's range are finished from all-gathered row blocks.
// d_in/d_out are device buffers; every rank is given the same batch and ends with the same results.
// ---------------------------------------------------------------------------------------------------------------
static int32_t place_sharded(mmp_fleet *f, PlaceCtx *c, const DeviceSnapshot &ds, const mmp_decision_in *d_in, int32_t n,
                             const FreshRow *d_fresh, int32_t n_fresh, const int32_t *d_extra, int32_t n_extra, mmp_decision_out *d_out,
                             int64_t now_ms, uint64_t seed, cudaStream_t st) {
  SnapshotView vw = ds.view;
  vw.n_extra = n_extra;  // per call: bounds of the decisions' extra[] slices (checked on the device, prepare_ctx_a)
  if (f->peers.ready && !f->peers.off && f->hs.cfg.shard_count > 1)
    return place_dealt(f, c, ds, d_in, n, d_fresh, n_fresh, d_extra, n_extra, d_out, now_ms, seed, st);
  if (!f->comm) { g_err = "instance-sharded fleet is not connected (mmp_shard_connect)"; return MMP_E_STATE; }
  // the key pass stages this shard's stored rows, the gather pass whole rows, both through k_place_lanes' landing stages
  const int ST = ds.view.excl_stride, NW = ds.view.row_words, widest = std::max(ST, NW);
  int ns = 0;
  if (!lanes_geometry(widest, ns)) {
    int limit = widest;
    while (limit > 0 && !lanes_geometry(limit, ns)) limit--;
    g_err = "instance shards: rows of " + std::to_string(widest) + " words are wider than the " + std::to_string(limit) +
            " words the collective path can stage (k_place_lanes)";
    return MMP_E_STATE;
  }
  NcclApi &nc = nccl_api();
  std::lock_guard<std::mutex> g(f->comm_mu);
  const int G = f->hs.cfg.shard_count;
  CK(c->d_open_flag.ensure((size_t)n));
  CK(c->d_open_idx.ensure((size_t)n * 4));
  CK(c->d_n_open.ensure(16));
  CK(cudaMemsetAsync(c->d_n_open.p, 0, sizeof(int), st));
  // 1-3. per-shard keys (the scoring kernel), the min-loc combine over NVLink, keys -> results
  PlaceArgs a{vw, d_in, n, d_fresh, n_fresh, d_extra, d_out, nullptr, nullptr, now_ms, seed, f->id_base.load()};
  a.emit_keys = 1;
  CK(launch_place(f, a, st));
  NK(nc.AllReduce(d_out, d_out, (size_t)n, ncclUint64, ncclMin, f->comm, st));
  k_shard_decode<<<(n + 255) / 256, 256, 0, st>>>(reinterpret_cast<uint64_t *>(d_out), n, c->d_open_flag.as<uint8_t>(), c->d_n_open.as<int>());
  f->launches++;
  CK(cudaGetLastError());
  int n_open = 0;
  CK(cudaMemcpyAsync(&n_open, c->d_n_open.p, sizeof(int), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (n_open == 0) return MMP_OK;
  f->open_decisions += n_open;
  // the open decisions as an ordered list, identical on every rank
  size_t tmp_bytes = 0;
  thrust::counting_iterator<int32_t> iota(0);
  CK(cub::DeviceSelect::Flagged(nullptr, tmp_bytes, iota, c->d_open_flag.as<uint8_t>(), c->d_open_idx.as<int32_t>(), c->d_n_open.as<int>(), n, st));
  CK(c->d_cub.ensure(tmp_bytes + 16));
  CK(cub::DeviceSelect::Flagged(c->d_cub.p, tmp_bytes, iota, c->d_open_flag.as<uint8_t>(), c->d_open_idx.as<int32_t>(), c->d_n_open.as<int>(), n, st));
  f->launches += 2;
  // 4. the open decisions, from whole rows: all-gather every shard's block of their exclusion rows (the same ordered
  // list on every rank), assemble, and run the same kernel on the assembled rows with the snapshot's whole rank range
  CK(c->d_blocks.ensure((size_t)n_open * ST * 4));
  CK(c->d_gathered.ensure((size_t)G * n_open * ST * 4));
  CK(c->d_rows.ensure((size_t)n_open * NW * 4));
  CK(c->d_in_open.ensure((size_t)n_open * sizeof(mmp_decision_in)));
  CK(c->d_out_open.ensure((size_t)n_open * sizeof(mmp_decision_out)));
  const int pack_blocks = (int)std::min<size_t>(((size_t)n_open * ST + 255) / 256, (size_t)f->sm_count * 8);
  k_shard_pack<<<std::max(pack_blocks, 1), 256, 0, st>>>(vw, d_in, c->d_open_idx.as<int32_t>(), n_open, c->d_blocks.as<uint32_t>(),
                                                         c->d_in_open.as<mmp_decision_in>());
  CK(cudaGetLastError());
  NK(nc.AllGather(c->d_blocks.p, c->d_gathered.p, (size_t)n_open * ST, ncclUint32, f->comm, st));
  const int asm_blocks = (int)std::min<size_t>(((size_t)n_open * NW + 255) / 256, (size_t)f->sm_count * 8);
  k_shard_assemble<<<std::max(asm_blocks, 1), 256, 0, st>>>(c->d_gathered.as<uint32_t>(), n_open, ST, G, NW, c->d_rows.as<uint32_t>());
  CK(cudaGetLastError());
  f->launches += 2;
  SnapshotView whole = vw;
  whole.excl = c->d_rows.as<uint32_t>(); whole.excl_ranks = nullptr;
  whole.excl_stride = NW; whole.word_lo = 0; whole.word_hi = NW;
  if (G > 1) { whole.nzw = ds.nzw_full.as<uint16_t>(); whole.nz_n = ds.nz_n_full.as<int32_t>(); }  // word lists over the whole row, not this shard's block
  PlaceArgs b{whole, c->d_in_open.as<mmp_decision_in>(), n_open, d_fresh, n_fresh, d_extra, c->d_out_open.as<mmp_decision_out>(),
              nullptr, nullptr, now_ms, seed, f->id_base.load()};
  b.orig_id = c->d_open_idx.as<int32_t>();
  CK(launch_place(f, b, st));
  k_shard_scatter<<<(n_open + 255) / 256, 256, 0, st>>>(c->d_out_open.as<mmp_decision_out>(), c->d_open_idx.as<int32_t>(), n_open, d_out);
  f->launches++;
  CK(cudaGetLastError());
  return MMP_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// the host side of a placement call: side tables, the sharded-or-not dispatch, the chunk pipeline
// ---------------------------------------------------------------------------------------------------------------
// Whether a call goes through place_sharded: always on an instance-sharded fleet, and for untraced calls on a fleet that
// connected a communicator with one shard (a traced call there takes the unsharded traced kernel).
static bool places_sharded(const mmp_fleet *f, bool traced) { return f->hs.cfg.shard_count > 1 || (f->comm && !traced); }

// The call's fresh rows and extra excludes into d_fresh / d_extra on st.  Both buffers hold at least one entry, so the
// kernels are given valid pointers when a call has none.
static int32_t stage_side_tables(PlaceCtx *c, const FreshRow *fresh, int32_t n_fresh, const int32_t *extra, int32_t n_extra, cudaStream_t st) {
  CK(c->d_fresh.ensure((size_t)std::max(n_fresh, 1) * sizeof(FreshRow)));
  CK(c->d_extra.ensure((size_t)std::max(n_extra, 1) * 4));
  if (n_fresh) CK(cudaMemcpyAsync(c->d_fresh.p, fresh, (size_t)n_fresh * sizeof(FreshRow), cudaMemcpyHostToDevice, st));
  if (n_extra) CK(cudaMemcpyAsync(c->d_extra.p, extra, (size_t)n_extra * 4, cudaMemcpyHostToDevice, st));
  return MMP_OK;
}

// Places the whole batch `a`, whose records, side tables and output are on the device, on stream st.  a.s.n_extra is the
// size of the call's extra[] table.
static int32_t place_on_device(mmp_fleet *f, PlaceCtx *c, const DeviceSnapshot &ds, const PlaceArgs &a, cudaStream_t st) {
  const bool traced = a.tr || a.cand;
  if (!places_sharded(f, traced)) { CK(launch_place(f, a, st)); return MMP_OK; }
  if (traced) { g_err = "traces are not available on an instance-sharded fleet"; return MMP_E_STATE; }
  return place_sharded(f, c, ds, a.in, a.n, a.fresh, a.n_fresh, a.extra, a.s.n_extra, a.out, a.now, a.seed, st);
}

// A large unsharded, untraced batch in chunks: chunk i goes to stream pipe[i % NPIPE] with slot-sort scratch set
// 1 + i % NPIPE, so that the H2D copy of chunk i+1, the kernel of chunk i and the D2H copy of chunk i-1 overlap (with
// pinned caller buffers these are true DMA).  `a` is the whole batch, its records in c->d_in and its results in c->d_out;
// the records are copied there chunk by chunk from `in` unless `in` is null.  Results go to `out` on the host.  Work
// queued on c->stream before the call (the side tables, records built on the device) completes before the first chunk.
static int32_t place_chunks(mmp_fleet *f, PlaceCtx *c, const PlaceArgs &a, int32_t chunk, const mmp_decision_in *in, mmp_decision_out *out) {
  CK(cudaEventRecord(c->ready, c->stream));
  for (int i = 0; i < PlaceCtx::NPIPE; i++) CK(cudaStreamWaitEvent(c->pipe[i], c->ready, 0));
  int ci = 0;
  for (int32_t lo = 0; lo < a.n; lo += chunk, ci++) {
    cudaStream_t ps = c->pipe[ci % PlaceCtx::NPIPE];
    PlaceArgs p = a;
    p.in = a.in + lo; p.out = a.out + lo; p.n = std::min(chunk, a.n - lo);
    p.id_base = a.id_base + (uint64_t)lo; p.sort_slot = 1 + ci % PlaceCtx::NPIPE;
    if (in) CK(cudaMemcpyAsync(c->d_in.as<mmp_decision_in>() + lo, in + lo, (size_t)p.n * sizeof(mmp_decision_in), cudaMemcpyHostToDevice, ps));
    CK(launch_place(f, p, ps));
    CK(cudaMemcpyAsync(out + lo, p.out, (size_t)p.n * sizeof(mmp_decision_out), cudaMemcpyDeviceToHost, ps));
  }
  for (int i = 0; i < PlaceCtx::NPIPE; i++) CK(cudaStreamSynchronize(c->pipe[i]));
  return MMP_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------------------------
extern "C" {

static void server_stop(mmp_fleet *f);

int32_t mmp_shard_unique_id(void *id128) {
  if (!id128) { g_err = "null argument"; return MMP_E_ARG; }
  NcclApi &nc = nccl_api();
  if (!nc.ok) { g_err = "libnccl.so.2 not found (needed only for instance-sharded fleets)"; return MMP_E_NCCL; }
  ncclUniqueId id;
  NK(nc.GetUniqueId(&id));
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  memcpy(id128, &id, sizeof(id));
  return MMP_OK;
}
int32_t mmp_shard_connect(mmp_fleet *f, const void *id128) {
  if (!f || !id128) { g_err = "null argument"; return MMP_E_ARG; }
  // (a single shard may connect too: its batches then take the same keys -> all-reduce -> decode path over whole rows)
  NcclApi &nc = nccl_api();
  if (!nc.ok) { g_err = "libnccl.so.2 not found"; return MMP_E_NCCL; }
  CK(cudaSetDevice(f->device));
  std::lock_guard<std::mutex> g(f->comm_mu);
  if (f->comm) { nc.CommDestroy(f->comm); f->comm = nullptr; }
  ncclUniqueId id;
  memcpy(&id, id128, sizeof(id));
  NK(nc.CommInitRank(&f->comm, f->hs.cfg.shard_count, id, f->hs.cfg.shard_rank));
  return MMP_OK;
}
int32_t mmp_shard_words(mmp_fleet *f, int32_t *word_lo, int32_t *word_hi) {
  if (!f) { g_err = "null fleet"; return MMP_E_ARG; }
  int32_t lo, hi, st;
  HostState::shard_words(f->hs.row_words(), f->hs.cfg.shard_rank, f->hs.cfg.shard_count, lo, hi, st);
  if (word_lo) *word_lo = lo;
  if (word_hi) *word_hi = hi;
  return st;
}
int64_t mmp_shard_open_decisions(mmp_fleet *f) { return f ? f->open_decisions.load() : 0; }

// ---- peer access between the instance shards (k_place_dealt) ----
struct ShardIpcBlob {
  uint32_t magic, rank, count, max_batch;
  uint64_t pid, bytes[4], ptr[4], off[4];  // off: offset of the buffer inside the allocation block its handle names
  int32_t device, pad;
  cudaIpcMemHandle_t h[4];  // excl of snapshot 0 / 1, the arena (flags + result buffers)
};
// cudaMalloc carves small allocations out of shared blocks and an IPC handle names the whole block: export the block's
// handle plus the buffer's offset in it, open every distinct block once
static int32_t ipc_block_offset(const void *p, uint64_t *off) {
  typedef int (*GetRange)(unsigned long long *, size_t *, unsigned long long);
  static GetRange fn = nullptr;
  if (!fn) {
    void *sym = nullptr;
    cudaDriverEntryPointQueryResult qr;
    CK(cudaGetDriverEntryPoint("cuMemGetAddressRange", &sym, cudaEnableDefault, &qr));
    if (!sym || qr != cudaDriverEntryPointSuccess) { g_err = "cuMemGetAddressRange not available"; return MMP_E_CUDA; }
    fn = reinterpret_cast<GetRange>(sym);
  }
  unsigned long long base = 0;
  size_t size = 0;
  if (fn(&base, &size, (unsigned long long)(uintptr_t)p) != 0) { g_err = "cuMemGetAddressRange failed"; return MMP_E_CUDA; }
  *off = (uint64_t)(uintptr_t)p - base;
  return MMP_OK;
}
static_assert(sizeof(ShardIpcBlob) <= MMP_SHARD_IPC_BYTES, "blob size");
int32_t mmp_shard_ipc_export(mmp_fleet *f, int32_t max_batch, void *blob) {
  if (!f || !blob || max_batch <= 0) { g_err = "bad argument"; return MMP_E_ARG; }
  const int G = f->hs.cfg.shard_count;
  if (G < 2 || G > MAX_SHARDS) { g_err = "peer access needs 2..16 instance shards"; return MMP_E_STATE; }
  CK(cudaSetDevice(f->device));
  std::lock_guard<std::mutex> g(f->ingest_mu);
  mmp_fleet::Peers &pr = f->peers;
  int32_t lo, hi, stw;
  HostState::shard_words(f->hs.row_words(), f->hs.cfg.shard_rank, G, lo, hi, stw);
  // the column blocks keep their address for the fleet's lifetime: both snapshots are sized for max_models rows now
  const size_t full = std::max(mmp_fleet::Peers::IPC_MIN_BYTES, (size_t)std::max(f->hs.cfg.max_models, 1) * stw * 4);
  for (int k = 0; k < 2; k++) {
    DevBuf &b = f->snaps[k].excl;
    if (b.p && b.cap < full) { g_err = "column block allocated before export is smaller than max_models rows"; return MMP_E_STATE; }
    if (!b.p) { CK(b.ensure(full)); CK(cudaMemset(b.p, 0, b.cap)); }
  }
  pr.ready = false;
  pr.max_batch = max_batch;
  CK(pr.arena.ensure(std::max(mmp_fleet::Peers::IPC_MIN_BYTES, (size_t)4096 + (size_t)2 * max_batch * sizeof(mmp_decision_out))));
  CK(pr.done.ensure(16)); CK(pr.err.ensure(16));
  CK(cudaMemset(pr.arena.p, 0, 4096)); CK(cudaMemset(pr.done.p, 0, 16)); CK(cudaMemset(pr.err.p, 0, 16));
  pr.step = 0;
  ShardIpcBlob bl;
  memset(&bl, 0, sizeof(bl));
  bl.magic = 0x4d4d5049u; bl.rank = (uint32_t)f->hs.cfg.shard_rank; bl.count = (uint32_t)G; bl.max_batch = (uint32_t)max_batch;
  bl.pid = (uint64_t)getpid(); bl.device = f->device;
  void *ptrs[3] = {f->snaps[0].excl.p, f->snaps[1].excl.p, pr.arena.p};
  const size_t bytes[3] = {f->snaps[0].excl.cap, f->snaps[1].excl.cap, pr.arena.cap};
  for (int k = 0; k < 3; k++) {
    bl.ptr[k] = (uint64_t)(uintptr_t)ptrs[k]; bl.bytes[k] = bytes[k];
    int32_t rco = ipc_block_offset(ptrs[k], &bl.off[k]);
    if (rco < 0) return rco;
    CK(cudaIpcGetMemHandle(&bl.h[k], ptrs[k]));
  }
  memset(blob, 0, MMP_SHARD_IPC_BYTES);
  memcpy(blob, &bl, sizeof(bl));
  return MMP_OK;
}
int32_t mmp_shard_ipc_import(mmp_fleet *f, const void *blobs) {
  if (!f || !blobs) { g_err = "bad argument"; return MMP_E_ARG; }
  const int G = f->hs.cfg.shard_count, me = f->hs.cfg.shard_rank;
  mmp_fleet::Peers &pr = f->peers;
  if (G < 2 || G > MAX_SHARDS || pr.max_batch <= 0) { g_err = "mmp_shard_ipc_export first"; return MMP_E_STATE; }
  CK(cudaSetDevice(f->device));
  std::lock_guard<std::mutex> g(f->ingest_mu);
  for (int q = 0; q < G; q++) {
    ShardIpcBlob bl;
    memcpy(&bl, (const unsigned char *)blobs + (size_t)q * MMP_SHARD_IPC_BYTES, sizeof(bl));
    if (bl.magic != 0x4d4d5049u || (int)bl.rank != q || (int)bl.count != G) { g_err = "blob of the wrong shard / fleet"; return MMP_E_ARG; }
    if ((int32_t)bl.max_batch != pr.max_batch) { g_err = "shards exported different max_batch"; return MMP_E_ARG; }
    if (q == me) continue;
    if (bl.pid == (uint64_t)getpid()) {  // the peer fleet lives in this process: its pointers are valid here once peer access is on
      int can = 0;
      CK(cudaDeviceCanAccessPeer(&can, f->device, bl.device));
      if (!can) { g_err = "no peer access between the shards' devices"; return MMP_E_CUDA; }
      cudaError_t e = cudaDeviceEnablePeerAccess(bl.device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { g_err = cudaGetErrorString(e); return MMP_E_CUDA; }
      (void)cudaGetLastError();
      for (int k = 0; k < 3; k++) pr.peer_base[q][k] = (void *)(uintptr_t)bl.ptr[k];
    } else {
      for (IpcMapping &m : pr.opened[q]) m.reset();
      void *block[3] = {};
      for (int k = 0; k < 3; k++) {
        int same = -1;
        for (int j = 0; j < k && same < 0; j++)
          if (bl.ptr[j] - bl.off[j] == bl.ptr[k] - bl.off[k]) same = j;  // the same block in the exporting process
        if (same >= 0) block[k] = block[same];
        else {
          CK(cudaIpcOpenMemHandle(pr.opened[q][k].put(), bl.h[k], cudaIpcMemLazyEnablePeerAccess));
          block[k] = pr.opened[q][k];
        }
        pr.peer_base[q][k] = (unsigned char *)block[k] + bl.off[k];
      }
    }
  }
  if (const char *t = getenv("MMP_SHARD_PEERS")) pr.off = atoi(t) == 0;
  pr.ready = true;
  return MMP_OK;
}
/* out[0] batches taken by the peer path, [1] row words read from peers' blocks, [2] result bytes stored to peers, [3] ready */
int32_t mmp_shard_peer_stats(mmp_fleet *f, int64_t *out4) {
  if (!f || !out4) { g_err = "bad argument"; return MMP_E_ARG; }
  mmp_fleet::Peers &pr = f->peers;
  unsigned long long words = 0;
  if (pr.arena.p) { CK(cudaSetDevice(f->device)); CK(cudaMemcpy(&words, pr.flag_buf() + MAX_SHARDS, 8, cudaMemcpyDeviceToHost)); }
  out4[0] = pr.batches; out4[1] = (int64_t)words; out4[2] = pr.result_bytes; out4[3] = pr.ready && !pr.off ? 1 : 0;
  return MMP_OK;
}

int32_t mmp_fleet_set_id_base(mmp_fleet *f, uint64_t id_base) {
  if (!f) { g_err = "null fleet"; return MMP_E_ARG; }
  f->id_base = id_base;
  return MMP_OK;
}

int32_t mmp_abi_version(void) { return MMP_ABI_VERSION; }
const char *mmp_last_error(mmp_fleet *) { return g_err.c_str(); }

int32_t mmp_fleet_create(const mmp_config *cfg, mmp_fleet **out) {
  if (!cfg || !out) { g_err = "null argument"; return MMP_E_ARG; }
  if (cfg->max_instances <= 0 || cfg->max_instances > 65536 || cfg->max_models <= 0) { g_err = "max_instances must be in [1, 65536] and max_models > 0"; return MMP_E_ARG; }
  if (cfg->shard_count < 1 || cfg->shard_rank < 0 || cfg->shard_rank >= cfg->shard_count) { g_err = "bad shard_rank/shard_count"; return MMP_E_ARG; }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev <= 0) {
    g_err = std::string("no usable CUDA device (libmmplace has no CPU path): ") + (e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
    return MMP_E_CUDA;
  }
  if (cfg->device < 0 || cfg->device >= ndev) { g_err = "device ordinal out of range"; return MMP_E_ARG; }
  auto f = std::make_unique<mmp_fleet>();
  f->device = cfg->device;
  CK(cudaSetDevice(f->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, f->device));
  f->sm_count = prop.multiProcessorCount;
  CK(cudaStreamCreateWithFlags(f->commit_stream.put(), cudaStreamNonBlocking));
  f->hs.init(*cfg);
  if (const char *t = getenv("MMP_KERNEL")) f->kernel = !strcmp(t, "tile") ? PlaceKernel::tile : !strcmp(t, "lanes") ? PlaceKernel::lanes : PlaceKernel::direct;
  if (const char *t = getenv("MMP_ONE")) f->one_mode = !strcmp(t, "lanes") ? 0 : (!strcmp(t, "small") ? 1 : (!strcmp(t, "server") ? 3 : 2));
  if (const char *t = getenv("MMP_COMMIT")) f->commit_host_only = strcmp(t, "host") == 0;
  if (const char *t = getenv("MMP_SORT_SLOTS")) { int v = atoi(t); if (v >= 0 && v <= 2) f->sort_slots = v; }
  if (const char *t = getenv("MMP_LANE_BUDGET")) { int v = atoi(t); if (v >= 1 && v <= 4096) f->lane_budget = v; }
  *out = f.release();
  return MMP_OK;
}

void mmp_fleet_destroy(mmp_fleet *f) {
  if (!f) return;
  cudaSetDevice(f->device);
  { std::lock_guard<std::mutex> lk(f->srv.mu); server_stop(f); }
  cudaDeviceSynchronize();
  if (f->comm && nccl_api().ok) { nccl_api().CommDestroy(f->comm); f->comm = nullptr; }
  delete f;  // (its members free the device buffers, streams, events, graphs, pinned buffers and IPC mappings they own)
}

#define NEED(f) do { if (!(f)) { g_err = "null fleet"; return MMP_E_ARG; } } while (0)
#define FWD(call) do { std::lock_guard<std::mutex> g_(f->ingest_mu); int32_t rc_ = (call); if (rc_ < 0) g_err = f->hs.err; return rc_; } while (0)

int32_t mmp_instance_upsert(mmp_fleet *f, int32_t idx, const mmp_instance_row *row, const char *id, const char *loc,
                            const char *zone, const char *const *labels, int32_t n_labels) {
  NEED(f);
  FWD(f->hs.upsert_instance(idx, row, id, loc, zone, labels, n_labels));
}
int32_t mmp_instance_update(mmp_fleet *f, int32_t idx, const mmp_instance_row *row) { NEED(f); FWD(f->hs.update_instance(idx, row)); }
int32_t mmp_instance_upsert_json(mmp_fleet *f, int32_t idx, const char *id, const char *json, int32_t active) {
  NEED(f);
  FWD(f->hs.upsert_instance_json(idx, id, json, active));
}
int32_t mmp_model_upsert_json(mmp_fleet *f, int32_t m, const char *json, int32_t size_units) { NEED(f); FWD(f->hs.set_model_json(m, json, size_units)); }
int32_t mmp_instance_remove(mmp_fleet *f, int32_t idx) { NEED(f); FWD(f->hs.remove_instance(idx)); }
int32_t mmp_types_set_json(mmp_fleet *f, const char *json) { NEED(f); FWD(f->hs.set_types_json(json)); }
int32_t mmp_type_id(mmp_fleet *f, const char *name) {
  NEED(f);
  if (!name) { g_err = "null type name"; return MMP_E_ARG; }
  std::lock_guard<std::mutex> g(f->ingest_mu);
  int32_t id = f->hs.intern_type(name);
  if (id < 0) { g_err = "more than 65534 model types"; return MMP_E_ARG; }
  return id;
}
int32_t mmp_replicasets_set(mmp_fleet *f, const char *const *p, int32_t n) { NEED(f); FWD(f->hs.set_replicasets(p, n)); }
int32_t mmp_model_times(mmp_fleet *f, int32_t m, const int64_t *edge_ts, int32_t n, int64_t last_unload_time) {
  NEED(f);
  FWD(f->hs.set_model_times(m, edge_ts, n, last_unload_time));
}
int32_t mmp_model_upsert(mmp_fleet *f, int32_t m, const mmp_model_row *row, const int32_t *ids, int32_t n) {
  NEED(f);
  FWD(f->hs.set_model(m, row, ids, n));
}
int32_t mmp_models_bulk(mmp_fleet *f, int32_t first, int32_t n, const mmp_model_row *rows, const int64_t *off, const int32_t *e) {
  NEED(f);
  if (n < 0 || !rows || !off || (off[n] > 0 && !e)) { g_err = "null argument"; return MMP_E_ARG; }
  std::lock_guard<std::mutex> g(f->ingest_mu);
  for (int32_t i = 0; i < n; i++) {
    int64_t k = off[i + 1] - off[i];
    if (k < 0 || k > 65536) { g_err = "bad edge offsets"; return MMP_E_ARG; }
    int32_t rc = f->hs.set_model(first + i, &rows[i], e + off[i], (int32_t)k);
    if (rc < 0) { g_err = f->hs.err; return rc; }
  }
  return MMP_OK;
}

// ---- commit: structural path (host build + upload of everything, live tables included) ----
static int32_t commit_structural(mmp_fleet *f, DeviceSnapshot &ds, cudaStream_t st) {
  f->hs.resolve_json_models();
  if (const char *m = f->hs.build_snapshot(ds.host)) { g_err = m; return MMP_E_ARG; }
  ds.host_stale = false;
  const HostSnapshot &h = ds.host;
  CK(upload_vec(ds.cand, h.cand, st)); CK(upload_vec(ds.pref, h.pref, st)); CK(upload_vec(ds.has_pref, h.has_pref, st));
  CK(upload_vec(ds.type_slot, h.type_slot_hp, st)); CK(upload_vec(ds.candx, h.candx, st)); CK(upload_vec(ds.full, h.full, st));
  CK(upload_vec(ds.rows, h.rows, st)); CK(upload_vec(ds.rank_of, h.rank_of, st)); CK(upload_vec(ds.csum, h.csum, st));
  CK(upload_vec(ds.lsum, h.lsum, st)); CK(upload_vec(ds.cap_col, h.cap_col, st));
  CK(upload_vec(ds.lthreads_col, h.lthreads_col, st)); CK(upload_vec(ds.linprog_col, h.linprog_col, st));
  CK(upload_vec(ds.part_of_rank, h.part_of_rank, st));
  CK(upload_vec(ds.count_col, h.count_col, st));
  CK(upload_vec(ds.cand_before, h.candx_before, st));
  CK(upload_vec(ds.nzw, h.nzw, st)); CK(upload_vec(ds.nz_n, h.nz_n, st));
  if (f->hs.cfg.shard_count > 1) { CK(upload_vec(ds.nzw_full, h.nzw_full, st)); CK(upload_vec(ds.nz_n_full, h.nz_n_full, st)); }
  // ---- the live tables later (non-structural) commits re-rank from ----
  LiveState &lv = f->live;
  const int32_t NI = f->hs.cfg.max_instances, NIW = (NI + 31) / 32, n = h.n_ranks, RW = h.row_words;
  lv.niw = NIW;
  std::vector<mmp_instance_row> rows((size_t)NI);
  std::vector<uint4> tie((size_t)NI, make_uint4(0, 0, 0, 0));
  std::vector<int2> meta((size_t)NI, make_int2(-1, 0));
  for (int32_t i = 0; i < NI; i++) rows[i] = f->hs.inst[i].present ? f->hs.inst[i].row : mmp_instance_row{};
  std::vector<uint32_t> cidx((size_t)h.n_slots * NIW, 0u), pidx((size_t)h.n_slots * NIW, 0u);
  for (int32_t r = 0; r < n; r++) {
    const int32_t i = h.rows[r].idx;
    tie[i] = make_uint4(h.tie_id[r], h.tie_loc[r], h.tie_zone[r], h.tie_lab[r]);
    meta[i] = make_int2(h.part_of_rank[r], 1 | (((h.rs[r >> 5] >> (r & 31)) & 1u) ? 2 : 0));
    for (int32_t sl = 0; sl < h.n_slots; sl++) {
      if ((h.cand[(size_t)sl * RW + (r >> 5)] >> (r & 31)) & 1u) cidx[(size_t)sl * NIW + (i >> 5)] |= 1u << (i & 31);
      if ((h.pref[(size_t)sl * RW + (r >> 5)] >> (r & 31)) & 1u) pidx[(size_t)sl * NIW + (i >> 5)] |= 1u << (i & 31);
    }
  }
  for (int32_t i = 0; i < NI; i++) if (f->hs.inst[i].present) meta[i].y |= 4;  // in the instance table (shutting-down records included)
  {  // type id -> partitions whose instances may host the type (typeSetStats MM:1432-1438; TCM:230-233, 700-716)
    const int32_t nt = (int32_t)h.type_slot.size();
    std::vector<int> off((size_t)nt + 1, 0), parts;
    for (int32_t ty = 0; ty < nt; ty++) {
      off[ty] = (int)parts.size();
      if (!h.tc_enabled || ty == 0) continue;  // no type constraints / an unconfigured name: the cluster's stats
      const std::string &name = f->hs.type_names[ty];
      auto it = f->hs.tc_config.find(name);
      if (it == f->hs.tc_config.end() || it->second.required.empty()) continue;  // hasStats only with required labels (TCM:706-716)
      const size_t before = parts.size();
      for (size_t p = 0; p < h.part_types.size(); p++)
        if (!std::binary_search(h.part_types[p].begin(), h.part_types[p].end(), name)) parts.push_back((int)p);
      if (parts.size() == before) parts.push_back(-1);  // a subset without instances: empty stats
    }
    off[nt] = (int)parts.size();
    if (parts.empty()) parts.push_back(-1);
    CK(upload_vec(lv.type_part_off, off, st)); CK(upload_vec(lv.type_parts, parts, st));
    CK(cudaStreamSynchronize(st));
    lv.n_type_ids = nt;
  }
  CK(upload_vec(lv.inst_rows, rows, st)); CK(upload_vec(lv.inst_tie, tie, st)); CK(upload_vec(lv.inst_meta, meta, st));
  CK(upload_vec(lv.cand_idx, cidx, st)); CK(upload_vec(lv.pref_idx, pidx, st));
  CK(cudaStreamSynchronize(st));  // the staging vectors above go out of scope
  lv.tmpl = h;
  lv.valid = true;
  f->structural_epoch++;
  return MMP_OK;
}

// ---- commit: device path.  Returns 1 when the fleet needs the host path after all (mixed versions, N1) ----
static int32_t commit_device(mmp_fleet *f, DeviceSnapshot &ds, cudaStream_t st) {
  LiveState &lv = f->live;
  const HostSnapshot &t = lv.tmpl;
  const int32_t NI = f->hs.cfg.max_instances, n = t.n_ranks, RW = t.row_words, NS = t.n_slots;
  // numeric instance updates since the last commit
  const int32_t nd = (int32_t)f->hs.dirty_inst.size();
  if (nd) {
    std::vector<mmp_instance_row> rows((size_t)nd);
    for (int32_t k = 0; k < nd; k++) rows[k] = f->hs.inst[f->hs.dirty_inst[k]].row;
    CK(upload_vec(lv.scratch_idx, f->hs.dirty_inst, st)); CK(upload_vec(lv.scratch_rows, rows, st));
    k_scatter_inst_rows<<<(nd + 255) / 256, 256, 0, st>>>(lv.scratch_idx.as<int32_t>(), lv.scratch_rows.as<mmp_instance_row>(), nd,
                                                          lv.inst_rows.as<mmp_instance_row>());
    f->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));  // staging vector
  }
  // sizes of the snapshot's tables (the live set did not change since the template was built)
  CK(ds.cand.ensure((size_t)NS * RW * 4)); CK(ds.pref.ensure((size_t)NS * RW * 4)); CK(ds.candx.ensure((size_t)NS * RW * 4));
  CK(ds.full.ensure((size_t)RW * 4)); CK(ds.rows.ensure((size_t)std::max(n, 1) * sizeof(RankRow))); CK(ds.rank_of.ensure((size_t)NI * 4));
  CK(ds.csum.ensure((size_t)RW * sizeof(WordSumI))); CK(ds.lsum.ensure((size_t)RW * sizeof(WordSumL)));
  CK(ds.cap_col.ensure((size_t)std::max(n, 1) * 8)); CK(ds.lthreads_col.ensure((size_t)std::max(n, 1) * 4));
  CK(ds.linprog_col.ensure((size_t)std::max(n, 1) * 4)); CK(ds.part_of_rank.ensure((size_t)std::max(n, 1) * 4));
  CK(ds.count_col.ensure((size_t)RW * 32 * 4)); CK(ds.cand_before.ensure((size_t)NS * 4));
  CK(ds.nzw.ensure((size_t)NS * RW * 2)); CK(ds.nz_n.ensure((size_t)NS * 4));
  CK(upload_vec(ds.has_pref, t.has_pref, st)); CK(upload_vec(ds.type_slot, t.type_slot_hp, st));
  CK(lv.keys.ensure((size_t)NI * sizeof(OrderKey))); CK(lv.rs_words.ensure((size_t)RW * 4)); CK(lv.flags.ensure(16 + (size_t)NS * 4));
  CK(cudaMemsetAsync(lv.flags.p, 0, 16, st));
  CK(cudaMemsetAsync(ds.full.p, 0, (size_t)RW * 4, st)); CK(cudaMemsetAsync(lv.rs_words.p, 0, (size_t)RW * 4, st));
  CK(cudaMemsetAsync(ds.count_col.p, 0, (size_t)RW * 32 * 4, st));
  const long long churn2 = (long long)((uint64_t)f->hs.cfg.min_churn_age_ms * 2u);
  const long long vers0 = n > 0 ? (long long)f->hs.inst[t.rows[0].idx].row.vers : 0;
  const int blocks = (NI + 127) / 128;
  k_rank_keys<<<blocks, 128, 0, st>>>(lv.inst_rows.as<mmp_instance_row>(), lv.inst_tie.as<uint4>(), lv.inst_meta.as<int2>(), NI,
                                     (long long)f->hs.cfg.min_space_units, lv.keys.as<OrderKey>(), vers0, lv.flags.as<int>());
  k_rank_init<<<blocks, 128, 0, st>>>(lv.inst_meta.as<int2>(), NI, ds.rank_of.as<int32_t>());
  {  // enough (i-block, j-slice) pairs to fill the SMs a few times over
    const int slices = std::max(1, std::min((NI + 127) / 128, (f->sm_count * 8 + blocks - 1) / blocks));
    k_rank_count<<<dim3((unsigned)blocks, (unsigned)slices), 128, 0, st>>>(lv.keys.as<OrderKey>(), lv.inst_meta.as<int2>(), NI, churn2, ds.rank_of.as<int32_t>());
  }
  f->launches++;
  k_build_rank_tables<<<blocks, 128, 0, st>>>(lv.inst_rows.as<mmp_instance_row>(), lv.inst_meta.as<int2>(), ds.rank_of.as<int32_t>(), NI,
                                             (long long)f->hs.cfg.min_space_units, ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(),
                                             ds.lthreads_col.as<int32_t>(), ds.linprog_col.as<int32_t>(), ds.part_of_rank.as<int32_t>(),
                                             ds.count_col.as<int32_t>(), ds.full.as<uint32_t>(), lv.rs_words.as<uint32_t>());
  k_word_summaries<<<(RW + 127) / 128, 128, 0, st>>>(ds.rows.as<RankRow>(), n, RW, ds.csum.as<WordSumI>(), ds.lsum.as<WordSumL>());
  k_permute_masks<<<(NS * RW + 127) / 128, 128, 0, st>>>(lv.cand_idx.as<uint32_t>(), lv.pref_idx.as<uint32_t>(), lv.niw, ds.rows.as<RankRow>(), n,
                                                        RW, NS, lv.rs_words.as<uint32_t>(), ds.cand.as<uint32_t>(), ds.candx.as<uint32_t>(),
                                                        ds.pref.as<uint32_t>());
  k_slot_lists<<<(NS + 31) / 32, 32, 0, st>>>(ds.cand.as<uint32_t>(), ds.candx.as<uint32_t>(), t.any_rs, RW, NS, t.word_lo, t.word_hi,
                                             ds.nzw.as<uint16_t>(), ds.nz_n.as<int32_t>(), ds.cand_before.as<int32_t>());
  if (f->hs.cfg.shard_count > 1) {
    CK(ds.nzw_full.ensure((size_t)NS * RW * 2)); CK(ds.nz_n_full.ensure((size_t)NS * 4));
    k_slot_lists<<<(NS + 31) / 32, 32, 0, st>>>(ds.cand.as<uint32_t>(), ds.candx.as<uint32_t>(), t.any_rs, RW, NS, 0, RW, ds.nzw_full.as<uint16_t>(),
                                               ds.nz_n_full.as<int32_t>(), lv.flags.as<int32_t>() + 2 /* scratch: cand_before of a whole row = 0 */);
    f->launches++;
  }
  f->launches += 6;
  CK(cudaGetLastError());
  int flags = 0;
  CK(cudaMemcpyAsync(&flags, lv.flags.p, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (flags & 1) return 1;
  // structural part of the host mirror; its rank-space vectors are downloaded on first use
  ds.host = HostSnapshot();
  ds.host.n_ranks = t.n_ranks; ds.host.row_words = t.row_words; ds.host.n_slots = t.n_slots; ds.host.any_rs = t.any_rs;
  ds.host.tc_enabled = t.tc_enabled; ds.host.has_pref = t.has_pref; ds.host.allowed_null = t.allowed_null;
  ds.host.type_slot = t.type_slot; ds.host.type_slot_hp = t.type_slot_hp; ds.host.word_lo = t.word_lo; ds.host.word_hi = t.word_hi;
  ds.host.excl_stride = t.excl_stride; ds.host.part_types = t.part_types; ds.host.part_type_ids = t.part_type_ids;
  ds.host_stale = true;
  return MMP_OK;
}

// rank-space vectors of a device-built snapshot, downloaded on first use (introspection, the reaper's host part)
static int32_t host_mirror(mmp_fleet *f, const DeviceSnapshot &cds, const HostSnapshot **out) {
  DeviceSnapshot &ds = const_cast<DeviceSnapshot &>(cds);
  std::lock_guard<std::mutex> g(f->mirror_mu);
  if (ds.host_stale) {
    HostSnapshot &h = ds.host;
    const int32_t n = h.n_ranks, RW = h.row_words, NS = h.n_slots, NI = f->hs.cfg.max_instances;
    h.rows.resize((size_t)n); h.rank_of.resize((size_t)NI); h.cand.resize((size_t)NS * RW); h.pref.resize((size_t)NS * RW);
    h.cap_col.resize((size_t)n); h.lthreads_col.resize((size_t)n); h.linprog_col.resize((size_t)n); h.part_of_rank.resize((size_t)n);
    if (n) {
      CK(cudaMemcpy(h.rows.data(), ds.rows.p, (size_t)n * sizeof(RankRow), cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h.cap_col.data(), ds.cap_col.p, (size_t)n * 8, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h.lthreads_col.data(), ds.lthreads_col.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h.linprog_col.data(), ds.linprog_col.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(h.part_of_rank.data(), ds.part_of_rank.p, (size_t)n * 4, cudaMemcpyDeviceToHost));
    }
    CK(cudaMemcpy(h.rank_of.data(), ds.rank_of.p, (size_t)NI * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(h.cand.data(), ds.cand.p, (size_t)NS * RW * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(h.pref.data(), ds.pref.p, (size_t)NS * RW * 4, cudaMemcpyDeviceToHost));
    ds.host_stale = false;
  }
  *out = &ds.host;
  return MMP_OK;
}

static int32_t sync_host_from_device(mmp_fleet *f, bool rows);  // churn_kernels.cuh: closed-loop changes on the device -> host tables
static int32_t commit_locked(mmp_fleet *f, bool rows_on_device);

int32_t mmp_fleet_commit(mmp_fleet *f) {
  NEED(f);
  std::lock_guard<std::mutex> g(f->ingest_mu);
  return commit_locked(f, false);
}
}  // extern "C"
// rows_on_device: called by mmp_churn_step after its republish, when lv.inst_rows is ahead of the host's instance rows
static int32_t commit_locked(mmp_fleet *f, bool rows_on_device) {
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  const auto t0 = std::chrono::steady_clock::now();
  DeviceSnapshot &ds = f->snaps[1 - f->cur];
  cudaStream_t st = f->commit_stream;
  LiveState &lv = f->live;
  bool structural = f->hs.structural_dirty || !lv.valid || f->commit_host_only;
  if (!structural) {
    rc = commit_device(f, ds, st);
    if (rc < 0) return rc;
    if (rc == 1) structural = true;  // mixed versions: the literal comparator needs the host's merge sort (N1)
  }
  if (structural) {
    // the host path builds from the host tables: first bring over what the closed loop changed on the device (either route:
    // a structural commit, or the device path's fallback above).  Outside a window the host rows are current -- the window
    // copied them back -- and may hold updates not yet scattered, so only the registry comes over.
    if (f->device_ahead) { rc = sync_host_from_device(f, rows_on_device); if (rc < 0) return rc; }
    rc = commit_structural(f, ds, st);
    if (rc < 0) return rc;
  }
  const HostSnapshot &h = ds.host;
  const int RW = h.row_words;
  const int32_t nm = f->hs.n_models_used;
  ds.n_models = nm;
  // ---- registry: model rows + edges live on the device; a commit sends only what changed on the host ----
  // A fresh allocation starts as the host holds a model that was never upserted: a zero row, no edges (-1).  A device-path
  // commit scatters only the dirty models, so an upsert past n_models_used leaves the rows in between to this initial state.
  const size_t models_cap0 = lv.models.cap, edges_cap0 = lv.edges.cap;
  CK(lv.models.ensure((size_t)std::max(f->hs.cfg.max_models, 1) * sizeof(mmp_model_row)));
  CK(lv.edges.ensure((size_t)std::max(f->hs.cfg.max_models, 1) * HostState::EDGE_INL * 4));
  if (lv.models.cap != models_cap0) CK(cudaMemsetAsync(lv.models.p, 0, lv.models.cap, st));
  if (lv.edges.cap != edges_cap0) CK(cudaMemsetAsync(lv.edges.p, 0xff, lv.edges.cap, st));
  if (!f->device_ahead) {
    f->churn.regs_from_host = true;
    if (structural || f->hs.all_models_dirty) {
      if (nm) {
        CK(cudaMemcpyAsync(lv.models.p, f->hs.models.data(), (size_t)nm * sizeof(mmp_model_row), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(lv.edges.p, f->hs.edge_inl.data(), (size_t)nm * HostState::EDGE_INL * 4, cudaMemcpyHostToDevice, st));
      }
    } else if (!f->hs.dirty_models.empty()) {
      const int32_t nd = (int32_t)f->hs.dirty_models.size();
      std::vector<mmp_model_row> rows((size_t)nd);
      std::vector<int4> ed((size_t)nd);
      for (int32_t k = 0; k < nd; k++) {
        const int32_t m = f->hs.dirty_models[k];
        rows[k] = f->hs.models[m];
        const int32_t *e = &f->hs.edge_inl[(size_t)m * HostState::EDGE_INL];
        ed[k] = make_int4(e[0], e[1], e[2], e[3]);
      }
      CK(upload_vec(lv.scratch_idx, f->hs.dirty_models, st)); CK(upload_vec(lv.scratch_rows, rows, st)); CK(upload_vec(lv.scratch_edges, ed, st));
      k_scatter_models<<<(nd + 255) / 256, 256, 0, st>>>(lv.scratch_idx.as<int32_t>(), lv.scratch_rows.as<mmp_model_row>(),
                                                         lv.scratch_edges.as<int4>(), nd, lv.models.as<mmp_model_row>(), lv.edges.as<int4>());
      f->launches++;
      CK(cudaGetLastError());
      CK(cudaStreamSynchronize(st));  // staging vectors
    }
    if (structural || f->hs.ovf_dirty || f->hs.times_dirty) {  // the overflow edges with their times (OvfEdge)
      std::vector<OvfEdge> ovf;
      f->hs.ovf_table(ovf);
      lv.n_ovf = (int32_t)ovf.size();
      CK(upload_vec(lv.ovf, ovf, st));
      CK(cudaStreamSynchronize(st));
    }
  }
  if (f->hs.times_dirty && !f->hs.edge_ts.empty()) {  // MR.instanceIds values / lastUnloadTime, when the host supplies them
    CK(upload_vec(lv.edge_ts, f->hs.edge_ts, st)); CK(upload_vec(lv.model_lul, f->hs.model_lul, st));
    CK(cudaStreamSynchronize(st));
    lv.have_times = true;
    f->hs.times_dirty = false;
  }
  // each snapshot keeps its own copy of the model rows so in-flight readers of the other epoch are undisturbed
  CK(ds.models.ensure((size_t)std::max(nm, 1) * sizeof(mmp_model_row)));
  if (nm) CK(cudaMemcpyAsync(ds.models.p, lv.models.p, (size_t)nm * sizeof(mmp_model_row), cudaMemcpyDeviceToDevice, st));
  // exclusion bitmap in rank space: zero, then scatter the device-resident loaded/failed lists (one write pass)
  const int ST = h.excl_stride;  // words per stored row: the whole row, or this instance shard's block
  // (instance-sharded: sized for max_models rows from the first commit on, so that the block keeps the address its peers mapped)
  CK(ds.excl.ensure(f->hs.cfg.shard_count > 1 ? std::max(mmp_fleet::Peers::IPC_MIN_BYTES, (size_t)std::max(nm, f->hs.cfg.max_models) * ST * 4)
                                              : (size_t)std::max(nm, 1) * ST * 4));
  // the excluded ranks of every model beside its row (k_place_direct reads them instead of the row): whole rows only
  const bool whole_rows = h.word_lo == 0 && h.word_hi == RW;
  if (whole_rows) CK(ds.excl_ranks.ensure((size_t)std::max(nm, 1) * 16));
  int4 *ranks = whole_rows ? ds.excl_ranks.as<int4>() : nullptr;
  // the row of every request-model decision (MMP_DF_REQUEST_MODEL): the stride is fixed for the fleet, so it is zeroed once
  // (cudaMalloc: 256-byte aligned, as the TMA copies of k_place_lanes and k_place need)
  if (whole_rows && !f->zero_row.p) {
    CK(f->zero_row.ensure((size_t)ST * 4));
    CK(cudaMemsetAsync(f->zero_row.p, 0, (size_t)ST * 4, st));
  }
  if (nm) {
    CK(cudaMemsetAsync(ds.excl.p, 0, (size_t)nm * ST * 4, st));
    k_build_bitmap<<<(nm + 255) / 256, 256, 0, st>>>(ds.excl.as<uint32_t>(), lv.edges.as<int4>(), ds.rank_of.as<int32_t>(), nm, ST,
                                                     h.word_lo, h.word_hi, ranks);
    f->launches++;
    CK(cudaGetLastError());
    if (lv.n_ovf) {
      k_build_bitmap_ovf<<<(lv.n_ovf + 255) / 256, 256, 0, st>>>(ds.excl.as<uint32_t>(), lv.ovf.as<OvfEdge>(), lv.n_ovf,
                                                                 ds.rank_of.as<int32_t>(), ST, h.word_lo, h.word_hi, ranks);
      f->launches++;
      CK(cudaGetLastError());
    }
  }
  if (f->hs.cfg.shard_count > 1 && nm) {  // the replicated front of every row (peer-access path: decisions are dealt across the shards)
    const int F = std::min(SHARD_FRONT_WORDS, RW);
    CK(ds.front.ensure((size_t)nm * F * 4));
    CK(cudaMemsetAsync(ds.front.p, 0, (size_t)nm * F * 4, st));
    k_build_bitmap<<<(nm + 255) / 256, 256, 0, st>>>(ds.front.as<uint32_t>(), lv.edges.as<int4>(), ds.rank_of.as<int32_t>(), nm, F, 0, F, nullptr);
    if (lv.n_ovf) k_build_bitmap_ovf<<<(lv.n_ovf + 255) / 256, 256, 0, st>>>(ds.front.as<uint32_t>(), lv.ovf.as<OvfEdge>(), lv.n_ovf, ds.rank_of.as<int32_t>(), F, 0, F, nullptr);
    f->launches += 2;
    CK(cudaGetLastError());
  }
  int n_sparse = 0;
  if (h.n_slots > 0) {
    CK(ds.sparse_dev.ensure(16));
    CK(cudaMemsetAsync(ds.sparse_dev.p, 0, 4, st));
    k_sparse_slots<<<(h.n_slots + 63) / 64, 64, 0, st>>>((h.any_rs ? ds.candx : ds.cand).as<uint32_t>(), RW, h.n_slots, h.word_lo, LANE_WIN, 24, ds.sparse_dev.as<int>());
    CK(cudaMemcpyAsync(&n_sparse, ds.sparse_dev.p, 4, cudaMemcpyDeviceToHost, st));
    f->launches++;
  }
  CK(cudaStreamSynchronize(st));
  ds.sparse_slots = h.n_slots > 0 && 2 * n_sparse >= h.n_slots;
  SnapshotView &v = ds.view;
  v.n_ranks = h.n_ranks; v.row_words = RW; v.n_models = nm; v.max_instances = f->hs.cfg.max_instances;
  v.any_rs = h.any_rs; v.n_type_ids = (int32_t)h.type_slot.size(); v.min_space = f->hs.cfg.min_space_units;
  v.word_lo = h.word_lo; v.word_hi = h.word_hi; v.excl_stride = ST; v.n_slots = h.n_slots; v.n_extra = 0;
  v.count_col = ds.count_col.as<int32_t>(); v.cand_before = ds.cand_before.as<int32_t>();
  v.nzw = ds.nzw.as<uint16_t>(); v.nz_n = ds.nz_n.as<int32_t>();
  v.excl = ds.excl.as<uint32_t>(); v.excl_ranks = ranks ? ds.excl_ranks.as<int32_t>() : nullptr;
  v.cand = ds.cand.as<uint32_t>(); v.pref = ds.pref.as<uint32_t>();
  v.has_pref = ds.has_pref.as<uint8_t>(); v.type_slot = ds.type_slot.as<uint16_t>(); v.candx = ds.candx.as<uint32_t>();
  v.full = ds.full.as<uint32_t>(); v.rows = ds.rows.as<RankRow>(); v.rank_of = ds.rank_of.as<int32_t>();
  v.csum = ds.csum.as<WordSumI>(); v.lsum = ds.lsum.as<WordSumL>(); v.models = ds.models.as<mmp_model_row>();
  v.zero_row = whole_rows ? f->zero_row.as<uint32_t>() : nullptr;
  {
    std::unique_lock<std::shared_mutex> w(f->snap_mu);  // waits for in-flight readers of the current epoch
    f->cur = 1 - f->cur;
    f->epoch++;
  }
  f->hs.clear_dirty();
  f->last_commit_path = structural ? 1 : 2;
  f->last_commit_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  return f->epoch;
}
extern "C" {
/* tuning / measurement knobs (the MMP_* environment variables, settable on a live fleet) */
int32_t mmp_tune(mmp_fleet *f, const char *key, int64_t value) {
  NEED(f);
  if (!key) { g_err = "null key"; return MMP_E_ARG; }
  if (!strcmp(key, "one_mode") && value >= 0 && value <= 3) f->one_mode = (int)value;
  else if (!strcmp(key, "server_life_us") && value >= 50 && value <= 1000000) f->srv.life_us = value;
  else if (!strcmp(key, "server_idle_us") && value >= 10 && value <= 1000000) f->srv.idle_us = value;
  else if (!strcmp(key, "direct") && (value == 0 || value == 1)) f->kernel = value ? PlaceKernel::direct : PlaceKernel::lanes;
  else if (!strcmp(key, "sort_slots") && value >= 0 && value <= 2) f->sort_slots = (int)value;
  else if (!strcmp(key, "lane_budget") && value >= 1 && value <= 4096) f->lane_budget = (int)value;
  else if (!strcmp(key, "split") && value >= 0 && value <= 2) f->split = (int)value;
  else if (!strcmp(key, "commit_host_only") && (value == 0 || value == 1)) f->commit_host_only = (int)value;
  else { g_err = "unknown key or value out of range"; return MMP_E_ARG; }
  return MMP_OK;
}
/* CUDA-event duration (ms) of the device part of the last call of a scan: "stats", "reaper", "lru_apply", "commit" */
int32_t mmp_last_timing(mmp_fleet *f, const char *key, double *ms) {
  NEED(f);
  if (!key || !ms) { g_err = "null argument"; return MMP_E_ARG; }
  if (!strcmp(key, "stats")) *ms = f->t_stats_ms;
  else if (!strcmp(key, "reaper")) *ms = f->t_reaper_ms;
  else if (!strcmp(key, "lru_apply")) *ms = f->t_lru_ms;
  else if (!strcmp(key, "lru_read")) *ms = f->t_lru_read_ms;
  else if (!strcmp(key, "prune")) *ms = f->t_prune_ms;
  else if (!strcmp(key, "commit")) *ms = f->last_commit_ms;
  else if (!strcmp(key, "dealt_kernel")) *ms = f->peers.t_kernel_ms;
  else if (!strcmp(key, "dealt_wait")) *ms = f->peers.t_wait_ms;
  else { g_err = "unknown key"; return MMP_E_ARG; }
  return MMP_OK;
}
/* which path the last commit took (1 = structural / host, 2 = device) and how long it took on the host clock */
int32_t mmp_commit_info(mmp_fleet *f, int32_t *path, double *ms) {
  NEED(f);
  if (path) *path = f->last_commit_path;
  if (ms) *ms = f->last_commit_ms;
  return MMP_OK;
}

// ---- the resident B = 1 server (k_place_server): post a request of up to 32 decisions, spin on the response ----
static void server_stop(mmp_fleet *f) {
  mmp_fleet::Server &sv = f->srv;
  if (!sv.mapped || !sv.running) return;
  volatile SrvLine0 *l0 = reinterpret_cast<volatile SrvLine0 *>(sv.mapped.get());
  sv.seq++;
  l0->seq = (sv.seq & 0x00ffffffffffffffull) | (0xffull << 56);  // kind 0xff: leave
  std::atomic_thread_fence(std::memory_order_seq_cst);
  cudaStreamSynchronize(sv.stream);
  sv.running = false;
}
// mapped buffer: [line 0][line 1][32 decisions][32 results][32 fresh rows][32 x MMP_MAX_EXTRA extras] ... [response line]
static int32_t place_server(mmp_fleet *f, const DeviceSnapshot &ds, const mmp_decision_in *in, int32_t n, const FreshRow *fresh, int32_t n_fresh,
                            const int32_t *extra, int32_t n_extra, mmp_decision_out *out, int64_t now_ms, uint64_t seed) {
  mmp_fleet::Server &sv = f->srv;
  if (!sv.mapped) {
    CK(cudaHostAlloc((void **)sv.mapped.put(), PlaceCtx::MAPPED_BYTES, cudaHostAllocMapped));
    memset(sv.mapped, 0, PlaceCtx::MAPPED_BYTES);
    CK(cudaStreamCreateWithFlags(sv.stream.put(), cudaStreamNonBlocking));
  }
  unsigned char *h = sv.mapped, *dbase = nullptr;
  CK(cudaHostGetDevicePointer((void **)&dbase, h, 0));
  const size_t g_in = 128, g_out = g_in + 32 * sizeof(mmp_decision_in), g_fr = g_out + 32 * sizeof(mmp_decision_out), g_ex = g_fr + 32 * sizeof(FreshRow),
               g_resp = PlaceCtx::MAPPED_BYTES - 64;
  static_assert(128 + 32 * (sizeof(mmp_decision_in) + sizeof(mmp_decision_out) + sizeof(FreshRow)) + 32 * MMP_MAX_EXTRA * 4 + 64 <= PlaceCtx::MAPPED_BYTES, "mapped layout");
  volatile SrvLine0 *l0 = reinterpret_cast<volatile SrvLine0 *>(h);
  volatile SrvLine1 *l1 = reinterpret_cast<volatile SrvLine1 *>(h + 64);
  volatile ServerResp *resp = reinterpret_cast<volatile ServerResp *>(h + g_resp);
  if (sv.running && sv.epoch != f->epoch) server_stop(f);  // its snapshot view is another epoch's
  // kind 1: one decision whose side tables are at most its own fresh row and a few extra excludes from the start of extra[]
  // (the shape of getNext on a request thread: a request-model decision carries its model's copies and failures there)
  const int32_t n_inline = n_extra == 0 ? 0 : in[0].extra_n;
  const bool single = n == 1 && (n_extra == 0 || (in[0].extra_off == 0 && n_inline >= 0 && n_inline <= SRV_INLINE_EXTRA && n_inline <= n_extra)) &&
                      (in[0].fresh < 0 || in[0].fresh == 0) && n_fresh <= 1;
  if (single) {
    mmp_decision_in d = in[0];
    if (n_fresh) { FreshRow fr = fresh[0]; memcpy((void *)&l1->fr, &fr, sizeof(fr)); }
    if (n_inline) memcpy((void *)l1->extra, extra, (size_t)n_inline * 4);
    l1->n = 1; l1->n_fresh = n_fresh; l1->n_extra = n_inline;
    memcpy((void *)&l0->d, &d, sizeof(d));
  } else {
    memcpy(h + g_in, in, (size_t)n * sizeof(mmp_decision_in));
    if (n_fresh) memcpy(h + g_fr, fresh, (size_t)n_fresh * sizeof(FreshRow));
    if (n_extra) memcpy(h + g_ex, extra, (size_t)n_extra * 4);
    l1->n = n; l1->n_fresh = n_fresh; l1->n_extra = n_extra;
  }
  l0->now = now_ms; l0->seed = seed; l0->id_base = f->id_base.load();
  auto launch = [&]() -> int32_t {
    if ((l0->seq >> 56) == 0xffull) l0->seq = resp->done_seq;  // (a "leave" left behind by server_stop is not for the new server)
    resp->alive = 1;
    std::atomic_thread_fence(std::memory_order_seq_cst);
    k_place_server<<<1, 32, 0, sv.stream>>>(ds.view, reinterpret_cast<volatile SrvLine0 *>(dbase), reinterpret_cast<volatile SrvLine1 *>(dbase + 64),
                                          reinterpret_cast<volatile ServerResp *>(dbase + g_resp), (const mmp_decision_in *)(dbase + g_in),
                                          (const FreshRow *)(dbase + g_fr), (const int32_t *)(dbase + g_ex), (mmp_decision_out *)(dbase + g_out),
                                          (unsigned long long)sv.life_us * 1000ull, (unsigned long long)sv.idle_us * 1000ull, f->lane_budget);
    CK(cudaGetLastError());
    sv.running = true; sv.epoch = f->epoch; sv.launches++; f->launches++;
    return MMP_OK;
  };
  if (!sv.running || resp->alive == 0) { int32_t rc = launch(); if (rc < 0) return rc; }
  sv.seq++;
  const uint64_t seq = (sv.seq & 0x00ffffffffffffffull) | ((uint64_t)(single ? 1 : 2) << 56);
  std::atomic_thread_fence(std::memory_order_seq_cst);
  l0->seq = seq;  // (the last store into line 0: a reader that sees it sees the request)
  std::atomic_thread_fence(std::memory_order_seq_cst);
  const auto t0 = std::chrono::steady_clock::now();
  for (uint32_t spins = 0;; spins++) {
    if (resp->done_seq == seq) break;
    if (resp->alive == 0) {  // the server's lifetime ended -- before or after it saw this request?
      CK(cudaStreamSynchronize(sv.stream));
      if (resp->done_seq == seq) break;
      int32_t rc = launch();
      if (rc < 0) return rc;
    }
    if ((spins & 0xfff) == 0xfff && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(2)) {
      server_stop(f);
      g_err = "the placement server did not answer within 2 s";
      return MMP_E_CUDA;
    }
  }
  std::atomic_thread_fence(std::memory_order_seq_cst);
  if (single) { out[0].target = resp->out0.target; out[0].n_candidates = resp->out0.n_candidates; }
  else memcpy(out, h + g_out, (size_t)n * sizeof(mmp_decision_out));
  sv.requests++;
  return MMP_OK;
}

// Tiny untraced, unsharded batches, zero-copy: the records, fresh rows (c->fresh_host) and extras are written into the
// context's pinned mapped buffer, and the kernel reads them and writes its results there, so a call is one launch and one
// synchronise with no copy calls.  The caller has checked that the batch fits the buffer.  A view with the call's own
// slot tables (`derived`: an exclude set) skips the resident server and the captured graph, which both hold the epoch's.
static int32_t place_mapped(mmp_fleet *f, PlaceCtx *c, const DeviceSnapshot &ds, const SnapshotView &vw, bool derived, const mmp_decision_in *in,
                            int32_t n, int32_t n_fresh, const int32_t *extra, int32_t n_extra, mmp_decision_out *out, int64_t now_ms, uint64_t seed) {
  const bool fits32 = n <= 32 && n_fresh <= 32 && (size_t)n_extra <= 32 * MMP_MAX_EXTRA && !derived;
  if (f->one_mode == 3 && fits32) {
    std::unique_lock<std::mutex> lk(f->srv.mu, std::try_to_lock);
    if (lk.owns_lock()) return place_server(f, ds, in, n, c->fresh_host.data(), n_fresh, extra, n_extra, out, now_ms, seed);
  }  // (taken by another caller: this call goes the graph way)
  // one 32-thread block as a replayed graph: the node's parameters are those of the epoch it was captured in (the snapshot
  // view by value, the fixed offsets of a layout for 32 decisions behind a SmallHdr); what changes per call -- now, seed,
  // id base, n -- is read from the header.  Other launches take the batch packed from offset 0.
  const bool graph = f->one_mode >= 2 && fits32;
  static_assert(64 + 32 * (sizeof(mmp_decision_in) + sizeof(mmp_decision_out) + sizeof(FreshRow)) + 32 * MMP_MAX_EXTRA * 4 <= PlaceCtx::MAPPED_BYTES, "mapped layout");
  const size_t rows = graph ? 32 : (size_t)n;
  const size_t o_in = graph ? 64 : 0, o_out = o_in + rows * sizeof(mmp_decision_in), o_fr = o_out + rows * sizeof(mmp_decision_out);
  const size_t o_ex = graph ? o_fr + 32 * sizeof(FreshRow) : (o_fr + (size_t)n_fresh * sizeof(FreshRow) + 15) / 16 * 16;
  unsigned char *h = c->mapped, *dbase = nullptr;
  CK(cudaHostGetDevicePointer((void **)&dbase, h, 0));
  memcpy(h + o_in, in, (size_t)n * sizeof(mmp_decision_in));
  if (n_fresh) memcpy(h + o_fr, c->fresh_host.data(), (size_t)n_fresh * sizeof(FreshRow));
  if (n_extra) memcpy(h + o_ex, extra, (size_t)n_extra * 4);
  const mmp_decision_in *d_in = (const mmp_decision_in *)(dbase + o_in);
  const FreshRow *d_fr = (const FreshRow *)(dbase + o_fr);
  const int32_t *d_ex = (const int32_t *)(dbase + o_ex);
  mmp_decision_out *d_out = (mmp_decision_out *)(dbase + o_out);
  cudaStream_t st = c->stream;
  if (graph) {
    SmallHdr *hd = reinterpret_cast<SmallHdr *>(h);
    hd->now = now_ms; hd->seed = seed; hd->id_base = f->id_base.load(); hd->n = n; hd->n_fresh = n_fresh; hd->n_extra = n_extra;
    if (c->graph_epoch != f->epoch || !c->graph_exec) {
      c->graph_exec.reset();
      c->graph.reset();  // (not inside the capture below)
      SnapshotView gv = ds.view;
      gv.n_extra = 32 * MMP_MAX_EXTRA;
      CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      k_place_small<<<1, 32, 0, st>>>(gv, d_in, 0, d_fr, 32, d_ex, d_out, 0, 0, 0, reinterpret_cast<const volatile SmallHdr *>(dbase), f->lane_budget);
      CK(cudaStreamEndCapture(st, c->graph.put()));
      CK(cudaGraphInstantiate(c->graph_exec.put(), c->graph, 0));
      c->graph_epoch = f->epoch;
    }
    CK(cudaGraphLaunch(c->graph_exec, st));
    f->launches++;
  } else if (f->one_mode == 0 || n > 512) {
    PlaceArgs a{vw, d_in, n, d_fr, n_fresh, d_ex, d_out, nullptr, nullptr, now_ms, seed, f->id_base.load()};
    CK(launch_place(f, a, st));
  } else {
    k_place_small<<<(n + 31) / 32, 32, 0, st>>>(vw, d_in, n, d_fr, n_fresh, d_ex, d_out, now_ms, seed, f->id_base.load(), nullptr, f->lane_budget);
    f->launches++;
    CK(cudaGetLastError());
  }
  CK(cudaStreamSynchronize(st));
  memcpy(out, h + o_out, (size_t)n * sizeof(mmp_decision_out));
  return MMP_OK;
}

// The call's view on the derived slot tables of an exclude set: k_exclude_slots clears the set's ranks from the snapshot's
// cand / candx / pref, k_slot_lists builds their compressed word lists.  Queued on st; the ids are in host memory.
static int32_t derive_exclude_tables(mmp_fleet *f, PlaceCtx *c, const int32_t *exclude, int32_t n_exclude, SnapshotView &vw, cudaStream_t st) {
  const int32_t NS = vw.n_slots, RW = vw.row_words;
  if (NS <= 0) return MMP_OK;  // (no live instance: no slot, nothing to derive)
  const size_t words = (size_t)NS * RW;
  CK(c->d_xids.ensure((size_t)n_exclude * 4));
  CK(c->d_xcand.ensure(words * 4)); CK(c->d_xcandx.ensure(words * 4)); CK(c->d_xpref.ensure(words * 4));
  CK(c->d_xnzw.ensure(words * 2)); CK(c->d_xnz_n.ensure((size_t)NS * 4)); CK(c->d_xbefore.ensure((size_t)NS * 4));
  CK(cudaMemcpyAsync(c->d_xids.p, exclude, (size_t)n_exclude * 4, cudaMemcpyHostToDevice, st));
  k_exclude_slots<<<NS, 256, (size_t)RW * 4, st>>>(c->d_xids.as<int32_t>(), n_exclude, vw.rank_of, RW, vw.cand, vw.candx, vw.pref,
                                                   c->d_xcand.as<uint32_t>(), c->d_xcandx.as<uint32_t>(), c->d_xpref.as<uint32_t>());
  k_slot_lists<<<(NS + 31) / 32, 32, 0, st>>>(c->d_xcand.as<uint32_t>(), c->d_xcandx.as<uint32_t>(), vw.any_rs, RW, NS, vw.word_lo, vw.word_hi,
                                             c->d_xnzw.as<uint16_t>(), c->d_xnz_n.as<int32_t>(), c->d_xbefore.as<int32_t>());
  f->launches += 2;
  CK(cudaGetLastError());
  vw.cand = c->d_xcand.as<uint32_t>(); vw.candx = c->d_xcandx.as<uint32_t>(); vw.pref = c->d_xpref.as<uint32_t>();
  vw.nzw = c->d_xnzw.as<uint16_t>(); vw.nz_n = c->d_xnz_n.as<int32_t>(); vw.cand_before = c->d_xbefore.as<int32_t>();
  return MMP_OK;
}

// The one host path of mmp_place_batch / _trace / _excluding / mmp_place_one.  exclude[0, n_exclude): the call-wide exclude
// set; with n_exclude == 0 the call takes exactly the route it takes without one.
static int32_t place_impl(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                          const int32_t *extra, int32_t n_extra, mmp_decision_out *out, mmp_decision_trace *trace,
                          uint32_t *cand_mask, int64_t now_ms, uint64_t seed, const int32_t *exclude = nullptr, int32_t n_exclude = 0) {
  NEED(f);
  if (n < 0 || (n > 0 && (!in || !out)) || n_fresh < 0 || n_extra < 0 || (n_fresh > 0 && !fresh) || (n_extra > 0 && !extra)) {
    g_err = "bad argument"; return MMP_E_ARG;
  }
  if (n_exclude < 0 || (n_exclude > 0 && !exclude)) { g_err = "bad exclude set"; return MMP_E_ARG; }
  for (int32_t k = 0; k < n_exclude; k++)
    if (exclude[k] < 0 || exclude[k] >= f->hs.cfg.max_instances) {
      g_err = "exclude set: instance index " + std::to_string(exclude[k]) + " outside [0, max_instances)"; return MMP_E_ARG;
    }
  if (n_exclude > 0 && places_sharded(f, trace || cand_mask)) {
    g_err = "an exclude set is not available on an instance-sharded fleet or one that connected a communicator"; return MMP_E_STATE;
  }
  if (n == 0) return MMP_OK;
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  if (f->epoch == 0) { g_err = "no committed snapshot (call mmp_fleet_commit)"; return MMP_E_EPOCH; }
  const DeviceSnapshot &ds = f->snaps[f->cur];
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  c->fresh_host.resize((size_t)n_fresh);
  for (int32_t i = 0; i < n_fresh; i++)
    if (const char *m = HostState::fresh_row(fresh[i], c->fresh_host[i])) { g_err = std::string("fresh row: ") + m; return MMP_E_ARG; }
  const int RW = ds.view.row_words;
  cudaStream_t st = c->stream;
  const bool traced = trace || cand_mask;
  const bool fast_paths = !traced && !places_sharded(f, traced);  // the mapped tiny-batch path and the chunk pipeline apply
  SnapshotView vw = ds.view;
  vw.n_extra = n_extra;  // per call: the device checks every decision's extra[] slice against it (prepare_ctx_a)
  if (n_exclude > 0 && (rc = derive_exclude_tables(f, c.get(), exclude, n_exclude, vw, st)) < 0) return rc;
  const size_t need = (size_t)n * (sizeof(mmp_decision_in) + sizeof(mmp_decision_out)) + (size_t)n_fresh * sizeof(FreshRow) + (size_t)n_extra * 4 + 64;
  if (fast_paths && need <= PlaceCtx::MAPPED_BYTES)
    return place_mapped(f, c.get(), ds, vw, n_exclude > 0, in, n, n_fresh, extra, n_extra, out, now_ms, seed);
  CK(c->d_in.ensure((size_t)n * sizeof(mmp_decision_in)));
  CK(c->d_out.ensure((size_t)n * sizeof(mmp_decision_out)));
  if (trace) CK(c->d_trace.ensure((size_t)n * sizeof(mmp_decision_trace)));
  if (cand_mask) CK(c->d_cand.ensure((size_t)n * 2 * RW * 4));
  if ((rc = stage_side_tables(c.get(), c->fresh_host.data(), n_fresh, extra, n_extra, st)) < 0) return rc;
  PlaceArgs a{vw, c->d_in.as<mmp_decision_in>(), n, c->d_fresh.as<FreshRow>(), n_fresh, c->d_extra.as<int32_t>(),
              c->d_out.as<mmp_decision_out>(), trace ? c->d_trace.as<mmp_decision_trace>() : nullptr,
              cand_mask ? c->d_cand.as<uint32_t>() : nullptr, now_ms, seed, f->id_base.load()};
  a.ctx = c.get();
  if (fast_paths && n > (1 << 17)) return place_chunks(f, c.get(), a, 1 << 17, in, out);
  CK(cudaMemcpyAsync(c->d_in.p, in, (size_t)n * sizeof(mmp_decision_in), cudaMemcpyHostToDevice, st));
  if (cand_mask) CK(cudaMemsetAsync(c->d_cand.p, 0, (size_t)n * 2 * RW * 4, st));
  if ((rc = place_on_device(f, c.get(), ds, a, st)) < 0) return rc;
  CK(cudaMemcpyAsync(out, c->d_out.p, (size_t)n * sizeof(mmp_decision_out), cudaMemcpyDeviceToHost, st));
  if (trace) CK(cudaMemcpyAsync(trace, c->d_trace.p, (size_t)n * sizeof(mmp_decision_trace), cudaMemcpyDeviceToHost, st));
  if (cand_mask) CK(cudaMemcpyAsync(cand_mask, c->d_cand.p, (size_t)n * 2 * RW * 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return MMP_OK;
}

int32_t mmp_place_batch(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                        const int32_t *extra, int32_t n_extra, mmp_decision_out *out, int64_t now_ms, uint64_t seed) {
  return place_impl(f, in, n, fresh, n_fresh, extra, n_extra, out, nullptr, nullptr, now_ms, seed);
}
int32_t mmp_place_batch_trace(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                              const int32_t *extra, int32_t n_extra, mmp_decision_out *out, mmp_decision_trace *trace,
                              uint32_t *cand_mask, int64_t now_ms, uint64_t seed) {
  return place_impl(f, in, n, fresh, n_fresh, extra, n_extra, out, trace, cand_mask, now_ms, seed);
}
int32_t mmp_place_batch_excluding(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                                  const int32_t *extra, int32_t n_extra, const int32_t *exclude, int32_t n_exclude, mmp_decision_out *out,
                                  mmp_decision_trace *trace, uint32_t *cand_mask, int64_t now_ms, uint64_t seed) {
  return place_impl(f, in, n, fresh, n_fresh, extra, n_extra, out, trace, cand_mask, now_ms, seed, exclude, n_exclude);
}
int32_t mmp_place_one(mmp_fleet *f, const mmp_decision_in *in, const mmp_instance_row *fresh, const int32_t *extra,
                      mmp_decision_out *out, int64_t now_ms, uint64_t seed) {
  if (!in) { g_err = "null decision"; return MMP_E_ARG; }
  int32_t nf = (fresh && in->fresh >= 0) ? in->fresh + 1 : 0;
  int32_t ne = (extra && in->extra_n > 0) ? in->extra_off + in->extra_n : 0;
  return place_impl(f, in, 1, fresh, nf, extra, ne, out, nullptr, nullptr, now_ms, seed);
}

int32_t mmp_place_sweep(mmp_fleet *f, int32_t first_model, int32_t n, const int32_t *self, int32_t self_stride,
                        const uint32_t *favour_bits, mmp_decision_out *out, int64_t now_ms, uint64_t seed) {
  NEED(f);
  if (n < 0 || first_model < 0 || (n > 0 && (!self || !out)) || (self_stride != 0 && self_stride != 1)) { g_err = "bad argument"; return MMP_E_ARG; }
  if (n == 0) return MMP_OK;
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  if (f->epoch == 0) { g_err = "no committed snapshot (call mmp_fleet_commit)"; return MMP_E_EPOCH; }
  const DeviceSnapshot &ds = f->snaps[f->cur];
  if ((int64_t)first_model + n > ds.n_models) { g_err = "sweep runs past the registry"; return MMP_E_ARG; }
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t st = c->stream;
  const size_t n_self = self_stride ? (size_t)n : 1, n_fav = favour_bits ? ((size_t)n + 31) / 32 : 0;
  CK(c->d_in.ensure((size_t)n * sizeof(mmp_decision_in)));
  CK(c->d_out.ensure((size_t)n * sizeof(mmp_decision_out)));
  if ((rc = stage_side_tables(c.get(), nullptr, 0, nullptr, 0, st)) < 0) return rc;
  CK(c->d_trace.ensure(n_self * 4 + n_fav * 4 + 16));  // scratch: self[] then favour bits
  int32_t *d_self = c->d_trace.as<int32_t>();
  uint32_t *d_fav = n_fav ? reinterpret_cast<uint32_t *>(d_self + n_self) : nullptr;
  CK(cudaMemcpyAsync(d_self, self, n_self * 4, cudaMemcpyHostToDevice, st));
  if (n_fav) CK(cudaMemcpyAsync(d_fav, favour_bits, n_fav * 4, cudaMemcpyHostToDevice, st));
  k_expand_sweep<<<(n + 255) / 256, 256, 0, st>>>(c->d_in.as<mmp_decision_in>(), n, first_model, d_self, self_stride, d_fav);
  f->launches++;
  CK(cudaGetLastError());
  PlaceArgs a{ds.view, c->d_in.as<mmp_decision_in>(), n, c->d_fresh.as<FreshRow>(), 0, c->d_extra.as<int32_t>(),
              c->d_out.as<mmp_decision_out>(), nullptr, nullptr, now_ms, seed, f->id_base.load()};
  a.ctx = c.get();
  // unsharded: the results of chunk k travel to the host while chunk k + 1 is scored
  if (!places_sharded(f, false)) return place_chunks(f, c.get(), a, 1 << 18, nullptr, out);
  if ((rc = place_on_device(f, c.get(), ds, a, st)) < 0) return rc;
  CK(cudaMemcpyAsync(out, c->d_out.p, (size_t)n * sizeof(mmp_decision_out), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return MMP_OK;
}

int32_t mmp_place_batch_device(mmp_fleet *f, const void *d_in, int32_t n, void *d_out, int64_t now_ms, uint64_t seed, float *kernel_ms) {
  NEED(f);
  if (n <= 0 || !d_in || !d_out) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  const DeviceSnapshot &ds = f->snaps[f->cur];
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  if ((rc = stage_side_tables(c.get(), nullptr, 0, nullptr, 0, c->stream)) < 0) return rc;
  PlaceArgs a{ds.view, (const mmp_decision_in *)d_in, n, c->d_fresh.as<FreshRow>(), 0, c->d_extra.as<int32_t>(),
              (mmp_decision_out *)d_out, nullptr, nullptr, now_ms, seed, f->id_base.load()};
  a.ctx = c.get();
  CK(cudaEventRecord(c->e0, c->stream));
  if ((rc = place_on_device(f, c.get(), ds, a, c->stream)) < 0) return rc;
  CK(cudaEventRecord(c->e1, c->stream));
  CK(cudaEventSynchronize(c->e1));
  if (kernel_ms) CK(cudaEventElapsedTime(kernel_ms, c->e0, c->e1));
  return MMP_OK;
}

int32_t mmp_device_alloc(mmp_fleet *f, int64_t bytes, void **out) {
  NEED(f);
  if (bytes <= 0 || !out) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f); if (rc < 0) return rc;
  CK(cudaMalloc(out, (size_t)bytes));
  return MMP_OK;
}
int32_t mmp_device_free(mmp_fleet *f, void *p) { NEED(f); int32_t rc = set_device(f); if (rc < 0) return rc; CK(cudaFree(p)); return MMP_OK; }
int32_t mmp_device_upload(mmp_fleet *f, void *dst, const void *src, int64_t bytes) {
  NEED(f); int32_t rc = set_device(f); if (rc < 0) return rc;
  CK(cudaMemcpy(dst, src, (size_t)bytes, cudaMemcpyHostToDevice));
  return MMP_OK;
}
int32_t mmp_device_download(mmp_fleet *f, void *dst, const void *src, int64_t bytes) {
  NEED(f); int32_t rc = set_device(f); if (rc < 0) return rc;
  CK(cudaMemcpy(dst, src, (size_t)bytes, cudaMemcpyDeviceToHost));
  return MMP_OK;
}
int32_t mmp_host_alloc(mmp_fleet *f, int64_t bytes, void **out) {
  NEED(f);
  if (bytes <= 0 || !out) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f); if (rc < 0) return rc;
  CK(cudaHostAlloc(out, (size_t)bytes, cudaHostAllocDefault));
  return MMP_OK;
}
int32_t mmp_host_free(mmp_fleet *f, void *p) { NEED(f); int32_t rc = set_device(f); if (rc < 0) return rc; CK(cudaFreeHost(p)); return MMP_OK; }
int32_t mmp_flush_l2(mmp_fleet *f) {
  NEED(f);
  int32_t rc = set_device(f); if (rc < 0) return rc;
  const size_t bytes = 128u << 20;  // > 2 x the 50 MB L2 of an H100
  CK(f->d_flush.ensure(bytes));
  CK(cudaMemsetAsync(f->d_flush.p, (int)(f->launches.load() & 0xff), bytes, 0));
  CK(cudaStreamSynchronize(0));
  return MMP_OK;
}

int32_t mmp_row_words(mmp_fleet *f) { NEED(f); return f->hs.row_words(); }
int32_t mmp_live_instances(mmp_fleet *f) { NEED(f); std::shared_lock<std::shared_mutex> rd(f->snap_mu); return f->snaps[f->cur].host.n_ranks; }
int32_t mmp_cluster_order(mmp_fleet *f, int32_t *out_idx, int32_t cap) {
  NEED(f);
  int32_t rc0 = set_device(f); if (rc0 < 0) return rc0;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  const HostSnapshot *hp = nullptr;
  rc0 = host_mirror(f, f->snaps[f->cur], &hp); if (rc0 < 0) return rc0;
  const HostSnapshot &h = *hp;
  for (int32_t r = 0; r < h.n_ranks && r < cap; r++) out_idx[r] = h.rows[r].idx;
  return h.n_ranks;
}
int32_t mmp_type_sets(mmp_fleet *f, int32_t type_id, int32_t n_idx, uint8_t *allowed, int32_t *allowed_null, uint8_t *preferred,
                      int32_t *preferred_null) {
  NEED(f);
  int32_t rc0 = set_device(f); if (rc0 < 0) return rc0;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  const HostSnapshot *hp = nullptr;
  rc0 = host_mirror(f, f->snaps[f->cur], &hp); if (rc0 < 0) return rc0;
  const HostSnapshot &s = *hp;
  if (type_id < 0 || type_id > 65535) { g_err = "bad type id"; return MMP_E_ARG; }
  // a name interned after this snapshot was committed had no configuration in it: it resolves like id 0
  int sl = s.type_slot[type_id < (int32_t)s.type_slot.size() ? type_id : 0];
  *allowed_null = s.allowed_null[sl]; *preferred_null = !s.has_pref[sl];
  for (int32_t i = 0; i < n_idx; i++) {
    int32_t r = i < (int32_t)s.rank_of.size() ? s.rank_of[i] : -1;
    allowed[i] = (r >= 0 && !s.allowed_null[sl]) ? (s.cand[(size_t)sl * s.row_words + (r >> 5)] >> (r & 31)) & 1u : 0;
    preferred[i] = (r >= 0) ? (s.pref[(size_t)sl * s.row_words + (r >> 5)] >> (r & 31)) & 1u : 0;
  }
  return MMP_OK;
}
int32_t mmp_instance_partition(mmp_fleet *f, int32_t idx) {
  NEED(f);
  int32_t rc0 = set_device(f); if (rc0 < 0) return rc0;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  const HostSnapshot *hp = nullptr;
  rc0 = host_mirror(f, f->snaps[f->cur], &hp); if (rc0 < 0) return rc0;
  const HostSnapshot &s = *hp;
  if (idx < 0 || idx >= (int32_t)s.rank_of.size() || s.rank_of[idx] < 0) return -1;
  return s.part_of_rank[s.rank_of[idx]];
}
int64_t mmp_kernel_launches(mmp_fleet *f) { return f ? f->launches.load() : 0; }

}  // extern "C"

// ---------------------------------------------------------------------------------------------------------------
// micro-batcher (SURVEY.md §8b plug point 1): many request threads, one submit thread, one mmp_place_batch per drain
// ---------------------------------------------------------------------------------------------------------------
struct mmp_batcher {
  mmp_fleet *f = nullptr;
  int32_t max_batch = 4096, max_wait_us = 50;
  uint64_t seed = 0;
  struct Req {
    mmp_decision_in in; mmp_instance_row fresh; bool has_fresh; int32_t extra[MMP_MAX_EXTRA]; int32_t n_extra;
    int64_t now_ms; mmp_decision_out out; int32_t rc; bool done;
  };
  std::mutex mu;
  std::condition_variable cv_submit, cv_done;
  std::vector<Req *> queue;
  bool stop = false;
  std::thread worker;
  std::atomic<uint32_t> next_id{1};
  std::atomic<int64_t> batches{0}, decisions{0};
  std::string err;

  void run() {
    std::vector<Req *> batch;
    std::vector<mmp_decision_in> in;
    std::vector<mmp_decision_out> out;
    std::vector<mmp_instance_row> fresh;
    std::vector<int32_t> extra;
    for (;;) {
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_submit.wait(lk, [&] { return stop || !queue.empty(); });
        if (stop && queue.empty()) return;
        if ((int32_t)queue.size() < max_batch && max_wait_us > 0)  // let concurrent callers pile up for one launch
          cv_submit.wait_for(lk, std::chrono::microseconds(max_wait_us), [&] { return stop || (int32_t)queue.size() >= max_batch; });
        batch.swap(queue);
      }
      const int32_t n = (int32_t)batch.size();
      in.resize(n); out.resize(n); fresh.clear(); extra.clear();
      for (int32_t i = 0; i < n; i++) {
        Req &r = *batch[i];
        in[i] = r.in;
        in[i].fresh = -1;
        if (r.has_fresh) { in[i].fresh = (int32_t)fresh.size(); fresh.push_back(r.fresh); }
        in[i].extra_off = (int32_t)extra.size();
        in[i].extra_n = r.n_extra;
        extra.insert(extra.end(), r.extra, r.extra + r.n_extra);
      }
      const int32_t rc = mmp_place_batch(f, in.data(), n, fresh.empty() ? nullptr : fresh.data(), (int32_t)fresh.size(),
                                         extra.empty() ? nullptr : extra.data(), (int32_t)extra.size(), out.data(), batch[0]->now_ms, seed);
      {
        std::lock_guard<std::mutex> lk(mu);
        if (rc < 0) err = mmp_last_error(f);
        for (int32_t i = 0; i < n; i++) { batch[i]->out = out[i]; batch[i]->rc = rc; batch[i]->done = true; }
      }
      cv_done.notify_all();
      batches++; decisions += n;
      batch.clear();
    }
  }
};

extern "C" {
int32_t mmp_batcher_create(mmp_fleet *f, int32_t max_batch, int32_t max_wait_us, uint64_t seed, mmp_batcher **out) {
  NEED(f);
  if (!out || max_batch < 1 || max_wait_us < 0) { g_err = "bad argument"; return MMP_E_ARG; }
  auto *b = new mmp_batcher();
  b->f = f; b->max_batch = max_batch; b->max_wait_us = max_wait_us; b->seed = seed;
  b->worker = std::thread([b] { b->run(); });
  *out = b;
  return MMP_OK;
}
void mmp_batcher_destroy(mmp_batcher *b) {
  if (!b) return;
  { std::lock_guard<std::mutex> lk(b->mu); b->stop = true; }
  b->cv_submit.notify_all();
  if (b->worker.joinable()) b->worker.join();
  delete b;
}
int32_t mmp_place_submit(mmp_batcher *b, const mmp_decision_in *in, const mmp_instance_row *fresh, const int32_t *extra, int64_t now_ms,
                         mmp_decision_out *out, uint32_t *decision_id) {
  if (!b || !in || !out) { g_err = "null argument"; return MMP_E_ARG; }
  if (in->extra_n < 0 || in->extra_n > MMP_MAX_EXTRA || (in->extra_n > 0 && (!extra || in->extra_off < 0))) { g_err = "bad extra slice"; return MMP_E_ARG; }
  mmp_batcher::Req r;
  r.in = *in;
  const uint32_t id = b->next_id.fetch_add(1) & 0xffffffu;
  r.in.flags = (r.in.flags & 0xffu) | MMP_DF_OWN_ID | (id << 8);
  r.has_fresh = fresh != nullptr && in->fresh >= 0;
  if (r.has_fresh) r.fresh = fresh[in->fresh];
  r.n_extra = in->extra_n;
  for (int32_t i = 0; i < r.n_extra; i++) r.extra[i] = extra[in->extra_off + i];
  r.now_ms = now_ms; r.done = false; r.rc = 0;
  {
    std::unique_lock<std::mutex> lk(b->mu);
    if (b->stop) { g_err = "batcher is shut down"; return MMP_E_STATE; }
    b->queue.push_back(&r);
    if ((int32_t)b->queue.size() == 1 || (int32_t)b->queue.size() >= b->max_batch) b->cv_submit.notify_one();
    b->cv_done.wait(lk, [&] { return r.done; });
    if (r.rc < 0) g_err = b->err;
  }
  *out = r.out;
  if (decision_id) *decision_id = id;
  return r.rc;
}
int32_t mmp_batcher_stats(mmp_batcher *b, int64_t *batches, int64_t *decisions) {
  if (!b) { g_err = "null batcher"; return MMP_E_ARG; }
  if (batches) *batches = b->batches.load();
  if (decisions) *decisions = b->decisions.load();
  return MMP_OK;
}
}  // extern "C"

#include "scan_kernels.cuh"
#include "churn_kernels.cuh"
#include "registry_kernels.cuh"

