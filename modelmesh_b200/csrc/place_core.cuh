// place_core.cuh — the placement decision in rank space, written once for two cooperative shapes:
//   * Coop32: one 32-lane warp per decision on sm_90a.  The decision's exclusion-bitmap row has been staged in shared
//     memory by a TMA bulk copy; the row is visited in windows of 32 consecutive words, one word per lane (1 024 ranks
//     per step), reductions are REDUX / SHFL / VOTE.
//   * Coop1: a single "lane", window = one word; compiled by g++ into the CPU-only test harness (tests/emul) so the
//     bitmask formulation can be checked against the oracle without a GPU.  It is NOT part of the shipped library.
//
// What is computed (reference: CacheMissForwardingLB.getNext, ModelMesh.java:4776-5004; quirk labels N1.. are those of
// SURVEY.md §8a / oracle/mm_oracle.cpp):
//   F      = cand[type] & ~excl[model] & ~extra (& ~replicaset-excluded, retried without if empty)   MM:4760-4805
//   best   = first set bit of F  (= argmin under PLACEMENT_ORDER, ranks are assigned at commit)       MM:4806
//   non-simple (a)/(b) preferred-instance handling as first-set / range queries                        MM:4822-4887
//   cut    = first rank in S whose walk test fails (MM:4913-4928, literal N2 semantics)               MM:4901-4937
//   shortlist = {best} ∪ (S below cut); rpm filter (MM:4957-4980); hash-indexed pick (MM:4981-4986, N4)
//
// The routine is written to be issue-efficient on the GPU: PLACEMENT_ORDER puts the answers near the front of the
// order and near `best`, so every query ("first member", "first violator", "how many below the cut", "k-th survivor")
// is a window scan that normally ends in its first window (~20 warp instructions), and single-rank questions ("is self
// in the filtered set?") are answered in O(1) from the staged row.  No per-lane copy of the row is kept in registers.
#pragma once
#include <stdint.h>

#include "../../include/mmplace.h"

#if defined(__CUDACC__)
#define MMP_HD __host__ __device__ __forceinline__
#define MMP_D __device__ __forceinline__
#else
#define MMP_HD inline
#endif

namespace mmp {

static constexpr uint32_t NONE_RANK = 0x7fffffffu;
static constexpr int32_t TARGET_INVALID = -3;  // malformed decision (bad model/self index or no fresh row for a non-live self; MMP_TARGET_INVALID)

struct RankRow {  // one per PLACEMENT_ORDER rank, 32 bytes
  int64_t lru;    // published lruTime (IR:37)
  int64_t rem;    // getRemaining() (IR:203-205)
  int32_t count;  // IR:39
  int32_t rpm;    // IR:51
  int32_t idx;    // instance index
  uint32_t flags; // bit0: isFull(rem)
};
// one 32-byte row as two 128-bit loads (device arrays are 256-byte aligned)
MMP_HD RankRow load_row(const RankRow *p) {
#if defined(__CUDA_ARCH__)
  const int4 a = __ldg(reinterpret_cast<const int4 *>(p)), b = __ldg(reinterpret_cast<const int4 *>(p) + 1);
  RankRow r;
  r.lru = (int64_t)(((uint64_t)(uint32_t)a.y << 32) | (uint32_t)a.x);
  r.rem = (int64_t)(((uint64_t)(uint32_t)a.w << 32) | (uint32_t)a.z);
  r.count = b.x; r.rpm = b.y; r.idx = b.z; r.flags = (uint32_t)b.w;
  return r;
#else
  return *p;
#endif
}
MMP_HD RankRow load_row_any(const RankRow *p) {  // generic address space (shared or global)
#if defined(__CUDA_ARCH__)
  const int4 a = reinterpret_cast<const int4 *>(p)[0], b = reinterpret_cast<const int4 *>(p)[1];
  RankRow r;
  r.lru = (int64_t)(((uint64_t)(uint32_t)a.y << 32) | (uint32_t)a.x);
  r.rem = (int64_t)(((uint64_t)(uint32_t)a.w << 32) | (uint32_t)a.z);
  r.count = b.x; r.rpm = b.y; r.idx = b.z; r.flags = (uint32_t)b.w;
  return r;
#else
  return *p;
#endif
}
struct WordSumI { int32_t lo, hi; };  // min/max count over the 32 ranks of a bitmap word
struct WordSumL { int64_t lo, hi; };  // min/max lruTime
struct FreshRow { int64_t lru, rem; int32_t count, rpm; };  // getFreshInstanceRecord() (MM:5369-5386), what the walk reads of it
// What k_place_split reads of a decision's model: one 16-byte entry per model, built at commit beside excl_ranks
// (make_split_key) and fixed for the epoch.  last_used: the snapshot's model row's; min_rank: the lowest live rank among
// its inline edges, INT32_MAX for none; slot: slot_key of its type id, SPLIT_KEY_OVF set for a model with overflow ids.
struct alignas(16) SplitKey { int64_t last_used; int32_t min_rank; uint32_t slot; };
static constexpr uint32_t SPLIT_KEY_OVF = 0x80000000u;

struct SnapshotView {  // pointers into HBM (or host vectors in the CPU harness)
  int32_t n_ranks, row_words, n_models, max_instances;
  int32_t any_rs, n_type_ids;
  // instance sharding (SURVEY.md §8e): this process holds words [word_lo, word_hi) of every exclusion row, stored at a
  // stride of excl_stride words; [0, row_words) and row_words when the fleet is not sharded
  int32_t word_lo, word_hi, excl_stride, n_slots;
  int32_t n_extra, pad_;       // PER CALL (set by the entry point, not by commit): number of entries in the call's extra[] table
  int64_t min_space;
  const uint32_t *excl;        // [n_models][excl_stride] loaded ∪ failed, bit = rank (word 0 of a stored row = row word word_lo)
  const int32_t *excl_ranks;   // [n_models][4] the ranks whose bits excl's row holds (see RowRanks); unsharded fleets only, else null
  const uint32_t *cand;        // [n_slots][row_words]  allowed(type) ∧ active
  const uint32_t *candx;       // [n_slots][row_words]  cand ∧ ¬(likely-replaced replicaset members)  (MM:4769-4770)
  const uint32_t *pref;        // [n_slots][row_words]
  const uint8_t *has_pref;     // [n_slots]
  const uint16_t *type_slot;   // [n_type_ids] mask slot | has_pref << 15
  const uint32_t *full;        // [row_words] isFull(remaining) (MM:4640-4642)
  const RankRow *rows;         // [n_ranks]
  const int32_t *rank_of;      // [max_instances]
  const WordSumI *csum;        // [row_words]
  const WordSumL *lsum;        // [row_words]
  const int32_t *count_col;    // [row_words*32] count by rank, 0 past the last rank (exact evaluation of a mixed word)
  const int32_t *cand_before;  // [n_slots] members of candx at ranks below word_lo*32 (instance-sharded; all 0 otherwise)
  const uint16_t *nzw;         // [n_slots][row_words] compressed word lists (see LaneTables), entries past nz_n[slot] unused
  const int32_t *nz_n;         // [n_slots]
  const mmp_model_row *models; // [n_models]
  const uint32_t *zero_row;    // [excl_stride] all zero: the exclusion row of an MMP_DF_REQUEST_MODEL decision; null on
                               // instance-sharded fleets, where such a decision is malformed
  const SplitKey *split_key;   // [n_models] what k_place_split reads of a model; unsharded fleets only (as excl_ranks), else null
};

// ---- where a decision's model comes from.  Unflagged: the committed registry (models[d.model], its exclusion row).
// MMP_DF_REQUEST_MODEL: the record the caller read for this request -- d.model is its type id, its loaded ∪ failed instances
// travel in extra[] -- so no registry state is read and the exclusion row is the all-zero one. ----
MMP_HD bool request_model(const mmp_decision_in &d) { return (d.flags & MMP_DF_REQUEST_MODEL) != 0; }
// the exclusion row a decision reads, as an int that lanes can exchange: its model's row (index clamped: a malformed
// decision is answered MMP_TARGET_INVALID, its row is fetched but never used) or ZERO_ROW
static constexpr int32_t ZERO_ROW = -3;
MMP_HD int32_t excl_row_id(const SnapshotView &s, int32_t model, uint32_t flags) {
  if ((flags & MMP_DF_REQUEST_MODEL) && s.zero_row) return ZERO_ROW;
  return (model >= 0 && model < s.n_models) ? model : 0;
}
MMP_HD const uint32_t *excl_row(const SnapshotView &s, int32_t id) {
  return id == ZERO_ROW ? s.zero_row : s.excl + (size_t)id * (size_t)s.excl_stride;
}

// ---- PLACEMENT_ORDER (MM:4646-4703) on numeric columns + dense string ranks.  Host: merge sort at a structural commit
// (host_state.hpp); device: rank = number of live instances that compare less (k_rank_count, the fast commit path). ----
struct OrderKey {
  int64_t vers, rem, lru, cap;
  int32_t count, free_threads, lip, rpm;
  uint32_t id_rank, loc_rank, zone_rank, labels_rank;
  bool full, shutting_down;
};
// literal restatement of MM:4646-4703 on OrderKey (shutting-down records never reach here, MM:1462-1464)
MMP_HD int compare_keys(const OrderKey &a, const OrderKey &b, int64_t churn2) {
  if (a.shutting_down != b.shutting_down) return a.shutting_down ? 1 : -1;
  if (a.vers != b.vers) {
    if (a.vers > b.vers) { if (!a.full || a.lru > churn2) return -1; }
    else if (!b.full || b.lru > churn2) return 1;
  }
  if (a.full != b.full) return a.full ? 1 : -1;
  if (a.full && a.lru != b.lru) return a.lru < b.lru ? -1 : 1;
  if (a.count != b.count) return a.count < b.count ? -1 : 1;  // counts validated to [0,1e9]: the int subtraction cannot wrap
  if (a.rem != b.rem) return a.rem > b.rem ? -1 : 1;
  if (!a.full && a.lru != b.lru) return a.lru < b.lru ? -1 : 1;
  if (a.free_threads != b.free_threads) return a.free_threads > b.free_threads ? -1 : 1;
  if (a.lip != b.lip) return a.lip < b.lip ? -1 : 1;
  if (a.cap != b.cap) return a.cap > b.cap ? -1 : 1;
  if (a.rpm != b.rpm) return a.rpm < b.rpm ? -1 : 1;
  if (a.id_rank != b.id_rank) return a.id_rank < b.id_rank ? -1 : 1;
  if (a.loc_rank != b.loc_rank) return a.loc_rank < b.loc_rank ? -1 : 1;
  if (a.zone_rank != b.zone_rank) return a.zone_rank < b.zone_rank ? -1 : 1;
  if (a.labels_rank != b.labels_rank) return a.labels_rank < b.labels_rank ? -1 : 1;
  return 0;
}

// ---- Java-semantics helpers (wrapping arithmetic, truncating division, saturating double->int) ----
MMP_HD int64_t jsub(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
MMP_HD int32_t jaddi(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
MMP_HD int32_t jmuli(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
MMP_HD int64_t age_of(int64_t t, int64_t now) { return t == 0 ? 0 : jsub(now, t); }  // MM:4162-4164
MMP_HD int32_t jd2i(double d) {
  if (d != d) return 0;
  if (d >= 2147483647.0) return 2147483647;
  if (d <= -2147483648.0) return (int32_t)0x80000000;
  return (int32_t)d;
}
MMP_HD double jmul_d(double a, double b) {
#if defined(__CUDA_ARCH__)
  return __dmul_rn(a, b);  // a plain IEEE multiply, never contracted
#else
  volatile double r = a * b;
  return r;
#endif
}
MMP_HD uint64_t hash64(uint64_t seed, uint64_t decision_id) {  // replaces ThreadLocalRandom (N4); same as the oracle's
  uint64_t z = seed + 0x9E3779B97F4A7C15ULL * (decision_id + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}
// index in [0, n) from the hash: multiply-shift on the high 32 bits (cheap on the GPU; the contract of N4)
MMP_HD uint32_t hash_index(uint64_t seed, uint64_t decision_id, uint32_t n) {
  return (uint32_t)(((hash64(seed, decision_id) >> 32) * (uint64_t)n) >> 32);
}
MMP_HD int ffs32(uint32_t x) {  // index of lowest set bit, x != 0
#if defined(__CUDA_ARCH__)
  return __ffs((int)x) - 1;
#else
  return __builtin_ctz(x);
#endif
}
MMP_HD int popc32(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return __popc(x);
#else
  return __builtin_popcount(x);
#endif
}
// position of the (n+1)-th set bit of w (n < popc(w))
MMP_HD int nth_bit(uint32_t w, uint32_t n) {  // halving search on popcounts (the __fns intrinsic is ~50 instructions)
  int pos = 0;
  uint32_t c = (uint32_t)popc32(w & 0xffffu);
  if (n >= c) { n -= c; pos = 16; w >>= 16; }
  c = (uint32_t)popc32(w & 0xffu);
  if (n >= c) { n -= c; pos += 8; w >>= 8; }
  c = (uint32_t)popc32(w & 0xfu);
  if (n >= c) { n -= c; pos += 4; w >>= 4; }
  c = (uint32_t)popc32(w & 0x3u);
  if (n >= c) { n -= c; pos += 2; w >>= 2; }
  if (n >= (w & 1u)) pos += 1;
  return pos;
}
// 0xffffffff << t with t clamped to [0, 32] (32 -> 0).  PTX shl clamps the shift amount, C does not.
MMP_HD uint32_t shl_ones(int32_t t) {
#if defined(__CUDA_ARCH__)
  uint32_t r;
  uint32_t tt = (uint32_t)max(t, 0);
  asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(0xffffffffu), "r"(tt));
  return r;
#else
  return t <= 0 ? 0xffffffffu : (t >= 32 ? 0u : (0xffffffffu << t));
#endif
}
// bits of the word whose first rank is `rank_base` that lie strictly above rank `lo` / strictly below rank `hi`
MMP_HD uint32_t mask_above(uint32_t rank_base, uint32_t lo) { return shl_ones((int32_t)lo - (int32_t)rank_base + 1); }
MMP_HD uint32_t mask_below(uint32_t rank_base, uint32_t hi) { return ~shl_ones((int32_t)hi - (int32_t)rank_base); }

// ---- the single-lane cooperative shape (CPU harness).  Scans step one word at a time (L = 1); the fast path's
// window values are arrays of WN words (WN = 32 or 16, the two tile widths the GPU kernel uses). ----
template <int WN_>
struct CoopHost {
  static constexpr uint32_t L = 1;
  static constexpr uint32_t WN = WN_;
  MMP_HD uint32_t lane() const { return 0; }
  MMP_HD uint32_t rmin(uint32_t x) const { return x; }
  MMP_HD uint32_t rsum(uint32_t x) const { return x; }
  MMP_HD int32_t rmin_i(int32_t x) const { return x; }
  MMP_HD bool rany(bool p) const { return p; }
  MMP_HD uint32_t exscan(uint32_t) const { return 0; }
  MMP_HD uint32_t shfl(uint32_t x, uint32_t) const { return x; }
  MMP_HD bool spend() const { return true; }    // scan budget (CoopLane only): one unit per row word visited
  MMP_HD bool bailed() const { return false; }
  template <class F> MMP_HD uint32_t eval_word(uint32_t wi, int32_t n_ranks, F &&f) const {
    uint32_t m = 0;
    for (int b = 0; b < 32; b++) {
      uint32_t r = wi * 32 + b;
      if ((int32_t)r < n_ranks && f(r)) m |= 1u << b;
    }
    return m;
  }
  // members of xm (a subset of word wi) for which f holds; only the lowest such bit is guaranteed to be reported
  template <class F> MMP_HD uint32_t eval_members(uint32_t wi, uint32_t xm, int32_t n_ranks, F &&f) const {
    return eval_word(wi, n_ranks, f) & xm;
  }
  // ---- window values (the GPU keeps one word per lane of the tile; here the WN words are an array) ----
  struct W { uint32_t v[WN_]; };
  template <class F> MMP_HD W wmap(uint32_t w0, uint32_t nw, F &&f) const {  // word wi = w0 + i, zero past the row
    W r;
    for (uint32_t i = 0; i < WN; i++) r.v[i] = (w0 + i < nw) ? f(w0 + i) : 0u;
    return r;
  }
  template <class F> MMP_HD W wmap1(uint32_t w0, const W &a, F &&f) const {
    W r;
    for (uint32_t i = 0; i < WN; i++) r.v[i] = f(w0 + i, a.v[i]);
    return r;
  }
  template <class F> MMP_HD W wmap2(uint32_t w0, const W &a, const W &b, F &&f) const {
    W r;
    for (uint32_t i = 0; i < WN; i++) r.v[i] = f(w0 + i, a.v[i], b.v[i]);
    return r;
  }
  MMP_HD uint32_t wfirst(uint32_t w0, const W &x) const {  // rank of the first set bit in the window
    for (uint32_t i = 0; i < WN; i++) if (x.v[i]) return (w0 + i) * 32u + (uint32_t)ffs32(x.v[i]);
    return NONE_RANK;
  }
  template <class F> MMP_HD uint32_t wmin(uint32_t w0, const W &x, F &&f) const {  // min over words of f(wi, word)
    uint32_t m = 0xffffffffu;
    for (uint32_t i = 0; i < WN; i++) { uint32_t t = f(w0 + i, x.v[i]); if (t < m) m = t; }
    return m;
  }
  MMP_HD uint32_t wpopc(const W &x) const { uint32_t c = 0; for (uint32_t i = 0; i < WN; i++) c += (uint32_t)popc32(x.v[i]); return c; }
  MMP_HD uint32_t wget(uint32_t w0, const W &x, uint32_t wi) const { return x.v[wi - w0]; }
  MMP_HD uint32_t wselect(uint32_t w0, const W &x, uint32_t kth) const {  // rank of the kth set bit; kth < wpopc(x)
    for (uint32_t i = 0; i < WN; i++) {
      uint32_t c = (uint32_t)popc32(x.v[i]);
      if (kth < c) return (w0 + i) * 32u + (uint32_t)nth_bit(x.v[i], kth);
      kth -= c;
    }
    return NONE_RANK;
  }
};
typedef CoopHost<32> Coop1;

// ---- one decision per GPU lane (k_place_lanes): the single-lane shape with a budget on the row words a decision may
// visit.  PLACEMENT_ORDER puts best and the shortlist at the front of the order, so almost every decision ends inside
// its first few words; a lane whose walk runs long gives up (bailed()) so that it does not hold up the other 31
// decisions of its warp, and that decision is redone cooperatively by the whole warp (Coop32).  Also compiled by g++
// into the CPU harness, which checks it against the oracle. ----
struct CoopLane {
  static constexpr uint32_t L = 1;
  mutable int32_t budget;
  MMP_HD explicit CoopLane(int32_t words) : budget(words) {}
  MMP_HD uint32_t lane() const { return 0; }
  MMP_HD uint32_t rmin(uint32_t x) const { return x; }
  MMP_HD uint32_t rsum(uint32_t x) const { return x; }
  MMP_HD int32_t rmin_i(int32_t x) const { return x; }
  MMP_HD bool rany(bool p) const { return p; }
  MMP_HD uint32_t exscan(uint32_t) const { return 0; }
  MMP_HD uint32_t shfl(uint32_t x, uint32_t) const { return x; }
  MMP_HD bool spend() const { return --budget >= 0; }
  MMP_HD bool bailed() const { return budget < 0; }
  template <class F> MMP_HD uint32_t eval_members(uint32_t wi, uint32_t xm, int32_t n_ranks, F &&f) const {
    while (xm) {  // ascending; the first hit is all the callers need
      const int b = ffs32(xm);
      const uint32_t r = wi * 32u + (uint32_t)b;
      if ((int32_t)r < n_ranks && f(r)) return 1u << b;
      xm &= xm - 1;
    }
    return 0u;
  }
  template <class F> MMP_HD uint32_t eval_word(uint32_t wi, int32_t n_ranks, F &&f) const { return eval_members(wi, 0xffffffffu, n_ranks, f); }
};

#if defined(__CUDACC__)
// ---- the cooperative shape on the GPU: a tile of T lanes (T = 32: one decision per warp; T = 16: two decisions per
// warp, each half-warp with its own 16-word window).  A window is T consecutive words of the row, one per lane. ----
template <int T>
struct CoopTile {
  static constexpr uint32_t L = T;
  static constexpr uint32_t WN = T;
  uint32_t lane_;  // lane within the tile
  uint32_t mask_;  // member mask of the tile
  uint32_t base_;  // first warp lane of the tile
  MMP_D CoopTile() {
    const uint32_t wl = threadIdx.x & 31;
    lane_ = wl & (T - 1);
    base_ = wl & ~(uint32_t)(T - 1);
    mask_ = T == 32 ? 0xffffffffu : (((1u << T) - 1u) << base_);
  }
  MMP_D uint32_t lane() const { return lane_; }
  MMP_D uint32_t rmin(uint32_t x) const { return __reduce_min_sync(mask_, x); }
  MMP_D uint32_t rsum(uint32_t x) const { return __reduce_add_sync(mask_, x); }
  MMP_D int32_t rmin_i(int32_t x) const { return __reduce_min_sync(mask_, x); }
  MMP_D bool rany(bool p) const { return (__ballot_sync(mask_, p) & mask_) != 0; }
  MMP_D uint32_t shfl(uint32_t x, uint32_t src) const { return __shfl_sync(mask_, x, (int)src, T); }
  MMP_D uint32_t exscan(uint32_t x) const {
    uint32_t v = x;
#pragma unroll
    for (int o = 1; o < T; o <<= 1) {
      uint32_t t = __shfl_up_sync(mask_, v, o, T);
      if (lane_ >= (uint32_t)o) v += t;
    }
    return v - x;
  }
  MMP_D bool spend() const { return true; }
  MMP_D bool bailed() const { return false; }
  template <class F> MMP_D uint32_t eval_members(uint32_t wi, uint32_t xm, int32_t n_ranks, F &&f) const {
    return eval_word(wi, n_ranks, f) & xm;
  }
  // exact 32-rank evaluation of one word by the tile (T = 16: two ranks per lane)
  template <class F> MMP_D uint32_t eval_word(uint32_t wi, int32_t n_ranks, F &&f) const {
    uint32_t m = 0;
#pragma unroll
    for (int h = 0; h < 32 / T; h++) {
      const uint32_t r = wi * 32 + h * T + lane_;
      const bool p = (int32_t)r < n_ranks && f(r);
      m |= ((__ballot_sync(mask_, p) >> base_) & (T == 32 ? 0xffffffffu : ((1u << T) - 1u))) << (h * T);
    }
    return m;
  }
  // ---- window values: one word per lane, in a register ----
  typedef uint32_t W;
  template <class F> MMP_D W wmap(uint32_t w0, uint32_t nw, F &&f) const { uint32_t wi = w0 + lane_; return wi < nw ? f(wi) : 0u; }
  template <class F> MMP_D W wmap1(uint32_t w0, W a, F &&f) const { return f(w0 + lane_, a); }
  template <class F> MMP_D W wmap2(uint32_t w0, W a, W b, F &&f) const { return f(w0 + lane_, a, b); }
  MMP_D uint32_t wfirst(uint32_t w0, W x) const { return rmin(x ? (w0 + lane_) * 32u + (uint32_t)ffs32(x) : NONE_RANK); }
  template <class F> MMP_D uint32_t wmin(uint32_t w0, W x, F &&f) const { return rmin(f(w0 + lane_, x)); }
  MMP_D uint32_t wpopc(W x) const { return rsum((uint32_t)popc32(x)); }
  MMP_D uint32_t wget(uint32_t w0, W x, uint32_t wi) const { return __shfl_sync(mask_, x, (int)(wi - w0), T); }
  MMP_D uint32_t wselect(uint32_t w0, W x, uint32_t kth) const {
    const uint32_t c = (uint32_t)popc32(x), pre = exscan(c);
    return rmin((kth >= pre && kth < pre + c) ? (w0 + lane_) * 32u + (uint32_t)nth_bit(x, kth - pre) : NONE_RANK);
  }
};
typedef CoopTile<32> Coop32;
#endif

// ---- window scans.  A row is visited C::L words at a time starting at the word that holds the lower bound; `word(wi)`
// returns word wi of the set being queried (range masks included).  Answers are almost always inside the first window
// (the shortlist is a short prefix after best), so a query costs one window: ~20 warp instructions, not a row pass. ----
template <class C, class W>
MMP_HD uint32_t scan_first(const C &co, uint32_t from_word, uint32_t end_word, W &&word) {
  for (uint32_t wb = from_word; wb < end_word; wb += C::L) {
    if (!co.spend()) break;
    const uint32_t wi = wb + co.lane();
    const uint32_t x = wi < end_word ? word(wi) : 0u;
    const uint32_t r = co.rmin(x ? wi * 32u + (uint32_t)ffs32(x) : NONE_RANK);
    if (r != NONE_RANK) return r;
  }
  return NONE_RANK;
}
// First rank whose per-rank predicate holds.  `cls(wi)` classifies a 32-rank word from its min/max summary: 0 = no rank
// violates, 1 = every rank violates, 2 = mixed; `eval(rank)` is the exact per-rank test.  Mixed words are resolved in
// ascending order by a cooperative 32-rank evaluation; the scan stops at the first hit.
template <class C, class W, class CLS, class EV>
MMP_HD uint32_t scan_first_violator(const C &co, uint32_t from_word, uint32_t end_word, int32_t n_ranks, W &&word, CLS &&cls, EV &&eval) {
  for (uint32_t wb = from_word; wb < end_word; wb += C::L) {
    if (!co.spend()) break;
    const uint32_t wi = wb + co.lane();
    const uint32_t x = wi < end_word ? word(wi) : 0u;
    uint32_t A = NONE_RANK, M = NONE_RANK;
    if (x) {
      const int c = cls(wi);
      if (c == 1) A = wi * 32u + (uint32_t)ffs32(x);
      else if (c == 2) M = wi;
    }
    uint32_t Amin = co.rmin(A), Mmin = co.rmin(M);
    while (Mmin != NONE_RANK && Mmin * 32u < Amin) {
      const uint32_t xm = co.shfl(x, Mmin - wb);
      const uint32_t vm = co.eval_members(Mmin, xm, n_ranks, eval);
      if (vm) { const uint32_t r = Mmin * 32u + (uint32_t)ffs32(vm); if (r < Amin) Amin = r; break; }
      if (M == Mmin) M = NONE_RANK;
      Mmin = co.rmin(M);
    }
    if (Amin != NONE_RANK) return Amin;
  }
  return NONE_RANK;
}
template <class C, class W>
MMP_HD uint32_t scan_count(const C &co, uint32_t from_word, uint32_t end_word, W &&word) {
  uint32_t mine = 0;
  for (uint32_t wb = from_word; wb < end_word; wb += C::L) {
    if (!co.spend()) break;
    const uint32_t wi = wb + co.lane();
    if (wi < end_word) mine += (uint32_t)popc32(word(wi));
  }
  return co.rsum(mine);
}
// rank of the kth (0-based) set bit in ascending rank order
template <class C, class W>
MMP_HD uint32_t scan_select(const C &co, uint32_t from_word, uint32_t end_word, W &&word, uint32_t kth) {
  for (uint32_t wb = from_word; wb < end_word; wb += C::L) {
    if (!co.spend()) break;
    const uint32_t wi = wb + co.lane();
    const uint32_t x = wi < end_word ? word(wi) : 0u;
    const uint32_t c = (uint32_t)popc32(x), tot = co.rsum(c);
    if (kth < tot) {
      const uint32_t pre = co.exscan(c);
      return co.rmin((kth >= pre && kth < pre + c) ? wi * 32u + (uint32_t)nth_bit(x, kth - pre) : NONE_RANK);
    }
    kth -= tot;
  }
  return NONE_RANK;
}

#define MMP_TF_FAST 256  // trace flag (not part of the ABI): resolved by the one-window fast path
#define MMP_TF_BAIL 512  // internal: a CoopLane walk ran out of budget; the result is void, redo cooperatively
#define MMP_TF_OPEN 1024 // instance-sharded: the walk ran off the end of this shard's rank range (unresolved here)

struct DecideOut {
  int32_t target, n_candidates;
  int32_t best, n_remaining, pick_index, flags, cut_rank, best_rank;
  int32_t first_rank;  // rank of the first filtered entry (before preferred handling): the min-loc key of a shard
  // decide_stream: every rank its answer depends on lies below reach (NONE_RANK: any rank may), so an exclusion or a self
  // at or beyond it leaves the answer as it is (k_slot_summary)
  int32_t reach;
};

// ---- instance-sharded combine (SURVEY.md §8e).  Every shard resolves the decision over its own rank range as if its
// first filtered entry were the global one and publishes ONE 64-bit key; the minimum over shards is the answer of the
// shard that holds the globally first entry (min-loc under PLACEMENT_ORDER), provided its walk stayed inside its range.
//   63      replicaset filter dropped (MM:4798-4802): any shard with a surviving entry under the filter sorts first
//   62..46  first_rank (0x1ffff = no entry in this shard)
//   45      open: the walk needs ranks beyond this shard (resolved by the row-gather pass)
//   44..27  target + 3        26..9  n_candidates        8..0  shard rank (diagnostics)
MMP_HD uint64_t shard_key(const DecideOut &o, int shard_rank) {
  if (o.target == TARGET_INVALID) return ((uint64_t)0 << 46) | ((uint64_t)(TARGET_INVALID + 3) << 27) | (uint64_t)(shard_rank & 511);
  if (o.first_rank < 0) return ~(uint64_t)0;
  const bool open = (o.flags & MMP_TF_OPEN) != 0;
  return ((uint64_t)((o.flags & MMP_TF_RS_RETRY) ? 1 : 0) << 63) | ((uint64_t)((uint32_t)o.first_rank & 0x1ffffu) << 46) |
         ((uint64_t)(open ? 1 : 0) << 45) | ((uint64_t)(uint32_t)((open ? MMP_TARGET_NONE : o.target) + 3) << 27) |
         ((uint64_t)(uint32_t)(open ? 0 : o.n_candidates) << 9) | (uint64_t)(shard_rank & 511);
}
MMP_HD bool shard_key_open(uint64_t k) { return k != ~(uint64_t)0 && ((k >> 45) & 1u) != 0; }
MMP_HD void shard_key_decode(uint64_t k, int32_t &target, int32_t &n_candidates) {
  if (k == ~(uint64_t)0) { target = MMP_TARGET_NONE; n_candidates = 0; return; }
  target = (int32_t)((k >> 27) & 0x3ffffu) - 3;
  n_candidates = (int32_t)((k >> 9) & 0x3ffffu);
}

// rpm-filter predicate of MM:4966-4974 for one recorded rpm
struct RpmFilter {
  int64_t ago;
  int32_t min_load, m11, m15;
  MMP_HD void init(int32_t min_rpm, int64_t last_used_ago) {
    ago = last_used_ago;
    min_load = min_rpm > 100 ? min_rpm : 100;                       // Math.max(100, instReqLoad.min())
    if (ago < 5000) {  // the 1.1x / 1.5x thresholds are only consulted for a model used in the last five seconds
      m11 = jd2i(jmul_d(1.1, (double)min_load));
      m15 = jd2i(jmul_d(1.5, (double)min_load));
    } else m11 = m15 = 2147483647;
  }
  MMP_HD bool drop(int32_t rpm) const {
    return rpm >= 100 && ((ago < -1000 && rpm > m11) || (ago < 5000 && rpm > m15) ||
                          (ago < 720000 && rpm > jmuli(min_load, 3)) || (ago < 86400000 && rpm > jmuli(min_load, 4)));
  }
};

// The end of a simple-case decision once its shortlist is known (MM:4957-4986): the rpm filter over best, the other
// members (N2: they all read the caller's record, other_rpm) and self (self_rpm), then the hash-indexed pick.  n_in =
// members of the shortlist besides best, self included when self_in_sl.  kind: the pick is best, self, or member kth of
// the shortlist in rank order (self left out when !keep_self).
enum { PICK_BEST = 0, PICK_SELF = 1, PICK_MEMBER = 2 };
struct PickOut { int32_t remaining; uint32_t index, kth; bool keep_best, keep_others, keep_self; int kind; };
MMP_HD PickOut pick_survivor(int32_t n_in, bool self_in_sl, int32_t best_rpm, int32_t other_rpm, int32_t self_rpm, int64_t last_used,
                             int64_t now, uint64_t seed, uint64_t decision_id) {
  PickOut p;
  p.keep_best = p.keep_others = p.keep_self = true; p.index = 0; p.kind = PICK_BEST;
  const int32_t n_others = n_in - (self_in_sl ? 1 : 0);
  const int32_t ccount = 1 + n_in;
  p.remaining = ccount;
  if (ccount > 1) {
    const int64_t ago = age_of(last_used, now);
    if (ago < 432000000LL) {  // FIVE_DAYS_MS
      int32_t mn = best_rpm;
      if (n_others > 0 && other_rpm < mn) mn = other_rpm;
      if (self_in_sl && self_rpm < mn) mn = self_rpm;
      RpmFilter rf; rf.init(mn, ago);
      p.keep_best = !rf.drop(best_rpm); p.keep_others = !rf.drop(other_rpm); p.keep_self = !rf.drop(self_rpm);
      p.remaining = (p.keep_best ? 1 : 0) + (p.keep_others ? n_others : 0) + ((self_in_sl && p.keep_self) ? 1 : 0);
    }
    p.index = p.remaining == 1 ? 0u : hash_index(seed, decision_id, (uint32_t)p.remaining);
  }
  p.kth = p.index;
  if (!(p.keep_best && p.kth == 0)) {
    if (p.keep_best) p.kth--;
    p.kind = p.keep_others ? PICK_MEMBER : PICK_SELF;  // without the others the only other survivor can be the self candidate
  }
  return p;
}
// what the caller is told about the instance the pick chose
MMP_HD int32_t target_of(int32_t cidx, const mmp_decision_in &d) {
  return (!(d.flags & MMP_DF_FAVOUR_SELF) && cidx == d.self) ? MMP_TARGET_SELF : cidx;
}

// Everything about one decision that does not need its bitmap row (72 bytes).  k_place lets lane j prepare the
// context of decision j of a 32-decision batch (the dependent gathers overlap across lanes) and stages it in shared memory.
struct DecisionCtx {
  mmp_decision_in d;
  int64_t last_used;
  FreshRow fr;         // the caller's fresh record (MM:5369), or its published row with rpm 0 (N7)
  int32_t self_rank;
  int32_t slot;        // type-constraint mask slot | (has_pref << 16); -1 = malformed decision, -2 = absent
  uint32_t self_bits;  // bit 0: self is in the slot's candidate mask (replicaset filter applied); bit 1: in its preferred mask
  int32_t self_count;  // published count of self (IR:39)
  int32_t xr[4];       // ranks of the first (up to 4) extra excludes, -1 = none / not live: all the lane routine needs of extra[]
};
static constexpr int LANE_MAX_EXTRA = 4;  // decisions with more extra excludes go to the cooperative general routine
MMP_HD int ctx_slot(const DecisionCtx &c) { return c.slot & 0xffff; }
// the id the hash-indexed pick (N4, MM:4981) is drawn with: the decision's position in the batch (+ id_base), or its own
// 24-bit id when the caller numbers its decisions itself (MMP_DF_OWN_ID: coalesced single decisions of many threads)
MMP_HD uint64_t pick_id(const mmp_decision_in &d, uint64_t positional) {
  return (d.flags & MMP_DF_OWN_ID) ? (uint64_t)(d.flags >> 8) : positional;
}
MMP_HD bool ctx_has_pref(const DecisionCtx &c) { return (c.slot >> 16) & 1; }

// The context is gathered in two steps so that a kernel can issue the first (two independent gathers that depend only on
// the decision record: the model row from HBM, rank_of[self]) a whole step ahead of the second (what depends on them).
struct CtxA { mmp_model_row mr; int32_t self_rank; int32_t ok; };
// whether a decision is well formed, from its record alone (no load): everything else is answered MMP_TARGET_INVALID
MMP_HD int32_t decision_ok(const SnapshotView &s, const mmp_decision_in &d) {
  // a request-model decision names a type id (mmp_type_id: [0, 65535)); its last_used can only come from the decision, and
  // only a fleet with the zero row (unsharded) takes it
  const bool req = request_model(d);
  int32_t ok = !(d.self < 0 || d.self >= s.max_instances);
  if (req ? (d.model < 0 || d.model >= 65535 || (d.flags & MMP_DF_MODEL_LAST_USED) || !s.zero_row) : (d.model < 0 || d.model >= s.n_models)) ok = 0;
  // the decision's slice of extra[] must lie inside the table the caller passed (at most 16 entries, MMP_MAX_EXTRA):
  // anything else is a malformed decision (MMP_TARGET_INVALID), never an out-of-bounds read
  if (d.extra_n < 0 || d.extra_n > 16 || (d.extra_n > 0 && (d.extra_off < 0 || (int64_t)d.extra_off + d.extra_n > (int64_t)s.n_extra))) ok = 0;
  return ok;
}
MMP_HD void prepare_ctx_a(const SnapshotView &s, const mmp_decision_in &d, CtxA &a) {
  const bool req = request_model(d);
  a.ok = decision_ok(s, d);
  a.self_rank = -1;
  a.mr.last_used = 0; a.mr.size_units = 0; a.mr.rpm = 0; a.mr.type_id = 0; a.mr.copy_count = 0; a.mr.fail_count = 0; a.mr.reserved = 0;
  if (a.ok && req) {
    a.mr.type_id = (uint16_t)d.model;  // (a type id past the snapshot's n_type_ids resolves as 0 in prepare_ctx_b, as a row's would)
#if defined(__CUDA_ARCH__)
    a.self_rank = __ldg(s.rank_of + d.self);
#else
    a.self_rank = s.rank_of[d.self];
#endif
  } else if (a.ok) {
#if defined(__CUDA_ARCH__)
    // the 24-byte model row is read once per decision: keep it out of L1, where the lane routine's tables live
    const int2 *mp = reinterpret_cast<const int2 *>(s.models + d.model);
    int2 v0, v1, v2;
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0,%1}, [%2];" : "=r"(v0.x), "=r"(v0.y) : "l"(mp));
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0,%1}, [%2];" : "=r"(v1.x), "=r"(v1.y) : "l"(mp + 1));
    asm volatile("ld.global.nc.L1::no_allocate.v2.s32 {%0,%1}, [%2];" : "=r"(v2.x), "=r"(v2.y) : "l"(mp + 2));
    a.mr.last_used = (int64_t)(((uint64_t)(uint32_t)v0.y << 32) | (uint32_t)v0.x);
    a.mr.size_units = v1.x; a.mr.rpm = v1.y;
    a.mr.type_id = (uint16_t)((uint32_t)v2.x & 0xffffu); a.mr.copy_count = (uint8_t)(((uint32_t)v2.x >> 16) & 0xffu);
    a.mr.fail_count = (uint8_t)((uint32_t)v2.x >> 24); a.mr.reserved = (uint32_t)v2.y;
    a.self_rank = __ldg(s.rank_of + d.self);
#else
    a.mr = s.models[d.model]; a.self_rank = s.rank_of[d.self];
#endif
  }
}
// the mask slot of a type id, resolved as prepare_ctx_b resolves it (an id the snapshot does not know is type 0): the key a
// slot-ordered batch is sorted by (prepare_ctx_b reads the whole type_slot entry, has_pref included)
MMP_HD uint32_t slot_key_of(const uint16_t *type_slot, int32_t n_type_ids, int32_t type_id) {
  return (uint32_t)type_slot[(type_id >= 0 && type_id < n_type_ids) ? type_id : 0] & 0x7fffu;
}
MMP_HD uint32_t slot_key(const SnapshotView &s, int32_t type_id) { return slot_key_of(s.type_slot, s.n_type_ids, type_id); }
// a model's SplitKey from its snapshot row and the epoch ranks of its inline edges (-1: none, or not live), overflow bit
// clear (k_build_bitmap; k_build_bitmap_ovf sets it)
MMP_HD SplitKey make_split_key(const mmp_model_row &mr, const int32_t rs[4], const uint16_t *type_slot, int32_t n_type_ids) {
  SplitKey k;
  k.last_used = mr.last_used;
  k.min_rank = INT32_MAX;
  for (int j = 0; j < 4; j++) if (rs[j] >= 0 && rs[j] < k.min_rank) k.min_rank = rs[j];
  k.slot = slot_key_of(type_slot, n_type_ids, mr.type_id);
  return k;
}
MMP_HD SplitKey load_split_key(const SplitKey *p) {  // read once per decision: kept out of L1 like the decision record
#if defined(__CUDA_ARCH__)
  int4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  SplitKey k;
  k.last_used = (int64_t)(((uint64_t)(uint32_t)v.y << 32) | (uint32_t)v.x);
  k.min_rank = v.z; k.slot = (uint32_t)v.w;
  return k;
#else
  return *p;
#endif
}
MMP_HD void prepare_ctx_b(const SnapshotView &s, const mmp_decision_in &d, const CtxA &a, const FreshRow *fresh_tab, int32_t n_fresh,
                          const int32_t *extra, DecisionCtx &c) {
  c.d = d; c.slot = -1; c.self_rank = -1; c.last_used = 0; c.self_bits = 0; c.self_count = 0;
  c.xr[0] = c.xr[1] = c.xr[2] = c.xr[3] = -1;
  c.fr.lru = 0; c.fr.rem = 0; c.fr.count = 0; c.fr.rpm = 0;
  if (!a.ok) return;
  const int tid = a.mr.type_id < s.n_type_ids ? a.mr.type_id : 0;
  c.last_used = (d.flags & MMP_DF_MODEL_LAST_USED) ? a.mr.last_used : d.last_used;
  c.self_rank = a.self_rank;
  const uint32_t ts = s.type_slot[tid];  // slot | has_pref << 15
  if (d.fresh >= 0 && d.fresh < n_fresh) c.fr = fresh_tab[d.fresh];
  else if (c.self_rank >= 0) { const RankRow sr = load_row(s.rows + c.self_rank); c.fr.lru = sr.lru; c.fr.rem = sr.rem; c.fr.count = sr.count; c.fr.rpm = 0; }
  else return;
  const int sl = (int)(ts & 0x7fffu);
  c.slot = sl | ((int)(ts >> 15) << 16);
  if (c.self_rank >= 0) {  // what the walk asks about self, gathered here so that it is not a dependent load inside the walk
    const size_t so = (size_t)sl * (size_t)s.row_words + ((uint32_t)c.self_rank >> 5);
    const uint32_t sh = (uint32_t)c.self_rank & 31u;
    c.self_bits = (((s.any_rs ? s.candx : s.cand)[so] >> sh) & 1u) | (((s.pref[so] >> sh) & 1u) << 1);
    c.self_count = s.count_col[c.self_rank];
  }
  if (d.extra_n > 0 && d.extra_n <= LANE_MAX_EXTRA) {  // (the slice was bounds-checked by prepare_ctx_a)
    for (int e = 0; e < LANE_MAX_EXTRA; e++)
      if (e < d.extra_n) { const int32_t x = extra[d.extra_off + e]; c.xr[e] = (x >= 0 && x < s.max_instances) ? s.rank_of[x] : -1; }
  }
}
MMP_HD void prepare_ctx(const SnapshotView &s, const mmp_decision_in &d, const FreshRow *fresh_tab, int32_t n_fresh,
                        const int32_t *extra, DecisionCtx &c) {
  CtxA a;
  prepare_ctx_a(s, d, a);
  prepare_ctx_b(s, d, a, fresh_tab, n_fresh, extra, c);
}

#define MMP_BAIL_CHECK do { if (co.bailed()) { o.flags |= MMP_TF_BAIL; o.target = MMP_TARGET_NONE; return; } } while (0)

// The common case of getNext resolved inside ONE window of C::WN words (32 words = 1 024 ranks for a warp-wide tile,
// 16 words for a half-warp tile) whose words stay in registers: best, the non-simple (a) probe, the cut, the shortlist
// count and the pick are all window reductions.  Returns false -- nothing written -- whenever the answer is not
// provably inside the window or the decision takes a path handled only by the general routine (extra excludes,
// replicaset retry, best full); the caller then runs decide_ctx.  Same semantics, same quirks; the tests compare both
// against the oracle.  TRACE = false skips the outputs only the trace needs.
template <bool TRACE, class C>
MMP_HD bool decide_fast(const SnapshotView &s, const DecisionCtx &c, const uint32_t *erow, int64_t now, uint64_t seed,
                        uint64_t decision_id, const C &co, DecideOut &o) {
  typedef typename C::W W;
  if (c.slot < 0 || c.d.extra_n != 0) return false;
  const uint32_t NW = (uint32_t)s.row_words;
  const mmp_decision_in &d = c.d;
  const uint32_t so = (uint32_t)ctx_slot(c) * NW;
  const uint32_t *CX = (s.any_rs ? s.candx : s.cand) + so;
  const uint32_t *P = s.pref + so;
  const bool favour_self = (d.flags & MMP_DF_FAVOUR_SELF) != 0;
  const int32_t self_rank = c.self_rank;
  uint32_t w0 = 0;
  W fw = co.wmap(w0, NW, [&](uint32_t wi) { return CX[wi] & ~erow[wi]; });
  const uint32_t b = co.wfirst(w0, fw);
  if (b == NONE_RANK) return false;  // deeper in the row, or empty (replicaset retry): general routine
  o.first_rank = (int32_t)b;
  if ((b >> 5) >= C::WN / 2) {       // re-centre so that the window starts at best's word
    w0 = b >> 5;
    fw = co.wmap(w0, NW, [&](uint32_t wi) { return CX[wi] & ~erow[wi]; });
  }
  const uint32_t wend = (w0 + C::WN < NW ? w0 + C::WN : NW) * 32u;  // ranks below wend are inside the window
  const bool to_row_end = w0 + C::WN >= NW;
  const RankRow rb = s.rows[b];
  bool us = rb.idx == d.self;
  const FreshRow fr = c.fr;
  int64_t best_rem = us ? fr.rem : rb.rem;
  int32_t best_count = us ? fr.count : rb.count, best_rpm = us ? fr.rpm : rb.rpm, best_idx = rb.idx;
  uint32_t best_rank = b;
  if (best_rem < s.min_space) return false;  // best full: general routine
  const bool has_pref = ctx_has_pref(c);
  W pw = co.wmap(w0, NW, [&](uint32_t wi) { return has_pref ? P[wi] : 0u; });
  bool simple = !has_pref || ((co.wget(w0, pw, b >> 5) >> (b & 31)) & 1u);
  uint32_t lo = b, hi = NONE_RANK;
  bool use_pref = has_pref && simple;
  if (!simple) {
    // non-simple (a) MM:4828-4852: the first later entry that is preferred or full decides: preferred -> new best
    // (even when it is also full, the preference test comes first), full and not preferred -> the replay stops there
    const W u = co.wmap2(w0, fw, pw, [&](uint32_t wi, uint32_t f, uint32_t p) { return f & mask_above(wi * 32u, b) & (p | s.full[wi]); });
    const uint32_t r1 = co.wfirst(w0, u);
    if (r1 == NONE_RANK) { if (!to_row_end) return false; }
    else if ((co.wget(w0, pw, r1 >> 5) >> (r1 & 31)) & 1u) {
      const RankRow rp = s.rows[r1];
      best_rank = r1; best_idx = rp.idx; best_rem = rp.rem; best_count = rp.count; best_rpm = rp.rpm;
      us = rp.idx == d.self;
      lo = r1; use_pref = true;
    } else hi = r1;
  }
  if (us && favour_self) {
    o.target = MMP_TARGET_SELF; o.n_candidates = 0;
    if (TRACE) { o.best = best_idx; o.best_rank = (int32_t)best_rank; o.n_remaining = 0; o.pick_index = 0;
                 o.flags = MMP_TF_SIMPLE | MMP_TF_FAST | MMP_TF_FAVOUR_EXIT; o.cut_rank = (int32_t)NONE_RANK; }
    return true;
  }
  // S inside the window
  const W sx = co.wmap2(w0, fw, pw, [&](uint32_t wi, uint32_t f, uint32_t p) {
    uint32_t m = f & mask_above(wi * 32u, lo) & mask_below(wi * 32u, hi);
    return use_pref ? (m & p) : m;
  });
  const bool s_in_window = hi != NONE_RANK ? hi <= wend : to_row_end;  // does the window hold all of S?
  const uint32_t sw_ = self_rank >= 0 ? (uint32_t)self_rank >> 5 : 0xffffffffu, sb_ = 1u << (self_rank & 31);
  bool self_in_s = false;
  if (self_rank >= 0 && (uint32_t)self_rank > lo && (uint32_t)self_rank < hi)
    self_in_s = (CX[sw_] & ~erow[sw_] & sb_) != 0 && (!use_pref || (P[sw_] & sb_) != 0);
  const int64_t q = best_rem >> 2;
  const bool c_self = fr.rem < s.min_space || fr.rem < q;
  bool self_viol = rb.rem < s.min_space || rb.rem < q;
  const int32_t thr = jaddi(best_count, best_count >> 2);
  auto cv = [&](int32_t cnt) { return cnt >= 10 && cnt > thr; };
  if (self_in_s && cv(s.rows[self_rank].count)) self_viol = true;
  uint32_t cut_others;
  if (c_self) {
    cut_others = co.wfirst(w0, co.wmap1(w0, sx, [&](uint32_t wi, uint32_t x) { return (self_in_s && wi == sw_) ? (x & ~sb_) : x; }));
  } else {
    // One key per word: (rank of its first member << 1) | mixed, for words whose count summary admits a violator.
    // The minimum key is the earliest word that can hold the cut: class 1 -> that member is the cut; mixed -> evaluate
    // the word's 32 ranks exactly, and on a miss drop the word and look again.
    W pend = co.wmap1(w0, sx, [&](uint32_t wi, uint32_t x) -> uint32_t {
      if (!x) return 0xffffffffu;
      const WordSumI m = s.csum[wi];
      if (!cv(m.hi)) return 0xffffffffu;
      return ((wi * 32u + (uint32_t)ffs32(x)) << 1) | (cv(m.lo) ? 0u : 1u);
    });
    cut_others = NONE_RANK;
    for (;;) {
      const uint32_t key = co.wmin(w0, pend, [](uint32_t, uint32_t k) { return k; });
      if (key == 0xffffffffu) break;
      if (!(key & 1u)) { cut_others = key >> 1; break; }
      const uint32_t mw = key >> 6;  // word index of the mixed word
      const uint32_t vm = co.eval_word(mw, s.n_ranks, [&](uint32_t r) { return cv(s.rows[r].count); }) & co.wget(w0, sx, mw);
      if (vm) { cut_others = mw * 32u + (uint32_t)ffs32(vm); break; }
      pend = co.wmap1(w0, pend, [&](uint32_t wi, uint32_t k) { return wi == mw ? 0xffffffffu : k; });
    }
  }
  const uint32_t cut_self = (self_in_s && self_viol) ? (uint32_t)self_rank : NONE_RANK;
  const uint32_t cut = cut_others < cut_self ? cut_others : cut_self;
  if (cut == NONE_RANK ? !s_in_window : cut > wend) return false;  // the walk continues past the window
  if (cut_others == NONE_RANK && !s_in_window) return false;       // an earlier violator may sit between wend and cut_self
  const bool self_in_sl = self_in_s && (uint32_t)self_rank < cut;
  if (favour_self && self_in_sl) {
    o.target = MMP_TARGET_SELF; o.n_candidates = 0;
    if (TRACE) { o.best = best_idx; o.best_rank = (int32_t)best_rank; o.n_remaining = 0; o.pick_index = 0;
                 o.flags = MMP_TF_SIMPLE | MMP_TF_FAST | MMP_TF_FAVOUR_EXIT; o.cut_rank = (int32_t)cut; }
    return true;
  }
  const W sl = co.wmap1(w0, sx, [&](uint32_t wi, uint32_t x) { return x & mask_below(wi * 32u, cut); });
  const int32_t n_in = (int32_t)co.wpopc(sl);
  const int32_t n_others = n_in - (self_in_sl ? 1 : 0);
  const int32_t ccount = 1 + n_in;
  bool keep_best = true, keep_others = true, keep_self = true;
  int32_t remaining = ccount;
  uint32_t index = 0;
  if (ccount > 1) {
    const int64_t ago = age_of(c.last_used, now);
    if (ago < 432000000LL) {
      int32_t mn = best_rpm;
      if (n_others > 0 && fr.rpm < mn) mn = fr.rpm;
      if (self_in_sl && rb.rpm < mn) mn = rb.rpm;
      RpmFilter rf; rf.init(mn, ago);
      keep_best = !rf.drop(best_rpm); keep_others = !rf.drop(fr.rpm); keep_self = !rf.drop(rb.rpm);
      remaining = (keep_best ? 1 : 0) + (keep_others ? n_others : 0) + ((self_in_sl && keep_self) ? 1 : 0);
    }
    index = remaining == 1 ? 0u : hash_index(seed, decision_id, (uint32_t)remaining);
  }
  uint32_t chosen_rank;
  uint32_t kth = index;
  if (keep_best && kth == 0) chosen_rank = best_rank;
  else {
    if (keep_best) kth--;
    if (!keep_others) chosen_rank = (uint32_t)self_rank;
    else {
      const bool drop_self = self_in_sl && !keep_self;
      chosen_rank = co.wselect(w0, co.wmap1(w0, sl, [&](uint32_t wi, uint32_t x) { return (drop_self && wi == sw_) ? (x & ~sb_) : x; }), kth);
    }
  }
  const int32_t cidx = chosen_rank == best_rank ? best_idx : s.rows[chosen_rank].idx;
  o.target = (!favour_self && cidx == d.self) ? MMP_TARGET_SELF : cidx;
  o.n_candidates = ccount;
  if (TRACE) {
    o.best = best_idx; o.best_rank = (int32_t)best_rank; o.n_remaining = remaining; o.pick_index = (int32_t)index;
    o.flags = MMP_TF_SIMPLE | MMP_TF_FAST | (keep_best ? MMP_TF_KEEP_BEST : 0) | (keep_others ? MMP_TF_KEEP_OTHERS : 0) |
              (keep_self ? MMP_TF_KEEP_SELF : 0);
    o.cut_rank = (int32_t)cut;
  }
  return true;
}

// What a lane of k_place_lanes reads besides its exclusion row: the snapshot's own tables (global memory: small, L1/L2
// resident) and, per type-constraint slot, the COMPRESSED WORD LIST nzw[slot][k] = index of the k-th row word in which the
// slot's candidate mask has any bit (within this process's word range).  A word without candidates contributes nothing to
// the filtered set F = cand & ~excl, so every walk of decide_stream steps through the list instead of through the row:
// on dense masks (C3: the list is 0, 1, 2, ...) nothing changes, on sparse ones (C5: a handful of candidates per type among
// 10 000 instances) a walk that crossed 50-300 empty words becomes a few steps.
// row words of a decision's window in k_place_lanes (shared with the commit path: nz_skip is computed for this width)
#define MMP_LANE_WIN 12
// decide_stream's per-lane slice of shared memory: the chunk of 8 steps beyond the window (21 words), then phase B's
// checkpoints for phase C, MMP_LANE_WIN / 2 words of u16 window counts (27: odd, a conflict-free lane stride)
#define MMP_CHUNK_WORDS 27
typedef uint16_t mark16 __attribute__((may_alias));  // (the window counts are u16s in a slice of u32 words)
struct LaneTables {
  const uint32_t *cx, *p;   // this decision's candidate (replicaset filter applied) and preferred mask rows, by absolute row word
  const uint32_t *full;
  const WordSumI *csum;
  const int32_t *count_col;
  const RankRow *rows;
  const uint16_t *nzw;      // [nz_n] ascending row-word indices with cx[w] != 0, all in [word_lo, word_hi)
  uint32_t nz_n;
  uint32_t nz_skip;         // list entries that lie inside the caller's window (k_place_lanes: entries < word_lo + MMP_LANE_WIN)
};
// SnapshotView::nz_n packs both: entries in the low 24 bits, nz_skip above
MMP_HD uint32_t nz_count(int32_t packed) { return (uint32_t)packed & 0xffffffu; }
MMP_HD uint32_t nz_skipped(int32_t packed) { return (uint32_t)packed >> 24; }
MMP_HD LaneTables lane_tables_global(const SnapshotView &s, int slot) {
  LaneTables t;
  const size_t so = (size_t)slot * (size_t)s.row_words;
  t.cx = (s.any_rs ? s.candx : s.cand) + so; t.p = s.pref + so; t.full = s.full; t.csum = s.csum; t.count_col = s.count_col;
  t.rows = s.rows;
  t.nzw = s.nzw + so; t.nz_n = nz_count(s.nz_n[slot]); t.nz_skip = nz_skipped(s.nz_n[slot]);
  return t;
}
// read-only table loads of the lane routine (ld.global.nc on the device)
template <class T> MMP_HD T ldro(const T *p) {
#if defined(__CUDA_ARCH__)
  return __ldg(p);
#else
  return *p;
#endif
}
MMP_HD WordSumI ldro_sum(const WordSumI *p) {
#if defined(__CUDA_ARCH__)
  const int2 v = __ldg(reinterpret_cast<const int2 *>(p));
  return WordSumI{v.x, v.y};
#else
  return *p;
#endif
}

// how the lane routine reads its tables: beyond the window through the read-only path from the snapshot's own arrays
// (TabGlob); inside the window through plain loads (TabWin) where the caller points them at shared-memory copies of the
// tables' window part (k_place_lanes, k_place_server), or through TabGlob too where its window tables are the global ones
struct TabWin {
  const LaneTables &t;
  MMP_HD uint32_t cx(uint32_t wi) const { return t.cx[wi]; }
  MMP_HD uint32_t p(uint32_t wi) const { return t.p[wi]; }
  MMP_HD uint32_t full(uint32_t wi) const { return t.full[wi]; }
  MMP_HD WordSumI csum(uint32_t wi) const { return t.csum[wi]; }
  MMP_HD RankRow row(uint32_t r) const { return load_row_any(t.rows + r); }
  MMP_HD int32_t idx(uint32_t r) const { return t.rows[r].idx; }
  // count test of a whole word against lim: 0 no rank reaches it, 1 every rank does, 2 mixed (look at the 32 counts)
  MMP_HD int cls(uint32_t wi, int32_t lim) const { const WordSumI m = t.csum[wi]; return m.hi < lim ? 0 : (m.lo >= lim ? 1 : 2); }
  MMP_HD uint32_t ge_mask(uint32_t wi, int32_t lim) const {  // bit j: count of rank wi*32 + j >= lim (32 counts, zero-padded past the last rank)
    uint32_t vm = 0;
#if defined(__CUDA_ARCH__)
    const int4 *cc = reinterpret_cast<const int4 *>(t.count_col + (size_t)wi * 32u);
#pragma unroll
    for (int jj = 0; jj < 8; jj++) {
      const int4 qq = cc[jj];
      vm |= ((qq.x >= lim ? 1u : 0u) | (qq.y >= lim ? 2u : 0u) | (qq.z >= lim ? 4u : 0u) | (qq.w >= lim ? 8u : 0u)) << (4 * jj);
    }
#else
    const int32_t *cc = t.count_col + (size_t)wi * 32u;
    for (int jj = 0; jj < 32; jj++) vm |= (cc[jj] >= lim ? 1u : 0u) << jj;
#endif
    return vm;
  }
};
struct TabGlob {
  const LaneTables &t;
  MMP_HD uint32_t cx(uint32_t wi) const { return ldro(t.cx + wi); }
  MMP_HD uint32_t p(uint32_t wi) const { return ldro(t.p + wi); }
  MMP_HD uint32_t full(uint32_t wi) const { return ldro(t.full + wi); }
  MMP_HD WordSumI csum(uint32_t wi) const { return ldro_sum(t.csum + wi); }
  MMP_HD RankRow row(uint32_t r) const { return load_row(t.rows + r); }
  MMP_HD int32_t idx(uint32_t r) const { return ldro(&t.rows[r].idx); }
  MMP_HD int cls(uint32_t wi, int32_t lim) const { const WordSumI m = ldro_sum(t.csum + wi); return m.hi < lim ? 0 : (m.lo >= lim ? 1 : 2); }
  MMP_HD uint32_t ge_mask(uint32_t wi, int32_t lim) const {
    uint32_t vm = 0;
#if defined(__CUDA_ARCH__)
    const int4 *cc = reinterpret_cast<const int4 *>(t.count_col + (size_t)wi * 32u);
#pragma unroll
    for (int jj = 0; jj < 8; jj++) {
      const int4 qq = __ldg(cc + jj);
      vm |= ((qq.x >= lim ? 1u : 0u) | (qq.y >= lim ? 2u : 0u) | (qq.z >= lim ? 4u : 0u) | (qq.w >= lim ? 8u : 0u)) << (4 * jj);
    }
#else
    const int32_t *cc = t.count_col + (size_t)wi * 32u;
    for (int jj = 0; jj < 32; jj++) vm |= (cc[jj] >= lim ? 1u : 0u) << jj;
#endif
    return vm;
  }
};
// a step beyond the window: its filtered word (candidates & ~exclusions), preferred word and count class were gathered
// when the chunk of 8 steps was (re)filled -- one round of independent loads per 8 steps instead of three dependent ones
// per step; the walk bodies see them through the same interface (cx() is the filtered word: they are handed e = 0)
struct TabChunk {
  uint32_t f, pw; int c; const TabGlob &g;
  MMP_HD uint32_t cx(uint32_t) const { return f; }
  MMP_HD uint32_t p(uint32_t) const { return pw; }
  MMP_HD uint32_t full(uint32_t wi) const { return g.full(wi); }
  MMP_HD int cls(uint32_t, int32_t) const { return c; }
  MMP_HD uint32_t ge_mask(uint32_t wi, int32_t lim) const { return g.ge_mask(wi, lim); }
};


// Instance-sharded early-out: an entry of the filtered set in a LOWER shard beats anything this shard can offer
// (min-loc under PLACEMENT_ORDER), and one must exist when the slot has more candidates below this shard's range than
// the decision can exclude (the model's loaded ∪ failed row plus its extra excludes).  models[].reserved = row size.
MMP_HD bool shard_cannot_win(const SnapshotView &s, const DecisionCtx &c, uint32_t n_row_bits) {
  if (s.word_lo == 0 || c.slot < 0) return false;
  return (int64_t)s.cand_before[ctx_slot(c)] > (int64_t)n_row_bits + (int64_t)(c.d.extra_n > 0 ? c.d.extra_n : 0);
}

// ---- how decide_stream reaches the part of a decision's exclusion row that is not in its window ----
// RowPtr: the stored row in this process's memory (word index relative to word_lo); p == nullptr: nothing beyond the window.
struct RowPtr {
  const uint32_t *p; uint32_t ws;
  MMP_HD bool ok() const { return p != nullptr; }
  MMP_HD uint32_t word(uint32_t wi) const { return ldro(p + (wi - ws)); }
};
// RowRanks (unsharded fleets): the row rebuilt in registers from the model's entry of excl_ranks -- the epoch ranks of its
// (at most 4) inline edges, -1 for no edge or an instance that is not live.  A model with overflow ids (more than the inline
// edges hold) has EXCL_RANKS_OVF in r[0] and must be read from its bitmap row instead.  16 bytes per decision, read in
// sweep order, where the row's words sit one 1 280-byte stride apart.
static constexpr int32_t EXCL_RANKS_OVF = -2;
MMP_HD uint32_t rank_bit_in(int32_t r, uint32_t wi) { return ((uint32_t)r >> 5) == wi ? 1u << (r & 31) : 0u; }  // (r < 0: no word)
struct RowRanks {
  int32_t r[4];
  MMP_HD bool ok() const { return true; }
  MMP_HD bool overflow() const { return r[0] == EXCL_RANKS_OVF; }
  MMP_HD uint32_t word(uint32_t wi) const { return rank_bit_in(r[0], wi) | rank_bit_in(r[1], wi) | rank_bit_in(r[2], wi) | rank_bit_in(r[3], wi); }
};
MMP_HD RowRanks load_ranks(const int32_t *p) {  // read once per decision: kept out of L1 like the decision record
  RowRanks k;
#if defined(__CUDA_ARCH__)
  asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(k.r[0]), "=r"(k.r[1]), "=r"(k.r[2]), "=r"(k.r[3]) : "l"(p));
#else
  for (int j = 0; j < 4; j++) k.r[j] = p[j];
#endif
  return k;
}
// RowDealt (instance-sharded fleets with peer access, SURVEY.md §8e): row words [0, front_words) are replicated on every
// shard, word wi beyond them lives in the column block of shard wi / block_words -- this GPU's HBM or a peer's, read through
// its NVLink-mapped pointer.
struct RowDealt {
  const uint32_t *front; const uint32_t *const *blocks; uint32_t front_words, block_words, stride; uint64_t model;
  uint32_t me; mutable uint32_t remote;  // remote = words this lane read from a peer's block (NVLink traffic accounting)
  MMP_HD bool ok() const { return true; }
  MMP_HD uint32_t word(uint32_t wi) const {
    if (wi < front_words) return ldro(front + model * front_words + wi);
    const uint32_t g = wi / block_words;
    if (g != me) remote++;
    return blocks[g][model * stride + (wi - g * block_words)];
  }
};

// ---- vote shapes for decide_stream: 32 decisions in lockstep on the GPU, one on the CPU harness ----
struct SoloVote { MMP_HD bool any(bool p) const { return p; } };
#if defined(__CUDACC__)
struct WarpVote { MMP_D bool any(bool p) const { return __any_sync(0xffffffffu, p) != 0; } };
#endif

// The common case of getNext for ONE DECISION PER LANE (k_place_lanes), written so that the 32 lanes of a warp stay
// converged: every phase is a walk whose loops are left by a warp vote, bodies are predicated on a per-lane state, and the
// scalar work between the walks is straight-line.  Phases:
//   A   first entry of F = cand & ~excl & ~extra (MM:4806)
//   A'  non-simple (a), MM:4828-4852: the first later entry that is preferred or full
//   B   the shortlist walk (MM:4901-4937): first member of S that fails its test; a word whose count summary is
//       "mixed" is evaluated exactly (32 counts) by the lanes that stop on one
//   C   the hash-indexed pick (MM:4981-4986): k-th member of the shortlist
// Every walk runs as two loops.  INSIDE THE WINDOW (steps k < win_words) step k is row word word_lo + k, dense: the word
// comes from the lane's window buffer (ewin[k]: k_place_lanes copies the first MMP_LANE_WIN words of the row out of the
// TMA landing stage when it hands the stage on) and the tables from Tw, which k_place_lanes points at shared-memory copies
// of the tables' window part -- two shared-memory loads per step, no bookkeeping; this is where every decision of a
// C3-like fleet ends.  BEYOND THE WINDOW a walk steps through the slot's compressed word list from its first entry past the
// window (list entry k + koff): the list and the row are read from global memory (row: the row has just been streamed, so
// it is an L2 hit) in chunks of 8 steps held in registers, refilled for all walking lanes at the same iteration (one vote),
// so that a long walk (C5: 100+ steps over sparse candidate masks) pays one L2 round trip per 8 steps; with !row.ok() the
// lane's attempt ends at the window's edge.
// Same semantics and quirks as decide_ctx (N2: the non-self test reads the caller's fresh record).  Returns false --
// and the caller redoes the decision with the cooperative general routine -- for everything outside the common case:
// malformed decision, more than LANE_MAX_EXTRA extra excludes, no entry (replicaset retry), a full best followed by preferred
// entries within its lruTime distance (non-simple (b) with preferred candidates), or
// a walk of more than `budget` steps.  Instance-sharded: a walk that needs ranks beyond this shard's range sets MMP_TF_OPEN.
// self_eword = the row word that holds self's bit (anywhere in the row).  Must be called by every lane of the vote group
// (active = false for lanes without a decision).
// AWT: how the window's tables Tw are read -- TabWin (plain loads: Tw points at shared memory) or TabGlob (Tw is global).
// chunk: the lane's shared-memory slice of MMP_CHUNK_WORDS words; every kernel passes one (only the CPU harness may leave
// it out).
template <class AWT = TabWin, class V, class R>
MMP_HD bool decide_stream(const SnapshotView &s, const LaneTables &Tw, const LaneTables &T, const DecisionCtx &c, bool active,
                          const uint32_t *ewin, uint32_t win_words, const R &row, uint32_t self_eword, int64_t now, uint64_t seed,
                          uint64_t decision_id, const V &vote, DecideOut &o, int32_t budget, uint32_t *chunk = nullptr) {
  o.target = MMP_TARGET_NONE; o.n_candidates = 0; o.best = -1; o.n_remaining = 0; o.pick_index = 0; o.flags = 0;
  o.cut_rank = (int32_t)NONE_RANK; o.best_rank = -1; o.first_rank = -1;
  const uint32_t NW = (uint32_t)s.row_words, WS = (uint32_t)s.word_lo, WE = (uint32_t)s.word_hi;
  const bool open_end = WE < NW;
  bool live = active && c.slot >= 0 && c.d.extra_n <= LANE_MAX_EXTRA;
  const mmp_decision_in &d = c.d;
  // virtual step positions: k < win_words is row word WS + k (window buffer, tables Tw); k >= win_words is list entry
  // k + koff (tables T): the list entries inside the window are skipped, the walk goes on with the first entry beyond it
  const uint32_t kz = win_words == 0 ? 0u : T.nz_skip;  // (the caller's window is the one nz_skip was counted for)
  const uint32_t koff = kz - win_words;                 // (mod 2^32)
  const uint32_t NZ = win_words + (T.nz_n - kz);        // virtual length of the walk
  const AWT AW{Tw};
  const TabGlob AG{T};
  const uint32_t win_end = WS + win_words;
  const bool favour_self = (d.flags & MMP_DF_FAVOUR_SELF) != 0;
  const int32_t self_rank = c.self_rank;
  const FreshRow fr = c.fr;
  int32_t left = budget;
  const bool has_x = d.extra_n > 0;
  auto xmask = [&](uint32_t wi) -> uint32_t {  // bits of word wi taken by the extra excludes
    uint32_t m = 0;
#pragma unroll
    for (int e = 0; e < LANE_MAX_EXTRA; e++) { const int32_t r = c.xr[e]; if (r >= 0 && ((uint32_t)r >> 5) == wi) m |= 1u << (r & 31); }
    return m;
  };
  auto pbit = [&](uint32_t r) -> bool { const uint32_t w = r >> 5; return ((w < win_end ? AW.p(w) : AG.p(w)) >> (r & 31)) & 1u; };
  auto row_of = [&](uint32_t r) -> RankRow { return (r >> 5) < win_end ? AW.row(r) : AG.row(r); };
  // ---- beyond the window: a chunk of 8 consecutive steps [base, base + 8) in registers ----
  uint32_t base = 0xfffffff0u;  // no chunk loaded
  // chunk storage, MMP_CHUNK_WORDS words per lane: [0,4) the list entries (u16 pairs), [4,12) filtered words cx & ~row,
  // [12,20) preferred words, [20] count classes against cls_lim (2 bits each), then phase B's checkpoints (mw below).
  // The caller hands a shared-memory slice (dynamic indexing is one load, and with no other candidate the compiler emits
  // every access to it as a shared-memory one); the CPU harness may leave it out.
#if defined(__CUDA_ARCH__)
  uint32_t *const ch = chunk;
#else
  uint32_t chunk_local[MMP_CHUNK_WORDS];
  uint32_t *const ch = chunk ? chunk : chunk_local;
#endif
  static_assert(MMP_CHUNK_WORDS >= 21 + MMP_LANE_WIN / 2, "slice too short for the checkpoints");
  // mw[k]: members of S' phase B counted before window step k < MMP_LANE_WIN (at most 32 * MMP_LANE_WIN: a u16)
  mark16 *const mw = reinterpret_cast<mark16 *>(ch + 21);
  int32_t cls_lim = 10;                             // the count limit the chunk's classes were computed for (phase B sets it and drops the chunk)
  auto wsel = [&](uint32_t j) -> uint32_t { return (ch[j >> 1] >> ((j & 1u) * 16u)) & 0xffffu; };
  auto refill = [&](uint32_t k) {
    base = k;
#pragma unroll
    for (uint32_t j = 0; j < 4; j++) {
      const uint32_t k0 = k + 2 * j, k1 = k0 + 1;
      const uint32_t lo16 = k0 < NZ ? (uint32_t)ldro(T.nzw + (k0 + koff)) : 0xffffu, hi16 = k1 < NZ ? (uint32_t)ldro(T.nzw + (k1 + koff)) : 0xffffu;
      ch[j] = lo16 | (hi16 << 16);
    }
    uint32_t cq = 0;
#pragma unroll
    for (uint32_t j = 0; j < 8; j++) {
      uint32_t f = 0, pw = 0;
      int cl = 0;
      if (k + j < NZ) {
        const uint32_t wi = wsel(j);
        f = AG.cx(wi) & ~row.word(wi); pw = AG.p(wi); cl = AG.cls(wi, cls_lim);
      }
      ch[4 + j] = f; ch[12 + j] = pw; cq |= (uint32_t)cl << (2u * j);
    }
    ch[20] = cq;
  };
  auto chunk_empty = [&]() -> bool { return (ch[4] | ch[5] | ch[6] | ch[7] | ch[8] | ch[9] | ch[10] | ch[11]) == 0u; };
  // One walk: BODY sees (K, wi, e) and sets go_ (true: next step).  WALKING is cleared when the lane stops: BODY said so, the
  // list ended (ENDED = true), or the budget / the reachable part of the row ran out (live = false).  CHARGE: the steps
  // count against the budget (phase C walks words phase B has paid for).  BULK (beyond the window only): an expression
  // that tries to take a freshly gathered chunk of 8 steps at once -- true: the 8 steps are done (its side effects are theirs).
  // MARK_W: a statement run before a window step's BODY (phase B's checkpoints).
#define MMP_WALK(K, WALKING, ENDED, CHARGE, BULK, MARK_W, BODY)                                                          \
  for (;;) { /* inside the window */                                                                                       \
    if (WALKING && K < win_words) {                                                                                        \
      if (CHARGE && left <= 0) { WALKING = false; live = false; }                                                          \
      else {                                                                                                               \
        const uint32_t wi = WS + K, e = ewin[K];                                                                           \
        const AWT &A = AW;                                                                                                 \
        bool go_;                                                                                                          \
        MARK_W;                                                                                                            \
        BODY;                                                                                                              \
        if (go_) { K++; if (CHARGE) left--; } else WALKING = false;                                                        \
      }                                                                                                                    \
    }                                                                                                                      \
    if (!vote.any(WALKING && K < win_words)) break;                                                                        \
  }                                                                                                                        \
  if (WALKING && K >= NZ) { WALKING = false; ENDED = true; }                                                               \
  if (WALKING && !row.ok()) { WALKING = false; live = false; }                                                              \
  if (vote.any(WALKING)) {                                                                                                 \
    for (;;) { /* beyond the window */                                                                                     \
      { const bool need_ = WALKING && K < NZ && (K - base) >= 8u; if (vote.any(need_)) { if (WALKING && K < NZ) refill(K); } } \
      if (WALKING) {                                                                                                       \
        if (K >= NZ) { WALKING = false; ENDED = true; }                                                                    \
        else if (CHARGE && left <= 0) { WALKING = false; live = false; }                                                   \
        else if (K == base && K + 8u <= NZ && (!CHARGE || left >= 8) && (BULK)) { K += 8u; if (CHARGE) left -= 8; }          \
        else {                                                                                                             \
          const uint32_t j_ = K - base, wi = wsel(j_), e = 0u;                                                              \
          const TabChunk A{ch[4u + j_], ch[12u + j_], (int)((ch[20] >> (2u * j_)) & 3u), AG};                                 \
          bool go_;                                                                                                        \
          BODY;                                                                                                            \
          if (go_) { K++; if (CHARGE) left--; } else WALKING = false;                                                      \
        }                                                                                                                  \
      }                                                                                                                    \
      if (!vote.any(WALKING)) break;                                                                                       \
    }                                                                                                                      \
  }

  // ---- A: first filtered entry ----
  uint32_t b = NONE_RANK, kb = 0;
  {
    uint32_t k = 0;
    bool walking = live, ended = false;
    MMP_WALK(k, walking, ended, true, (!has_x && chunk_empty()), (void)0, {
      uint32_t x = A.cx(wi) & ~e;
      if (has_x) x &= ~xmask(wi);
      if (x) { b = wi * 32u + (uint32_t)ffs32(x); kb = k; }
      go_ = x == 0;
    })
    (void)ended;
  }
  if (b == NONE_RANK) live = false;  // none in reach: the general routine decides (replicaset retry, null)
  RankRow rb; rb.lru = 0; rb.rem = 0; rb.count = 0; rb.rpm = 0; rb.idx = -1; rb.flags = 0;
  bool us = false, simple = true, use_pref = false;
  int64_t best_rem = 0, best_lru = 0;
  bool best_full = false;
  int32_t best_count = 0, best_rpm = 0, best_idx = -1;
  uint32_t best_rank = b, lo = b, hi = NONE_RANK, k_lo = kb;
  // the highest rank a phase's answer rests on (o.reach).  A phase that finds nothing counts for nothing: exclusions only
  // take entries out of F, so it would find nothing with them either.
  uint32_t dep = b;
  if (live) {
    rb = row_of(b);
    us = rb.idx == d.self;
    best_rem = us ? fr.rem : rb.rem; best_count = us ? fr.count : rb.count; best_rpm = us ? fr.rpm : rb.rpm; best_idx = rb.idx;
    best_lru = us ? fr.lru : rb.lru;
    best_full = best_rem < s.min_space;  // MM:4811
    const bool has_pref = ctx_has_pref(c);
    simple = !has_pref || pbit(b);
    use_pref = has_pref && simple;  // best is preferred: preference is treated as required (MM:4905-4907)
  }
  // ---- A': non-simple (a) ----
  uint32_t r1 = NONE_RANK, k1 = kb;
  {
    const uint32_t b_w = b >> 5, m_b = mask_above(b_w * 32u, b);
    uint32_t k = kb;
    bool walking = live && !simple && !best_full, ended = false;
    MMP_WALK(k, walking, ended, true, false, (void)0, {
      uint32_t x = A.cx(wi) & ~e & (A.p(wi) | A.full(wi));
      if (has_x) x &= ~xmask(wi);
      if (wi == b_w) x &= m_b;
      if (x) { r1 = wi * 32u + (uint32_t)ffs32(x); k1 = k; }
      go_ = x == 0;
    })
    (void)ended;
    if (r1 != NONE_RANK && r1 > dep) dep = r1;
  }
  bool open = false;
  // ---- A'': non-simple (b), MM:4853-4887 -- a full best that is not one of its type's preferred instances.  kb = the first
  // later entry whose lruTime is "far" from the best's (more than 2 min and more than a quarter of the best's age; each entry
  // tested on its OWN published lruTime); a preferred entry before kb makes the preferred ones the candidates (the general
  // routine takes those decisions), none means "no preference" logic over the entries before kb ----
  {
    const int64_t a4 = age_of(best_lru, now) / 4;
    auto far = [&](int64_t l) { const int64_t diff = jsub(l, best_lru); return diff > 120000 && diff > a4; };
    const uint32_t b_w = b >> 5, m_b = mask_above(b_w * 32u, b);
    uint32_t k = kb, kb_rank = NONE_RANK;
    bool pref_before = false;
    const bool case_b = live && !simple && best_full;
    bool walking = case_b, ended = false;
    MMP_WALK(k, walking, ended, true, false, (void)0, {
      uint32_t x = A.cx(wi) & ~e;
      if (has_x) x &= ~xmask(wi);
      if (wi == b_w) x &= m_b;
      go_ = true;
      if (x) {
        const int64_t l_lo = ldro(&s.lsum[wi].lo);
        const int64_t l_hi = ldro(&s.lsum[wi].hi);
        uint32_t v = 0;  // the members of x that are far
        if (far(l_hi)) {
          if (far(l_lo)) v = x;
          else for (uint32_t t = x; t; t &= t - 1) { const uint32_t bt = (uint32_t)ffs32(t); if (far(ldro(&T.rows[wi * 32u + bt].lru))) v |= 1u << bt; }
        }
        const uint32_t near_ = v ? (x & mask_below(wi * 32u, wi * 32u + (uint32_t)ffs32(v))) : x;  // members before the first far one
        if (near_ & A.p(wi)) { pref_before = true; go_ = false; }
        else if (v) { kb_rank = wi * 32u + (uint32_t)ffs32(v); go_ = false; }
      }
    })
    if (kb_rank != NONE_RANK && kb_rank > dep) dep = kb_rank;
    if (case_b && live) {
      if (pref_before) live = false;                      // the preferred entries within the distance are the candidates: general routine
      else if (kb_rank == NONE_RANK && open_end) open = true;  // the deciding entry is in a later shard
      else hi = kb_rank;                                  // no preferred one in range: rewind, "no preference" logic (use_pref stays false)
    }
    (void)ended;
  }
  if (live && !simple && !best_full) {
    if (r1 == NONE_RANK) open = open_end;  // else: neither kind follows, "no preference" logic over the whole remainder
    else if (pbit(r1)) {
      const RankRow rp = row_of(r1);
      best_rank = r1; best_idx = rp.idx; best_rem = rp.rem; best_count = rp.count; best_rpm = rp.rpm;
      us = rp.idx == d.self;
      lo = r1; k_lo = k1; use_pref = true;
    } else hi = r1;
  }
  bool done = false;
  int32_t fl = MMP_TF_SIMPLE | MMP_TF_FAST | (best_full ? MMP_TF_BEST_FULL : 0);
  if (live && !open && us && favour_self) { o.target = MMP_TARGET_SELF; fl |= MMP_TF_FAVOUR_EXIT; done = true; }
  // ---- the walk's per-decision constants ----
  bool walk = live && !open && !done;
  bool self_in_s = false, c_self = false, self_viol = false;
  uint32_t sw_ = 0xffffffffu, sb_ = 0;
  int32_t cv_min = 10;  // cv(cnt) = cnt >= 10 && cnt > thr (MM:4924-4927) = cnt >= max(10, thr + 1); thr <= 1.25e9 by the input domain
  auto cv = [&](int32_t cnt) { return cnt >= cv_min; };
  if (walk) {
    if (self_rank >= 0 && (uint32_t)self_rank > lo && (uint32_t)self_rank < hi) {
      const uint32_t w = (uint32_t)self_rank >> 5, bit = 1u << (self_rank & 31);
      // self may sit anywhere in the row: its mask bits were gathered with the context, its row word by the caller
      bool in = w - WS < WE - WS && (c.self_bits & 1u) != 0 && (self_eword & bit) == 0 && (!use_pref || (c.self_bits & 2u) != 0);
      if (in && has_x) in = (xmask(w) & bit) == 0;  // an explicitly excluded self never passes the filter (MM:4780-4781)
      if (in) { self_in_s = true; sw_ = w; sb_ = bit; }
    }
    if (best_full) {  // a full best: the distance test is on lruTime (MM:4862-4866), N2: the caller's record for every non-self member
      const int64_t a10 = age_of(best_lru, now) / 10;
      const int64_t df = jsub(fr.lru, best_lru), ds = jsub(rb.lru, best_lru);
      c_self = df > 45000 && df > a10;
      self_viol = ds > 45000 && ds > a10;
    } else {
      const int64_t q = best_rem >> 2;
      c_self = fr.rem < s.min_space || fr.rem < q;
      self_viol = rb.rem < s.min_space || rb.rem < q;
    }
    const int32_t thr = jaddi(best_count, best_count >> 2);
    cv_min = thr >= 9 ? thr + 1 : 10;
    if (!best_full && self_in_s && cv(c.self_count)) self_viol = true;
  }
  const uint32_t cut_self = (self_in_s && self_viol) ? (uint32_t)self_rank : NONE_RANK;
  // S' = F restricted to (lo, lim), lim = min(hi, cut_self): nothing at or beyond a failing self can be a candidate
  const uint32_t lim = hi < cut_self ? hi : cut_self;
  uint32_t stop_w = WE;
  if (lim != NONE_RANK) { const uint32_t e = (lim + 31u) >> 5; stop_w = e < WE ? e : WE; }
  // a word of S': only the word that holds lo and the one that holds lim are cut (none beyond lim's is ever visited)
  const uint32_t lo_w = lo >> 5, m_lo = mask_above(lo_w * 32u, lo);
  const uint32_t lim_w = lim >> 5, m_lim = mask_below(lim_w * 32u, lim);  // lim == NONE_RANK: lim_w is no real word
  auto Sw = [&](const auto &A, uint32_t wi, uint32_t e) -> uint32_t {
    uint32_t m = A.cx(wi) & ~e;
    if (has_x) m &= ~xmask(wi);
    if (wi == lo_w) m &= m_lo;
    if (wi == lim_w) m &= m_lim;
    return use_pref ? (m & A.p(wi)) : m;
  };
  // a gathered chunk whose 8 words need none of the special masks: strictly between lo's word and lim's, self's word not among them
  auto chunk_plain = [&]() -> bool { const uint32_t w0 = wsel(0), w7 = wsel(7); return w0 > lo_w && w7 < lim_w && (sw_ < w0 || sw_ > w7); };
  auto chunk_members = [&]() -> uint32_t {  // members of S' in such a chunk
    uint32_t n = 0;
#pragma unroll
    for (int j = 0; j < 8; j++) n += (uint32_t)popc32(use_pref ? (ch[4 + j] & ch[12 + j]) : ch[4 + j]);
    return n;
  };
  // ---- B: first member of S' that fails its walk test, counting the members before it ----
  uint32_t cut_others = NONE_RANK, n_in = 0;
  cls_lim = cv_min; base = 0xfffffff0u;  // (a chunk gathered by an earlier phase carries classes for another limit)
  auto bulk_b = [&]() -> bool {  // no member of the chunk can fail: count them all at once
    const uint32_t n = chunk_members();
    if (c_self) return n == 0;                    // (every non-self member fails: only an empty chunk passes)
    if (!best_full && ch[20] != 0u) return false;  // a word whose counts may reach the limit: step by step
    n_in += n;
    return true;
  };
  // checkpoints for phase C: n_in before every window step phase B takes (the first MMP_LANE_WIN)
  uint32_t k_b = k_lo;  // where phase B stopped
  {
    uint32_t k = k_lo;
    bool walking = walk, ended = false;
    MMP_WALK(k, walking, ended, true, (!has_x && chunk_plain() && bulk_b()), if (k < MMP_LANE_WIN) mw[k] = (uint16_t)n_in, {
      go_ = true;
      if (wi >= stop_w) { ended = true; go_ = false; }  // the walk's natural end (everything at or beyond lim)
      else {
        const uint32_t x = Sw(A, wi, e);
        int cls = 0;  // 0: no member fails, 1: every member (but a passing self) fails, 2: look at the counts
        uint32_t v = x;
        if (c_self) { if (wi == sw_) v &= ~sb_; cls = v ? 1 : 0; }
        else if (x && !best_full) cls = A.cls(wi, cv_min);  // (a full best: no count test, the walk runs to the end of S)
        if (cls == 2) {  // exact evaluation of a mixed word: 32 counts, zero-padded past the last rank
          const uint32_t vm = A.ge_mask(wi, cv_min);
          v = vm & x;
          cls = v ? 1 : 0;
        }
        if (cls == 0) n_in += (uint32_t)popc32(x);
        else {
          cut_others = wi * 32u + (uint32_t)ffs32(v);
          n_in += (uint32_t)popc32(x & mask_below(wi * 32u, cut_others));
          go_ = false;
        }
      }
    })
    if (walk && live && ended && cut_others == NONE_RANK && lim == NONE_RANK && open_end) open = true;
    k_b = k;
    if (cut_others != NONE_RANK) { if (cut_others > dep) dep = cut_others; }
    else if (walk && (lim == NONE_RANK || lim > dep)) dep = lim;  // every member of S' below lim counted
  }
  walk = walk && live && !open;
  const uint32_t cut = cut_others < cut_self ? cut_others : cut_self;
  const bool self_in_sl = self_in_s && (uint32_t)self_rank < cut;
  bool keep_best = true, keep_others = true, keep_self = true, sel = false;
  int32_t remaining = 0, ccount = 0;
  uint32_t index = 0, kth = 0, chosen_rank = best_rank;
  if (walk) {
    if (favour_self && self_in_sl) { o.target = MMP_TARGET_SELF; fl |= MMP_TF_FAVOUR_EXIT; done = true; }
    else {
      ccount = 1 + (int32_t)n_in;
      const PickOut pk = pick_survivor((int32_t)n_in, self_in_sl, best_rpm, fr.rpm, rb.rpm, c.last_used, now, seed, decision_id);
      keep_best = pk.keep_best; keep_others = pk.keep_others; keep_self = pk.keep_self;
      remaining = pk.remaining; index = pk.index; kth = pk.kth;
      if (pk.kind == PICK_SELF) chosen_rank = (uint32_t)self_rank;
      else sel = pk.kind == PICK_MEMBER;
    }
  }
  // ---- C: k-th survivor in rank order, walked from the last checkpoint of phase B that lies before it (words phase B
  // has visited: the budget is not charged again) ----
  {
    const bool drop_self = self_in_sl && !keep_self;
    const uint32_t cut_w = cut >> 5, m_cut = mask_below(cut_w * 32u, cut);
    uint32_t k = k_lo;
    if (sel) {
      // phase B counted self (a member of S') where phase C drops it: one fewer before every checkpoint past self's word
      uint32_t n0 = 0;
      const uint32_t mark_end = win_words < MMP_LANE_WIN ? win_words : MMP_LANE_WIN;  // (k_place_lanes: windows up to 20 words)
      if (k_lo < mark_end) {  // the window steps phase B took and counted: [k_lo, min(k_b, mark_end - 1)], counts ascending from 0
        uint32_t hi_k = k_b < mark_end ? k_b : mark_end - 1u;
        while (k < hi_k) {
          const uint32_t mid = (k + hi_k + 1u) >> 1;
          const uint32_t n = (uint32_t)mw[mid] - ((drop_self && sw_ < WS + mid) ? 1u : 0u);
          if (n <= kth) k = mid;
          else hi_k = mid - 1u;
        }
        n0 = (uint32_t)mw[k] - ((drop_self && sw_ < WS + k) ? 1u : 0u);
      }
      kth -= n0;
    }
    bool walking = sel, ended = false;
    auto bulk_c = [&]() -> bool { const uint32_t n = chunk_members(); if (kth < n) return false; kth -= n; return true; };
    MMP_WALK(k, walking, ended, false, (!has_x && chunk_plain() && wsel(7) < cut_w && bulk_c()), (void)0, {
      uint32_t x = Sw(A, wi, e);
      if (wi == cut_w) x &= m_cut;
      if (drop_self && wi == sw_) x &= ~sb_;
      const uint32_t n = (uint32_t)popc32(x);
      go_ = true;
      if (kth < n) { chosen_rank = wi * 32u + (uint32_t)nth_bit(x, kth); go_ = false; }
      else kth -= n;
    })
    if (sel && ended) live = false;  // cannot happen: kth < number of survivors, all in visited words
  }
#undef MMP_WALK
  if (!active) return true;
  if (!live) return false;
  o.first_rank = (int32_t)b;
  o.best = best_idx; o.best_rank = (int32_t)best_rank;
  if (open) { o.flags = MMP_TF_OPEN; return true; }
  if (!done) {
    const int32_t cidx = chosen_rank == best_rank ? best_idx : ((int32_t)chosen_rank == self_rank ? d.self : ((chosen_rank >> 5) < win_end ? AW.idx(chosen_rank) : AG.idx(chosen_rank)));
    o.target = target_of(cidx, d);
    o.n_candidates = ccount;
    o.n_remaining = remaining; o.pick_index = (int32_t)index;
    fl |= (keep_best ? MMP_TF_KEEP_BEST : 0) | (keep_others ? MMP_TF_KEEP_OTHERS : 0) | (keep_self ? MMP_TF_KEEP_SELF : 0);
  }
  o.cut_rank = (int32_t)(walk || (done && cut != NONE_RANK) ? cut : NONE_RANK);
  o.flags = fl;
  o.reach = (int32_t)(dep == NONE_RANK ? NONE_RANK : dep + 1u);
  return true;
}

// One getNext.  erow: this decision's exclusion row, readable by every lane (shared memory on the GPU) until the
// routine returns.  cand_rows (optional, trace): [2][row_words] receives the candidate mask (other than best) and the
// survivor mask.
template <class C>
MMP_HD void decide_ctx(const SnapshotView &s, const DecisionCtx &c, const uint32_t *erow, const int32_t *extra, int64_t now,
                       uint64_t seed, uint64_t decision_id, const C &co, DecideOut &o, uint32_t *cand_rows) {
  o.target = MMP_TARGET_NONE; o.n_candidates = 0; o.best = -1; o.n_remaining = 0; o.pick_index = 0; o.flags = 0;
  o.cut_rank = (int32_t)NONE_RANK; o.best_rank = -1; o.first_rank = -1;
  const uint32_t NW = (uint32_t)s.row_words;
  // this process's part of the row: words [WS, WE); erow[0] is row word WS.  Not sharded: [0, NW).
  const uint32_t WS = (uint32_t)s.word_lo, WE = (uint32_t)s.word_hi;
  const bool open_end = WE < NW;  // ranks from WE*32 on live in another shard
  if (c.slot < 0) { o.target = TARGET_INVALID; return; }
  const mmp_decision_in &d = c.d;
  const int slot = ctx_slot(c);
  const bool favour_self = (d.flags & MMP_DF_FAVOUR_SELF) != 0;
  const int32_t self_rank = c.self_rank;
  const FreshRow fr = c.fr;
  const uint32_t *CAND = s.cand + (size_t)slot * NW;
  const uint32_t *P = s.pref + (size_t)slot * NW;
  const int n_extra = d.extra_n < 16 ? d.extra_n : 16;
  auto end_for = [&](uint32_t hi_rank) -> uint32_t {  // one past the last word that can hold a rank < hi_rank
    if (hi_rank == NONE_RANK) return WE;
    uint32_t e = (hi_rank + 31u) >> 5;
    return e < WE ? e : WE;
  };
  auto emit_rows = [&](auto &&w0f, auto &&w1f) {  // trace only
    for (uint32_t wb = WS; wb < WE; wb += C::L) {
      uint32_t wi = wb + co.lane();
      if (wi < WE) { cand_rows[wi] = w0f(wi); cand_rows[NW + wi] = w1f(wi); }
    }
  };

  // ---- filter (MM:4760-4771): candx already excludes likely-replaced replicaset members ----
  const uint32_t *CX = s.any_rs ? s.candx + (size_t)slot * NW : CAND;
  // word wi of the filtered set F
  auto Fw = [&](uint32_t wi) -> uint32_t {  // wi in [WS, WE)
    uint32_t m = CX[wi] & ~erow[wi - WS];
    for (int e = 0; e < n_extra; e++) {
      int32_t x = extra[d.extra_off + e];
      if (x >= 0 && x < s.max_instances) { int32_t r = s.rank_of[x]; if (r >= 0 && (uint32_t)(r >> 5) == wi) m &= ~(1u << (r & 31)); }
    }
    return m;
  };
  uint32_t b = scan_first(co, WS, WE, Fw);
  MMP_BAIL_CHECK;
  if (b == NONE_RANK && s.any_rs) {
    // MM:4798-4802: nothing survives; run the filter again without the replicaset exclusion
    o.flags |= MMP_TF_RS_RETRY;
    CX = CAND;
    b = scan_first(co, WS, WE, Fw);
    MMP_BAIL_CHECK;
  }
  if (b == NONE_RANK) return;  // null
  // a rank outside this shard's range reads as "not in the filtered set": it can only be asked about self, and self
  // matters to a walk only below the cut, i.e. inside the range whenever the walk is resolved here
  auto in_filter = [&](uint32_t r) -> bool { return ((r >> 5) - WS) < (WE - WS) && ((Fw(r >> 5) >> (r & 31)) & 1u); };
  auto pref_bit = [&](uint32_t r) -> bool { return (P[r >> 5] >> (r & 31)) & 1u; };

  const RankRow rb = s.rows[b];  // bestEntry.getValue()
  bool us = rb.idx == d.self;    // excluded self never passes the filter, so !excludeSelf is implied
  int64_t best_rem = us ? fr.rem : rb.rem, best_lru = us ? fr.lru : rb.lru;
  int32_t best_count = us ? fr.count : rb.count, best_rpm = us ? fr.rpm : rb.rpm, best_idx = rb.idx;
  uint32_t best_rank = b;
  const bool best_full = best_rem < s.min_space;
  if (best_full) o.flags |= MMP_TF_BEST_FULL;
  const bool has_pref = ctx_has_pref(c);
  bool simple = !has_pref || pref_bit(b);
  uint32_t lo = b, hi = NONE_RANK;
  bool use_pref = has_pref && simple;  // best is preferred: preference is treated as required (MM:4905-4907)
  o.best = best_idx; o.best_rank = (int32_t)b; o.first_rank = (int32_t)b;
#define MMP_OPEN_EXIT do { o.flags |= MMP_TF_OPEN; o.target = MMP_TARGET_NONE; o.n_candidates = 0; return; } while (0)

  if (!simple) {
    if (!best_full) {
      // non-simple (a) MM:4828-4852: first later entry that is preferred, unless a full one comes first.
      // One fused scan: stop at the first window that holds either.
      uint32_t p1 = NONE_RANK, f1 = NONE_RANK;
      for (uint32_t wb = b >> 5; wb < WE; wb += C::L) {
        if (!co.spend()) break;
        const uint32_t wi = wb + co.lane();
        uint32_t xp = 0, xf = 0;
        if (wi < WE) {
          const uint32_t x = Fw(wi) & mask_above(wi * 32u, b), pw = P[wi];
          xp = x & pw; xf = x & s.full[wi] & ~pw;
        }
        p1 = co.rmin(xp ? wi * 32u + (uint32_t)ffs32(xp) : NONE_RANK);
        f1 = co.rmin(xf ? wi * 32u + (uint32_t)ffs32(xf) : NONE_RANK);
        if (p1 != NONE_RANK || f1 != NONE_RANK) break;
      }
      MMP_BAIL_CHECK;
      if (open_end && p1 == NONE_RANK && f1 == NONE_RANK) MMP_OPEN_EXIT;  // the deciding entry is in a later shard
      if (p1 < f1) {
        const RankRow rp = s.rows[p1];
        best_rank = p1; best_idx = rp.idx; best_rem = rp.rem; best_lru = rp.lru; best_count = rp.count; best_rpm = rp.rpm;
        us = rp.idx == d.self;
        lo = p1; use_pref = true;
        o.best = best_idx; o.best_rank = (int32_t)p1;
      } else hi = f1;
      simple = true;
    } else {
      // non-simple (b) MM:4853-4887
      const int64_t oldest = best_lru, a4 = age_of(oldest, now) / 4;
      auto viol = [&](int64_t l) { int64_t diff = jsub(l, oldest); return diff > 120000 && diff > a4; };
      const uint32_t kb = scan_first_violator(co, b >> 5, WE, s.n_ranks,
          [&](uint32_t wi) { return Fw(wi) & mask_above(wi * 32u, b); },
          [&](uint32_t wi) { WordSumL m = s.lsum[wi]; return !viol(m.hi) ? 0 : (viol(m.lo) ? 1 : 2); },
          [&](uint32_t r) { return viol(s.rows[r].lru); });
      MMP_BAIL_CHECK;
      if (open_end && kb == NONE_RANK) MMP_OPEN_EXIT;
      const uint32_t endb = end_for(kb);
      auto Cw = [&](uint32_t wi) { return Fw(wi) & P[wi] & mask_above(wi * 32u, b) & mask_below(wi * 32u, kb); };
      const uint32_t firstp = scan_first(co, b >> 5, endb, Cw);
      MMP_BAIL_CHECK;
      if (firstp != NONE_RANK) {
        // only preferred instances within the age distance are candidates; each records its own published rpm
        o.flags |= MMP_TF_PREF_B;
        const bool self_in = self_rank >= 0 && (uint32_t)self_rank > b && (uint32_t)self_rank < kb && pref_bit((uint32_t)self_rank) &&
                             in_filter((uint32_t)self_rank);
        if (self_in && favour_self) {  // N8: returns null
          o.flags |= MMP_TF_FAVOUR_EXIT;
          if (cand_rows) emit_rows(Cw, [](uint32_t) { return 0u; });
          return;
        }
        const int32_t ccount = (int32_t)scan_count(co, firstp >> 5, endb, Cw);
        MMP_BAIL_CHECK;
        o.n_candidates = ccount;
        uint32_t chosen;
        if (ccount == 1) {
          chosen = firstp; o.n_remaining = 1;
          if (cand_rows) emit_rows(Cw, Cw);
        } else {
          int32_t remaining = ccount;
          const int64_t ago = age_of(c.last_used, now);
          const bool filter = ago < 432000000LL;
          RpmFilter rf;
          rf.init(100, ago);
          if (filter) {
            int32_t mn = 2147483647;
            for (uint32_t wb = firstp >> 5; wb < endb; wb += C::L) {
              if (!co.spend()) break;
              const uint32_t wi = wb + co.lane();
              uint32_t w = wi < endb ? Cw(wi) : 0u;
              while (w) { int bt = ffs32(w); w &= w - 1; int32_t v = s.rows[wi * 32 + bt].rpm; if (v < mn) mn = v; }
            }
            rf.init(co.rmin_i(mn), ago);
          }
          auto Kw = [&](uint32_t wi) {  // candidates that survive the rpm filter
            uint32_t w = Cw(wi), keep = w;
            if (filter) while (w) { int bt = ffs32(w); w &= w - 1; if (rf.drop(s.rows[wi * 32 + bt].rpm)) keep &= ~(1u << bt); }
            return keep;
          };
          if (filter) remaining = (int32_t)scan_count(co, firstp >> 5, endb, Kw);
          uint32_t index = remaining == 1 ? 0u : hash_index(seed, decision_id, (uint32_t)remaining);
          chosen = scan_select(co, firstp >> 5, endb, Kw, index);
          MMP_BAIL_CHECK;
          o.n_remaining = remaining; o.pick_index = (int32_t)index;
          if (cand_rows) emit_rows(Cw, Kw);
        }
        int32_t cidx = s.rows[chosen].idx;
        o.target = (!favour_self && cidx == d.self) ? MMP_TARGET_SELF : cidx;
        return;
      }
      hi = kb; simple = true;  // no preferred in range: rewind, "no preference" logic over the replayed prefix
    }
  }
  // ---- simple case MM:4889-4938 ----
  o.flags |= MMP_TF_SIMPLE;
  if (us && favour_self) { o.flags |= MMP_TF_FAVOUR_EXIT; o.target = MMP_TARGET_SELF; return; }
  // S = F restricted to ranks in (lo, hi) and, when preference is binding, to preferred instances
  const uint32_t from = lo >> 5, end = end_for(hi);
  auto Sw = [&](uint32_t wi) -> uint32_t {
    uint32_t m = Fw(wi) & mask_above(wi * 32u, lo) & mask_below(wi * 32u, hi);
    if (use_pref) m &= P[wi];
    return m;
  };
  const bool self_in_s = self_rank >= 0 && (uint32_t)self_rank > lo && (uint32_t)self_rank < hi &&
                         (!use_pref || pref_bit((uint32_t)self_rank)) && in_filter((uint32_t)self_rank);
  const int64_t oldest = best_lru;
  bool c_self, self_viol;
  uint32_t cut_others = NONE_RANK;
  // the non-self walk test reads the caller's fresh record (N2), so it is one constant per decision
  if (best_full) {
    const int64_t a10 = age_of(oldest, now) / 10;
    int64_t df = jsub(fr.lru, oldest), ds = jsub(rb.lru, oldest);
    c_self = df > 45000 && df > a10;
    self_viol = ds > 45000 && ds > a10;
  } else {
    const int64_t q = best_rem >> 2;
    c_self = fr.rem < s.min_space || fr.rem < q;
    self_viol = rb.rem < s.min_space || rb.rem < q;
  }
  const int32_t thr = jaddi(best_count, best_count >> 2);
  auto cv = [&](int32_t cnt) { return cnt >= 10 && cnt > thr; };  // MM:4924-4927, always on the candidate's own count
  if (!best_full && self_in_s && cv(s.rows[self_rank].count)) self_viol = true;
  if (c_self) {
    // every non-self candidate fails: the walk stops at the first member of S other than self
    cut_others = scan_first(co, from, end, Sw);
    if (self_in_s && cut_others == (uint32_t)self_rank)
      cut_others = scan_first(co, (uint32_t)self_rank >> 5, end, [&](uint32_t wi) { return Sw(wi) & mask_above(wi * 32u, (uint32_t)self_rank); });
  } else if (!best_full) {
    // a self member that fails the count test is reported here too; it then also sets self_viol: same cut
    cut_others = scan_first_violator(co, from, end, s.n_ranks, Sw,
        [&](uint32_t wi) { WordSumI m = s.csum[wi]; return !cv(m.hi) ? 0 : (cv(m.lo) ? 1 : 2); },
        [&](uint32_t r) { return cv(s.rows[r].count); });
  }
  MMP_BAIL_CHECK;
  const uint32_t cut_self = (self_in_s && self_viol) ? (uint32_t)self_rank : NONE_RANK;
  const uint32_t cut = cut_others < cut_self ? cut_others : cut_self;
  o.cut_rank = (int32_t)cut;
  if (open_end && cut == NONE_RANK && hi == NONE_RANK) MMP_OPEN_EXIT;  // the shortlist runs on into the next shard
  const bool self_in_sl = self_in_s && (uint32_t)self_rank < cut;
  if (favour_self && self_in_sl) { o.flags |= MMP_TF_FAVOUR_EXIT; o.target = MMP_TARGET_SELF; return; }
  const uint32_t endc = cut == NONE_RANK ? end : (end_for(cut) < end ? end_for(cut) : end);
  auto SLw = [&](uint32_t wi) -> uint32_t { return Sw(wi) & mask_below(wi * 32u, cut); };  // candidates other than best
  const int32_t n_in = (int32_t)scan_count(co, from, endc, SLw);
  MMP_BAIL_CHECK;
  const int32_t n_others = n_in - (self_in_sl ? 1 : 0);
  const int32_t ccount = 1 + n_in;
  o.n_candidates = ccount;
  bool keep_best = true, keep_others = true, keep_self = true;
  int32_t remaining = ccount;
  uint32_t index = 0;
  if (ccount > 1) {
    const int64_t ago = age_of(c.last_used, now);
    if (ago < 432000000LL) {  // FIVE_DAYS_MS
      int32_t mn = best_rpm;
      if (n_others > 0 && fr.rpm < mn) mn = fr.rpm;
      if (self_in_sl && rb.rpm < mn) mn = rb.rpm;
      RpmFilter rf; rf.init(mn, ago);
      keep_best = !rf.drop(best_rpm); keep_others = !rf.drop(fr.rpm); keep_self = !rf.drop(rb.rpm);
      remaining = (keep_best ? 1 : 0) + (keep_others ? n_others : 0) + ((self_in_sl && keep_self) ? 1 : 0);
    }
    index = remaining == 1 ? 0u : hash_index(seed, decision_id, (uint32_t)remaining);
  }
  o.n_remaining = remaining; o.pick_index = (int32_t)index;
  o.flags |= (keep_best ? MMP_TF_KEEP_BEST : 0) | (keep_others ? MMP_TF_KEEP_OTHERS : 0) | (keep_self ? MMP_TF_KEEP_SELF : 0);
  // survivors in rank order: best first (its rank precedes all of S), then S below the cut
  const uint32_t sw = self_rank >= 0 ? (uint32_t)self_rank >> 5 : NONE_RANK, sb = 1u << (self_rank & 31);
  auto SVw = [&](uint32_t wi) -> uint32_t {
    uint32_t v = keep_others ? SLw(wi) : 0u;
    if (self_in_sl && wi == sw) v = keep_self ? (v | sb) : (v & ~sb);
    return v;
  };
  if (cand_rows) emit_rows(SLw, SVw);
  uint32_t chosen_rank;
  uint32_t kth = index;
  if (keep_best && kth == 0) chosen_rank = best_rank;
  else {
    if (keep_best) kth--;
    if (!keep_others) chosen_rank = (uint32_t)self_rank;  // the only other survivor can be the self candidate
    else chosen_rank = scan_select(co, from, endc, SVw, kth);
    MMP_BAIL_CHECK;
  }
  const int32_t cidx = chosen_rank == best_rank ? best_idx : s.rows[chosen_rank].idx;
  o.target = (!favour_self && cidx == d.self) ? MMP_TARGET_SELF : cidx;
}

// ---- two-pass placement of a large batch (k_slot_summary, k_place_split; DESIGN.md §5.2).  For a type slot, a plain
// decision's best, shortlist and their order depend on the decision only through its exclusions and self when those lie
// below the walk's reach, and through its own record only as c_self (N2: one test for every member other than self).
// The summary is that decision worked out once per slot for each value of c_self; a decision whose exclusions and self
// all lie at or past the reach is answered from it by the pick arithmetic alone. ----
static constexpr int SPLIT_CAP = 256;  // shortlist members a summary lists; a longer shortlist is walked
struct SlotSummary {
  int64_t best_rem, best_lru;  // what c_self is tested against: the best's remaining, and the first entry's lruTime when it is full
  int32_t best_idx, best_rpm, best_full;
  int32_t reach[2];            // by c_self: DecideOut::reach; -1: the decisions of this slot are walked
  int32_t n_in[2];             // shortlist members besides best
  int32_t pad_;
};

// The summary of type slot `slot` for c_self = cs, and its shortlist members (instance indices, rank order) into
// members[0, SPLIT_CAP): decide_stream on a decision without exclusions, with a self that is not live and a record
// that makes c_self come out as cs.  Called by every lane of the vote group (active = false for lanes without a slot);
// ewin: win_words zero words.
template <class V>
MMP_HD void slot_summary(const SnapshotView &s, const LaneTables &T, int slot, bool active, int cs, const uint32_t *ewin,
                         uint32_t win_words, int64_t now, const V &vote, uint32_t *chunk, SlotSummary &sum, int32_t *members) {
  DecisionCtx c;
  c.d.model = 0; c.d.self = -1; c.d.last_used = 0; c.d.flags = 0; c.d.fresh = -1; c.d.extra_off = 0; c.d.extra_n = 0;
  c.last_used = 0; c.self_rank = -1; c.self_bits = 0; c.self_count = 0;
  c.xr[0] = c.xr[1] = c.xr[2] = c.xr[3] = -1;
  c.slot = active ? (slot | ((s.has_pref[slot] ? 1 : 0) << 16)) : -1;
  // c_self against a best with room tests remaining: this record makes it come out as cs
  c.fr.lru = 0; c.fr.rem = cs ? INT64_MIN : INT64_MAX; c.fr.count = 0; c.fr.rpm = 0;
  RowRanks none;
  none.r[0] = none.r[1] = none.r[2] = none.r[3] = -1;
  // first pass: the best (phases A, A', A'' do not read the caller's record of a self that is not live), and the
  // shortlist when the best has room
  DecideOut o;
  bool ok = decide_stream<TabGlob>(s, T, T, c, active, ewin, win_words, none, 0u, now, 0, 0, vote, o, 0x3fffffff, chunk) && active &&
            o.best_rank >= 0 && !(o.flags & MMP_TF_OPEN);
  RankRow r0, rb;
  r0.lru = r0.rem = 0; r0.rpm = 0; rb = r0; rb.idx = -1;
  bool full = false;
  if (ok) {
    r0 = load_row(s.rows + o.first_rank);
    rb = load_row(s.rows + o.best_rank);
    full = r0.rem < s.min_space;  // (a full first entry is never replaced as best: A' runs for a best with room only)
    if (full) {
      const int64_t a10 = age_of(r0.lru, now) / 10;
      c.fr.lru = cs ? (int64_t)((uint64_t)r0.lru + (uint64_t)((a10 > 45000 ? a10 : 45000) + 1)) : r0.lru;
    }
  }
  // second pass, for a full best: c_self tests lruTime against the best's, which the record now forces to come out as cs
  const bool again = ok && full;
  DecideOut ox;
  const bool ok2 = decide_stream<TabGlob>(s, T, T, c, again, ewin, win_words, none, 0u, now, 0, 0, vote, ox, 0x3fffffff, chunk);
  const DecideOut &o2 = again ? ox : o;
  ok = ok && (!again || ok2) && o2.best_rank == o.best_rank && !(o2.flags & (MMP_TF_OPEN | MMP_TF_FAVOUR_EXIT)) && o2.n_candidates >= 1 &&
       o2.n_candidates - 1 <= SPLIT_CAP;
  const int32_t n_in = ok ? o2.n_candidates - 1 : 0;
  if (ok) {  // the members: S' strictly between best and the cut (no cut: the end of S, one below the reach)
    const uint32_t lo = (uint32_t)o2.best_rank;
    const uint32_t lim = o2.cut_rank != (int32_t)NONE_RANK ? (uint32_t)o2.cut_rank : (o2.reach == (int32_t)NONE_RANK ? NONE_RANK : (uint32_t)o2.reach - 1u);
    const bool use_pref = (c.slot >> 16) && ((T.p[lo >> 5] >> (lo & 31)) & 1u);
    int32_t k = 0;
    for (uint32_t w = lo >> 5; w < (uint32_t)s.row_words && w * 32u < lim && k <= n_in; w++) {
      uint32_t x = T.cx[w] & (use_pref ? T.p[w] : 0xffffffffu) & mask_above(w * 32u, lo) & mask_below(w * 32u, lim);
      for (; x; x &= x - 1u) {
        if (k < SPLIT_CAP) members[k] = s.rows[w * 32u + (uint32_t)ffs32(x)].idx;
        k++;
      }
    }
    ok = k == n_in;
  }
  if (!active) return;
  if (cs == 0) { sum.best_rem = rb.rem; sum.best_lru = r0.lru; sum.best_idx = rb.idx; sum.best_rpm = rb.rpm; sum.best_full = full ? 1 : 0; sum.pad_ = 0; }
  sum.reach[cs] = ok ? o2.reach : -1;
  sum.n_in[cs] = n_in;
}

// The fast answer of k_place_split: a valid, unflagged decision without extra excludes whose model has no overflow ids
// and whose exclusions and self all lie at or past its slot's reach for its c_self.  ok: decision_ok of d; self_rank:
// rank_of[d.self]; k: its model's SplitKey (read only when ok and not a request-model decision).  Returns false, with
// nothing written, for every other decision.
MMP_HD bool split_answer(const SnapshotView &s, const mmp_decision_in &d, int32_t ok, int32_t self_rank, const SplitKey &k,
                         const FreshRow *fresh, int32_t n_fresh, const SlotSummary *sums, const int32_t *members, int64_t now,
                         uint64_t seed, uint64_t decision_id, mmp_decision_out &out) {
  if (!ok || request_model(d) || d.extra_n != 0 || (k.slot & SPLIT_KEY_OVF)) return false;
  FreshRow fr;  // (as prepare_ctx_b)
  if (d.fresh >= 0 && d.fresh < n_fresh) fr = fresh[d.fresh];
  else if (self_rank >= 0) { const RankRow sr = load_row(s.rows + self_rank); fr.lru = sr.lru; fr.rem = sr.rem; fr.count = sr.count; fr.rpm = 0; }
  else return false;
  const int slot = (int)k.slot;
  const SlotSummary &sm = sums[slot];
  int cs;
  if (sm.best_full) {  // (decide_stream's c_self)
    const int64_t a10 = age_of(sm.best_lru, now) / 10, df = jsub(fr.lru, sm.best_lru);
    cs = df > 45000 && df > a10;
  } else cs = fr.rem < s.min_space || fr.rem < (sm.best_rem >> 2);
  const int32_t reach = sm.reach[cs];
  if (reach < 0 || (self_rank >= 0 && self_rank < reach) || k.min_rank < reach) return false;
  const int32_t n_in = sm.n_in[cs];
  const int64_t last_used = (d.flags & MMP_DF_MODEL_LAST_USED) ? k.last_used : d.last_used;
  const PickOut pk = pick_survivor(n_in, false, sm.best_rpm, fr.rpm, sm.best_rpm, last_used, now, seed, decision_id);
  if (pk.kind == PICK_SELF) return false;
  const int32_t cidx = pk.kind == PICK_BEST ? sm.best_idx : members[((size_t)slot * 2 + (size_t)cs) * SPLIT_CAP + pk.kth];
  out.target = target_of(cidx, d);
  out.n_candidates = 1 + n_in;
  return true;
}
// The same answer for a caller that holds the decision's model row and excluded ranks instead of its SplitKey (the CPU
// harness): a: prepare_ctx_a of d; row: its model's excl_ranks entry.  The key is made from them as the commit makes it.
MMP_HD bool split_answer(const SnapshotView &s, const mmp_decision_in &d, const CtxA &a, const RowRanks &row, const FreshRow *fresh,
                         int32_t n_fresh, const SlotSummary *sums, const int32_t *members, int64_t now, uint64_t seed,
                         uint64_t decision_id, mmp_decision_out &out) {
  if (!a.ok || request_model(d)) return false;
  SplitKey k = make_split_key(a.mr, row.r, s.type_slot, s.n_type_ids);
  if (row.overflow()) k.slot |= SPLIT_KEY_OVF;
  return split_answer(s, d, a.ok, a.self_rank, k, fresh, n_fresh, sums, members, now, seed, decision_id, out);
}

}  // namespace mmp
