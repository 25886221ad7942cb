// scan_kernels.cuh — batch scans (plug points 3 and 4 of include/mmplace.h): ClusterStats reductions, the reaper's
// registry sweep + top-K selection, and the per-instance time-ordered weighted LRU.  Included at the end of mmplace.cu.
#pragma once

// ---------------------------------------------------------------------------------------------------------------
// ClusterStats (MM:1570-1591) per prohibited-type-set partition: InstanceSetStatsTracker.add (ISST:63-72) as a
// segmented reduction over the rank-ordered instance columns.  acc layout per partition: [cap, free, count|copies]
// ---------------------------------------------------------------------------------------------------------------
struct StatsAcc { unsigned long long cap, free; int count, copies; };

// One pass over the rank-ordered instance columns (~50 B per instance).  Every block accumulates into shared-memory slots
// (one per partition + the cluster) and publishes each slot it touched with one global atomic: a handful of global atomics
// per block instead of eight per instance.
static constexpr int STATS_SMEM_PARTS = 511;
__global__ void k_stats(const RankRow *__restrict__ rows, const int64_t *__restrict__ cap_col,
                        const int32_t *__restrict__ part_of_rank, int n_ranks, int64_t min_space, StatsAcc *acc,
                        long long *min_lru, int n_parts) {
  __shared__ StatsAcc sacc[STATS_SMEM_PARTS + 1];
  const bool use_smem = n_parts <= STATS_SMEM_PARTS;
  if (use_smem)
    for (int i = threadIdx.x; i <= n_parts; i += blockDim.x) sacc[i] = StatsAcc{0ull, 0ull, 0, 0};
  __syncthreads();
  long long lmin = 0x7fffffffffffffffLL;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n_ranks; r += gridDim.x * blockDim.x) {
    RankRow row = rows[r];
    int p = part_of_rank[r] + 1;  // slot 0 = whole cluster
    unsigned long long cap = (unsigned long long)cap_col[r];
    unsigned long long fr = row.rem < min_space ? 0ull : (unsigned long long)row.rem;  // only non-full instances (ISST:67-71)
    StatsAcc *dst = use_smem ? sacc : acc;
    atomicAdd(&dst[0].cap, cap); atomicAdd(&dst[0].free, fr); atomicAdd(&dst[0].count, 1); atomicAdd(&dst[0].copies, row.count);
    atomicAdd(&dst[p].cap, cap); atomicAdd(&dst[p].free, fr); atomicAdd(&dst[p].count, 1); atomicAdd(&dst[p].copies, row.count);
    if (row.lru > 0 && row.lru < lmin) lmin = row.lru;  // ISST.addLru (ISST:57-61)
  }
  for (int o = 16; o > 0; o >>= 1) {
    long long t = __shfl_xor_sync(0xffffffffu, lmin, o);
    if (t < lmin) lmin = t;
  }
  if ((threadIdx.x & 31) == 0 && lmin != 0x7fffffffffffffffLL) atomicMin(min_lru, lmin);
  if (use_smem) {
    __syncthreads();
    for (int i = threadIdx.x; i <= n_parts; i += blockDim.x) {
      const StatsAcc v = sacc[i];
      if (v.count) { atomicAdd(&acc[i].cap, v.cap); atomicAdd(&acc[i].free, v.free); atomicAdd(&acc[i].count, v.count); atomicAdd(&acc[i].copies, v.copies); }
    }
  }
}

struct StatsResult {
  std::vector<mmp_cluster_stats> parts;  // [0] cluster, [1+p] partition p
};

static int32_t run_stats(mmp_fleet *f, const DeviceSnapshot &ds, StatsResult &res) {
  const HostSnapshot &h = ds.host;
  const int np = (int)h.part_types.size();
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  size_t bytes = (size_t)(np + 1) * sizeof(StatsAcc) + 8;
  CK(c->d_trace.ensure(bytes));
  CK(cudaMemsetAsync(c->d_trace.p, 0, bytes, c->stream));
  long long *d_min = reinterpret_cast<long long *>(c->d_trace.as<char>() + (size_t)(np + 1) * sizeof(StatsAcc));
  const long long init = 0x7fffffffffffffffLL;
  CK(cudaMemcpyAsync(d_min, &init, 8, cudaMemcpyHostToDevice, c->stream));
  CK(cudaEventRecord(c->e0, c->stream));
  if (h.n_ranks > 0) {
    int grid = std::min(f->sm_count, (h.n_ranks + 255) / 256);
    k_stats<<<grid, 256, 0, c->stream>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(), ds.part_of_rank.as<int32_t>(), h.n_ranks,
                                        f->hs.cfg.min_space_units, c->d_trace.as<StatsAcc>(), d_min, np);
    f->launches++;
    CK(cudaGetLastError());
  }
  CK(cudaEventRecord(c->e1, c->stream));
  std::vector<StatsAcc> acc(np + 1);
  long long mn = 0;
  CK(cudaMemcpyAsync(acc.data(), c->d_trace.p, (size_t)(np + 1) * sizeof(StatsAcc), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(&mn, d_min, 8, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  { float ms = 0; if (cudaEventElapsedTime(&ms, c->e0, c->e1) == cudaSuccess) f->t_stats_ms = ms; }
  res.parts.resize(np + 1);
  for (int i = 0; i <= np; i++) {
    mmp_cluster_stats &s = res.parts[i];
    s.total_capacity = (int64_t)acc[i].cap; s.total_free = (int64_t)acc[i].free; s.instance_count = acc[i].count;
    s.model_copy_count = acc[i].copies;
    // quirk N10: every subset's LRU is recomputed over all cluster instances (MM:1519-1541)
    s.global_lru = acc[i].count > 0 || i == 0 ? (int64_t)mn : INT64_MAX;
  }
  return MMP_OK;
}

// PARTITION_STATS_COMP (TCM:264-271): free desc, lru asc, capacity desc; partition id breaks remaining ties
static std::vector<int> partition_order(const StatsResult &res) {
  std::vector<int> ord;
  for (int p = 1; p < (int)res.parts.size(); p++)
    if (res.parts[p].instance_count > 0) ord.push_back(p - 1);
  std::stable_sort(ord.begin(), ord.end(), [&](int a, int b) {
    const mmp_cluster_stats &x = res.parts[a + 1], &y = res.parts[b + 1];
    if (x.total_free != y.total_free) return x.total_free > y.total_free;
    if (x.global_lru != y.global_lru) return x.global_lru < y.global_lru;
    if (x.total_capacity != y.total_capacity) return x.total_capacity > y.total_capacity;
    return a < b;
  });
  return ord;
}

// ---------------------------------------------------------------------------------------------------------------
// Reaper: registry sweep (MM:6536-6590 candidate rule MM:6574-6577) + bounded most-recently-used selection
// (MM:6675-6698) as  flag/compact -> bitonic sort by (lastUsed desc, model asc) -> first-of-run.
// ---------------------------------------------------------------------------------------------------------------
// key: ~biased(lastUsed), so that ascending keys = descending time.  One thread per model: 24 B read, 1 + 8 B written.
__global__ void k_reaper_flag(const mmp_model_row *__restrict__ models, int n_models, const uint8_t *__restrict__ type_excluded,
                              int n_type_ids, const uint8_t *__restrict__ taken, long long global_lru, int need_cutoff,
                              long long cutoff, uint8_t *__restrict__ flag, unsigned long long *__restrict__ key) {
  int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  mmp_model_row r = models[m];
  bool ok = r.copy_count == 0 && r.fail_count < 2 && (global_lru == 0 || r.last_used > global_lru);  // MM:6574-6577
  if (ok && taken && taken[m]) ok = false;                                                           // allCandidates.set(i, null)
  if (ok && r.type_id < n_type_ids && type_excluded[r.type_id]) ok = false;                          // MM:6681-6683
  if (ok && need_cutoff && !(r.last_used > cutoff)) ok = false;                                      // MM:6685-6687
  flag[m] = ok ? 1 : 0;
  key[m] = ~((unsigned long long)r.last_used ^ 0x8000000000000000ull);
}
// keep the first record of every equal-lastUsed run (TreeSet<ModelToLoad> drops equal keys, MM:6405-6408), in order
__global__ void k_unique_mark(const unsigned long long *__restrict__ keys, int n, uint8_t *__restrict__ flags) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

static int32_t reaper_impl(mmp_fleet *f, int32_t partition, int64_t now, uint8_t *taken, int32_t *out_models, int32_t cap) {
  if (!out_models || cap < 0) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  const DeviceSnapshot &ds = f->snaps[f->cur];
  const HostSnapshot *hp = nullptr;
  rc = host_mirror(f, ds, &hp);
  if (rc < 0) return rc;
  const HostSnapshot &h = *hp;
  const int np = (int)h.part_types.size();
  if (partition >= np || (partition >= 0 && !h.tc_enabled)) { g_err = "no such partition"; return MMP_E_ARG; }
  StatsResult sr;
  rc = run_stats(f, ds, sr);
  if (rc < 0) return rc;
  const mmp_cluster_stats &g = sr.parts[0];
  if (!(g.total_capacity > 0)) return 0;                                   // MM:6456
  const int64_t global_lru = g.total_free > 0 ? 0 : g.global_lru;          // MM:6460
  const mmp_cluster_stats &st = partition < 0 ? g : sr.parts[partition + 1];
  // triggerProactiveLoadsForInstanceSubset MM:6616-6664
  int32_t free_count = 0, total_count = 0;
  if (st.total_capacity > 0 && st.total_free > 0) {
    int32_t size_est;
    const int32_t def = f->hs.cfg.default_model_size_units;
    if (st.model_copy_count < 3) size_est = def;
    else {
      int32_t avg = (int32_t)jsub(st.total_capacity, st.total_free) / st.model_copy_count;
      size_est = st.model_copy_count > 10 ? avg : jaddi(avg, def) / 2;
    }
    if (size_est == 0) { g_err = "size estimate is zero (the reference would throw ArithmeticException)"; return MMP_E_ARG; }
    int64_t space = 0;
    for (int32_t r = 0; r < h.n_ranks; r++) {
      if (partition >= 0 && h.part_of_rank[r] != partition) continue;
      int32_t max_loads = (int32_t)((uint32_t)jmuli(h.lthreads_col[r], 50) - (uint32_t)h.linprog_col[r]);
      if (max_loads <= 0) continue;
      int64_t avail = jsub(h.rows[r].rem, h.cap_col[r] / 8);
      if (avail > 0) space = (int64_t)((uint64_t)space + (uint64_t)std::min<int64_t>(avail, (int64_t)jmuli(max_loads, size_est)));
    }
    space /= 2;
    free_count = (int32_t)(space / size_est);
    int64_t d = (int64_t)((uint64_t)20 * (uint64_t)(int64_t)size_est);
    total_count = std::max(free_count, d == 0 ? 0 : (int32_t)(d == -1 ? -st.total_capacity : st.total_capacity / d));
  }
  const int64_t cutoff = st.global_lru == INT64_MAX ? 0
      : (int64_t)((uint64_t)st.global_lru + (uint64_t)std::max<int64_t>(age_of(st.global_lru, now) / 3, 1200000));
  if (total_count <= 0) return 0;
  // prohibited types of this partition -> per type id flag
  std::vector<uint8_t> excl(h.type_slot.size(), 0);
  if (partition >= 0)  // ids as interned when this epoch was committed: the ingest-side name table is never read here
    for (int32_t tid : h.part_type_ids[partition])
      if (tid >= 0 && tid < (int32_t)excl.size()) excl[tid] = 1;
  const int nm = ds.n_models;
  if (nm == 0) return 0;
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t s = c->stream;
  // Registry sweep -> candidates compacted in model order (stable) -> radix sort by ~lastUsed (stable: equal times keep the
  // lower model index first) -> first of every equal-time run (N12) -> only the first `total_count` survivors leave the device.
  // All on the device; the host applies the emission rule (MM:6711-6719) to at most total_count records.
  const size_t n8 = (size_t)nm * 8, n4 = (size_t)nm * 4;
  CK(c->d_in.ensure(2 * n8 + 64));        // keys[nm], keys_sel[nm]
  CK(c->d_out.ensure(2 * n8 + 64));       // keys_sorted[nm], keys_uniq[nm]
  CK(c->d_trace.ensure(4 * n4 + 64));     // idx_sel, idx_sorted, idx_uniq, (spare)
  CK(c->d_cand.ensure((size_t)nm + 64));  // flags
  CK(c->d_extra.ensure(excl.size() + 16));
  CK(c->d_fresh.ensure((size_t)nm + 16));
  CK(c->d_n_open.ensure(16));
  unsigned long long *keys = c->d_in.as<unsigned long long>(), *keys_sel = keys + nm;
  unsigned long long *keys_sorted = c->d_out.as<unsigned long long>(), *keys_uniq = keys_sorted + nm;
  int32_t *idx_sel = c->d_trace.as<int32_t>(), *idx_sorted = idx_sel + nm, *idx_uniq = idx_sorted + nm;
  uint8_t *flags = c->d_cand.as<uint8_t>();
  int *d_n = c->d_n_open.as<int>();
  CK(cudaMemcpyAsync(c->d_extra.p, excl.data(), excl.size(), cudaMemcpyHostToDevice, s));
  if (taken) CK(cudaMemcpyAsync(c->d_fresh.p, taken, (size_t)nm, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(c->e0, s));
  k_reaper_flag<<<(nm + 255) / 256, 256, 0, s>>>(ds.models.as<mmp_model_row>(), nm, c->d_extra.as<uint8_t>(), (int)excl.size(),
                                               taken ? c->d_fresh.as<uint8_t>() : nullptr, global_lru, free_count > 0 ? 0 : 1, cutoff, flags, keys);
  f->launches++;
  CK(cudaGetLastError());
  thrust::counting_iterator<int32_t> iota(0);
  size_t t1 = 0, t2 = 0, t3 = 0;
  CK(cub::DeviceSelect::Flagged(nullptr, t1, keys, flags, keys_sel, d_n, nm, s));
  CK(cub::DeviceSelect::Flagged(nullptr, t2, iota, flags, idx_sel, d_n, nm, s));
  CK(cub::DeviceRadixSort::SortPairs(nullptr, t3, keys_sel, keys_sorted, idx_sel, idx_sorted, nm, 0, 64, s));
  CK(c->d_cub.ensure(std::max(t1, std::max(t2, t3)) + 64));
  CK(cub::DeviceSelect::Flagged(c->d_cub.p, t1, keys, flags, keys_sel, d_n, nm, s));
  CK(cub::DeviceSelect::Flagged(c->d_cub.p, t2, iota, flags, idx_sel, d_n, nm, s));
  int ncand = 0;
  CK(cudaMemcpyAsync(&ncand, d_n, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  f->launches += 2;
  if (ncand == 0) return 0;
  CK(cub::DeviceRadixSort::SortPairs(c->d_cub.p, t3, keys_sel, keys_sorted, idx_sel, idx_sorted, ncand, 0, 64, s));
  k_unique_mark<<<(ncand + 255) / 256, 256, 0, s>>>(keys_sorted, ncand, flags);
  CK(cub::DeviceSelect::Flagged(c->d_cub.p, t1, keys_sorted, flags, keys_uniq, d_n, ncand, s));
  CK(cub::DeviceSelect::Flagged(c->d_cub.p, t2, idx_sorted, flags, idx_uniq, d_n, ncand, s));
  f->launches += 4;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->e1, s));
  int nuniq = 0;
  CK(cudaMemcpyAsync(&nuniq, d_n, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  { float ms = 0; if (cudaEventElapsedTime(&ms, c->e0, c->e1) == cudaSuccess) f->t_reaper_ms = ms; }
  const int take = std::min(nuniq, total_count);
  std::vector<unsigned long long> hk((size_t)take);
  std::vector<int32_t> hm((size_t)take);
  if (take) {
    CK(cudaMemcpyAsync(hk.data(), keys_uniq, (size_t)take * 8, cudaMemcpyDeviceToHost, s));
    CK(cudaMemcpyAsync(hm.data(), idx_uniq, (size_t)take * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  int64_t emitted = 0;
  int32_t free_left = free_count;
  for (int i = 0; i < take; i++) {
    const int64_t ts = (int64_t)((~hk[i]) ^ 0x8000000000000000ull);
    if (free_left > 0) free_left--;          // MM:6713-6714
    else if (ts < cutoff) break;             // MM:6715-6717
    const int32_t m = hm[i];
    if (taken) taken[m] = 1;
    if (emitted < cap) out_models[emitted] = m;
    emitted++;
  }
  return (int32_t)std::min<int64_t>(emitted, INT32_MAX);
}

// ---------------------------------------------------------------------------------------------------------------
// Time-ordered weighted LRU (CLHM + LinkedDeque), one warp per instance, events applied in order.
// An entry's position in the reference's deque is represented by the key (lastUsed, seq): LinkedDeque.insert (LD:258-288)
// links after every element with lastUsed <= ts  ==  a fresh, larger seq; reposition (LD:243-255) keeps the node in
// place when its successor's lastUsed >= the new time  ==  keep the position (seq just below the successor's when the
// times tie).  Eviction (CLHM:329-352) pops the minimum key while weightedSize > capacity.
// ---------------------------------------------------------------------------------------------------------------
struct LruView {
  long long *ts; long long *seq; int *weight; int *model;   // [n][slots]
  long long *loadts;                                        // [n][slots] registration time of the copy (MR.instanceIds value), -1: not registered
  long long *cap, *wsize, *seqctr; int *count;              // [n]
  long long *pin;                                           // [n] oldestTime() as a setCapacity left it (N14), LRU_PIN_NONE
  int n, slots;
};
// CLHM caches oldestTime and refreshes it after every write and read (updateOldestTime, CLHM:444, 463), but setCapacity
// (CLHM:305-316) evicts without refreshing it: until the next refresh oldestTime() reports the head from before the
// evictions (quirk N14).  The pin holds that value; LRU_PIN_NONE (a byte pattern, so cudaMemset clears the column) means
// oldestTime() is the head of the deque.
#define LRU_PIN_NONE ((long long)0x8080808080808080ULL)

// one event of an instance's cache, as the kernels see it
enum { LEV_INSERT = 0, LEV_TOUCH = 1, LEV_RESIZE = 2, LEV_REMOVE = 3, LEV_SET_CAPACITY = 4, LEV_LOAD = 5, LEV_SEED = 6 };
struct LruEv {
  int op, model, weight, order;  // order: what an eviction reports as its cause (event index / position in the epoch's trace)
  int dec, pad;                  // LEV_LOAD: index of the placement decision that sent the load here
  long long last_used, t;        // t: the event's own clock (churn epochs), or the registration time of a LEV_SEED entry
};
struct EvictRec { int instance, model; long long last_used; int weight, order, reload, seq; };
struct Follow { int model, exclude; long long last_used; int weight, order, seq, inst; };  // a queued ensureLoadedElsewhere (MM:2922, 6905)

// per-decision outcome of a checked load (the statuses of oracle/mm_sim.inc)
enum { CH_ACCEPTED = 0, CH_NOWHERE = 1, CH_CHURN = 2, CH_FALLTHRU = 3, CH_EARLY = 4, CH_GROW_EVICTED = 5, CH_EXISTS = 6, CH_SKIPPED = 7,
       CH_INVALID = 8, CH_EVICTED_LATER = 9 };

// What the closed loop hooks into the LRU kernel (null pointers / enabled = 0 for a plain mmp_lru_apply)
struct ChurnHooks {
  int enabled;
  long long min_space, min_churn_age, load_timeout;
  int *status;                     // [n_decisions] CH_*
  const int *dec_target;           // [n_decisions] instance the decision resolved to
  const int *dec_of_model;         // [n_models] this epoch's decision for the model, -1
  const int4 *edges;               // [n_models] registered instances (first copy_count = loaded)
  const mmp_model_row *models;
  unsigned *rm_mask;               // [n_models] bit j: edge j is deregistered at the end of the epoch
  const unsigned char *type_ok;    // [n_type_ids] the type set is < 95 % full (MM:2918-2920)
  int n_type_ids;
  Follow *next; int *n_next; int next_cap;
  unsigned char *force_publish;    // [n_instances]
};

__device__ __forceinline__ bool key_less(long long t1, long long s1, long long t2, long long s2) { return t1 < t2 || (t1 == t2 && s1 < s2); }

// warp argmin of (ts, seq) over alive slots with key > (lo_t, lo_s) when bounded; returns slot or -1
__device__ int lru_min_slot(const LruView &v, int inst, int lane, bool bounded, long long lo_t, long long lo_s, long long *out_t, long long *out_s) {
  const size_t base = (size_t)inst * v.slots;
  long long bt = 0x7fffffffffffffffLL, bs = 0x7fffffffffffffffLL;
  int bi = -1;
  for (int i = lane; i < v.slots; i += 32) {
    if (v.model[base + i] < 0) continue;
    long long t = v.ts[base + i], s = v.seq[base + i];
    if (bounded && !key_less(lo_t, lo_s, t, s)) continue;
    if (bi < 0 || key_less(t, s, bt, bs)) { bt = t; bs = s; bi = i; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    long long t2 = __shfl_xor_sync(0xffffffffu, bt, o), s2 = __shfl_xor_sync(0xffffffffu, bs, o);
    int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    if (i2 >= 0 && (bi < 0 || key_less(t2, s2, bt, bs))) { bt = t2; bs = s2; bi = i2; }
  }
  *out_t = bt; *out_s = bs;
  return bi;
}
__device__ int lru_find(const LruView &v, int inst, int lane, int model, int *free_slot) {
  const size_t base = (size_t)inst * v.slots;
  int found = -1, fr = -1;
  for (int i = lane; i < v.slots; i += 32) {
    int m = v.model[base + i];
    if (m == model) found = i;
    if (m < 0 && fr < 0) fr = i;
  }
  found = __reduce_max_sync(0xffffffffu, found);
  unsigned ufr = fr < 0 ? 0x7fffffffu : (unsigned)fr;
  ufr = __reduce_min_sync(0xffffffffu, ufr);
  *free_slot = ufr == 0x7fffffffu ? -1 : (int)ufr;
  return found;
}

// One warp per instance applies its events in order.  LEV_LOAD is loadLocal's admission (a11): churn guard MM:3872-3884,
// placeholder insert (INSERTION_WEIGHT = 1, MM:5011, 5061), immediate-eviction fall-through MM:5145-5148, early reject
// MM:5185-5190, registration, inflate to the predicted size + grow-then-check MM:2094-2106.  With hooks.enabled every eviction
// also runs the eviction listener's bookkeeping (onEviction MM:2875-2931): deregistration mark, the reload-elsewhere rule (a12).
__global__ void k_lru_events(LruView v, const LruEv *__restrict__ ev, const int *__restrict__ ev_order, const int *__restrict__ inst_off,
                             long long now_param, int use_ev_time, ChurnHooks hk, EvictRec *out, int out_cap, int *out_n, int *err, int stage_slots) {
  const int lane = threadIdx.x & 31;
  const int inst = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (inst >= v.n) return;
  const int p0 = inst_off[inst], p1 = inst_off[inst + 1];
  if (p0 >= p1) return;
  // An instance with many events (the pod that holds a hot model: its touches are serial) works on a copy of its slot arrays
  // in shared memory -- every event scans the slots twice (find the model, find the successor / the oldest) -- and writes
  // them back at the end.  stage_slots = slots the block's dynamic shared memory has room for per warp (0: no staging).
  extern __shared__ __align__(16) unsigned char lru_smem[];
  LruView sv = v;
  int hi = inst;                 // the instance index the helpers see (0 on the staged copy)
  size_t base = (size_t)inst * v.slots;
  const bool staged = stage_slots >= v.slots && (p1 - p0) >= 12;
  if (staged) {
    unsigned char *mine = lru_smem + (size_t)(threadIdx.x >> 5) * (size_t)stage_slots * 32u;
    long long *s_ts = reinterpret_cast<long long *>(mine), *s_seq = s_ts + stage_slots, *s_lt = s_seq + stage_slots;
    int *s_w = reinterpret_cast<int *>(s_lt + stage_slots), *s_m = s_w + stage_slots;
    for (int i = lane; i < v.slots; i += 32) {
      s_ts[i] = sv.ts[base + i]; s_seq[i] = sv.seq[base + i]; s_lt[i] = sv.loadts[base + i]; s_w[i] = sv.weight[base + i]; s_m[i] = sv.model[base + i];
    }
    __syncwarp();
    sv.ts = s_ts; sv.seq = s_seq; sv.loadts = s_lt; sv.weight = s_w; sv.model = s_m;
    hi = 0; base = 0;
  }
  long long wsize = v.wsize[inst], capacity = v.cap[inst], ctr = v.seqctr[inst], pin = v.pin[inst];
  int count = v.count[inst];
  int evseq = 0;
  // evict() CLHM:329-352 + the listener; returns through *self_gone whether `watch_model` was among the victims
  auto evict_loop = [&](const LruEv &e, long long now, int watch_model, bool *self_gone) {
    while (wsize > capacity) {
      long long t, s;
      const int victim = lru_min_slot(sv, hi, lane, false, 0, 0, &t, &s);
      if (victim < 0) break;
      const int w = sv.weight[base + victim], m = sv.model[base + victim];
      const long long lt = sv.loadts[base + victim];
      __syncwarp();
      if (m == watch_model && self_gone) *self_gone = true;
      if (lane == 0) {
        sv.model[base + victim] = -1;
        int reload = 0;
        if (hk.enabled) {
          const bool in_registry = lt >= 0;
          const bool attempt = in_registry && (now - lt) > 2 * hk.load_timeout;  // MM:2901
          if (in_registry) {
            const int4 ed = hk.edges[m];
            const int cc = hk.models[m].copy_count;
            const int es[4] = {ed.x, ed.y, ed.z, ed.w};
            for (int j = 0; j < 4 && j < cc; j++) if (es[j] == inst) atomicOr(&hk.rm_mask[m], 1u << j);
          }
          const int k2 = hk.dec_of_model[m];
          if (k2 >= 0 && hk.dec_target[k2] == inst && hk.status[k2] == CH_ACCEPTED) hk.status[k2] = CH_EVICTED_LATER;
          const int ty = hk.models[m].type_id;
          if (attempt && hk.type_ok[ty < hk.n_type_ids ? ty : 0]) {  // MM:2916-2922
            reload = 1;
            const int q = atomicAdd(hk.n_next, 1);
            if (q < hk.next_cap) hk.next[q] = Follow{m, inst, t, w, e.order, evseq, inst};
          }
          hk.force_publish[inst] = 1;
        }
        const int pos = atomicAdd(out_n, 1);
        if (pos < out_cap) out[pos] = EvictRec{inst, m, t, w, e.order, reload, evseq};
      }
      evseq++;
      __syncwarp();
      wsize -= (w < 0 ? -w : w); count--;
    }
  };
  LruEv e_next = ev[ev_order[p0]];
  for (int p = p0; p < p1; p++) {
    const LruEv e = e_next;
    if (p + 1 < p1) e_next = ev[ev_order[p + 1]];  // (the next event's two dependent loads fly while this one is applied)
    const long long now = use_ev_time ? e.t : now_param;
    int free_slot;
    int slot = (e.op == LEV_SET_CAPACITY) ? -1 : lru_find(sv, hi, lane, e.model, &free_slot);
    // oldestTime() (N14) for a SET_CAPACITY, which keeps it, and for the churn guard of a load into a cache with less than
    // min_space free (MM:3872-3884); one call site of the slot scan for both keeps the kernel's code as small as before
    const bool guard = e.op == LEV_LOAD && hk.min_churn_age > 0 && capacity - wsize < hk.min_space;
    if (e.op == LEV_SET_CAPACITY || guard) {
      long long lru = pin, s;
      if (lru == LRU_PIN_NONE && lru_min_slot(sv, hi, lane, false, 0, 0, &lru, &s) < 0) lru = -1;
      if (!guard) { pin = lru; capacity = e.last_used; evict_loop(e, now, -1, nullptr); continue; }
      if (lru >= 0 && lru != 0x7fffffffffffffffLL && (lru == 0 ? 0 : now - lru) < hk.min_churn_age) { if (lane == 0) hk.status[e.dec] = CH_CHURN; continue; }
    }
    if (e.op == LEV_LOAD && slot >= 0) { if (lane == 0) hk.status[e.dec] = CH_EXISTS; }  // putIfAbsent found an entry: afterRead below
    if ((e.op == LEV_INSERT || e.op == LEV_SEED || e.op == LEV_LOAD) && slot < 0) {
      if (free_slot < 0) { if (lane == 0) atomicExch(err, 1); continue; }
      const int w0 = e.op == LEV_LOAD ? 1 : e.weight;  // INSERTION_WEIGHT MM:5011
      if (lane == 0) {
        sv.model[base + free_slot] = e.model; sv.weight[base + free_slot] = w0;
        sv.ts[base + free_slot] = e.last_used == 0 ? now : e.last_used;   // Node ctor: touch(time) (CLHM:1352-1360)
        sv.seq[base + free_slot] = ++ctr;
        sv.loadts[base + free_slot] = e.op == LEV_SEED ? e.t : -1;
      } else ++ctr;
      __syncwarp();
      wsize += w0; count++;                                              // AddTask (CLHM:601-610)
      pin = LRU_PIN_NONE;                                                // afterWrite: updateOldestTime (CLHM:444)
      bool gone = false;
      evict_loop(e, now, e.model, &gone);
      if (e.op != LEV_LOAD) continue;
      if (lane == 0 && hk.enabled) hk.force_publish[inst] = 1;
      if (gone) { if (lane == 0) hk.status[e.dec] = CH_FALLTHRU; continue; }  // MM:5145-5148
      // early reject MM:5185-5190 (capacity, weightedSize, oldestTime after the placeholder went in)
      long long ot, os;
      const int oi = lru_min_slot(sv, hi, lane, false, 0, 0, &ot, &os);
      const long long oldest = oi < 0 ? -1 : ot;
      const long long abs_size = e.weight < 0 ? -(long long)e.weight : (long long)e.weight;
      if (abs_size > capacity || (e.last_used > 0 && abs_size > capacity - wsize && e.last_used < oldest)) {
        if (lane == 0) { sv.model[base + free_slot] = -1; hk.status[e.dec] = CH_EARLY; }  // ce.remove()
        __syncwarp();
        wsize -= 1; count--;
        continue;
      }
      if (lane == 0) { sv.loadts[base + free_slot] = now; hk.status[e.dec] = CH_ACCEPTED; sv.weight[base + free_slot] = e.weight; }  // MM:5203, 2100
      __syncwarp();
      wsize += (long long)e.weight - 1;
      gone = false;
      evict_loop(e, now, e.model, &gone);
      if (gone && lane == 0) hk.status[e.dec] = CH_GROW_EVICTED;          // MM:2102-2106
      continue;
    }
    if ((e.op == LEV_INSERT || e.op == LEV_TOUCH || e.op == LEV_LOAD || e.op == LEV_SEED) && slot >= 0) {
      // afterRead -> touch + reposition (CLHM:383-388, 477-505; LD:243-255), then updateOldestTime (CLHM:463)
      pin = LRU_PIN_NONE;
      long long old_t = sv.ts[base + slot], old_s = sv.seq[base + slot];
      long long lu = e.last_used > 0 ? (old_t > e.last_used ? old_t : e.last_used) : now;
      if (lu != old_t) {
        long long nt, ns;
        // (times only move forward through max(); a smaller "now" than the entry's time can move it backwards)
        bool moved_back = lu < old_t;
        int nx = moved_back ? -1 : lru_min_slot(sv, hi, lane, true, old_t, old_s, &nt, &ns);
        bool stay = !moved_back && (nx < 0 || nt >= lu);
        if (moved_back) {
          // prev.lastUsed <= lu fails in general: unlink + insert (LD:253-254)
          if (lane == 0) { sv.ts[base + slot] = lu; sv.seq[base + slot] = ctr + 1; }
          ++ctr;
        } else if (stay) {
          if (lane == 0) { sv.ts[base + slot] = lu; if (nx >= 0 && nt == lu) sv.seq[base + slot] = ns - 1; }
        } else {
          if (lane == 0) { sv.ts[base + slot] = lu; sv.seq[base + slot] = ctr + 1; }
          ++ctr;
        }
        __syncwarp();
      }
    } else if (e.op == LEV_RESIZE && slot >= 0) {
      int oldw = sv.weight[base + slot];
      if (lane == 0) sv.weight[base + slot] = e.weight;
      __syncwarp();
      if (e.weight != oldw) pin = LRU_PIN_NONE;                          // no UpdateTask for an unchanged weight
      wsize += (long long)e.weight - oldw;                               // UpdateTask (CLHM:643-651), quiet
      evict_loop(e, now, -1, nullptr);
    } else if (e.op == LEV_REMOVE && slot >= 0) {
      int w = sv.weight[base + slot];
      const long long lt = sv.loadts[base + slot];
      if (lane == 0) {
        sv.model[base + slot] = -1;
        if (hk.enabled) {
          hk.force_publish[inst] = 1;
          if (lt >= 0) {  // deregisterModel
            const int4 ed = hk.edges[e.model];
            const int cc = hk.models[e.model].copy_count;
            const int es[4] = {ed.x, ed.y, ed.z, ed.w};
            for (int j = 0; j < 4 && j < cc; j++) if (es[j] == inst) atomicOr(&hk.rm_mask[e.model], 1u << j);
          }
        }
      }
      __syncwarp();
      wsize -= (w < 0 ? -w : w); count--;                                // RemovalTask + makeDead (CLHM:614-628, 561-570)
      pin = LRU_PIN_NONE;
    }
  }
  if (staged) {
    __syncwarp();
    const size_t gb = (size_t)inst * v.slots;
    for (int i = lane; i < v.slots; i += 32) {
      v.ts[gb + i] = sv.ts[i]; v.seq[gb + i] = sv.seq[i]; v.loadts[gb + i] = sv.loadts[i]; v.weight[gb + i] = sv.weight[i]; v.model[gb + i] = sv.model[i];
    }
  }
  if (lane == 0) { v.wsize[inst] = wsize; v.cap[inst] = capacity; v.seqctr[inst] = ctr; v.count[inst] = count; v.pin[inst] = pin; }
}

__global__ void k_lru_state(LruView v, long long *oldest, long long *weighted, int *count) {
  const int lane = threadIdx.x & 31;
  const int inst = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (inst >= v.n) return;
  long long t, s;
  int slot = lru_min_slot(v, inst, lane, false, 0, 0, &t, &s);
  const long long pin = v.pin[inst];
  if (lane == 0) { oldest[inst] = pin != LRU_PIN_NONE ? pin : slot < 0 ? -1 : t; weighted[inst] = v.wsize[inst]; count[inst] = v.count[inst]; }
}

// dynamic shared memory of a k_lru_events launch with 4 warps per block: room for every warp's staged slot arrays (32 B per
// slot), or none when the instance caches are too large for it
static int lru_stage_slots(mmp_fleet *f, size_t *smem) {
  static std::atomic<bool> attr_set[64];
  const size_t tot = (size_t)f->lru_slots * 32u * 4u;
  *smem = 0;
  if (f->lru_slots <= 0 || tot > (size_t)200 * 1024) return 0;
  if (!attr_set[f->device & 63].load()) {
    if (cudaFuncSetAttribute(k_lru_events, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
    attr_set[f->device & 63] = true;
  }
  *smem = tot;
  return f->lru_slots;
}
static LruView lru_view(mmp_fleet *f) {
  LruView v;
  v.ts = f->lru_ts.as<long long>(); v.seq = f->lru_seq.as<long long>(); v.weight = f->lru_weight.as<int>(); v.model = f->lru_model.as<int>();
  v.loadts = f->lru_loadts.as<long long>();
  v.cap = f->lru_cap.as<long long>(); v.wsize = f->lru_wsize.as<long long>(); v.seqctr = f->lru_seqctr.as<long long>();
  v.count = f->lru_count.as<int>(); v.pin = f->lru_pin.as<long long>(); v.n = f->lru_n; v.slots = f->lru_slots;
  return v;
}

extern "C" {

int32_t mmp_stats(mmp_fleet *f, mmp_cluster_stats *out, int32_t *part_ids, int32_t cap) {
  NEED(f);
  if (!out || !part_ids || cap < 1) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  const DeviceSnapshot &ds = f->snaps[f->cur];
  StatsResult sr;
  rc = run_stats(f, ds, sr);
  if (rc < 0) return rc;
  int n = 0;
  out[n] = sr.parts[0]; part_ids[n] = -1; n++;
  if (ds.host.tc_enabled)
    for (int p : partition_order(sr)) {
      if (n < cap) { out[n] = sr.parts[p + 1]; part_ids[n] = p; }
      n++;
    }
  return n;
}

int32_t mmp_reaper_select(mmp_fleet *f, int32_t partition, int64_t now_ms, uint8_t *taken, int32_t *out_models, int32_t cap) {
  NEED(f);
  return reaper_impl(f, partition, now_ms, taken, out_models, cap);
}

int32_t mmp_lru_init(mmp_fleet *f, int32_t n, const int64_t *capacity, int32_t slots) {
  NEED(f);
  if (n <= 0 || !capacity || slots <= 0 || slots > (1 << 20)) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  size_t tot = (size_t)n * slots;
  CK(f->lru_ts.ensure(tot * 8)); CK(f->lru_seq.ensure(tot * 8)); CK(f->lru_weight.ensure(tot * 4)); CK(f->lru_model.ensure(tot * 4));
  CK(f->lru_loadts.ensure(tot * 8));
  CK(cudaMemset(f->lru_loadts.p, 0xff, tot * 8));
  CK(f->lru_cap.ensure((size_t)n * 8)); CK(f->lru_wsize.ensure((size_t)n * 8)); CK(f->lru_seqctr.ensure((size_t)n * 8)); CK(f->lru_count.ensure((size_t)n * 4));
  CK(f->lru_pin.ensure((size_t)n * 8));
  CK(cudaMemset(f->lru_pin.p, 0x80, (size_t)n * 8));  // LRU_PIN_NONE
  CK(cudaMemset(f->lru_model.p, 0xff, tot * 4));
  CK(cudaMemset(f->lru_wsize.p, 0, (size_t)n * 8)); CK(cudaMemset(f->lru_count.p, 0, (size_t)n * 4));
  std::vector<long long> ctr((size_t)n, 1LL << 40);
  CK(cudaMemcpy(f->lru_seqctr.p, ctr.data(), (size_t)n * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(f->lru_cap.p, capacity, (size_t)n * 8, cudaMemcpyHostToDevice));
  f->lru_n = n; f->lru_slots = slots;
  return MMP_OK;
}

static int32_t lru_apply_impl(mmp_fleet *f, const mmp_lru_event *ev, int32_t n, int64_t now_ms, mmp_eviction *out, int32_t cap,
                              int32_t *status) {
  NEED(f);
  if (n < 0 || (n > 0 && !ev) || cap < 0 || (cap > 0 && !out)) { g_err = "bad argument"; return MMP_E_ARG; }
  if (f->lru_n == 0) { g_err = "mmp_lru_init not called"; return MMP_E_STATE; }
  if (n == 0) return 0;
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  // group events by instance, keeping their order (counting sort)
  std::vector<int> off((size_t)f->lru_n + 1, 0), order((size_t)n);
  std::vector<LruEv> lev((size_t)n);
  for (int32_t i = 0; i < n; i++) {
    if (ev[i].instance < 0 || ev[i].instance >= f->lru_n || ev[i].op < 0 || ev[i].op > MMP_LRU_LOAD || ev[i].last_used < 0 ||
        (ev[i].op != MMP_LRU_SET_CAPACITY && ev[i].model < 0)) { g_err = "bad LRU event"; return MMP_E_ARG; }
    off[ev[i].instance + 1]++;
    lev[i] = LruEv{ev[i].op, ev[i].model, ev[i].weight, i, i, 0, ev[i].last_used, now_ms};
  }
  for (int i = 0; i < f->lru_n; i++) off[i + 1] += off[i];
  { std::vector<int> pos(off.begin(), off.end() - 1); for (int32_t i = 0; i < n; i++) order[pos[ev[i].instance]++] = i; }
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t s = c->stream;
  CK(c->d_in.ensure((size_t)n * sizeof(LruEv)));
  CK(c->d_extra.ensure((size_t)n * 4));
  CK(c->d_fresh.ensure(off.size() * 4));
  CK(c->d_out.ensure((size_t)std::max(cap, 1) * sizeof(EvictRec)));
  CK(c->d_trace.ensure(16 + (size_t)n * 4));
  CK(cudaMemcpyAsync(c->d_in.p, lev.data(), (size_t)n * sizeof(LruEv), cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(c->d_extra.p, order.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(c->d_fresh.p, off.data(), off.size() * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(c->d_trace.p, 0, 16, s));
  CK(cudaMemsetAsync(c->d_trace.as<char>() + 16, 0xff, (size_t)n * 4, s));  // status -1: not a load
  ChurnHooks hk{};
  hk.enabled = 0;
  hk.min_space = f->hs.cfg.min_space_units; hk.min_churn_age = f->hs.cfg.min_churn_age_ms;
  hk.status = c->d_trace.as<int>() + 4;
  const int warps_per_block = 4;
  const int grid = (f->lru_n + warps_per_block - 1) / warps_per_block;
  size_t lsm = 0;
  const int lst = lru_stage_slots(f, &lsm);
  CK(cudaEventRecord(c->e0, s));
  k_lru_events<<<grid, warps_per_block * 32, lsm, s>>>(lru_view(f), c->d_in.as<LruEv>(), c->d_extra.as<int>(), c->d_fresh.as<int>(), now_ms, 0, hk,
                                                      c->d_out.as<EvictRec>(), cap, c->d_trace.as<int>(), c->d_trace.as<int>() + 1, lst);
  CK(cudaEventRecord(c->e1, s));
  f->launches++;
  CK(cudaGetLastError());
  int hdr[2] = {0, 0};
  CK(cudaMemcpyAsync(hdr, c->d_trace.p, 8, cudaMemcpyDeviceToHost, s));
  if (status) CK(cudaMemcpyAsync(status, c->d_trace.as<char>() + 16, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  { float ms = 0; if (cudaEventElapsedTime(&ms, c->e0, c->e1) == cudaSuccess) f->t_lru_ms = ms; }
  if (hdr[1]) { g_err = "LRU slot capacity exceeded for some instance (raise slots_per_instance)"; return MMP_E_NOMEM; }
  int got = std::min(hdr[0], cap);
  std::vector<EvictRec> tmp((size_t)got);
  if (got) CK(cudaMemcpy(tmp.data(), c->d_out.p, (size_t)got * sizeof(EvictRec), cudaMemcpyDeviceToHost));
  // each instance's evictions were appended in its own order (seq); group by instance keeping that order
  std::sort(tmp.begin(), tmp.end(), [](const EvictRec &a, const EvictRec &b) { return a.instance != b.instance ? a.instance < b.instance : a.seq < b.seq; });
  for (int i = 0; i < got; i++) out[i] = mmp_eviction{tmp[i].instance, tmp[i].model, tmp[i].last_used, tmp[i].weight, tmp[i].order};
  return hdr[0];
}

int32_t mmp_lru_apply(mmp_fleet *f, const mmp_lru_event *ev, int32_t n, int64_t now_ms, mmp_eviction *out, int32_t cap) {
  return lru_apply_impl(f, ev, n, now_ms, out, cap, nullptr);
}
int32_t mmp_lru_apply_status(mmp_fleet *f, const mmp_lru_event *ev, int32_t n, int64_t now_ms, mmp_eviction *out, int32_t cap,
                             int32_t *status) {
  return lru_apply_impl(f, ev, n, now_ms, out, cap, status);
}

int32_t mmp_lru_state(mmp_fleet *f, int32_t n, int64_t *oldest, int64_t *weighted, int32_t *count) {
  NEED(f);
  if (n != f->lru_n || !oldest || !weighted || !count) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  CK(c->d_in.ensure((size_t)n * 8)); CK(c->d_out.ensure((size_t)n * 8)); CK(c->d_extra.ensure((size_t)n * 4));
  k_lru_state<<<(n + 3) / 4, 128, 0, c->stream>>>(lru_view(f), c->d_in.as<long long>(), c->d_out.as<long long>(), c->d_extra.as<int>());
  f->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(oldest, c->d_in.p, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(weighted, c->d_out.p, (size_t)n * 8, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaMemcpyAsync(count, c->d_extra.p, (size_t)n * 4, cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  return MMP_OK;
}

}  // extern "C"
