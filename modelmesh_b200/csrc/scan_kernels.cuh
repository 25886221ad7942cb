// scan_kernels.cuh — batch scans (plug points 3 and 4 of include/mmplace.h): ClusterStats reductions, the reaper's
// registry sweep + top-K selection, and the per-instance time-ordered weighted LRU.  Included at the end of mmplace.cu.
#pragma once
#include <cuda/std/tuple>
#include <thrust/iterator/transform_iterator.h>

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
  event_ms(c.get(), f->t_stats_ms);
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
// The reaper's proactive loads (MM:6456-6494, 6574-6577, 6616-6747) for mmp_reaper_select and the closed loop's REAPER
// events, on the caller's stream against one snapshot: the stats of k_stats -> per-partition plan and PARTITION_STATS_COMP
// order (k_rp_plan) -> candidates (k_rp_flag, compaction) -> one radix sort by (lastUsed desc, model asc) -> spaceToFill per
// partition (k_rp_space) -> one block walks the sorted list per run and partition (k_rp_walk; reaper_pass, the closed loop).
// mmp_reaper_select's one run in one partition runs the same stages with its filter in k_rp_flag and k_rp_pick for the walk.
// ---------------------------------------------------------------------------------------------------------------
// the candidate rule of the registry sweep (MM:6574-6577): no loaded copy, fewer than 2 failed loads, used after globalLru
// (0 when the cluster has free space)
__device__ __forceinline__ bool reaper_candidate(const mmp_model_row &r, long long global_lru) {
  return r.copy_count == 0 && r.fail_count < 2 && (global_lru == 0 || r.last_used > global_lru);
}
// one slot per partition (the whole cluster when the pass runs without type constraints), as run_stats reports them
struct RpPart { long long cap, free, glru; int copies, count, size_est, pad; };
struct RpPlan { int go, n_order; long long global_lru; };
MMP_HD long long rp_last_used(unsigned long long key) { return (long long)((~key) ^ 0x8000000000000000ull); }
// One run at clock t in one partition (MM:6621-6664): the free-space count, totalProactiveLoadCount and the lastUsed cutoff from
// the plan and spaceToFill.  false: the size estimate is 0 and spaceToFill / sizeEstimate throws (MM:6651)
MMP_HD bool rp_counts(const RpPart &p, unsigned long long space, long long t, int &free_count, int &total, long long &cutoff) {
  free_count = 0; total = 0;
  if (p.cap > 0 && p.free > 0) {
    if (p.size_est == 0) return false;
    const long long fill = (long long)space / 2;
    free_count = (int32_t)(fill / p.size_est);
    const long long d = (long long)(20ull * (unsigned long long)(long long)p.size_est);
    const int32_t cap_count = d == 0 ? 0 : (int32_t)(d == -1 ? -p.cap : p.cap / d);
    total = free_count > cap_count ? free_count : cap_count;
  }
  const long long a3 = age_of(p.glru, t) / 3;
  cutoff = p.glru == 0x7fffffffffffffffLL ? 0 : (long long)((unsigned long long)p.glru + (unsigned long long)(a3 > 1200000 ? a3 : 1200000));
  return true;
}
// the emission rule (MM:6711-6719) for the k-th counted entry of a run in a partition
MMP_HD bool rp_emits(int k, int free_count, int total, long long last_used, long long cutoff) {
  return k < total && (k < free_count || !(last_used < cutoff));
}

// slot >= 0: the runs walk that partition alone, whatever its stats.  Also zeroes the spaceToFill sums k_rp_space adds into.
__global__ void k_rp_plan(const StatsAcc *__restrict__ acc, const long long *__restrict__ min_lru, int n_slots, int tc, int slot,
                          int def_size, RpPart *__restrict__ parts, int *__restrict__ order, RpPlan *__restrict__ plan,
                          unsigned long long *__restrict__ space) {
  const long long mn = *min_lru;
  for (int s = threadIdx.x; s < n_slots; s += blockDim.x) {
    space[s] = 0;
    const StatsAcc a = acc[tc ? 1 + s : 0];
    RpPart p{(long long)a.cap, (long long)a.free, (a.count > 0 || !tc) ? mn : 0x7fffffffffffffffLL, a.copies, a.count, 0, 0};
    if (p.copies < 3) p.size_est = def_size;  // MM:6622-6629
    else {
      const int32_t avg = (int32_t)jsub(p.cap, p.free) / p.copies;
      p.size_est = p.copies > 10 ? avg : jaddi(avg, def_size) / 2;
    }
    parts[s] = p;
  }
  __syncthreads();
  // PARTITION_STATS_COMP (TCM:264-271) as partition_order: free desc, lru asc, capacity desc, partition id; with instances only
  __shared__ int n_in;
  if (threadIdx.x == 0) n_in = 0;
  __syncthreads();
  for (int s = threadIdx.x; s < n_slots; s += blockDim.x) {
    const RpPart x = parts[s];
    if (tc && x.count == 0) continue;
    int rank = 0;
    for (int o = 0; o < n_slots; o++) {
      const RpPart y = parts[o];
      if (o == s || (tc && y.count == 0)) continue;
      rank += y.free != x.free ? y.free > x.free : y.glru != x.glru ? y.glru < x.glru : y.cap != x.cap ? y.cap > x.cap : o < s;
    }
    order[rank] = s;
    atomicAdd(&n_in, 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {  // MM:6456-6463
    plan->go = (long long)acc[0].cap > 0;
    plan->global_lru = (long long)acc[0].free > 0 ? 0 : mn;
    plan->n_order = slot < 0 ? n_in : 1;
    if (slot >= 0) order[0] = slot;
  }
}
// With a filter (mmp_reaper_select: one run in one partition) the candidates are only those the run may select: not taken
// (allCandidates.set(i, null)), type allowed in the partition (MM:6681-6683), used after the cutoff without free space (MM:6685-6687)
struct RpFilter { const uint8_t *taken, *type_excluded; int n_type_ids, need_cutoff; long long cutoff; };
__global__ void k_rp_flag(const mmp_model_row *__restrict__ models, int n_models, const RpPlan *__restrict__ plan, RpFilter flt,
                          uint8_t *__restrict__ flag) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  const RpPlan p = *plan;
  const mmp_model_row r = models[m];
  bool ok = p.go && reaper_candidate(r, p.global_lru);
  if (ok && flt.taken && flt.taken[m]) ok = false;
  if (ok && r.type_id < flt.n_type_ids && flt.type_excluded[r.type_id]) ok = false;
  if (ok && flt.need_cutoff && !(r.last_used > flt.cutoff)) ok = false;
  flag[m] = ok ? 1 : 0;
}
// sort keys of the compacted candidates (in model order), ~biased(lastUsed) so that ascending keys = descending time; the
// positions past them sort last
__global__ void k_rp_keys(const mmp_model_row *__restrict__ models, const int *__restrict__ idx, const int *__restrict__ n_cand, int n,
                          unsigned long long *__restrict__ key) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  key[i] = i < *n_cand ? ~((unsigned long long)models[idx[i]].last_used ^ 0x8000000000000000ull) : ~0ull;
}
// spaceToFill (MM:6633-6649) per partition: one segmented reduction over the rank-ordered instance columns, in the reference's
// wrapping int / long arithmetic (the sum wraps too, so the order of the additions does not matter)
__global__ void k_rp_space(const RankRow *__restrict__ rows, const int64_t *__restrict__ cap_col, const int32_t *__restrict__ lthreads,
                           const int32_t *__restrict__ linprog, const int32_t *__restrict__ part_of_rank, int n_ranks, int tc, int n_slots,
                           const RpPart *__restrict__ parts, unsigned long long *__restrict__ space) {
  __shared__ unsigned long long sacc[STATS_SMEM_PARTS + 1];
  const bool use_smem = n_slots <= STATS_SMEM_PARTS + 1;
  if (use_smem) for (int i = threadIdx.x; i < n_slots; i += blockDim.x) sacc[i] = 0ull;
  __syncthreads();
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n_ranks; r += gridDim.x * blockDim.x) {
    const int s = tc ? part_of_rank[r] : 0;
    if (s < 0 || s >= n_slots) continue;
    const int32_t max_loads = (int32_t)((uint32_t)jmuli(lthreads[r], 50) - (uint32_t)linprog[r]);
    if (max_loads <= 0) continue;
    const int64_t avail = jsub(rows[r].rem, cap_col[r] / 8);
    if (avail <= 0) continue;
    const int64_t lim = (int64_t)jmuli(max_loads, parts[s].size_est);
    atomicAdd(use_smem ? &sacc[s] : &space[s], (unsigned long long)(avail < lim ? avail : lim));
  }
  if (use_smem) {
    __syncthreads();
    for (int i = threadIdx.x; i < n_slots; i += blockDim.x) if (sacc[i]) atomicAdd(&space[i], sacc[i]);
  }
}
// The selection of every run (clock run_t[r]), one after the other, by one block: for each partition in the plan's order, the
// sorted candidates are walked in chunks of RP_WALK.  Per chunk: eligible = not taken by
// this run, type allowed in the partition (MM:6681-6683) and (free space or lastUsed > cutoff) (MM:6685-6688); of an
// equal-lastUsed run of eligible entries only the first counts (N12; a block-wide max scan finds each entry's previous
// eligible entry); the counted entries take ranks k by a block-wide sum scan, and the first totalProactiveLoadCount of them
// go through the emission rule (MM:6711-6719), which, the list being in descending lastUsed, emits a prefix of them.  The walk
// stops at the count, at the rule's break, or (full partition) at the first entry at or under the cutoff.  Emitted models are
// tagged taken and appended as (model, run).  sel_off = [the runs' offsets | total].
constexpr int RP_WALK = 1024;
__global__ void __launch_bounds__(RP_WALK) k_rp_walk(const mmp_model_row *__restrict__ models, const unsigned long long *__restrict__ skey,
                                                      const int *__restrict__ sidx, const int *__restrict__ n_cand, const RpPlan *__restrict__ plan,
                                                      const RpPart *__restrict__ parts, const int *__restrict__ order,
                                                      const unsigned long long *__restrict__ space, int tc, const int *__restrict__ pt_off,
                                                      const int *__restrict__ pt_ids, const long long *__restrict__ run_t, int n_rp, int gen0,
                                                      int *__restrict__ taken, int2 *__restrict__ sel, long long sel_cap, int *__restrict__ sel_off) {
  using Scan = cub::BlockScan<int, RP_WALK>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ unsigned long long chunk_key[RP_WALK];
  const int tid = threadIdx.x;
  const int ncand = *n_cand;
  const RpPlan P = *plan;
  long long out = 0;
  for (int r = 0; r < n_rp; r++) {
    if (tid == 0) sel_off[r] = (int)out;
    const int gen = gen0 + r;
    const long long t = run_t[r];
    for (int oi = 0; P.go && ncand > 0 && oi < P.n_order; oi++) {
      const int s = order[oi];
      const RpPart p = parts[s];
      int free_count, total;
      long long cutoff;
      if (!rp_counts(p, space[s], t, free_count, total, cutoff)) break;  // the exception: the run ends here
      if (total <= 0) continue;
      const int *ex = tc ? pt_ids + pt_off[s] : nullptr;
      const int nex = tc ? pt_off[s + 1] - pt_off[s] : 0;
      int kept = 0, emitted = 0;
      bool have_prev = false;
      unsigned long long prev_key = 0;
      for (int base = 0; base < ncand; base += RP_WALK) {
        const int i = base + tid;
        int m = -1;
        unsigned long long key = ~0ull;
        bool elig = false;
        if (i < ncand) {
          m = sidx[i]; key = skey[i];
          elig = taken[m] != gen && (free_count > 0 || rp_last_used(key) > cutoff);
          if (elig && nex) {  // the partition's prohibited type ids, sorted
            const int ty = models[m].type_id;
            int lo = 0, hi = nex;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (ex[mid] < ty) lo = mid + 1; else hi = mid; }
            elig = !(lo < nex && ex[lo] == ty);
          }
        }
        chunk_key[tid] = key;
        int prev, last;
        Scan(tmp).ExclusiveScan(elig ? tid : -1, prev, -1, cub::Max(), last);
        __syncthreads();
        const bool hp = prev >= 0 || have_prev;
        const unsigned long long pk = prev >= 0 ? chunk_key[prev] : prev_key;
        const int first = elig && !(hp && pk == key) ? 1 : 0;
        int j, n_first;
        Scan(tmp).ExclusiveSum(first, j, n_first);
        const int k = kept + j;
        const bool emit = first && rp_emits(k, free_count, total, rp_last_used(key), cutoff);
        const int n_emit = __syncthreads_count(emit);
        if (emit) {
          taken[m] = gen;
          const long long pos = out + k;
          if (pos < sel_cap) sel[pos] = make_int2(m, r);
        }
        kept += n_first; emitted += n_emit;
        if (last >= 0) { have_prev = true; prev_key = chunk_key[last]; }
        bool stop = n_emit < n_first || kept >= total || base + RP_WALK >= ncand;
        if (free_count == 0 && rp_last_used(chunk_key[RP_WALK - 1]) <= cutoff) stop = true;  // nothing eligible past it
        __syncthreads();
        if (stop) break;
      }
      out += emitted;
    }
  }
  if (tid == 0) sel_off[n_rp] = (int)out;
}

// mmp_reaper_select's run over its filtered candidates, sorted: only the first of an equal-lastUsed run counts (N12, an entry
// whose key differs from its predecessor's); rank[i] = the counted entries before i.  The emission rule then emits a prefix of
// the counted entries (the list descends in lastUsed): out[k] = the k-th, n_out = how many.
struct RpFirst {
  const unsigned long long *key;
  __device__ int operator()(int i) const { return i == 0 || key[i] != key[i - 1] ? 1 : 0; }
};
__global__ void k_rp_pick(const unsigned long long *__restrict__ skey, const int *__restrict__ sidx, const int *__restrict__ rank, int n,
                          int free_count, int total, long long cutoff, int *__restrict__ out, int *__restrict__ n_out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long key = skey[i];
  if (i > 0 && skey[i - 1] == key) return;
  const int k = rank[i];
  if (!rp_emits(k, free_count, total, rp_last_used(key), cutoff)) return;
  out[k] = sidx[i];
  atomicMax(n_out, k + 1);
}

// The pass's stages, on stream st after k_stats filled acc / min_lru for the snapshot ds.  tc = 0: one slot, the whole
// cluster with no type exclusion; slot >= 0: the runs take that partition alone.
struct RpBufs { RpPart *parts; unsigned long long *space; RpPlan *plan; int *order; };
// plan and PARTITION_STATS_COMP order (k_rp_plan), spaceToFill per partition (k_rp_space)
static int32_t rp_plan_stage(mmp_fleet *f, const DeviceSnapshot &ds, int tc, int slot, const StatsAcc *acc, const long long *min_lru,
                             RpScratch &rs, cudaStream_t st, RpBufs &b) {
  const HostSnapshot &h = ds.host;
  const int ns = tc ? (int)h.part_types.size() : 1;
  const size_t parts_b = (size_t)ns * sizeof(RpPart), space_b = (size_t)ns * 8;
  CK(rs.plan.ensure(parts_b + space_b + sizeof(RpPlan) + (size_t)ns * 4 + 16));
  b.parts = rs.plan.as<RpPart>();
  b.space = reinterpret_cast<unsigned long long *>(rs.plan.as<char>() + parts_b);
  b.plan = reinterpret_cast<RpPlan *>(rs.plan.as<char>() + parts_b + space_b);
  b.order = reinterpret_cast<int *>(b.plan + 1);
  k_rp_plan<<<1, 256, 0, st>>>(acc, min_lru, ns, tc, slot, f->hs.cfg.default_model_size_units, b.parts, b.order, b.plan, b.space);
  if (h.n_ranks > 0)
    k_rp_space<<<std::min(f->sm_count, (h.n_ranks + 255) / 256), 256, 0, st>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(),
                                                                            ds.lthreads_col.as<int32_t>(), ds.linprog_col.as<int32_t>(),
                                                                            ds.part_of_rank.as<int32_t>(), h.n_ranks, tc, ns, b.parts, b.space);
  f->launches += 1 + (h.n_ranks > 0);
  CK(cudaGetLastError());
  return MMP_OK;
}
// the candidates (k_rp_flag) compacted in model order into rs.idx, their count behind the sorted indices; cub_tmp is sized for
// the compaction and for a sort of every model
static int32_t rp_candidates(mmp_fleet *f, const mmp_model_row *models, int NM, const RpPlan *plan, const RpFilter &flt, RpScratch &rs,
                             DevBuf &cub_tmp, cudaStream_t st, int **d_n) {
  const size_t nmx = (size_t)std::max(NM, 1);
  CK(rs.keys.ensure(nmx * 16)); CK(rs.idx.ensure(nmx * 8 + 16)); CK(rs.flag.ensure(nmx));
  unsigned long long *keys = rs.keys.as<unsigned long long>();
  int *idx = rs.idx.as<int>();
  *d_n = idx + 2 * nmx;
  k_rp_flag<<<(int)((nmx + 255) / 256), 256, 0, st>>>(models, NM, plan, flt, rs.flag.as<uint8_t>());
  thrust::counting_iterator<int32_t> iota(0);
  size_t t1 = 0, t2 = 0;
  CK(cub::DeviceSelect::Flagged(nullptr, t1, iota, rs.flag.as<uint8_t>(), idx, *d_n, NM, st));
  CK(cub::DeviceRadixSort::SortPairs(nullptr, t2, keys, keys + nmx, idx, idx + nmx, NM, 0, 64, st));
  CK(cub_tmp.ensure(std::max(t1, t2) + 16));
  CK(cub::DeviceSelect::Flagged(cub_tmp.p, t1, iota, rs.flag.as<uint8_t>(), idx, *d_n, NM, st));
  f->launches += 2;
  CK(cudaGetLastError());
  return MMP_OK;
}
// the first n compacted entries by (lastUsed desc, model asc) (k_rp_keys + a stable radix sort) into rs.keys + nmx / rs.idx + nmx
static int32_t rp_sort(mmp_fleet *f, const mmp_model_row *models, int NM, int n, RpScratch &rs, DevBuf &cub_tmp, cudaStream_t st) {
  const size_t nmx = (size_t)std::max(NM, 1);
  unsigned long long *keys = rs.keys.as<unsigned long long>();
  int *idx = rs.idx.as<int>();
  k_rp_keys<<<(int)((std::max(n, 1) + 255) / 256), 256, 0, st>>>(models, idx, idx + 2 * nmx, n, keys);
  size_t t = cub_tmp.cap;
  CK(cub::DeviceRadixSort::SortPairs(cub_tmp.p, t, keys, keys + nmx, idx, idx + nmx, n, 0, 64, st));
  f->launches += 3;
  CK(cudaGetLastError());
  return MMP_OK;
}

// The closed loop's selection for the runs run_t (their clocks): every run walks the partitions in PARTITION_STATS_COMP
// order over all the candidates, sorted once (k_rp_walk).  Run r tags the models it selects gen + 1 + r in rs.taken, which the
// caller fills (tags other than the run's own do not count as taken); gen advances past the tags used.  Selections land in
// rs.sel as (model, run) in emission order, their offsets per run in rs.off.  The total is read back (one synchronisation);
// a second walk follows only when the selections outgrow rs.sel.
static int32_t reaper_pass(mmp_fleet *f, const DeviceSnapshot &ds, const mmp_model_row *models, int n_models, int tc,
                           const StatsAcc *acc, const long long *min_lru, const std::vector<long long> &run_t, int32_t &gen,
                           RpScratch &rs, DevBuf &cub_tmp, cudaStream_t st, int32_t *n_sel) {
  const HostSnapshot &h = ds.host;
  const int NM = n_models, R = (int)run_t.size(), ns = tc ? (int)h.part_types.size() : 1;
  const size_t nmx = (size_t)std::max(NM, 1);
  // one upload: the runs' clocks, then each partition's prohibited type ids of this epoch, sorted: [offsets (ns + 1) | ids]
  std::vector<int> pt((size_t)ns + 1, 0);
  for (int p = 0; tc && p < ns; p++) {
    std::vector<int> ids;
    for (int32_t tid : h.part_type_ids[p]) if (tid >= 0 && tid < (int32_t)h.type_slot.size()) ids.push_back(tid);
    std::sort(ids.begin(), ids.end());
    pt.insert(pt.end(), ids.begin(), ids.end());
    pt[p + 1] = pt[p] + (int)ids.size();
  }
  std::vector<long long> up(run_t);
  up.resize((size_t)R + (pt.size() + 1) / 2);
  memcpy(up.data() + R, pt.data(), pt.size() * 4);
  CK(upload_vec(rs.runs, up, st));
  const long long *d_t = rs.runs.as<long long>();
  const int *pt_off = reinterpret_cast<const int *>(d_t + R), *pt_ids = pt_off + ns + 1;
  CK(rs.sel.ensure(nmx * sizeof(int2)));  // (one run selects each model at most once)
  CK(rs.off.ensure((size_t)(R + 1) * 4));
  RpBufs b;
  int *d_n = nullptr;
  int32_t rc = rp_plan_stage(f, ds, tc, -1, acc, min_lru, rs, st, b);
  if (rc == MMP_OK) rc = rp_candidates(f, models, NM, b.plan, RpFilter{}, rs, cub_tmp, st, &d_n);
  if (rc == MMP_OK) rc = rp_sort(f, models, NM, NM, rs, cub_tmp, st);  // (the positions past the candidates sort last)
  if (rc < 0) return rc;
  const unsigned long long *skeys = rs.keys.as<unsigned long long>() + nmx;
  const int *sidx = rs.idx.as<int>() + nmx;
  int *d_off = rs.off.as<int>();
  for (int pass = 0;; pass++) {
    const long long sel_cap = (long long)(rs.sel.cap / sizeof(int2));
    k_rp_walk<<<1, RP_WALK, 0, st>>>(models, skeys, sidx, d_n, b.plan, b.parts, b.order, b.space, tc, pt_off, pt_ids, d_t, R, gen + 1,
                                     rs.taken.as<int>(), rs.sel.as<int2>(), sel_cap, d_off);
    f->launches++;
    CK(cudaGetLastError());
    gen += R;
    int total = 0;
    CK(cudaMemcpyAsync(&total, d_off + R, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (total <= sel_cap) { *n_sel = total; return MMP_OK; }
    if (pass) { g_err = "internal: the reaper's selections changed between two walks"; return MMP_E_STATE; }
    CK(rs.sel.ensure((size_t)total * sizeof(int2)));
  }
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
  const int4 *edges;               // [n_models] registrations 0-3 (first copy_count = loaded)
  const mmp_model_row *models;
  unsigned *rm_mask;               // [n_models] bit j < 4: registration j is deregistered at the end of the epoch; RM_OVF: a later one is
  const unsigned char *type_ok;    // [n_type_ids] the type set is < 95 % full (MM:2918-2920)
  int n_type_ids;
  Follow *next; int *n_next; int next_cap;
  unsigned char *force_publish;    // [n_instances]
};
// the hooks' overflow registrations (LiveState::ovf), a launch argument of their own after the others: as fields of ChurnHooks
// they move every later argument, and the compiler gives the kernel another register allocation
struct OvfHooks {
  const OvfEdge *ovf; int n_ovf;
  unsigned char *dead;             // [n_ovf] the overflow registration is deregistered at the end of the epoch
};
#define RM_OVF (1u << 4)

// deregisterModel / the listener's deregistration (MM:2875-2931): mark the model's loaded copy on `inst` at whatever position it
// holds.  Copies of one model on different instances are marked by different warps of the same launch: bits by atomicOr, and
// each overflow position has a flag byte of its own.  OVF = false (no overflow table) compiles the four inline positions only.
template <bool OVF>
__device__ __forceinline__ void churn_deregister(const ChurnHooks &hk, const OvfHooks &ov, int m, int inst) {
  const int4 ed = hk.edges[m];
  const int cc = hk.models[m].copy_count;
  const int es[4] = {ed.x, ed.y, ed.z, ed.w};
  for (int j = 0; j < 4 && j < cc; j++) if (es[j] == inst) atomicOr(&hk.rm_mask[m], 1u << j);
  if (OVF && cc > 4) {
    const RegTables R{hk.edges, nullptr, ov.ovf, ov.n_ovf};
    const ModelRegs g = model_regs(R, m, (unsigned)cc);
    for (int j = 4; j < cc; j++) {
      long long ts;
      if (reg_at(R, g, j, ts) == inst) { ov.dead[g.ovf0 + j - 4] = 1; atomicOr(&hk.rm_mask[m], RM_OVF); }
    }
  }
}

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
// OVF: the hooks' registry has an overflow table (a model may hold more than four registrations).
template <bool OVF>
__global__ void k_lru_events(LruView v, const LruEv *__restrict__ ev, const int *__restrict__ ev_order, const int *__restrict__ inst_off,
                             long long now_param, int use_ev_time, ChurnHooks hk, EvictRec *out, int out_cap, int *out_n, int *err, int stage_slots,
                             OvfHooks ov) {
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
          if (in_registry) churn_deregister<OVF>(hk, ov, m, inst);
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
          if (lt >= 0) churn_deregister<OVF>(hk, ov, e.model, inst);  // deregisterModel
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

// ---------------------------------------------------------------------------------------------------------------
// Read side: descendingMapWithCutoff / descendingLruMap (CLHM:1226-1260, 1087-1116), getLastUsedTime / getWeight
// (CLHM:742-771).  The walk from the MRU end stops at the first node with 0 < lastUsed < usedSince.  The deque is in (ts, seq)
// order, so the walk returns every entry with ts >= used_since, and the entries with ts <= 0 (which lie below every positive
// time) only when no entry has 0 < ts < used_since.  The kernels only read the slot arrays k_lru_events writes.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool lru_read_passes(long long ts, long long used_since, bool stops) {
  return ts >= used_since || (ts <= 0 && !stops);
}

// one warp per listed cache: the length of its walk (cnt[k]) and whether the walk stops before its end (stops[k]);
// cnt[n] is left for the caller to zero, so the exclusive scan of cnt[0 .. n] is the offsets array
__global__ void k_lru_read_count(LruView v, const int *__restrict__ inst, int n, long long used_since, long long *__restrict__ cnt,
                                 unsigned char *__restrict__ stops) {
  const int lane = threadIdx.x & 31;
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (k >= n) return;
  const size_t base = (size_t)inst[k] * v.slots;
  int since = 0, nonpos = 0;
  bool stop = false;
  for (int i = lane; i < v.slots; i += 32) {
    if (v.model[base + i] < 0) continue;
    const long long t = v.ts[base + i];
    since += t >= used_since;
    nonpos += t <= 0 && t < used_since;
    stop |= t > 0 && t < used_since;
  }
  stop = __any_sync(0xffffffffu, stop);
  since = __reduce_add_sync(0xffffffffu, since);
  nonpos = __reduce_add_sync(0xffffffffu, nonpos);
  if (lane == 0) { cnt[k] = since + (stop ? 0 : nonpos); stops[k] = stop; }
}

__device__ __forceinline__ mmp_lru_entry lru_read_entry(const LruView &v, size_t at, int loop) {
  return mmp_lru_entry{v.model[at], v.weight[at], v.ts[at], loop ? v.loadts[at] : -1};
}

// One block per listed cache whose walk has at most LRU_READ_SMEM entries and starts before `cap`: the passing entries go to
// shared memory, and each one's rank is the number of entries with a larger (ts, seq) key.  Keys are unique within a cache
// (a fresh seq per insert or move, the successor's seq - 1 for a tie with it), so the ranks are a permutation.
static constexpr int LRU_READ_SMEM = 2048;  // 20 B per entry: 40 KB of static shared memory
__global__ void __launch_bounds__(256) k_lru_read_emit(LruView v, const int *__restrict__ inst, const long long *__restrict__ off,
                                                       const unsigned char *__restrict__ stops, long long used_since, int loop,
                                                       mmp_lru_entry *__restrict__ out, long long cap) {
  __shared__ long long s_ts[LRU_READ_SMEM], s_seq[LRU_READ_SMEM];
  __shared__ int s_slot[LRU_READ_SMEM];
  __shared__ int s_n;
  const int k = blockIdx.x;
  const long long o = off[k], c = off[k + 1] - o;
  if (c == 0 || c > LRU_READ_SMEM || o >= cap) return;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  const size_t base = (size_t)inst[k] * v.slots;
  const bool stop = stops[k];
  for (int i = threadIdx.x; i < v.slots; i += blockDim.x) {
    if (v.model[base + i] < 0) continue;
    const long long t = v.ts[base + i];
    if (!lru_read_passes(t, used_since, stop)) continue;
    const int p = atomicAdd(&s_n, 1);
    s_ts[p] = t; s_seq[p] = v.seq[base + i]; s_slot[p] = i;
  }
  __syncthreads();
  for (int p = threadIdx.x; p < (int)c; p += blockDim.x) {
    const long long t = s_ts[p], q = s_seq[p];
    int r = 0;
    for (int j = 0; j < (int)c; j++) r += key_less(t, q, s_ts[j], s_seq[j]);
    if (o + r < cap) out[o + r] = lru_read_entry(v, base + s_slot[p], loop);
  }
}

// The global-memory path, for walks longer than LRU_READ_SMEM: the passing entries of every such cache are keyed
// (segment, ~ts, ~seq), sorted ascending by one radix sort, and a position's rank is its distance from its segment's start.
struct LruReadKey { unsigned seg; unsigned long long nts, nseq; };
struct LruReadKeyParts {
  __host__ __device__ ::cuda::std::tuple<unsigned &, unsigned long long &, unsigned long long &> operator()(LruReadKey &k) const {
    return {k.seg, k.nts, k.nseq};
  }
};
__device__ __forceinline__ unsigned long long lru_desc_bits(long long x) { return ~((unsigned long long)x ^ 0x8000000000000000ull); }

// one block per segment (listed cache big[b]): its passing entries, keyed, from seg_off[b] on
__global__ void k_lru_read_gather(LruView v, const int *__restrict__ inst, const unsigned char *__restrict__ stops, long long used_since,
                                  const int *__restrict__ big, const long long *__restrict__ seg_off, LruReadKey *__restrict__ keys,
                                  int *__restrict__ slot_of) {
  __shared__ int s_n;
  const int b = blockIdx.x, k = big[b];
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  const size_t base = (size_t)inst[k] * v.slots;
  const bool stop = stops[k];
  for (int i = threadIdx.x; i < v.slots; i += blockDim.x) {
    if (v.model[base + i] < 0) continue;
    const long long t = v.ts[base + i];
    if (!lru_read_passes(t, used_since, stop)) continue;
    const long long p = seg_off[b] + atomicAdd(&s_n, 1);
    keys[p] = LruReadKey{(unsigned)b, lru_desc_bits(t), lru_desc_bits(v.seq[base + i])};
    slot_of[p] = i;
  }
}
__global__ void k_lru_read_scatter(LruView v, const int *__restrict__ inst, const long long *__restrict__ off, const int *__restrict__ big,
                                   const long long *__restrict__ seg_off, const LruReadKey *__restrict__ keys, const int *__restrict__ slot_of,
                                   long long total, int loop, mmp_lru_entry *__restrict__ out, long long cap) {
  const long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= total) return;
  const unsigned b = keys[p].seg;
  const int k = big[b];
  const long long dst = off[k] + (p - seg_off[b]);
  if (dst < cap) out[dst] = lru_read_entry(v, (size_t)inst[k] * v.slots + slot_of[p], loop);
}

// one warp per (instance, model) query
__global__ void k_lru_lookup(LruView v, int n, const int *__restrict__ inst, const int *__restrict__ model, int loop,
                             long long *__restrict__ last_used, int *__restrict__ weight, long long *__restrict__ load_ts) {
  const int lane = threadIdx.x & 31;
  const int q = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (q >= n) return;
  const int m = model[q];
  int fr;
  const int slot = m < 0 ? -1 : lru_find(v, inst[q], lane, m, &fr);  // (a negative key would match a free slot)
  if (lane) return;
  const size_t at = (size_t)inst[q] * v.slots + (slot < 0 ? 0 : slot);
  const long long t = slot < 0 ? -1 : v.ts[at];
  last_used[q] = t <= 0 ? -1 : t;
  weight[q] = slot < 0 ? -1 : v.weight[at];
  load_ts[q] = slot < 0 || !loop ? -1 : v.loadts[at];
}

// dynamic shared memory of a k_lru_events launch with 4 warps per block: room for every warp's staged slot arrays (32 B per
// slot), or none when the instance caches are too large for it
static int lru_stage_slots(mmp_fleet *f, size_t *smem) {
  static std::atomic<bool> attr_set[64];
  const size_t tot = (size_t)f->lru_slots * 32u * 4u;
  *smem = 0;
  if (f->lru_slots <= 0 || tot > (size_t)200 * 1024) return 0;
  if (!attr_set[f->device & 63].load()) {
    if (cudaFuncSetAttribute(k_lru_events<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess ||
        cudaFuncSetAttribute(k_lru_events<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024) != cudaSuccess) { (void)cudaGetLastError(); return 0; }
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

// One run at now_ms on the lease's stream, in one partition: -1 is the whole cluster without type exclusion (on a constrained
// fleet too), p >= 0 that partition alone.  The pass's stages with a read-back after each: the plan (the call ends when the
// run has nothing to select), the candidates the run may select (k_rp_flag with its filter: ends when there are none), their
// sort, and k_rp_pick, the walk's N12 and emission rule over one run's list in parallel.
int32_t mmp_reaper_select(mmp_fleet *f, int32_t partition, int64_t now_ms, uint8_t *taken, int32_t *out_models, int32_t cap) {
  NEED(f);
  if (!out_models || cap < 0) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::shared_lock<std::shared_mutex> rd(f->snap_mu);
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  const DeviceSnapshot &ds = f->snaps[f->cur];
  const HostSnapshot &h = ds.host;
  const int np = (int)h.part_types.size(), nm = ds.n_models, tc = partition >= 0 ? 1 : 0;
  if (partition >= np || (partition >= 0 && !h.tc_enabled)) { g_err = "no such partition"; return MMP_E_ARG; }
  if (nm == 0) return 0;
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t s = c->stream;
  RpScratch &rs = c->rp;
  const mmp_model_row *models = ds.models.as<mmp_model_row>();
  // stats: [acc (np + 1) | the cluster's LRU, from Long.MAX_VALUE (ISST)]
  const size_t acc_b = (size_t)(np + 1) * sizeof(StatsAcc);
  CK(c->d_trace.ensure(acc_b + 8));
  long long *d_min = reinterpret_cast<long long *>(c->d_trace.as<char>() + acc_b);
  static const long long lru_init = 0x7fffffffffffffffLL;
  CK(cudaMemsetAsync(c->d_trace.p, 0, acc_b, s));
  CK(cudaMemcpyAsync(d_min, &lru_init, 8, cudaMemcpyHostToDevice, s));
  if (h.n_ranks > 0) {
    k_stats<<<std::min(f->sm_count, (h.n_ranks + 255) / 256), 256, 0, s>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(),
                                                                          ds.part_of_rank.as<int32_t>(), h.n_ranks, f->hs.cfg.min_space_units,
                                                                          c->d_trace.as<StatsAcc>(), d_min, np);
    f->launches++;
  }
  RpBufs b;
  const int slot = tc ? partition : 0, ns = tc ? np : 1;
  rc = rp_plan_stage(f, ds, tc, slot, c->d_trace.as<StatsAcc>(), d_min, rs, s, b);
  if (rc < 0) return rc;
  // one read-back of [parts | space | plan] (b's layout in rs.plan)
  std::vector<char> hb((size_t)ns * (sizeof(RpPart) + 8) + sizeof(RpPlan));
  CK(cudaMemcpyAsync(hb.data(), rs.plan.p, hb.size(), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  RpPart part;
  RpPlan plan;
  unsigned long long space;
  memcpy(&part, hb.data() + (size_t)slot * sizeof(RpPart), sizeof(RpPart));
  memcpy(&space, hb.data() + (size_t)ns * sizeof(RpPart) + (size_t)slot * 8, 8);
  memcpy(&plan, hb.data() + (size_t)ns * (sizeof(RpPart) + 8), sizeof(RpPlan));
  if (!plan.go) return 0;  // MM:6456
  int free_count = 0, total = 0;
  long long cutoff = 0;
  const bool counted = rp_counts(part, space, now_ms, free_count, total, cutoff);
  if (counted && total <= 0) return 0;
  auto timed = [&](int32_t r) {  // t_reaper_ms: from the candidate sweep to the last stage run
    event_ms(c.get(), f->t_reaper_ms);
    return r;
  };
  // the candidates: those of the base rule alone when the size estimate is 0 (the reference throws only when there is one,
  // MM:6470), else those this run may select
  RpFilter flt{};
  std::vector<uint8_t> excl(tc ? h.type_slot.size() : 0, 0);
  if (counted) {
    for (int32_t tid : tc ? h.part_type_ids[partition] : std::vector<int32_t>())
      if (tid >= 0 && tid < (int32_t)excl.size()) excl[tid] = 1;
    CK(c->d_extra.ensure(excl.size() + 16));
    if (!excl.empty()) CK(cudaMemcpyAsync(c->d_extra.p, excl.data(), excl.size(), cudaMemcpyHostToDevice, s));
    if (taken) {
      CK(c->d_fresh.ensure((size_t)nm));
      CK(cudaMemcpyAsync(c->d_fresh.p, taken, (size_t)nm, cudaMemcpyHostToDevice, s));
    }
    flt = RpFilter{taken ? c->d_fresh.as<uint8_t>() : nullptr, c->d_extra.as<uint8_t>(), (int)excl.size(), free_count > 0 ? 0 : 1, cutoff};
  }
  int *d_n = nullptr;
  CK(cudaEventRecord(c->e0, s));
  rc = rp_candidates(f, models, nm, b.plan, flt, rs, c->d_cub, s, &d_n);
  if (rc < 0) return rc;
  int ncand = 0;
  CK(cudaMemcpyAsync(&ncand, d_n, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(c->e1, s));
  CK(cudaStreamSynchronize(s));
  if (ncand == 0) return timed(0);
  if (!counted) { timed(0); g_err = "size estimate is zero (the reference would throw ArithmeticException)"; return MMP_E_ARG; }
  rc = rp_sort(f, models, nm, ncand, rs, c->d_cub, s);
  if (rc < 0) return rc;
  const size_t nmx = (size_t)nm;
  int *rank = rs.idx.as<int>();  // (the unsorted indices are spent)
  int *out = reinterpret_cast<int *>(rs.keys.as<unsigned long long>());
  CK(rs.sel.ensure(16));
  int *d_out_n = rs.sel.as<int>();
  auto first = thrust::make_transform_iterator(thrust::counting_iterator<int>(0), RpFirst{rs.keys.as<unsigned long long>() + nmx});
  size_t t = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, t, first, rank, ncand, s));
  CK(c->d_cub.ensure(t + 16));
  CK(cub::DeviceScan::ExclusiveSum(c->d_cub.p, t, first, rank, ncand, s));
  CK(cudaMemsetAsync(d_out_n, 0, 4, s));
  k_rp_pick<<<(ncand + 255) / 256, 256, 0, s>>>(rs.keys.as<unsigned long long>() + nmx, rs.idx.as<int>() + nmx, rank, ncand, free_count,
                                                total, cutoff, out, d_out_n);
  f->launches += 2;
  CK(cudaGetLastError());
  int n = 0;
  CK(cudaMemcpyAsync(&n, d_out_n, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(c->e1, s));
  CK(cudaStreamSynchronize(s));
  timed(0);
  std::vector<int32_t> sel((size_t)n);
  if (n) {
    CK(cudaMemcpyAsync(sel.data(), out, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
  }
  for (int32_t i = 0; i < n; i++) {  // every selection is taken, those past cap too
    if (taken) taken[sel[i]] = 1;
    if (i < cap) out_models[i] = sel[i];
  }
  return n;
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
  f->lru_n = n; f->lru_slots = slots; f->lru_loop = false;
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
  k_lru_events<false><<<grid, warps_per_block * 32, lsm, s>>>(lru_view(f), c->d_in.as<LruEv>(), c->d_extra.as<int>(), c->d_fresh.as<int>(), now_ms, 0, hk,
                                                      c->d_out.as<EvictRec>(), cap, c->d_trace.as<int>(), c->d_trace.as<int>() + 1, lst, OvfHooks{});
  CK(cudaEventRecord(c->e1, s));
  f->launches++;
  CK(cudaGetLastError());
  int hdr[2] = {0, 0};
  CK(cudaMemcpyAsync(hdr, c->d_trace.p, 8, cudaMemcpyDeviceToHost, s));
  if (status) CK(cudaMemcpyAsync(status, c->d_trace.as<char>() + 16, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  event_ms(c.get(), f->t_lru_ms);
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

int32_t mmp_lru_read(mmp_fleet *f, const int32_t *instances, int32_t n, int64_t used_since, int64_t *offsets, mmp_lru_entry *out,
                     int64_t cap) {
  NEED(f);
  if (n < 0 || (n > 0 && !offsets) || cap < 0 || (cap > 0 && !out)) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  if (f->lru_n == 0) { g_err = "mmp_lru_init not called"; return MMP_E_STATE; }
  std::vector<int32_t> inst((size_t)n);
  for (int32_t k = 0; k < n; k++) {
    inst[k] = instances ? instances[k] : k;
    if (inst[k] < 0 || inst[k] >= f->lru_n) { g_err = "instance index out of range"; return MMP_E_ARG; }
  }
  if (n == 0) { if (offsets) offsets[0] = 0; return MMP_OK; }
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t s = c->stream;
  const LruView v = lru_view(f);
  const int loop = f->lru_loop ? 1 : 0;
  // d_in: instances; d_trace: per-cache counts, then the offsets; d_cand: stop flags
  const size_t n1 = (size_t)n + 1;
  CK(c->d_in.ensure((size_t)n * 4));
  CK(c->d_trace.ensure(2 * n1 * 8));
  CK(c->d_cand.ensure((size_t)n));
  long long *d_cnt = c->d_trace.as<long long>(), *d_off = d_cnt + n1;
  int *d_inst = c->d_in.as<int>();
  unsigned char *d_stop = c->d_cand.as<unsigned char>();
  size_t tscan = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, tscan, d_cnt, d_off, (int)n1, s));
  CK(c->d_cub.ensure(tscan + 64));
  CK(cudaMemcpyAsync(d_inst, inst.data(), (size_t)n * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemsetAsync(d_cnt + n, 0, 8, s));
  CK(cudaEventRecord(c->e0, s));
  k_lru_read_count<<<(n + 3) / 4, 128, 0, s>>>(v, d_inst, n, used_since, d_cnt, d_stop);
  CK(cub::DeviceScan::ExclusiveSum(c->d_cub.p, tscan, d_cnt, d_off, (int)n1, s));
  CK(cudaEventRecord(c->e1, s));
  f->launches += 2;
  CK(cudaGetLastError());
  std::vector<int64_t> off(n1);
  CK(cudaMemcpyAsync(off.data(), d_off, n1 * 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  float ms_count = 0;
  event_ms(c.get(), ms_count);
  const int64_t total = off[n], written = std::min(total, cap);
  // the walks longer than the shared-memory path holds, among those that start before cap: one segment each
  std::vector<int32_t> big;
  std::vector<int64_t> seg_off(1, 0);
  for (int32_t k = 0; k < n; k++)
    if (off[k] < cap && off[k + 1] - off[k] > LRU_READ_SMEM) { big.push_back(k); seg_off.push_back(seg_off.back() + off[k + 1] - off[k]); }
  const int64_t n_sort = seg_off.back();
  if (written > 0) {
    CK(c->d_out.ensure((size_t)written * sizeof(mmp_lru_entry)));
    mmp_lru_entry *d_out = c->d_out.as<mmp_lru_entry>();
    // d_extra: big + seg_off; d_fresh: keys in / out; d_rows: slots in / out
    LruReadKey *k_in = nullptr, *k_out = nullptr;
    int *s_in = nullptr, *s_out = nullptr, *d_big = nullptr;
    long long *d_seg = nullptr;
    size_t tsort = 0;
    if (n_sort > 0) {
      CK(c->d_extra.ensure(seg_off.size() * 8 + big.size() * 4));
      CK(c->d_fresh.ensure((size_t)n_sort * 2 * sizeof(LruReadKey)));
      CK(c->d_rows.ensure((size_t)n_sort * 2 * 4));
      d_seg = c->d_extra.as<long long>(); d_big = reinterpret_cast<int *>(d_seg + seg_off.size());
      k_in = c->d_fresh.as<LruReadKey>(); k_out = k_in + n_sort;
      s_in = c->d_rows.as<int>(); s_out = s_in + n_sort;
      CK(cub::DeviceRadixSort::SortPairs(nullptr, tsort, k_in, k_out, s_in, s_out, n_sort, LruReadKeyParts{}, s));
      CK(c->d_cub.ensure(tsort + 64));
      CK(cudaMemcpyAsync(d_seg, seg_off.data(), seg_off.size() * 8, cudaMemcpyHostToDevice, s));
      CK(cudaMemcpyAsync(d_big, big.data(), big.size() * 4, cudaMemcpyHostToDevice, s));
    }
    CK(cudaEventRecord(c->e0, s));
    k_lru_read_emit<<<n, 256, 0, s>>>(v, d_inst, d_off, d_stop, used_since, loop, d_out, cap);
    f->launches++;
    if (n_sort > 0) {
      k_lru_read_gather<<<(int)big.size(), 256, 0, s>>>(v, d_inst, d_stop, used_since, d_big, d_seg, k_in, s_in);
      CK(cub::DeviceRadixSort::SortPairs(c->d_cub.p, tsort, k_in, k_out, s_in, s_out, n_sort, LruReadKeyParts{}, s));
      k_lru_read_scatter<<<(unsigned)((n_sort + 255) / 256), 256, 0, s>>>(v, d_inst, d_off, d_big, d_seg, k_out, s_out, n_sort, loop, d_out, cap);
      f->launches += 3;
    }
    CK(cudaEventRecord(c->e1, s));
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(out, d_out, (size_t)written * sizeof(mmp_lru_entry), cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    float ms = 0;
    event_ms(c.get(), ms);
    ms_count += ms;
  }
  f->t_lru_read_ms = ms_count;
  std::memcpy(offsets, off.data(), n1 * 8);
  return MMP_OK;
}

int32_t mmp_lru_lookup(mmp_fleet *f, int32_t n, const int32_t *instance, const int32_t *model, int64_t *last_used, int32_t *weight,
                       int64_t *load_ts) {
  NEED(f);
  if (n < 0 || (n > 0 && (!instance || !model || !last_used || !weight || !load_ts))) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  if (f->lru_n == 0) { g_err = "mmp_lru_init not called"; return MMP_E_STATE; }
  for (int32_t q = 0; q < n; q++)
    if (instance[q] < 0 || instance[q] >= f->lru_n) { g_err = "instance index out of range"; return MMP_E_ARG; }
  if (n == 0) return MMP_OK;
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t s = c->stream;
  // d_in: instances, models; d_out: last_used, load_ts; d_extra: weights
  CK(c->d_in.ensure((size_t)n * 8)); CK(c->d_out.ensure((size_t)n * 16)); CK(c->d_extra.ensure((size_t)n * 4));
  int *d_inst = c->d_in.as<int>(), *d_model = d_inst + n;
  long long *d_lu = c->d_out.as<long long>(), *d_lt = d_lu + n;
  CK(cudaMemcpyAsync(d_inst, instance, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  CK(cudaMemcpyAsync(d_model, model, (size_t)n * 4, cudaMemcpyHostToDevice, s));
  k_lru_lookup<<<(n + 3) / 4, 128, 0, s>>>(lru_view(f), n, d_inst, d_model, f->lru_loop ? 1 : 0, d_lu, c->d_extra.as<int>(), d_lt);
  f->launches++;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(last_used, d_lu, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(load_ts, d_lt, (size_t)n * 8, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(weight, c->d_extra.p, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  return MMP_OK;
}

}  // extern "C"
