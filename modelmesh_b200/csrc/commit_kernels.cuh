// commit_kernels.cuh — the device side of mmp_fleet_commit (SURVEY.md §8f-1: handleInstanceTableChange MM:1455-1568 at fleet
// scale).  Included by mmplace.cu.
//
// A commit is STRUCTURAL when the set of live instances, their strings / labels / siMap membership, the type configuration
// or the replicaset list changed: string ranks, type-constraint set algebra and partitions are then rebuilt on the host
// (HostState::build_snapshot) and uploaded, together with the DEVICE-RESIDENT LIVE TABLES every later commit works from:
//   inst_rows [NI] mmp_instance_row        the published numeric columns (IR:37-73), by instance index
//   inst_tie  [NI] uint4                   dense ranks of id / location / zone / labels (tie-break chain MM:4697-4700)
//   inst_meta [NI] int2                    {partition id, bit0 live | bit1 likely-replaced replicaset member | bit2 in the instance table}
//   cand_idx / pref_idx [n_slots][NIW]     type-constraint masks over instance INDEX (allowed ∧ active / preferred)
//   edges [NM][4], models [NM]             the registry: loaded ∪ failed instance indices (first copy_count = loaded) + rows
// Every other commit -- numeric instance updates (the common KV event), model-record changes, the closed loop of
// churn_kernels.cuh -- scatters its deltas into those tables and rebuilds the snapshot ON THE DEVICE:
//   k_rank_keys + k_rank_count   PLACEMENT_ORDER rank of every live instance = number of live instances that compare less
//                                under the literal comparator (mmp::compare_keys, MM:4646-4703): O(N^2) compares, 10^8 at
//                                10 k instances, a fraction of a millisecond; no sort, no host round trip
//   k_build_rank_tables, k_word_summaries, k_permute_masks, k_slot_lists   the rank-space tables of DESIGN.md §4
//   cudaMemset + k_build_bitmap  the exclusion bitmap from the device-resident edges: one write pass over the bitmap
//                                (the floor of any scheme that keeps two consistent epochs) -- no edge upload, no host sort
#pragma once

struct LiveState {
  DevBuf inst_rows, inst_tie, inst_meta, cand_idx, pref_idx, edges, models, keys, rs_words, flags, scratch_idx, scratch_rows,
      scratch_edges;
  DevBuf ovf;                                 // [n_ovf] OvfEdge: registrations 4, 5, ... of every model, sorted by (model, position)
  DevBuf edge_ts, model_lul;                  // MR.instanceIds / failedIn values and MR.lastUnloadTime (registry_kernels.cuh), when given
  bool have_times = false;
  DevBuf type_part_off, type_parts;           // type id -> partitions whose instances may host the type (typeSetStats MM:1432-1438)
  int32_t n_type_ids = 0;
  int32_t n_ovf = 0, niw = 0;
  bool valid = false;           // a structural commit has populated the tables
  mmp::HostSnapshot tmpl;       // the last structural snapshot: everything that does not depend on the numeric columns
};

// A model's registrations in the order of its last upsert (loaded first, then failed): positions 0-3 are the inline edges and
// their times, positions 4, 5, ... the model's slice of the overflow table, found by a lower_bound on its model column.  Only
// models with more than four registrations search.
struct RegTables { const int4 *edges; const long long *edge_ts; const OvfEdge *ovf; int n_ovf; };
struct ModelRegs { int m, ovf0; int4 e; };
__device__ __forceinline__ ModelRegs model_regs(const RegTables &R, int m, unsigned reserved) {
  ModelRegs g{m, 0, R.edges[m]};
  if (reserved > 4u) {
    int lo = 0, hi = R.n_ovf;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (R.ovf[mid].model < m) lo = mid + 1; else hi = mid; }
    g.ovf0 = lo;
  }
  return g;
}
// registration j of the model -> its instance (-1: none) and its load / failure time (0: unknown)
__device__ __forceinline__ int reg_at(const RegTables &R, const ModelRegs &g, int j, long long &ts) {
  if (j < 4) {
    ts = R.edge_ts ? R.edge_ts[(size_t)g.m * 4 + j] : 0;
    return j == 0 ? g.e.x : j == 1 ? g.e.y : j == 2 ? g.e.z : g.e.w;
  }
  const int q = g.ovf0 + j - 4;
  if (q >= R.n_ovf || R.ovf[q].model != g.m) { ts = 0; return -1; }
  ts = R.ovf[q].ts;
  return R.ovf[q].inst;
}
static RegTables reg_tables(const LiveState &lv) {
  return RegTables{lv.edges.as<int4>(), lv.have_times ? lv.edge_ts.as<long long>() : nullptr, lv.ovf.as<OvfEdge>(), lv.n_ovf};
}

// scratch of the reaper's selection pass (reaper_pass, scan_kernels.cuh), owned by its caller: sort keys, model indices and
// their count, candidate flags, the per-partition plan, the runs' clocks with the partitions' prohibited type ids, the
// selections and their offsets per run; taken[m] holds the tag of the last run that selected model m
struct RpScratch { DevBuf keys, idx, flag, plan, runs, sel, off, taken; };

// state of the closed loop (churn_kernels.cuh), owned by the fleet
struct ChurnState {
  bool on = false;
  int64_t load_timeout_ms = 0;
  DevBuf last_published, first_ev, dec_of_model, rm_mask, add_inst, used_t, force_publish, type_ok, stats_acc;
  DevBuf carry, next_carry, counters;
  DevBuf ev, is_dec, dec_pos, dec_in, dec_out, dec_meta, dec_target, extra, status, lev, keys, vals, keys2, vals2, cub_tmp, off, evict, fkeys,
      fvals, rows_changed;
  DevBuf ovf_dead, ovf_next, ovf_count;  // the registry phase's re-lay of LiveState::ovf (churn_kernels.cuh)
  // the reaper pass of a window with MMP_CHURN_REAPER events (churn_kernels.cuh): its scratch, the events' trace indices and
  // their selections' first-decision flags; rp_gen: the last tag in rp.taken (tags grow across windows: no reset per run)
  RpScratch rp;
  DevBuf rp_ev, rp_fpos;
  int32_t rp_gen = 0;
  int32_t n_carry = 0;
  // what the step's host side knows of the registry without reading it back: the loop only removes loaded copies or loads the
  // first one of a model without any, so the largest copy count does not grow past max(it, 1) and the failed loads of a model
  // stay as they are.  Taken from the host tables when they were last uploaded (regs_from_host).
  bool regs_from_host = true, deep_failed = false;
  int32_t max_copies = 1;
  // last step's phase timings (ms, between these events on the step's stream; created by mmp_churn_init)
  Event phase_ev[9];  // [7], [8]: around the reaper pass
  float t_classify = 0, t_place = 0, t_route = 0, t_apply = 0, t_registry = 0, t_commit = 0, t_total = 0;
  int32_t last_lru_events = 0;
};


// the PLACEMENT_ORDER key of a live instance's published record (HostState::build_snapshot builds the same on the host)
__device__ __forceinline__ OrderKey order_key(const mmp_instance_row &r, const uint4 &t, long long min_space) {
  OrderKey k;
  k.vers = r.vers;
  k.rem = r.capacity - r.used > 0 ? r.capacity - r.used : 0;  // IR:203-205
  k.lru = r.lru_time; k.cap = r.capacity; k.count = r.count;
  k.free_threads = (int32_t)((uint32_t)r.l_threads - (uint32_t)r.l_in_prog);
  k.lip = r.l_in_prog; k.rpm = r.rpm;
  k.id_rank = t.x; k.loc_rank = t.y; k.zone_rank = t.z; k.labels_rank = t.w;
  k.full = k.rem < min_space;
  k.shutting_down = false;
  return k;
}

__global__ void k_rank_keys(const mmp_instance_row *__restrict__ rows, const uint4 *__restrict__ tie, const int2 *__restrict__ meta,
                            int n_idx, long long min_space, OrderKey *__restrict__ keys, long long vers0, int *__restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_idx) return;
  const mmp_instance_row r = rows[i];
  keys[i] = order_key(r, tie[i], min_space);
  if ((meta[i].y & 1) && r.vers != vers0) atomicOr(flags, 1);  // mixed versions: the comparator may be non-transitive (N1): host path
}

// rank_of[i] = #{ live j : compare_keys(j, i) < 0 }, keys tiled through shared memory.  The j range is cut into gridDim.y
// slices (N threads alone would leave most SMs idle: 79 blocks at 10 k instances); rank_of must hold 0 for live and -1 for
// other indices on entry (k_rank_init), every slice adds its count
__global__ void k_rank_init(const int2 *__restrict__ meta, int n_idx, int32_t *__restrict__ rank_of) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_idx) rank_of[i] = (meta[i].y & 1) ? 0 : -1;
}
__global__ void __launch_bounds__(128) k_rank_count(const OrderKey *__restrict__ keys, const int2 *__restrict__ meta, int n_idx,
                                                    long long churn2, int32_t *__restrict__ rank_of) {
  __shared__ OrderKey tile[128];
  __shared__ int live_t[128];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool mine = i < n_idx && (meta[i].y & 1);
  OrderKey me;
  if (i < n_idx) me = keys[i];
  const int per = ((n_idx + (int)gridDim.y - 1) / (int)gridDim.y + 127) / 128 * 128;
  const int j0 = (int)blockIdx.y * per, j1 = min(n_idx, j0 + per);
  int cnt = 0;
  for (int base = j0; base < j1; base += 128) {
    const int j = base + threadIdx.x;
    live_t[threadIdx.x] = (j < j1) ? (meta[j].y & 1) : 0;
    if (j < j1) tile[threadIdx.x] = keys[j];
    __syncthreads();
    if (mine) {
      const int lim = min(128, j1 - base);
      for (int t = 0; t < lim; t++)
        if (live_t[t] && compare_keys(tile[t], me, churn2) < 0) cnt++;
    }
    __syncthreads();
  }
  if (mine && cnt) atomicAdd(&rank_of[i], cnt);
}

__global__ void k_build_rank_tables(const mmp_instance_row *__restrict__ rows_in, const int2 *__restrict__ meta,
                                    const int32_t *__restrict__ rank_of, int n_idx, long long min_space, RankRow *__restrict__ rows,
                                    int64_t *__restrict__ cap_col, int32_t *__restrict__ lthreads, int32_t *__restrict__ linprog,
                                    int32_t *__restrict__ part_of_rank, int32_t *__restrict__ count_col, uint32_t *__restrict__ full,
                                    uint32_t *__restrict__ rs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_idx) return;
  const int r = rank_of[i];
  if (r < 0) return;
  const mmp_instance_row in = rows_in[i];
  RankRow o;
  o.lru = in.lru_time;
  o.rem = in.capacity - in.used > 0 ? in.capacity - in.used : 0;
  o.count = in.count; o.rpm = in.rpm; o.idx = i;
  const bool is_full = o.rem < min_space;
  o.flags = is_full ? 1u : 0u;
  rows[r] = o;
  cap_col[r] = in.capacity; lthreads[r] = in.l_threads; linprog[r] = in.l_in_prog;
  part_of_rank[r] = meta[i].x;
  count_col[r] = in.count;
  if (is_full) atomicOr(&full[r >> 5], 1u << (r & 31));
  if (meta[i].y & 2) atomicOr(&rs[r >> 5], 1u << (r & 31));
}

__global__ void k_word_summaries(const RankRow *__restrict__ rows, int n_ranks, int row_words, WordSumI *__restrict__ csum,
                                 WordSumL *__restrict__ lsum) {
  const int w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= row_words) return;
  WordSumI c{INT32_MAX, INT32_MIN};
  WordSumL l{INT64_MAX, INT64_MIN};
  for (int b = 0; b < 32; b++) {
    const int r = w * 32 + b;
    if (r >= n_ranks) break;
    const RankRow x = rows[r];
    c.lo = min(c.lo, x.count); c.hi = max(c.hi, x.count);
    l.lo = x.lru < l.lo ? x.lru : l.lo; l.hi = x.lru > l.hi ? x.lru : l.hi;
  }
  csum[w] = c; lsum[w] = l;
}

// type-constraint masks: instance-index space -> rank space (one thread per (slot, row word))
__global__ void k_permute_masks(const uint32_t *__restrict__ cand_idx, const uint32_t *__restrict__ pref_idx, int niw,
                                const RankRow *__restrict__ rows, int n_ranks, int row_words, int n_slots,
                                const uint32_t *__restrict__ rs, uint32_t *__restrict__ cand, uint32_t *__restrict__ candx,
                                uint32_t *__restrict__ pref) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_slots * row_words) return;
  const int sl = t / row_words, w = t - sl * row_words;
  uint32_t c = 0, p = 0;
  for (int b = 0; b < 32; b++) {
    const int r = w * 32 + b;
    if (r >= n_ranks) break;
    const int idx = rows[r].idx;
    c |= ((cand_idx[(size_t)sl * niw + (idx >> 5)] >> (idx & 31)) & 1u) << b;
    p |= ((pref_idx[(size_t)sl * niw + (idx >> 5)] >> (idx & 31)) & 1u) << b;
  }
  cand[t] = c; pref[t] = p; candx[t] = c & ~rs[w];
}

// compressed word lists (LaneTables) and the instance-shard early-out counts, one thread per slot
__global__ void k_slot_lists(const uint32_t *__restrict__ cand, const uint32_t *__restrict__ candx, int any_rs, int row_words,
                             int n_slots, int word_lo, int word_hi, uint16_t *__restrict__ nzw, int32_t *__restrict__ nz_n,
                             int32_t *__restrict__ cand_before) {
  const int sl = blockIdx.x * blockDim.x + threadIdx.x;
  if (sl >= n_slots) return;
  const uint32_t *cx = (any_rs ? candx : cand) + (size_t)sl * row_words;
  uint16_t *out = nzw + (size_t)sl * row_words;
  int k = 0, before = 0, skip = 0;
  for (int w = 0; w < word_lo; w++) before += __popc(candx[(size_t)sl * row_words + w]);
  for (int w = word_lo; w < word_hi; w++)
    if (cx[w]) { out[k++] = (uint16_t)w; if (w < word_lo + MMP_LANE_WIN) skip++; }
  nz_n[sl] = k | (skip << 24);
  for (; k < row_words; k++) out[k] = 0xffff;
  cand_before[sl] = before;
}

// A call-wide exclude set (mmp_place_batch_excluding): the snapshot's per-slot candidate, replicaset-filtered and preferred
// masks with the set's ranks cleared, into the call's own tables.  An excluded instance then leaves the filter exactly as one
// the type does not allow (MM:4760-4771), so the decision routine runs unchanged on a view of these tables.  One block per
// type slot; each builds the set's rank-space mask in shared memory (row_words words, at most 8 KB) from the instance
// indices, which the host has checked against [0, max_instances).  Indices of instances that are not live have no rank.
__global__ void k_exclude_slots(const int32_t *__restrict__ ids, int n_ids, const int32_t *__restrict__ rank_of, int row_words,
                                const uint32_t *__restrict__ cand, const uint32_t *__restrict__ candx, const uint32_t *__restrict__ pref,
                                uint32_t *__restrict__ x_cand, uint32_t *__restrict__ x_candx, uint32_t *__restrict__ x_pref) {
  extern __shared__ uint32_t xm[];
  for (int w = threadIdx.x; w < row_words; w += blockDim.x) xm[w] = 0u;
  __syncthreads();
  for (int k = threadIdx.x; k < n_ids; k += blockDim.x) {
    const int r = rank_of[ids[k]];
    if (r >= 0) atomicOr(&xm[r >> 5], 1u << (r & 31));
  }
  __syncthreads();
  const size_t so = (size_t)blockIdx.x * row_words;
  for (int w = threadIdx.x; w < row_words; w += blockDim.x) {
    const uint32_t keep = ~xm[w];
    x_cand[so + w] = cand[so + w] & keep;
    x_candx[so + w] = candx[so + w] & keep;
    x_pref[so + w] = pref[so + w] & keep;
  }
}

// deltas of a non-structural commit
__global__ void k_scatter_inst_rows(const int32_t *__restrict__ idx, const mmp_instance_row *__restrict__ src, int n,
                                    mmp_instance_row *__restrict__ rows) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) rows[idx[t]] = src[t];
}
__global__ void k_scatter_models(const int32_t *__restrict__ ids, const mmp_model_row *__restrict__ rows, const int4 *__restrict__ edges,
                                 int n, mmp_model_row *__restrict__ models, int4 *__restrict__ edge_inl) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < n) { models[ids[t]] = rows[t]; edge_inl[ids[t]] = edges[t]; }
}
