// registry_kernels.cuh — the registry-side batch scans (SURVEY.md §8a row a14, §8f-2): the scale-up / scale-down arithmetic of
// the rate-tracking and janitor tasks (MM:5640-5806, 5835-5870, 6197-6335) evaluated for a batch of cache entries against the
// fleet state in HBM, and the registry prune sweep of the reaper (pruneModelRegistry MM:6524-6609, pruneMissingInstances
// MM:6752-6784) as ONE pass over the registry -- the part the reference's author notes "have seen it take ~10min".
// Oracle: orc_rate_task_eval / orc_janitor_eval / orc_prune_missing (oracle/mm_sim.inc).  Included by mmplace.cu.
#pragma once

struct TypeStat { long long cap, free, lru; int count, copies; };

// typeSetStats (MM:1432-1438, TCM:230-233) per type id from the per-partition accumulators of k_stats
__global__ void k_type_stats(const StatsAcc *__restrict__ acc, const long long *__restrict__ min_lru, const int *__restrict__ type_part_off,
                             const int *__restrict__ type_parts, int n_type_ids, TypeStat *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_type_ids) return;
  TypeStat s{0, 0, 0x7fffffffffffffffLL, 0, 0};
  const int a = type_part_off[t], b = type_part_off[t + 1];
  const long long glru = *min_lru;
  if (a == b) { s.cap = (long long)acc[0].cap; s.free = (long long)acc[0].free; s.count = acc[0].count; s.copies = acc[0].copies; s.lru = glru; }
  else if (type_parts[a] >= 0) {
    for (int j = a; j < b; j++) {
      const StatsAcc x = acc[1 + type_parts[j]];
      s.cap += (long long)x.cap; s.free += (long long)x.free; s.count += x.count; s.copies += x.copies;
      if (x.count > 0) s.lru = glru;  // N10: every subset's LRU is recomputed over all cluster instances (MM:1519-1541)
    }
  }
  out[t] = s;
}

struct ScaleTables {
  const mmp_model_row *models; const int4 *edges; const long long *edge_ts; const long long *model_lul;
  const int32_t *rank_of; const RankRow *rows; const int32_t *part_of_rank; const uint4 *inst_tie;
  const TypeStat *type_stats; const StatsAcc *part_acc; const long long *min_lru; const int *sorted_rpm;
  int n_ranks, n_models, n_type_ids, max_instances, tc_enabled;
};

__device__ __forceinline__ int count_rpm_above(const int *sorted, int n, int thr) {  // #{rpm > thr} in an ascending array
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (sorted[mid] <= thr) lo = mid + 1; else hi = mid; }
  return n - lo;
}
__device__ __forceinline__ long long ts_of(const ScaleTables &T, int model, int j) { return T.edge_ts ? T.edge_ts[(size_t)model * 4 + j] : 0; }

// one thread per cache entry: rateTrackingTask's loop body (MM:5684-5806) and removeModelCopies (MM:6197-6335)
__global__ void k_scale_eval(ScaleTables T, const mmp_scale_in *__restrict__ in, int n, mmp_scale_params p, mmp_scale_out *__restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const mmp_scale_in e = in[r];
  mmp_scale_out o;
  o.action = 0; o.copies_to_load = 0; o.load_last_used = 0; o.rpm = 0; o.i1 = e.i1; o.i2 = e.i2; o.set_heavy = 0; o.remove = 0;
  if (e.model < 0 || e.model >= T.n_models || e.instance < 0 || e.instance >= T.max_instances) { o.action = -1; out[r] = o; return; }
  const mmp_model_row mr = T.models[e.model];
  if (mr.reserved > 4u) { o.action = -1; out[r] = o; return; }  // more registered instances than the inline list holds: host path
  const int4 ed = T.edges[e.model];
  const int es[4] = {ed.x, ed.y, ed.z, ed.w};
  const int loaded = mr.copy_count < 4 ? mr.copy_count : 4, n_edges = (int)mr.reserved, failed = n_edges - loaded;
  const int self_rank = T.rank_of[e.instance];
  const long long time_delta = p.now - p.last_check_time;
  // ---------------- scale-up (rateTrackingTask) ----------------
  do {
    const int inst_count = T.n_ranks;
    if (inst_count < 2) break;
    const int ty = mr.type_id < T.n_type_ids ? mr.type_id : 0;
    const TypeStat cs = T.type_stats[ty];
    int suitable = inst_count;
    if (T.tc_enabled) { suitable = cs.count; if (suitable < 2) break; }
    const int thr = p.scale_up_rpm_threshold, heavy = (int)((unsigned)thr * 3u) / 4;
    const int rpm = (int)((e.count * 60000LL) / time_delta);
    o.rpm = rpm;
    if (rpm > heavy) o.set_heavy = 1;
    if (loaded == 0) break;
    int cand = suitable - (loaded + failed);
    if (cand <= 0) break;
    if (loaded == 1) {
      const int lower = p.iteration - p.second_copy_max_age_iters, upper = p.iteration - p.second_copy_min_age_iters;
      const int i1 = e.i1, i2 = e.i2;
      bool in1 = false, in2 = false;
      if (i2 >= lower && i1 <= upper) { in1 = i1 >= lower; in2 = i2 <= upper; }
      if (in2 || !in1) o.i1 = i2;
      o.i2 = p.iteration;
      if (in1 || in2) {
        if (cs.cap == 0) break;  // the reference's ArithmeticException -> entry skipped (MM:5797)
        if ((10 * cs.free) / cs.cap >= 1 || (p.now - cs.lru) > p.second_copy_lru_threshold_ms) {
          o.action = 1; o.copies_to_load = 1; o.load_last_used = p.last_check_time;
          break;
        }
      }
    }
    if (rpm < thr) break;
    const long long cutoff = p.now - (time_delta + p.rate_check_interval_ms + 2 * p.assume_completed_ms);
    bool recent = false;
    for (int j = 0; j < loaded; j++) if (es[j] != e.instance && ts_of(T, e.model, j) > cutoff) recent = true;  // loadedSince MM:5858-5870
    if (recent) break;
    const int our_rpm = self_rank >= 0 ? T.rows[self_rank].rpm : 0;
    const int max_rpm = max((int)((unsigned)thr * 4u), (int)((unsigned)our_rpm - 2u * (unsigned)thr));   // getExcludeSet MM:5835-5856
    int excluded = count_rpm_above(T.sorted_rpm, T.n_ranks, max_rpm) - ((self_rank >= 0 && our_rpm > max_rpm) ? 1 : 0);
    if (excluded != 0) {
      int holding = 0;
      for (int j = 0; j < n_edges; j++) {
        const int i = es[j];
        if (i < 0 || i == e.instance) continue;
        const int rk = T.rank_of[i];
        if (rk >= 0 && T.rows[rk].rpm > max_rpm) holding++;
      }
      cand -= (excluded - holding);
      cand -= excluded;
      if (cand <= 0) break;
    }
    int copies = min(rpm / thr, cand);
    if (copies > 2) copies = min(copies, suitable / 3);
    o.action = 2; o.copies_to_load = copies; o.load_last_used = p.now + 20000;
  } while (false);
  // ---------------- scale-down (janitor: removeModelCopies) ----------------
  do {
    if (!p.can_remove || e.last_used == 0 || loaded < 2) break;
    // instanceSetStats(): the local instance's partition with type constraints, else the cluster (MM:1440-1446, TCM:236-239)
    long long cap, fr;
    const long long glru = *T.min_lru;
    if (T.tc_enabled) {
      if (self_rank < 0 || (e.flags & MMP_SCALE_NO_LOCAL_STATS)) break;  // EMPTY_STATS: totalCapacity == 0 (quirk N13, mmplace.h)
      const StatsAcc a = T.part_acc[1 + T.part_of_rank[self_rank]];
      cap = (long long)a.cap; fr = (long long)a.free;
    } else { cap = (long long)T.part_acc[0].cap; fr = (long long)T.part_acc[0].free; }
    if (cap == 0 || (fr * 100) / cap > 5) break;
    // the first other copy in instance-ID order that is in the table and not shutting down (MM:6236-6245)
    int other = -1;
    unsigned best_id = 0xffffffffu;
    for (int j = 0; j < loaded; j++) {
      const int i = es[j];
      if (i < 0 || i == e.instance || T.rank_of[i] < 0) continue;
      const unsigned idr = T.inst_tie[i].x;
      if (idr < best_id) { best_id = idr; other = i; }
    }
    if (other < 0) break;
    if (loaded == 2) {
      const long long cache_age = p.now - glru;
      long long scale_down_age = cache_age / 10;
      if (e.last_heavy == 0 || (p.now - e.last_heavy) < cache_age / 5) scale_down_age = p.second_copy_remove_max_age_ms < scale_down_age ? (long long)p.second_copy_remove_max_age_ms : scale_down_age;
      if ((p.now - e.last_used) > scale_down_age) {
        if (self_rank < 0) break;
        if (T.rank_of[other] > self_rank) break;  // PLACEMENT_ORDER.compare(other, this) > 0: the other pod should flush it (MM:6328)
        o.remove = 1;
      }
      break;
    }
    const long long lul = T.model_lul ? T.model_lul[e.model] : 0;
    if (lul > 0 && p.now - lul < 8 * p.rate_check_interval_ms) break;
    bool recent = false;
    for (int j = 0; j < loaded; j++) if (ts_of(T, e.model, j) > p.now - 1800000LL) recent = true;
    if (recent) break;
    long long min_age = (3 * glru + 10400000LL) / 100;
    if (min_age < 600000LL) min_age = 600000LL; else if (min_age > 18000000LL) min_age = 18000000LL;
    if (p.now - e.last_heavy < min_age) break;
    const long long since = p.now - p.last_check_time;
    if (since < p.rate_check_interval_ms / 10) break;
    const long long rpm2 = (e.count * 60000LL) / since;
    if (rpm2 > ((long long)p.scale_up_rpm_threshold * 2) / 3) break;
    o.remove = 1;
  } while (false);
  out[r] = o;
}

// the reaper's prune pass: one thread per model record, 24 B row + 16 B edges + 32 B edge times.  missing_since = the
// `missings` map by instance index (0 = absent); first-seen-missing instances are stamped (atomicCAS), pruned entries reported.
__global__ void k_registry_prune(const mmp_model_row *__restrict__ models, const int4 *__restrict__ edges, const long long *__restrict__ edge_ts,
                                 const int2 *__restrict__ inst_meta, int n_models, int max_instances, int self, long long now,
                                 long long assume_gone, long long *__restrict__ missing_since, int *__restrict__ out_models,
                                 unsigned char *__restrict__ out_masks, int cap, int *__restrict__ out_n) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  const mmp_model_row mr = models[m];
  const int n_edges = mr.reserved < 4u ? (int)mr.reserved : 4;
  if (n_edges == 0) return;
  const int4 ed = edges[m];
  const int es[4] = {ed.x, ed.y, ed.z, ed.w};
  unsigned mask = 0;
  for (int j = 0; j < n_edges; j++) {
    const int i = es[j];
    if (i < 0 || i >= max_instances || i == self) continue;
    if (now - (edge_ts ? edge_ts[(size_t)m * 4 + j] : 0) < assume_gone) continue;   // ignore recently loaded
    if (inst_meta[i].y & 4) continue;                                               // the instance is in the table
    const long long since = atomicCAS(reinterpret_cast<unsigned long long *>(&missing_since[i]), 0ull, (unsigned long long)now);
    if (since != 0 && (now - since) > assume_gone) mask |= 1u << j;
  }
  if (mask) {
    const int q = atomicAdd(out_n, 1);
    if (q < cap) { out_models[q] = m; out_masks[q] = (unsigned char)mask; }
  }
}

__global__ void k_extract_rpm(const RankRow *__restrict__ rows, int n, int *__restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) out[r] = rows[r].rpm;
}

extern "C" {

int32_t mmp_scale_eval(mmp_fleet *f, const mmp_scale_in *in, int32_t n, const mmp_scale_params *params, mmp_scale_out *out) {
  NEED(f);
  if (n < 0 || (n > 0 && (!in || !out)) || !params) { g_err = "bad argument"; return MMP_E_ARG; }
  if (params->now - params->last_check_time <= 0 || params->scale_up_rpm_threshold <= 0) { g_err = "now must be after last_check_time and the threshold positive"; return MMP_E_ARG; }
  if (n == 0) return MMP_OK;
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);  // reads the live registry tables a commit rewrites
  if (f->epoch == 0 || !f->live.valid) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  const DeviceSnapshot &ds = f->snaps[f->cur];
  LiveState &lv = f->live;
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t st = c->stream;
  const int np = (int)ds.host.part_types.size(), nr = ds.host.n_ranks, nt = lv.n_type_ids;
  const size_t acc_bytes = (size_t)(np + 1) * sizeof(StatsAcc) + 8;
  CK(c->d_trace.ensure(acc_bytes + (size_t)std::max(nt, 1) * sizeof(TypeStat) + 64));
  CK(c->d_fresh.ensure((size_t)std::max(nr, 1) * 8 + 64));
  CK(c->d_in.ensure((size_t)n * sizeof(mmp_scale_in)));
  CK(c->d_out.ensure((size_t)n * sizeof(mmp_scale_out)));
  StatsAcc *acc = c->d_trace.as<StatsAcc>();
  long long *d_min = reinterpret_cast<long long *>(c->d_trace.as<char>() + (size_t)(np + 1) * sizeof(StatsAcc));
  TypeStat *tstats = reinterpret_cast<TypeStat *>(c->d_trace.as<char>() + ((acc_bytes + 15) / 16) * 16);
  int *rpm_raw = c->d_fresh.as<int>(), *rpm_sorted = rpm_raw + std::max(nr, 1);
  CK(cudaMemsetAsync(c->d_trace.p, 0, acc_bytes, st));
  const long long init = 0x7fffffffffffffffLL;
  CK(cudaMemcpyAsync(d_min, &init, 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(c->d_in.p, in, (size_t)n * sizeof(mmp_scale_in), cudaMemcpyHostToDevice, st));
  if (nr > 0) {
    k_stats<<<std::min(f->sm_count, (nr + 255) / 256), 256, 0, st>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(), ds.part_of_rank.as<int32_t>(), nr,
                                                                     f->hs.cfg.min_space_units, acc, d_min, np);
    k_extract_rpm<<<(nr + 255) / 256, 256, 0, st>>>(ds.rows.as<RankRow>(), nr, rpm_raw);
    size_t tmp = 0;
    CK(cub::DeviceRadixSort::SortKeys(nullptr, tmp, rpm_raw, rpm_sorted, nr, 0, 32, st));
    CK(c->d_cub.ensure(tmp + 16));
    CK(cub::DeviceRadixSort::SortKeys(c->d_cub.p, tmp, rpm_raw, rpm_sorted, nr, 0, 32, st));
    f->launches += 3;
  }
  k_type_stats<<<(std::max(nt, 1) + 127) / 128, 128, 0, st>>>(acc, d_min, lv.type_part_off.as<int>(), lv.type_parts.as<int>(), nt, tstats);
  ScaleTables T;
  T.models = lv.models.as<mmp_model_row>(); T.edges = lv.edges.as<int4>();
  T.edge_ts = lv.have_times ? lv.edge_ts.as<long long>() : nullptr; T.model_lul = lv.have_times ? lv.model_lul.as<long long>() : nullptr;
  T.rank_of = ds.rank_of.as<int32_t>(); T.rows = ds.rows.as<RankRow>(); T.part_of_rank = ds.part_of_rank.as<int32_t>();
  T.inst_tie = lv.inst_tie.as<uint4>(); T.type_stats = tstats; T.part_acc = acc; T.min_lru = d_min; T.sorted_rpm = rpm_sorted;
  T.n_ranks = nr; T.n_models = f->hs.n_models_used; T.n_type_ids = nt; T.max_instances = f->hs.cfg.max_instances; T.tc_enabled = ds.host.tc_enabled;
  k_scale_eval<<<(n + 127) / 128, 128, 0, st>>>(T, c->d_in.as<mmp_scale_in>(), n, *params, c->d_out.as<mmp_scale_out>());
  f->launches += 2;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, c->d_out.p, (size_t)n * sizeof(mmp_scale_out), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return MMP_OK;
}

int32_t mmp_registry_prune(mmp_fleet *f, int32_t self, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, int32_t *out_models,
                           uint8_t *out_masks, int32_t cap) {
  NEED(f);
  if (!missing_since || cap < 0 || (cap > 0 && (!out_models || !out_masks))) { g_err = "bad argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  if (!f->live.valid) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  LiveState &lv = f->live;
  const int32_t nm = f->hs.n_models_used, NI = f->hs.cfg.max_instances;
  if (nm == 0) return 0;
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t st = c->stream;
  CK(c->d_in.ensure((size_t)NI * 8)); CK(c->d_out.ensure((size_t)std::max(cap, 1) * 4)); CK(c->d_extra.ensure((size_t)std::max(cap, 1)));
  CK(c->d_n_open.ensure(16));
  CK(cudaMemcpyAsync(c->d_in.p, missing_since, (size_t)NI * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(c->d_n_open.p, 0, 4, st));
  CK(cudaEventRecord(c->e0, st));
  k_registry_prune<<<(nm + 255) / 256, 256, 0, st>>>(lv.models.as<mmp_model_row>(), lv.edges.as<int4>(), lv.have_times ? lv.edge_ts.as<long long>() : nullptr,
                                                    lv.inst_meta.as<int2>(), nm, NI, self, now_ms, assume_gone_ms, c->d_in.as<long long>(),
                                                    c->d_out.as<int>(), c->d_extra.as<unsigned char>(), cap, c->d_n_open.as<int>());
  CK(cudaEventRecord(c->e1, st));
  f->launches++;
  CK(cudaGetLastError());
  int n_out = 0;
  CK(cudaMemcpyAsync(&n_out, c->d_n_open.p, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(missing_since, c->d_in.p, (size_t)NI * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  { float ms = 0; if (cudaEventElapsedTime(&ms, c->e0, c->e1) == cudaSuccess) f->t_prune_ms = ms; }
  const int got = std::min(n_out, cap);
  if (got) {
    std::vector<int32_t> ms((size_t)got);
    std::vector<uint8_t> mk((size_t)got);
    CK(cudaMemcpy(ms.data(), c->d_out.p, (size_t)got * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(mk.data(), c->d_extra.p, (size_t)got, cudaMemcpyDeviceToHost));
    std::vector<int32_t> ord((size_t)got);
    for (int i = 0; i < got; i++) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](int a, int b) { return ms[a] < ms[b]; });  // registry order
    for (int i = 0; i < got; i++) { out_models[i] = ms[ord[i]]; out_masks[i] = mk[ord[i]]; }
  }
  return n_out;
}

}  // extern "C"
