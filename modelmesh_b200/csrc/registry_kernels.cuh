// registry_kernels.cuh — the registry-side batch scans (SURVEY.md §8a row a14, §8f-2): the scale-up / scale-down arithmetic of
// the rate-tracking and janitor tasks (MM:5640-5806, 5835-5870, 6197-6335) evaluated for a batch of cache entries against the
// fleet state in HBM, and the registry prune sweep of the reaper (pruneModelRegistry MM:6524-6609, pruneMissingInstances
// MM:6752-6784) as ONE pass over the registry -- the part the reference's author notes "have seen it take ~10min".
// Oracle: orc_rate_task_eval / orc_janitor_eval / orc_prune_missing (oracle/mm_sim.inc).  Included by mmplace.cu.
#pragma once
#include <cub/block/block_scan.cuh>

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
  const mmp_model_row *models; RegTables R; const long long *model_lul;
  const int32_t *rank_of; const RankRow *rows; const int32_t *part_of_rank; const uint4 *inst_tie;
  const mmp_instance_row *inst_rows; long long min_space, churn2;  // PLACEMENT_ORDER keys of the live instances
  const TypeStat *type_stats; const StatsAcc *part_acc; const long long *min_lru; const int *sorted_rpm;
  int n_ranks, n_models, n_type_ids, max_instances, tc_enabled;
};

// Java long arithmetic: wraps
__device__ __forceinline__ long long jmul64(long long a, long long b) { return (long long)((unsigned long long)a * (unsigned long long)b); }
__device__ __forceinline__ long long jadd64(long long a, long long b) { return (long long)((unsigned long long)a + (unsigned long long)b); }

// how many of a model's registrations are loaded copies: the first copy_count of them (up to four registrations, a copy count
// past them reads the inline positions, as the four-edge list always did).  -1 for a copy count saturated at 255 over more
// than 255 registrations, where the loaded copies end is unknown (mmplace.h): k_scale_eval answers -1, the pod tasks
// MMP_*_UNDECIDED
__device__ __forceinline__ int loaded_copies(const mmp_model_row &mr) {
  if (mr.copy_count == 255 && mr.reserved > 255u) return -1;
  return min((int)mr.copy_count, max((int)mr.reserved, 4));
}

__device__ __forceinline__ int count_rpm_above(const int *sorted, int n, int thr) {  // #{rpm > thr} in an ascending array
  int lo = 0, hi = n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (sorted[mid] <= thr) lo = mid + 1; else hi = mid; }
  return n - lo;
}

// getExcludeSet's bound (MM:5835-5856): instances whose published rpm is above it are excluded from a scale-up's loads.
// k_scale_eval counts them, k_rate_heavy lists them.  our_rpm: the pod's published rpm (0 when it is not in the snapshot)
__device__ __forceinline__ int exclude_set_max_rpm(int thr, int our_rpm) {
  return max((int)((unsigned)thr * 4u), (int)((unsigned)our_rpm - 2u * (unsigned)thr));
}

// removeModelCopies (MM:6197-6335) with canRemove = true for `instance`'s copy of `model` (who-drops-the-copy by PLACEMENT_ORDER
// MM:6314-6335 included): k_scale_eval's scale-down and the janitor's registry pass (k_janitor_eval) both run it.  g / loaded:
// the model's registrations and how many of them are loaded copies; self_rank: `instance`'s rank in the snapshot (-1: none).
// rereg (mmp_janitor_task's registry pass): the cache pass re-registered `instance` at rereg_ts; `added` of the loaded copies
// are that registration, past the committed ones (0 where it replaced the time of `instance`'s committed copy)
__device__ __forceinline__ bool scale_down_removes(const ScaleTables &T, const mmp_scale_params &p, int instance, int model, long long last_used,
                                                   long long last_heavy, long long count, int flags, const ModelRegs &g, int loaded,
                                                   int self_rank, bool rereg = false, long long rereg_ts = 0, int added = 0) {
  long long ts;
  if (last_used == 0 || loaded < 2) return false;
  // instanceSetStats(): the local instance's partition with type constraints, else the cluster (MM:1440-1446, TCM:236-239)
  long long cap, fr;
  const long long glru = *T.min_lru;
  if (T.tc_enabled) {
    if (self_rank < 0 || (flags & MMP_SCALE_NO_LOCAL_STATS)) return false;  // EMPTY_STATS: totalCapacity == 0 (quirk N13, mmplace.h)
    const StatsAcc a = T.part_acc[1 + T.part_of_rank[self_rank]];
    cap = (long long)a.cap; fr = (long long)a.free;
  } else { cap = (long long)T.part_acc[0].cap; fr = (long long)T.part_acc[0].free; }
  if (cap == 0 || jmul64(fr, 100) / cap > 5) return false;
  // the first other copy in instance-ID order that is in the table and not shutting down (MM:6236-6245)
  int other = -1;
  unsigned best_id = 0xffffffffu;
  for (int j = 0; j < loaded - added; j++) {
    const int i = reg_at(T.R, g, j, ts);
    if (i < 0 || i == instance || T.rank_of[i] < 0) continue;
    const unsigned idr = T.inst_tie[i].x;
    if (idr < best_id) { best_id = idr; other = i; }
  }
  if (other < 0) return false;
  if (loaded == 2) {
    const long long cache_age = jsub(p.now, glru);
    long long scale_down_age = cache_age / 10;
    if (last_heavy == 0 || jsub(p.now, last_heavy) < cache_age / 5) scale_down_age = p.second_copy_remove_max_age_ms < scale_down_age ? (long long)p.second_copy_remove_max_age_ms : scale_down_age;
    if (jsub(p.now, last_used) > scale_down_age) {
      if (self_rank < 0) return false;
      // PLACEMENT_ORDER.compare(other, this) > 0: the other pod should flush it (MM:6328).  The comparator, not the ranks:
      // with mixed versions (quirk N1) it is no total order, and the snapshot's linear order contradicts it on some pair
      if (compare_keys(order_key(T.inst_rows[other], T.inst_tie[other], T.min_space),
                       order_key(T.inst_rows[instance], T.inst_tie[instance], T.min_space), T.churn2) > 0) return false;
      return true;
    }
    return false;
  }
  const long long lul = T.model_lul ? T.model_lul[model] : 0;
  if (lul > 0 && jsub(p.now, lul) < jmul64(8, p.rate_check_interval_ms)) return false;
  bool recent = rereg && added && rereg_ts > jsub(p.now, 1800000LL);
  for (int j = 0; j < loaded - added; j++) {
    if (reg_at(T.R, g, j, ts) == instance && rereg) ts = rereg_ts;
    if (ts > jsub(p.now, 1800000LL)) recent = true;
  }
  if (recent) return false;
  long long min_age = jadd64(jmul64(3, glru), 10400000LL) / 100;
  if (min_age < 600000LL) min_age = 600000LL; else if (min_age > 18000000LL) min_age = 18000000LL;
  if (jsub(p.now, last_heavy) < min_age) return false;
  const long long since = jsub(p.now, p.last_check_time);
  if (since < p.rate_check_interval_ms / 10) return false;
  const long long rpm2 = jmul64(count, 60000) / since;
  if (rpm2 > ((long long)p.scale_up_rpm_threshold * 2) / 3) return false;
  return true;
}

// one thread per cache entry: rateTrackingTask's loop body (MM:5684-5806) and removeModelCopies (MM:6197-6335)
__global__ void k_scale_eval(ScaleTables T, const mmp_scale_in *__restrict__ in, int n, mmp_scale_params p, mmp_scale_out *__restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const mmp_scale_in e = in[r];
  mmp_scale_out o;
  o.action = 0; o.copies_to_load = 0; o.load_last_used = 0; o.rpm = 0; o.i1 = e.i1; o.i2 = e.i2; o.set_heavy = 0; o.remove = 0;
  if (e.model < 0 || e.model >= T.n_models || e.instance < 0 || e.instance >= T.max_instances) { o.action = -1; out[r] = o; return; }
  const mmp_model_row mr = T.models[e.model];
  const int loaded = loaded_copies(mr);
  if (loaded < 0) { o.action = -1; out[r] = o; return; }
  const ModelRegs g = model_regs(T.R, e.model, mr.reserved);
  long long ts;
  const int n_edges = (int)mr.reserved, failed = n_edges - loaded;
  const int self_rank = T.rank_of[e.instance];
  const long long time_delta = jsub(p.now, p.last_check_time);
  // ---------------- scale-up (rateTrackingTask) ----------------
  do {
    const int inst_count = T.n_ranks;
    if (inst_count < 2) break;
    const int ty = mr.type_id < T.n_type_ids ? mr.type_id : 0;
    const TypeStat cs = T.type_stats[ty];
    int suitable = inst_count;
    if (T.tc_enabled) { suitable = cs.count; if (suitable < 2) break; }
    const int thr = p.scale_up_rpm_threshold, heavy = (int)((unsigned)thr * 3u) / 4;
    const int rpm = (int)(jmul64(e.count, 60000) / time_delta);
    o.rpm = rpm;
    if (rpm > heavy) o.set_heavy = 1;
    if (loaded == 0) break;
    int cand = suitable - (loaded + failed);
    if (cand <= 0) break;
    if (loaded == 1) {
      const int lower = (int)((unsigned)p.iteration - (unsigned)p.second_copy_max_age_iters);
      const int upper = (int)((unsigned)p.iteration - (unsigned)p.second_copy_min_age_iters);
      const int i1 = e.i1, i2 = e.i2;
      bool in1 = false, in2 = false;
      if (i2 >= lower && i1 <= upper) { in1 = i1 >= lower; in2 = i2 <= upper; }
      if (in2 || !in1) o.i1 = i2;
      o.i2 = p.iteration;
      if (in1 || in2) {
        if (cs.cap == 0) break;  // the reference's ArithmeticException -> entry skipped (MM:5797)
        if (jmul64(10, cs.free) / cs.cap >= 1 || jsub(p.now, cs.lru) > p.second_copy_lru_threshold_ms) {
          o.action = 1; o.copies_to_load = 1; o.load_last_used = p.last_check_time;
          break;
        }
      }
    }
    if (rpm < thr) break;
    const long long cutoff = jsub(p.now, jadd64(jadd64(time_delta, p.rate_check_interval_ms), jmul64(2, p.assume_completed_ms)));
    bool recent = false;
    for (int j = 0; j < loaded; j++) if (reg_at(T.R, g, j, ts) != e.instance && ts > cutoff) recent = true;  // loadedSince MM:5858-5870
    if (recent) break;
    const int our_rpm = self_rank >= 0 ? T.rows[self_rank].rpm : 0;
    const int max_rpm = exclude_set_max_rpm(thr, our_rpm);
    int excluded = count_rpm_above(T.sorted_rpm, T.n_ranks, max_rpm) - ((self_rank >= 0 && our_rpm > max_rpm) ? 1 : 0);
    if (excluded != 0) {
      int holding = 0;
      for (int j = 0; j < n_edges; j++) {
        const int i = reg_at(T.R, g, j, ts);
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
  if (p.can_remove && scale_down_removes(T, p, e.instance, e.model, e.last_used, e.last_heavy, e.count, e.flags, g, loaded, self_rank)) o.remove = 1;
  out[r] = o;
}

// the reaper's prune pass: one thread per model record, 24 B row + 16 B edges + 32 B edge times (+ 16 B per overflow
// registration).  missing_since = the `missings` map by instance index (0 = absent); first-seen-missing instances are stamped
// (atomicCAS), pruned entries reported.  walk_ovf = 0: the first four registrations, one (model, mask) per model with pruned
// entries (mmp_registry_prune); 1: every registration, one PrunedReg per pruned one, in no order (mmp_registry_prune_ids).
// With a view (mmp_reaper_run, walk_ovf = 1) every model's row is also written as the reaper's loop sees it after the prune
// and repairLastUsedTimeIfNeeded (MM:6837-6850): a pruned registration at a position < copy_count leaves copy_count, any
// other fail_count; a last_used of Long.MAX_VALUE becomes now - 3 x LASTUSED_AGE_ON_ADD_MS, the model listed as repaired.
struct PrunedReg { int32_t model, pos, inst; };
struct PruneView { mmp_model_row *rows; int *repaired, *n_repaired; };
__global__ void k_registry_prune(RegTables R, const mmp_model_row *__restrict__ models, const int2 *__restrict__ inst_meta, int n_models,
                                 int max_instances, int self, long long now, long long assume_gone, long long *__restrict__ missing_since,
                                 int walk_ovf, int *__restrict__ out_models, unsigned char *__restrict__ out_masks, PrunedReg *__restrict__ out_regs,
                                 int cap, int *__restrict__ out_n, PruneView view) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  const mmp_model_row mr = models[m];
  const int n_edges = walk_ovf || mr.reserved < 4u ? (int)mr.reserved : 4;
  if (n_edges == 0 && !view.rows) return;
  const ModelRegs g = model_regs(R, m, walk_ovf ? mr.reserved : 0u);
  unsigned mask = 0;
  int gone_loaded = 0, gone_failed = 0;
  for (int j = 0; j < n_edges; j++) {
    long long ts;
    const int i = reg_at(R, g, j, ts);
    if (i < 0 || i >= max_instances || i == self) continue;
    if (now - ts < assume_gone) continue;        // ignore recently loaded
    if (inst_meta[i].y & 4) continue;            // the instance is in the table
    const long long since = atomicCAS(reinterpret_cast<unsigned long long *>(&missing_since[i]), 0ull, (unsigned long long)now);
    if (since == 0 || (now - since) <= assume_gone) continue;
    if (!walk_ovf) { mask |= 1u << j; continue; }
    if (j < mr.copy_count) gone_loaded++; else gone_failed++;
    const int q = atomicAdd(out_n, 1);
    if (q < cap) out_regs[q] = PrunedReg{m, j, i};
  }
  if (mask) {
    const int q = atomicAdd(out_n, 1);
    if (q < cap) { out_models[q] = m; out_masks[q] = (unsigned char)mask; }
  }
  if (view.rows) {
    mmp_model_row v = mr;
    v.copy_count = (uint8_t)max((int)mr.copy_count - gone_loaded, 0);
    v.fail_count = (uint8_t)max((int)mr.fail_count - gone_failed, 0);
    if (mr.last_used == 0x7fffffffffffffffLL) {
      v.last_used = jsub(now, 3LL * 3600000LL);
      view.repaired[atomicAdd(view.n_repaired, 1)] = m;
    }
    view.rows[m] = v;
  }
}

__global__ void k_extract_rpm(const RankRow *__restrict__ rows, int n, int *__restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n) out[r] = rows[r].rpm;
}

// One prune pass (k_registry_prune) over the live registry.  It keeps every record -- walk_ovf = 0: one (model, mask) per
// model; 1: every pruned registration (at most 4 per model + the overflow table) -- so that the caller can hand out the first
// ones in order.  `read(ctx, n)` copies the records out once missing_since is back; n = the kernel's count.
template <class Read>
static int32_t registry_prune(mmp_fleet *f, int32_t self, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, bool walk_ovf,
                              Read read) {
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
  CK(c->d_in.ensure((size_t)NI * 8));
  const int32_t cap = walk_ovf ? nm * HostState::EDGE_INL + lv.n_ovf : nm;
  if (walk_ovf) CK(c->d_out.ensure((size_t)cap * sizeof(PrunedReg)));
  else { CK(c->d_out.ensure((size_t)cap * 4)); CK(c->d_extra.ensure((size_t)cap)); }
  CK(c->d_n_open.ensure(16));
  CK(cudaMemcpyAsync(c->d_in.p, missing_since, (size_t)NI * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(c->d_n_open.p, 0, 4, st));
  CK(cudaEventRecord(c->e0, st));
  k_registry_prune<<<(nm + 255) / 256, 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), lv.inst_meta.as<int2>(), nm, NI, self, now_ms,
                                                    assume_gone_ms, c->d_in.as<long long>(), walk_ovf ? 1 : 0, c->d_out.as<int>(),
                                                    c->d_extra.as<unsigned char>(), c->d_out.as<PrunedReg>(), cap, c->d_n_open.as<int>(),
                                                    PruneView{});
  CK(cudaEventRecord(c->e1, st));
  f->launches++;
  CK(cudaGetLastError());
  int n_out = 0;
  CK(cudaMemcpyAsync(&n_out, c->d_n_open.p, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(missing_since, c->d_in.p, (size_t)NI * 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  event_ms(c.get(), f->t_prune_ms);
  return read(c.get(), n_out);
}

// mmp_reaper_run's decisions: selection k (rs.sel, emission order) is getNext(model, self = leader, lastUsed = the model's
// row in the view, i.e. the repaired value where repaired), no flags, no extra excludes
__global__ void k_reaper_decisions(const int2 *__restrict__ sel, int n, const mmp_model_row *__restrict__ view, int leader,
                                   mmp_decision_in *__restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const int m = sel[k].x;
  out[k] = mmp_decision_in{m, leader, view[m].last_used, 0u, -1, 0, 0};
}
// ... and its loads, from the placed decisions
__global__ void k_reaper_loads(const mmp_decision_in *__restrict__ in, const mmp_decision_out *__restrict__ res, int n,
                               mmp_reaper_load *__restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  out[k] = mmp_reaper_load{in[k].model, res[k].target, res[k].n_candidates, 0, in[k].last_used};
}
// the reaper's cleanup of its `missings` map after the registry loop (MM:6601-6607)
__global__ void k_missing_cleanup(long long *__restrict__ missing_since, const int2 *__restrict__ inst_meta, int n, long long now,
                                  long long assume_gone) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long v = missing_since[i];
  if (v != 0 && (jsub(now, v) > assume_gone || (inst_meta[i].y & 4))) missing_since[i] = 0;
}

// the tables k_scale_eval and k_janitor_eval read: the snapshot's, the live registry's, and the call's stats (the type-set
// stats and the sorted rpm column only the scale-up reads: NULL where no scale-up runs)
static ScaleTables scale_tables(mmp_fleet *f, const DeviceSnapshot &ds, LiveState &lv, const StatsAcc *acc, const long long *d_min,
                                const TypeStat *tstats, const int *rpm_sorted) {
  ScaleTables T;
  T.models = lv.models.as<mmp_model_row>(); T.R = reg_tables(lv);
  T.model_lul = lv.have_times ? lv.model_lul.as<long long>() : nullptr;
  T.rank_of = ds.rank_of.as<int32_t>(); T.rows = ds.rows.as<RankRow>(); T.part_of_rank = ds.part_of_rank.as<int32_t>();
  T.inst_tie = lv.inst_tie.as<uint4>(); T.inst_rows = lv.inst_rows.as<mmp_instance_row>();
  T.min_space = f->hs.cfg.min_space_units; T.churn2 = (long long)((uint64_t)f->hs.cfg.min_churn_age_ms * 2u);
  T.type_stats = tstats; T.part_acc = acc; T.min_lru = d_min; T.sorted_rpm = rpm_sorted;
  T.n_ranks = ds.host.n_ranks; T.n_models = f->hs.n_models_used; T.n_type_ids = lv.n_type_ids; T.max_instances = f->hs.cfg.max_instances;
  T.tc_enabled = ds.host.tc_enabled;
  return T;
}

// The pod-task calls index their entries by model in the context's per-model slot array (max_models ints, -1 = no entry):
// k_slot_claim takes entry k's model slot (atomicCAS -1 -> k) and raises *dup where another entry holds it; k_slot_release
// gives the same slots back, so the array is filled with -1 only when it is allocated.  mmp_janitor_run and mmp_rate_run
// launch the pair; k_shutdown_plan / k_evict_plan claim and k_shutdown_pack / k_evict_pack release in their own launches.
template <class Entry>
__global__ void k_slot_claim(const Entry *entries, int n, int *slot, int *dup) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n && atomicCAS(&slot[entries[k].model], -1, k) != -1) *dup = 1;
}
template <class Entry>
__global__ void k_slot_release(const Entry *entries, int n, int *slot) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < n) slot[entries[k].model] = -1;
}

// mmp_janitor_run: the registry loop of one pod's janitor task (MM:6013-6145).  The pod's entries are indexed by model in
// slot[] (k_slot_claim); a second entry of one model is reported through cnt[JC_DUP].
enum { JC_EDITS = 0, JC_CANDS = 1, JC_REFS = 2, JC_DUP = 3 };
struct JanitorCand { int model, entry, edit, removes; long long reg_ts; };  // reg_ts: the time of self's loaded registration
// mmp_janitor_task: a model's record as the cache pass left it, per entry beside the entry's slot -- its lastUsed, and where
// the pass re-registered the pod, self's loaded registration time and whether it added a loaded copy
struct JanitorOv { long long last_used, reg_ts; int rereg, added; };
struct JanitorBufs {
  const mmp_janitor_entry *entries; int *slot;
  const JanitorOv *ov;                 // mmp_janitor_task: per entry (NULL for mmp_janitor_run: the committed records)
  const int *halt;                     // mmp_janitor_task: nonzero when the cache pass stopped (no registry pass)
  mmp_janitor_edit *edits;             // one per model at most, in no order
  unsigned long long *keys; int *vals; // candidate keys (last_used; ~0 past the candidates) and their JanitorCand index
  JanitorCand *cand;
  int *cnt;                            // JC_*
  mmp_janitor_report *report;
};
// a deregistration's record changes (the janitor's MM:6059-6073, deregisterModel's MM:2955-2957): updateLastUnloadTime where
// self's loaded copy left the record's cc loaded copies (MR:260-262), and updateLastUsed(lu) where use_lu (MR:239-246; the
// callers decide what lu is and when it applies).  k_janitor_sweep, k_janitor_walk and k_evict_plan all make it
__device__ __forceinline__ void dereg_record_edit(bool unregistered, bool use_lu, long long lu, int cc, long long now, int64_t &lu_rec,
                                                  int64_t &lul) {
  if (unregistered) lul = cc - 1 <= 2 ? 0 : now;
  if (use_lu && lu > lu_rec) lu_rec = lu;
}
// the record of entry k's model as the registry pass reads it: the cache pass's (J.ov) where there is one, else the committed
__device__ __forceinline__ JanitorOv janitor_record(const JanitorBufs &J, const mmp_model_row &mr, int k) {
  return J.ov && k >= 0 ? J.ov[k] : JanitorOv{mr.last_used, 0, 0, 0};
}
// one thread per model record, in the shape of k_registry_prune: self's loaded and failed registrations, remLoaded / remFailed
// (MM:6028-6053), the record changes of the edit (MM:6059-6073), REMOVE_LOCAL (MM:6089-6091) and the scale-down candidates
// (MM:6092-6100) with their last_used as the key
__global__ void k_janitor_sweep(RegTables R, const mmp_model_row *__restrict__ models, const long long *__restrict__ model_lul, int n_models,
                                int self, long long now, long long expiry_ms, JanitorBufs J) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models || (J.halt && *J.halt)) return;
  const mmp_model_row mr = models[m];
  const int n_regs = (int)mr.reserved;
  const int k_ov = J.ov ? J.slot[m] : -1;
  const JanitorOv rec = janitor_record(J, mr, k_ov);  // (a re-registration may give a model its first registration)
  if (n_regs == 0 && !rec.rereg) return;
  const int cc = mr.copy_count + rec.added;
  const ModelRegs g = model_regs(R, m, mr.reserved);
  int loaded_pos = -1;
  bool failed = false;
  long long loaded_ts = 0, failed_ts = 0;
  for (int j = 0; j < n_regs; j++) {
    long long ts;
    if (reg_at(R, g, j, ts) != self) continue;
    if (j < mr.copy_count) { if (loaded_pos < 0) { loaded_pos = j; loaded_ts = ts; } }
    else if (!failed) { failed = true; failed_ts = ts; }
  }
  if (rec.rereg) { loaded_pos = max(loaded_pos, 0); loaded_ts = rec.reg_ts; failed = false; }  // (put, removeLoadFailure)
  if (loaded_pos < 0 && !failed) return;
  atomicAdd(&J.cnt[JC_REFS], 1);
  const long long lul0 = model_lul[m];
  if (loaded_copies(mr) < 0) {  // where the loaded copies end is unknown (mmp_scale_eval's -1)
    J.edits[atomicAdd(&J.cnt[JC_EDITS], 1)] = mmp_janitor_edit{m, MMP_JE_UNDECIDED, rec.last_used, lul0};
    return;
  }
  const int k = J.ov ? k_ov : J.slot[m];
  mmp_janitor_entry ce{};
  if (k >= 0) ce = J.entries[k];
  const bool has = k >= 0, ce_failed = has && (ce.flags & MMP_JANITOR_FAILED), loaded = loaded_pos >= 0;
  const bool rem_loaded = loaded && (!has || ce_failed);
  bool rem_failed = false;
  if (failed) {
    if (has && !ce_failed) rem_failed = true;
    else {
      const long long lu = has ? ce.last_used : -1;
      // IN_USE_LOAD_FAILURE_EXPIRY_MS when used in the last SHORT_EXPIRY_RECENT_USE_TIME_MS (MM:221, 280)
      const long long expiry = lu > 0 && jsub(now, lu) < 180000LL ? expiry_ms / 2 : expiry_ms;
      rem_failed = jsub(now, failed_ts) > expiry;
    }
  }
  unsigned what = 0;
  int64_t lu_rec = rec.last_used, lul = lul0;
  if (rem_loaded || rem_failed) {
    if (rem_loaded) what |= MMP_JE_UNREGISTER;
    if (rem_failed) what |= MMP_JE_DROP_FAILURE;
    dereg_record_edit(rem_loaded, has, ce.last_used, cc, now, lu_rec, lul);  // updateLastUsed(lastUsed) where lastUsed > 0
  }
  if (rem_failed && ce_failed) what |= MMP_JE_REMOVE_LOCAL;
  int q = -1;
  if (what) J.edits[q = atomicAdd(&J.cnt[JC_EDITS], 1)] = mmp_janitor_edit{m, what, lu_rec, lul};
  if (loaded && !rem_loaded && ce.last_used > 0) {  // (an entry that is present and not failed)
    const int c = atomicAdd(&J.cnt[JC_CANDS], 1);
    J.keys[c] = (unsigned long long)ce.last_used;
    J.vals[c] = c;
    J.cand[c] = JanitorCand{m, k, q, 0, loaded_ts};
  }
}
// removeModelCopies of every candidate with canRemove = true, and removeLocalModelCopyAsync's check of the registration time
// against the entry's loadTimestamp (MM:6347-6349); the budget walk decides which of them run
__global__ void k_janitor_eval(ScaleTables T, mmp_scale_params p, int self, int flags, JanitorBufs J, int n) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n || c >= J.cnt[JC_CANDS]) return;
  const JanitorCand x = J.cand[c];
  const mmp_janitor_entry ce = J.entries[x.entry];
  const mmp_model_row mr = T.models[x.model];
  const ModelRegs g = model_regs(T.R, x.model, mr.reserved);
  const JanitorOv rec = janitor_record(J, mr, x.entry);
  const int loaded = loaded_copies(mr) + rec.added;  // (>= 0: k_janitor_sweep makes no candidate of a saturated record)
  J.cand[c].removes = scale_down_removes(T, p, self, x.model, ce.last_used, ce.last_heavy, ce.count, flags, g, loaded, T.rank_of[self],
                                         rec.rereg, rec.reg_ts, rec.added) &&
                      x.reg_ts == ce.load_ts;
}
// one thread: the TreeSet(VALUE_COMP) over the sorted candidates (of an equal-last_used run the first model in index order,
// quirk N15) and the budget of MM:6117-6140; SCALE_DOWN joins the model's edit or adds one; the report
__global__ void k_janitor_walk(JanitorBufs J, const mmp_model_row *__restrict__ models, long long budget, long long now) {
  const int nc = J.cnt[JC_CANDS];
  int n_edits = J.cnt[JC_EDITS], kept = 0, removed = 0;
  long long weight_removed = 0;
  for (int s = 0; s < nc;) {
    const unsigned long long key = J.keys[s];
    int best = J.vals[s];
    for (s++; s < nc && J.keys[s] == key; s++)
      if (J.cand[J.vals[s]].model < J.cand[best].model) best = J.vals[s];
    kept++;
    const JanitorCand x = J.cand[best];
    const mmp_janitor_entry ce = J.entries[x.entry];
    if (!((removed == 0 || ce.weight <= budget) && x.removes)) continue;
    removed++;
    budget -= ce.weight;
    weight_removed += ce.weight;
    // the async removal's record changes (MM:6363-6365) on the record after this run's edit of it
    const mmp_model_row mr = models[x.model];
    const JanitorOv rec = janitor_record(J, mr, x.entry);
    const int cc = mr.copy_count + rec.added;
    mmp_janitor_edit &e = x.edit >= 0 ? J.edits[x.edit] : J.edits[n_edits++];
    if (x.edit < 0) e = mmp_janitor_edit{x.model, 0u, rec.last_used, 0};
    e.what |= MMP_JE_SCALE_DOWN;
    dereg_record_edit(true, true, ce.last_used, cc, now, e.last_used, e.last_unload_time);
  }
  *J.report = mmp_janitor_report{J.cnt[JC_REFS], n_edits, kept, removed, weight_removed};
}

// mmp_janitor_task's cache pass (MM:5892-6008).  k_jt_plan gives every entry the action the loop would take if it reached
// the entry, the registry pass's copy of it (last_used -1 where it is removed) and its record after the action (JanitorOv,
// read beside the entry's slot); k_jt_order (one block, in entry order) adds the out-of-order scan and cuts the entries
// past the stop.  JtHdr.stop: the first qualifying Long.MAX_VALUE entry (atomicMin from 0x7f7f7f7f, > 2^24: none);
// halt: the registry pass does not run.  The header, the counters and the actions come back in one copy.
struct JtHdr { mmp_janitor_task_report rep; int stop, halt, pad[2]; };
static_assert(sizeof(JtHdr) == 96, "the counters follow the header");
constexpr long long JT_LONG_MAX = 0x7fffffffffffffffLL;
// updateLastUsedTimeInRegistryIfStale (MM:6165-6183; last_used is never Long.MAX_VALUE here) on the record rec
__device__ __forceinline__ void jt_stale_update(long long lu, long long min_stale, JanitorOv &rec, unsigned &what) {
  if (jsub(lu, rec.last_used) < min_stale) return;
  what |= MMP_JC_STALE_UPDATE;
  if (lu > rec.last_used) rec.last_used = lu;  // updateLastUsed (MR:239-246)
}
// one thread per entry: the loop body of MM:5904-5997 past the out-of-order log line
__global__ void k_jt_plan(RegTables R, const mmp_model_row *__restrict__ models, int n_models, const mmp_janitor_task_entry *__restrict__ te,
                          int n, int self, long long now, long long window, long long min_stale, mmp_janitor_entry *__restrict__ ent,
                          JanitorOv *__restrict__ ov, mmp_janitor_cache_action *__restrict__ out, JtHdr *__restrict__ hdr) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  mmp_janitor_entry e = te[r].e;
  const long long lu = e.last_used;
  const bool has_rec = e.model < n_models;  // registry.get / getStrong: the committed record, none for a model never upserted
  const mmp_model_row mr = has_rec ? models[e.model] : mmp_model_row{};
  JanitorOv rec{mr.last_used, 0, 0, 0};
  unsigned what = 0;
  long long shown = 0, replaced = -1;
  if (e.flags & MMP_JANITOR_NOT_DONE) {
    what = MMP_JC_NOT_DONE;
  } else if (lu <= 0) {
    what = MMP_JC_NOT_CACHED;
  } else if (lu == JT_LONG_MAX) {  // forceSetLastUsedTime, repairLastUsedTimeIfNeeded and the task's return (quirk N16)
    what = MMP_JC_STOP;
    shown = jsub(now, 3LL * 3600000LL);
    if (has_rec && mr.last_used == JT_LONG_MAX) { what |= MMP_JC_REPAIR; rec.last_used = shown; }
    atomicMin(&hdr->stop, r);
  } else if (jsub(now, lu) < window) {  // new or recently used
    if (has_rec) jt_stale_update(lu, min_stale, rec, what);
  } else if (has_rec && loaded_copies(mr) < 0) {
    what = MMP_JC_UNDECIDED;
  } else {
    // the pod's first loaded and first failed registration, as k_janitor_sweep finds them
    bool loaded_at = false, failed_at = false;
    long long loaded_ts = 0, failed_ts = 0;
    if (has_rec) {
      const ModelRegs g = model_regs(R, e.model, mr.reserved);
      for (int j = 0; j < (int)mr.reserved; j++) {
        long long ts;
        if (reg_at(R, g, j, ts) != self) continue;
        if (j < mr.copy_count) { if (!loaded_at) { loaded_at = true; loaded_ts = ts; } }
        else if (!failed_at) { failed_at = true; failed_ts = ts; }
      }
    }
    const bool failed = e.flags & MMP_JANITOR_FAILED;
    if (has_rec && (failed ? failed_at && failed_ts == te[r].load_complete_ts : loaded_at && loaded_ts == e.load_ts)) {
      jt_stale_update(lu, min_stale, rec, what);
    } else if (!has_rec || (e.flags & (MMP_JANITOR_NOT_LIVE | MMP_JANITOR_UNLOAD_RECENT))) {
      what = MMP_JC_REMOVE;
      e.last_used = -1;  // getLastUsedTime of a key no longer in the cache (MM:6045, 6068, 6094)
    } else {  // instanceIds.put(self, loadTimestamp), removeLoadFailure(self), updateLastUsed(lastUsed)
      what = MMP_JC_REREGISTER;
      if (!failed && loaded_at) replaced = loaded_ts;
      rec = JanitorOv{max(rec.last_used, lu), e.load_ts, 1, loaded_at ? 0 : 1};
    }
  }
  ent[r] = e;
  ov[r] = rec;
  out[r] = mmp_janitor_cache_action{e.model, what, (what & MMP_JC_STOP) ? shown : rec.last_used, replaced};
}
// One block over the entries in order, a tile of JT_ORDER_THREADS at a time: lastLastUsed (MM:5900, 5913-5917) is the
// last_used of the previous qualifying entry, found by an exclusive max-scan of the qualifying indices; the entries past the
// stop are not reached (their record's own lastUsed); the counts per bit and the report's flags
constexpr int JT_ORDER_THREADS = 512;
struct JtMax { __device__ __forceinline__ int operator()(int a, int b) const { return a > b ? a : b; } };
__global__ void __launch_bounds__(JT_ORDER_THREADS) k_jt_order(const mmp_janitor_task_entry *__restrict__ te, int n,
                                                               const mmp_model_row *__restrict__ models, int n_models,
                                                               mmp_janitor_cache_action *__restrict__ out, JtHdr *__restrict__ hdr) {
  using Scan = cub::BlockScan<int, JT_ORDER_THREADS>;
  __shared__ typename Scan::TempStorage tmp;
  __shared__ int carry, cnt[10];
  if (threadIdx.x < 10) cnt[threadIdx.x] = 0;
  if (threadIdx.x == 0) carry = -1;
  __syncthreads();
  const int stop = hdr->stop;
  for (int base = 0; base < n; base += JT_ORDER_THREADS) {
    const int r = base + threadIdx.x;
    int q = -1;
    long long lu = 0;
    if (r < n) {
      const mmp_janitor_entry e = te[r].e;
      lu = e.last_used;
      if (!(e.flags & MMP_JANITOR_NOT_DONE) && lu > 0) q = r;
    }
    const int before = carry;
    int prev, tile_max;
    Scan(tmp).ExclusiveScan(q, prev, before, JtMax(), tile_max);
    if (r < n) {
      mmp_janitor_cache_action a = out[r];
      if (r > stop) {
        a = mmp_janitor_cache_action{a.model, MMP_JC_NOT_REACHED, a.model < n_models ? models[a.model].last_used : 0, -1};
        out[r] = a;
      } else if (q >= 0 && prev >= 0 && lu > te[prev].e.last_used) {
        a.what |= MMP_JC_OUT_OF_ORDER;
        out[r].what = a.what;
      }
#pragma unroll
      for (int b = 0; b < 10; b++)
        if (a.what & (1u << b)) atomicAdd(&cnt[b], 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) carry = max(before, tile_max);
    __syncthreads();
  }
  if (threadIdx.x < 10) (&hdr->rep.n_not_done)[threadIdx.x] = cnt[threadIdx.x];
  if (threadIdx.x == 0) {
    const bool stopped = stop < n;
    hdr->rep.stopped_at = stopped ? stop : -1;
    hdr->rep.registry_ran = !stopped;
    hdr->rep.cache_changed = cnt[7] > 0;  // MMP_JC_REMOVE
    hdr->halt = stopped;
  }
}

// Lays a call's scratch out in one device buffer: take<T>(n) hands out room for n T's, each 16-byte aligned after the one
// before.  carve() runs a layout twice: once to size the buffer, which it ensures at that total, then to hand out the
// pointers, so no pointer is taken into a buffer that ensure() may still move.
struct Carve {
  uintptr_t base;
  size_t off = 0;
  template <class T> T *take(size_t n) { const size_t o = off; off += (n * sizeof(T) + 15) / 16 * 16; return reinterpret_cast<T *>(base + o); }
};
template <class Layout> static int32_t carve(DevBuf &buf, Layout layout) {
  Carve size{0};
  layout(size);
  CK(buf.ensure(size.off));
  Carve k{reinterpret_cast<uintptr_t>(buf.p)};
  layout(k);
  return MMP_OK;
}

// the epoch's type-set stats, queued on st: k_stats (the per-partition accumulators and the global LRU, into c->d_trace) and
// k_type_stats per type id.  queue_scale_eval and mmp_evict_run read them
struct TypeSetStats { StatsAcc *acc; long long *d_min; TypeStat *types; };
static int32_t queue_type_stats(mmp_fleet *f, PlaceCtx *c, const DeviceSnapshot &ds, LiveState &lv, TypeSetStats &S, cudaStream_t st) {
  const int np = (int)ds.host.part_types.size(), nr = ds.host.n_ranks, nt = lv.n_type_ids;
  const int32_t rc = carve(c->d_trace, [&](Carve &k) { S.acc = k.take<StatsAcc>(np + 1); S.d_min = k.take<long long>(1); S.types = k.take<TypeStat>(std::max(nt, 1)); });
  if (rc < 0) return rc;
  CK(cudaMemsetAsync(S.acc, 0, (size_t)(np + 1) * sizeof(StatsAcc), st));
  static const long long init = 0x7fffffffffffffffLL;
  CK(cudaMemcpyAsync(S.d_min, &init, 8, cudaMemcpyHostToDevice, st));
  if (nr > 0) {
    k_stats<<<std::min(f->sm_count, (nr + 255) / 256), 256, 0, st>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(), ds.part_of_rank.as<int32_t>(), nr,
                                                                     f->hs.cfg.min_space_units, S.acc, S.d_min, np);
    f->launches++;
  }
  k_type_stats<<<(std::max(nt, 1) + 127) / 128, 128, 0, st>>>(S.acc, S.d_min, lv.type_part_off.as<int>(), lv.type_parts.as<int>(), nt, S.types);
  f->launches++;
  CK(cudaGetLastError());
  return MMP_OK;
}

// mmp_scale_eval's device part, queued on st: the type-set stats (queue_type_stats), the sorted rpm column (into rpm) and
// k_scale_eval of in[0, n) into out (both on the device).  mmp_rate_run runs the same.
static int32_t queue_scale_eval(mmp_fleet *f, PlaceCtx *c, const DeviceSnapshot &ds, LiveState &lv, const mmp_scale_in *in, int32_t n,
                                const mmp_scale_params &params, DevBuf &rpm, mmp_scale_out *out, cudaStream_t st) {
  const int nr = ds.host.n_ranks;
  TypeSetStats S;
  const int32_t rc = queue_type_stats(f, c, ds, lv, S, st);
  if (rc < 0) return rc;
  CK(rpm.ensure((size_t)std::max(nr, 1) * 8 + 64));
  int *rpm_raw = rpm.as<int>(), *rpm_sorted = rpm_raw + std::max(nr, 1);
  if (nr > 0) {
    k_extract_rpm<<<(nr + 255) / 256, 256, 0, st>>>(ds.rows.as<RankRow>(), nr, rpm_raw);
    size_t tmp = 0;
    CK(cub::DeviceRadixSort::SortKeys(nullptr, tmp, rpm_raw, rpm_sorted, nr, 0, 32, st));
    CK(c->d_cub.ensure(tmp + 16));
    CK(cub::DeviceRadixSort::SortKeys(c->d_cub.p, tmp, rpm_raw, rpm_sorted, nr, 0, 32, st));
    f->launches += 2;
  }
  const ScaleTables T = scale_tables(f, ds, lv, S.acc, S.d_min, S.types, rpm_sorted);
  k_scale_eval<<<(n + 127) / 128, 128, 0, st>>>(T, in, n, params, out);
  f->launches++;
  CK(cudaGetLastError());
  return MMP_OK;
}

// mmp_rate_run: one pod's rate-tracking task (MM:5619-5858).  After k_scale_eval, k_rate_heavy lists getExcludeSet and
// k_rate_plan (one block) applies checkLoadFailureCount and numbers the decisions: each entry's second copy (per entry, an
// inactive record where there is none) and decision 0 of each scale-up chain (compacted in entry order).  The host reads the
// counts back once, then places the second copies under the epoch's tables and the chains round by round under the tables
// derived for the heavy set; k_rate_step builds round j from round j - 1.  An inactive decision has model -1: a malformed
// record, answered MMP_TARGET_INVALID without a walk.  The pod's entries are indexed by model in slot[] (k_slot_claim) only
// to find two entries of one model.
struct RateHdr { int n_heavy, dup, n_second, n_scale_up, n_refused, n_sec_place, n_chain, longest; long long n_ids; };
struct RateChain { int entry, copies, id0, len; };  // len: the decisions the chain places at most (min(copies, MMP_RATE_CHAIN_MAX))
struct RateBufs {
  const mmp_scale_in *entries; const mmp_scale_out *sout; int *slot;
  mmp_decision_in *sec;    // per entry
  mmp_decision_in *c0;     // per chain: decision 0
  RateChain *chains;
  int32_t *extra;          // [the pod | MMP_MAX_EXTRA per chain: its targets so far]
  int32_t *heavy;
  RateHdr *hdr;
};
__device__ __forceinline__ mmp_decision_in rate_inactive(int pod) { return mmp_decision_in{-1, pod, 0, 0u, -1, 0, 0}; }
// getExcludeSet (MM:5835-5856): the instances of the snapshot other than the pod whose published rpm is above the bound, in
// no order (the derived tables do not depend on it)
__global__ void k_rate_heavy(const int32_t *__restrict__ rank_of, const RankRow *__restrict__ rows, int max_instances, int pod, int thr,
                             RateBufs B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= max_instances || i == pod) return;
  const int rk = rank_of[i];
  if (rk < 0) return;
  const int pr = rank_of[pod];
  if (rows[rk].rpm > exclude_set_max_rpm(thr, pr >= 0 ? rows[pr].rpm : 0)) B.heavy[atomicAdd(&B.hdr->n_heavy, 1)] = i;
}
// checkLoadFailureCount (MM:3771, 4607-4627): 3 or more failure records (the registrations past the `loaded` copies) whose time
// is after fail_since refuse the load.  dropped: how many of those records the caller's own edit removed first (k_evict_plan:
// the pod's failure record that deregisterModel dropped).  k_rate_plan, k_shutdown_plan and k_evict_plan all ask it
__device__ __forceinline__ bool load_failures_refuse(const RegTables &R, const ModelRegs &g, int loaded, int n_edges, long long fail_since,
                                                     int dropped = 0) {
  int recent = -dropped;
  long long ts;
  for (int j = loaded; j < n_edges; j++) {
    reg_at(R, g, j, ts);
    if (ts > fail_since) recent++;
  }
  return recent >= 3;
}
// One block over the entries in order, a tile of RATE_PLAN_THREADS at a time: checkLoadFailureCount (load_failures_refuse), the ids (exclusive prefix sum of the decisions per entry) and the round-0 records
constexpr int RATE_PLAN_THREADS = 512;
__global__ void __launch_bounds__(RATE_PLAN_THREADS) k_rate_plan(RegTables R, const mmp_model_row *__restrict__ models, RateBufs B, int n,
                                                                 int pod, long long fail_since, int fresh) {
  using IdScan = cub::BlockScan<long long, RATE_PLAN_THREADS>;
  using ChainScan = cub::BlockScan<int, RATE_PLAN_THREADS>;
  __shared__ union { typename IdScan::TempStorage ids; typename ChainScan::TempStorage chains; } tmp;
  __shared__ long long ids_before;
  __shared__ int chains_before, tot[5];  // n_second, n_scale_up, n_refused, n_sec_place, longest
  if (threadIdx.x < 5) tot[threadIdx.x] = 0;
  if (threadIdx.x == 0) { ids_before = 0; chains_before = 0; B.extra[0] = pod; }
  __syncthreads();
  for (int base = 0; base < n; base += RATE_PLAN_THREADS) {
    const int r = base + threadIdx.x;
    int len = 0, chain = 0, favour = 0, model = -1;
    mmp_scale_out o{};
    if (r < n) {
      o = B.sout[r];
      model = B.entries[r].model;
      if (o.action == 1 || o.action == 2) {
        const mmp_model_row mr = models[model];
        const ModelRegs g = model_regs(R, model, mr.reserved);
        const int n_edges = (int)mr.reserved, loaded = loaded_copies(mr);  // (>= 0: k_scale_eval answered -1 for a saturated record)
        long long ts;
        atomicAdd(&tot[o.action == 1 ? 0 : 1], 1);
        if (load_failures_refuse(R, g, loaded, n_edges, fail_since)) atomicAdd(&tot[2], 1);
        else if (o.action == 1) { len = 1; atomicAdd(&tot[3], 1); }
        else if (o.copies_to_load > 0) {
          len = min(o.copies_to_load, MMP_RATE_CHAIN_MAX);
          chain = 1;
          for (int j = 0; j < loaded; j++) if (reg_at(R, g, j, ts) == pod) favour = 1;
          atomicMax(&tot[4], len);
        }
      }
    }
    long long id, ids_tile;
    int q, chains_tile;
    IdScan(tmp.ids).ExclusiveSum((long long)len, id, ids_tile);
    __syncthreads();
    ChainScan(tmp.chains).ExclusiveSum(chain, q, chains_tile);
    id += ids_before;
    q += chains_before;
    if (r < n) {
      const unsigned own = MMP_DF_OWN_ID | ((unsigned)id << 8);
      B.sec[r] = len && !chain ? mmp_decision_in{model, pod, o.load_last_used, MMP_DF_FAVOUR_SELF | own, fresh, 0, 1} : rate_inactive(pod);
      if (chain) {
        B.chains[q] = RateChain{r, o.copies_to_load, (int)id, len};
        B.c0[q] = mmp_decision_in{model, pod, o.load_last_used, (favour ? MMP_DF_FAVOUR_SELF : 0u) | own, fresh, 1 + q * MMP_MAX_EXTRA, 0};
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) { ids_before += ids_tile; chains_before += chains_tile; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    RateHdr *h = B.hdr;
    h->n_second = tot[0]; h->n_scale_up = tot[1]; h->n_refused = tot[2]; h->n_sec_place = tot[3]; h->longest = tot[4];
    h->n_chain = chains_before; h->n_ids = ids_before;
  }
}
// round j >= 1 of every chain from round j - 1: self = target j - 1 (the pod for MMP_TARGET_SELF), appended to the chain's
// extras; a chain whose target was MMP_TARGET_NONE / INVALID, or that has placed its len decisions, goes inactive
__global__ void k_rate_step(const mmp_decision_in *__restrict__ prev, const mmp_decision_out *__restrict__ res,
                            const RateChain *__restrict__ chains, int n_chain, int j, int pod, int fresh, int32_t *__restrict__ extra,
                            mmp_decision_in *__restrict__ next) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_chain) return;
  mmp_decision_in d = prev[q];
  const int t = res[q].target;
  const RateChain ch = chains[q];
  if (d.model < 0 || t == MMP_TARGET_NONE || t == MMP_TARGET_INVALID || j >= ch.len) { next[q] = rate_inactive(pod); return; }
  const int s = t == MMP_TARGET_SELF ? pod : t;
  extra[d.extra_off + j - 1] = s;
  d.self = s;
  d.fresh = s == pod ? fresh : -1;
  d.extra_n = j;
  d.flags = MMP_DF_FAVOUR_SELF | MMP_DF_OWN_ID | ((unsigned)(ch.id0 + j) << 8);
  next[q] = d;
}

// mmp_shutdown_run: one pod's pre-shutdown migration (MM:6990-7047).  k_shutdown_plan classifies every entry and writes its
// decision, or rate_inactive's record where there is none; launch_place answers all n; k_shutdown_pack adds the answers and
// the wait test.  The entries take their model's slot of slot[] in k_shutdown_plan and give it back in k_shutdown_pack, a
// later launch on the same stream: two entries of one model are found without a launch of their own.
// mmp_shutdown_run's and mmp_evict_run's header: the report and the duplicate flag (48 B: the actions follow it in one copy
// back, pack_copy_back)
template <class Report> struct PackHdr { Report rep; int dup, pad[3]; };
static_assert(sizeof(PackHdr<mmp_shutdown_report>) == 48 && sizeof(PackHdr<mmp_evict_report>) == 48, "the actions follow the header");
struct SdBufs {
  const mmp_shutdown_entry *entries; int *slot;
  mmp_decision_in *dec; const mmp_decision_out *res;
  PackHdr<mmp_shutdown_report> *hdr; mmp_shutdown_action *out;
  int32_t *extra;  // [the pod]
};
// one thread per entry: foundOther (MM:6968-6976), the registry test over every registration (MM:7007-7010), willBeSkipped
// (MM:7011-7014), the task body up to its getNext (MM:7017-7032) with checkLoadFailureCount
__global__ void k_shutdown_plan(RegTables R, const mmp_model_row *__restrict__ models, const int32_t *__restrict__ rank_of, int n_ranks,
                                SdBufs B, int n, int pod, long long cutoff, long long fail_since, int fresh) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  const bool found_other = n_ranks - (rank_of[pod] >= 0 ? 1 : 0) > 0;
  if (r == 0) { B.hdr->rep.found_other = found_other; B.extra[0] = pod; }
  if (r >= n) return;
  const mmp_shutdown_entry e = B.entries[r];
  if (atomicCAS(&B.slot[e.model], -1, r) != -1) B.hdr->dup = 1;
  unsigned what = 0;
  long long lru = 0;
  if (found_other) {
    const mmp_model_row mr = models[e.model];
    const ModelRegs g = model_regs(R, e.model, mr.reserved);
    const int n_edges = (int)mr.reserved, loaded = loaded_copies(mr);
    bool registered = false;
    long long ts;
    for (int j = 0; j < loaded && !registered; j++) registered = reg_at(R, g, j, ts) == pod;
    if (loaded < 0) {
      what = MMP_SD_UNDECIDED;
    } else if (!registered) {
      what = MMP_SD_NOT_REGISTERED;
    } else {
      atomicAdd(&B.hdr->rep.n_registered, 1);
      if (e.lru_t < cutoff) { what |= MMP_SD_STALE; atomicAdd(&B.hdr->rep.will_be_skipped, 1); }
      if (!(e.flags & (MMP_SD_ENTRY_GONE | MMP_SD_ENTRY_FAILED))) {
        lru = e.lru_t != 0 ? e.lru_t : e.last_used;
        if (lru >= 0) what |= MMP_SD_REMOVE_LOCAL;
        if (e.flags & MMP_SD_ENTRY_ABORTED) what |= MMP_SD_DEREGISTER_NOW;
        if (lru > 0) {
          if (load_failures_refuse(R, g, loaded, n_edges, fail_since)) { what |= MMP_SD_REFUSED; atomicAdd(&B.hdr->rep.n_refused, 1); }
          else what |= MMP_SD_PLACED;
        }
      }
    }
  }
  B.dec[r] = (what & MMP_SD_PLACED) ? mmp_decision_in{e.model, pod, lru, MMP_DF_FAVOUR_SELF | MMP_DF_OWN_ID | ((unsigned)r << 8), fresh, 0, 1}
                                    : rate_inactive(pod);
  B.out[r] = mmp_shutdown_action{e.model, what, MMP_TARGET_INVALID, 0, lru};
}
// one thread per entry: the answer, Status.LOADING && lruTime >= cutoff (MM:7037-7038) as a target that is an instance
__global__ void k_shutdown_pack(SdBufs B, int n, long long cutoff) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  mmp_shutdown_action a = B.out[r];
  B.slot[a.model] = -1;
  if (!(a.what & MMP_SD_PLACED)) return;
  const mmp_decision_out o = B.res[r];
  a.target = o.target;
  a.n_candidates = o.n_candidates;
  atomicAdd(&B.hdr->rep.n_placed, 1);
  if (o.target == MMP_TARGET_NONE) atomicAdd(&B.hdr->rep.n_none, 1);
  else if (o.target >= 0 && a.last_used >= cutoff) { a.what |= MMP_SD_WAIT; atomicAdd(&B.hdr->rep.n_wait, 1); }
  B.out[r] = a;
}

// mmp_evict_run: one pod's eviction listener (MM:2867-2933) for a burst of evictions.  The type-set stats come from
// queue_type_stats; k_evict_plan makes every entry's deregistration edit and decides its reload, writing the decision or
// rate_inactive's record; launch_place answers all n; k_evict_pack adds the answers and the report.  The entries take their
// model's slot of slot[] in k_evict_plan and give it back in k_evict_pack, as mmp_shutdown_run's do.
struct EvBufs {
  const mmp_evict_entry *entries; int *slot;
  mmp_decision_in *dec; const mmp_decision_out *res;
  PackHdr<mmp_evict_report> *hdr; mmp_evict_action *out;
  int32_t *extra;  // [the pod]
};
// one thread per entry: the pod's registrations over every registration of the model, deregisterModel's edit (MM:2948-2957,
// the record arithmetic through dereg_record_edit), attemptReload on the record before it (MM:2886-2896), the rebalance gate
// (MM:2918-2920) and ensureLoadedElsewhere up to its getNext on the record after it: a live copy elsewhere, then
// checkLoadFailureCount without the failure record the edit dropped
__global__ void k_evict_plan(RegTables R, const mmp_model_row *__restrict__ models, const long long *__restrict__ model_lul,
                             const int32_t *__restrict__ rank_of, const TypeStat *__restrict__ type_stats, int n_type_ids, EvBufs B, int n,
                             int pod, long long now, long long reload_age, long long fail_since, int fresh) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0) B.extra[0] = pod;
  if (r >= n) return;
  const mmp_evict_entry e = B.entries[r];
  if (atomicCAS(&B.slot[e.model], -1, r) != -1) B.hdr->dup = 1;
  const mmp_model_row mr = models[e.model];
  const int loaded = loaded_copies(mr);
  if (loaded < 0) {
    B.dec[r] = rate_inactive(pod);
    B.out[r] = mmp_evict_action{e.model, MMP_EV_UNDECIDED, MMP_TARGET_INVALID, 0, mr.last_used, model_lul[e.model]};
    return;
  }
  const ModelRegs g = model_regs(R, e.model, mr.reserved);
  const int n_edges = (int)mr.reserved;
  // the pod's first loaded and first failed registration (as k_janitor_sweep finds them), and a loaded copy on another ranked
  // instance
  int loaded_at = -1, failed_at = -1;
  long long loaded_ts = 0, failed_ts = 0;
  bool live_elsewhere = false;
  for (int j = 0, top = max(loaded, n_edges); j < top; j++) {
    long long ts;
    const int i = reg_at(R, g, j, ts);
    if (i == pod) {
      if (j < loaded) { if (loaded_at < 0) { loaded_at = j; loaded_ts = ts; } }
      else if (failed_at < 0) { failed_at = j; failed_ts = ts; }
    } else if (j < loaded && i >= 0 && rank_of[i] >= 0) {
      live_elsewhere = true;
    }
  }
  const bool unreg = loaded_at >= 0 && loaded_ts == e.load_ts, drop = failed_at >= 0 && failed_ts == e.load_complete_ts;
  unsigned what = (unreg ? MMP_EV_UNREGISTER : 0u) | (drop ? MMP_EV_DROP_FAILURE : 0u);
  int64_t lu_rec = mr.last_used, lul = model_lul[e.model];
  if (unreg || drop) dereg_record_edit(unreg, true, e.last_used == 0 ? now : e.last_used, mr.copy_count, now, lu_rec, lul);
  if (!(e.flags & MMP_EV_ENTRY_FAILED) && (loaded_at >= 0 || failed_at >= 0) && jsub(now, loaded_at >= 0 ? loaded_ts : failed_ts) > reload_age) {
    what |= MMP_EV_RELOAD;
    const TypeStat cs = type_stats[mr.type_id < n_type_ids ? mr.type_id : 0];
    if (!(cs.cap > 0 && cs.count > 1 && jmul64(20, cs.free) / cs.cap >= 1)) what |= MMP_EV_CLUSTER_FULL;
    else if (live_elsewhere) what |= MMP_EV_LOADED_ELSEWHERE;
    else if (load_failures_refuse(R, g, loaded, n_edges, fail_since, drop && failed_ts > fail_since)) what |= MMP_EV_REFUSED;
    else what |= MMP_EV_PLACED;
  }
  B.dec[r] = (what & MMP_EV_PLACED) ? mmp_decision_in{e.model, pod, e.last_used, MMP_DF_FAVOUR_SELF | MMP_DF_OWN_ID | ((unsigned)r << 8), fresh, 0, 1}
                                    : rate_inactive(pod);
  B.out[r] = mmp_evict_action{e.model, what, MMP_TARGET_INVALID, 0, lu_rec, lul};
}
// one thread per entry: the answer, and the report (one counter per MMP_EV_* bit below MMP_EV_UNDECIDED, in bit order, then
// n_none)
__global__ void k_evict_pack(EvBufs B, int n) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  mmp_evict_action a = B.out[r];
  B.slot[a.model] = -1;
  int32_t *cnt = &B.hdr->rep.n_unregister;
#pragma unroll
  for (int b = 0; b < 7; b++)
    if (a.what & (1u << b)) atomicAdd(cnt + b, 1);
  if (!(a.what & MMP_EV_PLACED)) return;
  const mmp_decision_out o = B.res[r];
  a.target = o.target;
  a.n_candidates = o.n_candidates;
  if (o.target == MMP_TARGET_NONE) atomicAdd(&B.hdr->rep.n_none, 1);
  B.out[r] = a;
}

// ---------------------------------------------------------------------------------------------------------------
// the host steps the pod-task calls share: mmp_reaper_run, mmp_janitor_run, mmp_rate_run, mmp_shutdown_run, mmp_evict_run
// ---------------------------------------------------------------------------------------------------------------
// MMP_E_ARG for the first entry whose model index is out of range or that `also` refuses (a message, else null)
template <class Entry> static int32_t entry_model(const Entry &e) { return e.model; }
static int32_t entry_model(const mmp_janitor_task_entry &e) { return e.e.model; }
template <class Entry, class Also>
static int32_t check_entries(const mmp_fleet *f, const Entry *entries, int32_t n, Also also) {
  for (int32_t k = 0; k < n; k++) {
    const int32_t m = entry_model(entries[k]);
    if (m < 0 || m >= f->hs.cfg.max_models) { g_err = "entry model index out of range"; return MMP_E_ARG; }
    if (const char *m = also(entries[k])) { g_err = m; return MMP_E_ARG; }
  }
  return MMP_OK;
}
template <class Entry> static int32_t check_entries(const mmp_fleet *f, const Entry *entries, int32_t n) {
  return check_entries(f, entries, n, [](const Entry &) -> const char * { return nullptr; });
}

static int32_t parse_fresh_self(const mmp_instance_row *fresh_self, FreshRow &fr) {
  if (fresh_self)
    if (const char *m = HostState::fresh_row(*fresh_self, fr)) { g_err = std::string("fresh row: ") + m; return MMP_E_ARG; }
  return MMP_OK;
}

// How a pod-task call opens, after its own argument checks.  It reads the registry as of the last commit and the epoch built
// from it: ingest_mu, then snap_mu shared (a commit's order: it flips the epoch under snap_mu while it holds ingest_mu), both
// held until the call returns.  Then the refusals: no committed snapshot; no registration times (TIMES); a fleet on which
// placing elsewhere is a collective call (PLACES).  Then the context lease and, for SLOTS, the per-model slot array.
class PodCall {
 public:
  enum : unsigned { TIMES = 1, PLACES = 2, SLOTS = 4 };
  PlaceCtx *c = nullptr;
  const DeviceSnapshot *ds = nullptr;
  LiveState *lv = nullptr;

  int32_t open(mmp_fleet *f, const char *name, unsigned need) {
    const int32_t rc = set_device(f);
    if (rc < 0) return rc;
    ingest_ = std::unique_lock<std::mutex>(f->ingest_mu);
    snap_ = std::shared_lock<std::shared_mutex>(f->snap_mu);
    if (f->epoch == 0 || !f->live.valid) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
    if ((need & TIMES) && !f->live.have_times) { g_err = "the committed registry has no registration times (mmp_model_times)"; return MMP_E_STATE; }
    if ((need & PLACES) && places_sharded(f, false)) {
      g_err = std::string(name) + " places on an unsharded fleet without a communicator (elsewhere placement is a collective call)";
      return MMP_E_STATE;
    }
    lease_.emplace(f);
    if (!*lease_) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
    c = lease_->get(); ds = &f->snaps[f->cur]; lv = &f->live;
    const size_t slot_b = (size_t)f->hs.cfg.max_models * 4;
    if ((need & SLOTS) && c->d_model_slot.cap < slot_b) {  // filled with -1 once; every call leaves it so
      CK(c->d_model_slot.ensure(slot_b));
      CK(cudaMemsetAsync(c->d_model_slot.p, 0xff, c->d_model_slot.cap, c->stream));
    }
    return MMP_OK;
  }

 private:
  std::unique_lock<std::mutex> ingest_;
  std::shared_lock<std::shared_mutex> snap_;
  std::optional<CtxLease> lease_;  // (after the locks: given back before they are released)
};

// The call's fresh row for the pod (none where fr is null) into d_fresh, and d_extra sized for n_extra excludes
static int32_t stage_fresh_self(PlaceCtx *c, const FreshRow *fr, size_t n_extra) {
  c->fresh_host.assign(fr ? 1 : 0, fr ? *fr : FreshRow{});
  const int32_t rc = stage_side_tables(c, c->fresh_host.data(), (int32_t)c->fresh_host.size(), nullptr, 0, c->stream);
  if (rc < 0) return rc;
  CK(c->d_extra.ensure(n_extra * 4));
  return MMP_OK;
}

// Places in[0, n) under the view v into out on the call's stream, with the fresh row and the extras stage_fresh_self staged
static cudaError_t place_staged(mmp_fleet *f, PlaceCtx *c, const SnapshotView &v, const mmp_decision_in *in, int n,
                                mmp_decision_out *out, int64_t now, uint64_t seed) {
  PlaceArgs a{v, in, n, c->d_fresh.as<FreshRow>(), (int)c->fresh_host.size(), c->d_extra.as<int32_t>(), out, nullptr, nullptr, now, seed,
              f->id_base.load()};
  a.ctx = c;
  return launch_place(f, a, c->stream);
}

// The end of mmp_shutdown_run and mmp_evict_run: e1, one copy back of [header | actions], the synchronise and the timer; then
// two entries of one model are refused, or the actions and the report are written
template <class Report, class Action>
static int32_t pack_copy_back(PlaceCtx *c, const PackHdr<Report> *hdr, int32_t n, float &t_ms, Action *out, Report *report) {
  CK(cudaEventRecord(c->e1, c->stream));
  std::vector<char> back(sizeof(PackHdr<Report>) + (size_t)n * sizeof(Action));
  CK(cudaMemcpyAsync(back.data(), hdr, back.size(), cudaMemcpyDeviceToHost, c->stream));
  CK(cudaStreamSynchronize(c->stream));
  event_ms(c, t_ms);
  PackHdr<Report> H;
  memcpy(&H, back.data(), sizeof(H));
  if (H.dup) { g_err = "two entries of one model"; return MMP_E_ARG; }
  if (n) memcpy(out, back.data() + sizeof(H), (size_t)n * sizeof(Action));
  *report = H.rep;
  return n;
}

// mmp_janitor_run's and mmp_janitor_task's registry pass, queued on the call's stream once the pod's entries are on the
// device: the stats (into acc / d_min, cleared by the caller), the slot claim, the sweep, the candidates' eval and sort, the
// budget walk (e1 is recorded after it) and the slot release
static int32_t queue_janitor_pass(mmp_fleet *f, PlaceCtx *c, const DeviceSnapshot &ds, LiveState &lv, const JanitorBufs &J, const JanitorBufs &Js,
                                  int32_t n, int32_t self, const mmp_janitor_params &p, StatsAcc *acc, long long *d_min) {
  const int32_t NM = ds.n_models, np = (int)ds.host.part_types.size(), nr = ds.host.n_ranks;
  cudaStream_t st = c->stream;
  if (nr > 0) {  // instanceSetStats / globalLru for the scale-down
    k_stats<<<std::min(f->sm_count, (nr + 255) / 256), 256, 0, st>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(), ds.part_of_rank.as<int32_t>(), nr,
                                                                     f->hs.cfg.min_space_units, acc, d_min, np);
    f->launches++;
  }
  if (n) { k_slot_claim<<<(n + 255) / 256, 256, 0, st>>>(J.entries, n, J.slot, J.cnt + JC_DUP); f->launches++; }
  if (NM) {
    k_janitor_sweep<<<(NM + 255) / 256, 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), lv.model_lul.as<long long>(), NM, self,
                                                      p.scale.now, p.load_failure_expiry_ms, J);
    f->launches++;
  }
  CK(cudaGetLastError());
  if (n) {  // the candidates (at most one per entry) by ascending last_used; eval before the sort reads them by JanitorCand index
    mmp_scale_params sp = p.scale;
    sp.can_remove = 1;
    k_janitor_eval<<<(n + 127) / 128, 128, 0, st>>>(scale_tables(f, ds, lv, acc, d_min, nullptr, nullptr), sp, self, (int)p.flags, J, n);
    size_t tmp = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp, J.keys, Js.keys, J.vals, Js.vals, n, 0, 64, st));
    CK(c->d_cub.ensure(tmp + 16));
    CK(cub::DeviceRadixSort::SortPairs(c->d_cub.p, tmp, J.keys, Js.keys, J.vals, Js.vals, n, 0, 64, st));
    f->launches += 2;
  }
  k_janitor_walk<<<1, 1, 0, st>>>(Js, lv.models.as<mmp_model_row>(), p.adjusted_capacity / 20, p.scale.now);
  CK(cudaEventRecord(c->e1, st));
  if (n) k_slot_release<<<(n + 255) / 256, 256, 0, st>>>(J.entries, n, J.slot);
  f->launches += n ? 2 : 1;
  CK(cudaGetLastError());
  return MMP_OK;
}
// the edits the first copy back brings: as many as a pod is likely to have (twice its entries + 1024: most edits are of
// models the pod holds); more take a second copy (janitor_edits_out)
static size_t janitor_first_edits(int32_t NM, int32_t n) { return (size_t)std::min<int64_t>(std::max(NM, 1), 2 * (int64_t)n + 1024); }
// the n_edits edits in model order into edits[0, cap): the first `first` from the copy back at hb, the rest from the device
static int32_t janitor_edits_out(const JanitorBufs &J, const char *hb, size_t first, int32_t n_edits, mmp_janitor_edit *edits, int32_t cap) {
  std::vector<mmp_janitor_edit> ed((size_t)n_edits);
  memcpy(ed.data(), hb, std::min(ed.size(), first) * sizeof(mmp_janitor_edit));
  if (ed.size() > first)
    CK(cudaMemcpy(ed.data() + first, J.edits + first, (ed.size() - first) * sizeof(mmp_janitor_edit), cudaMemcpyDeviceToHost));
  std::sort(ed.begin(), ed.end(), [](const mmp_janitor_edit &a, const mmp_janitor_edit &b) { return a.model < b.model; });
  if (cap > 0 && n_edits) memcpy(edits, ed.data(), (size_t)std::min(n_edits, cap) * sizeof(mmp_janitor_edit));
  return MMP_OK;
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
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  cudaStream_t st = c->stream;
  CK(c->d_in.ensure((size_t)n * sizeof(mmp_scale_in)));
  CK(c->d_out.ensure((size_t)n * sizeof(mmp_scale_out)));
  CK(cudaMemcpyAsync(c->d_in.p, in, (size_t)n * sizeof(mmp_scale_in), cudaMemcpyHostToDevice, st));
  if ((rc = queue_scale_eval(f, c.get(), f->snaps[f->cur], f->live, c->d_in.as<mmp_scale_in>(), n, *params, c->d_fresh,
                             c->d_out.as<mmp_scale_out>(), st)) < 0)
    return rc;
  CK(cudaMemcpyAsync(out, c->d_out.p, (size_t)n * sizeof(mmp_scale_out), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return MMP_OK;
}

int32_t mmp_registry_prune(mmp_fleet *f, int32_t self, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, int32_t *out_models,
                           uint8_t *out_masks, int32_t cap) {
  NEED(f);
  if (!missing_since || cap < 0 || (cap > 0 && (!out_models || !out_masks))) { g_err = "bad argument"; return MMP_E_ARG; }
  return registry_prune(f, self, now_ms, assume_gone_ms, missing_since, false, [&](PlaceCtx *c, int n_out) -> int32_t {
    if (n_out == 0) return 0;
    std::vector<int32_t> ms((size_t)n_out);
    std::vector<uint8_t> mk((size_t)n_out);
    CK(cudaMemcpy(ms.data(), c->d_out.p, (size_t)n_out * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(mk.data(), c->d_extra.p, (size_t)n_out, cudaMemcpyDeviceToHost));
    std::vector<int32_t> ord((size_t)n_out);
    for (int i = 0; i < n_out; i++) ord[i] = i;
    std::sort(ord.begin(), ord.end(), [&](int a, int b) { return ms[a] < ms[b]; });  // model order: one record per model
    for (int i = 0; i < std::min(n_out, cap); i++) { out_models[i] = ms[ord[i]]; out_masks[i] = mk[ord[i]]; }
    return n_out;
  });
}

int32_t mmp_registry_prune_ids(mmp_fleet *f, int32_t self, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, int32_t *out_models,
                               int32_t *out_instances, int32_t cap) {
  NEED(f);
  if (!missing_since || cap < 0 || assume_gone_ms < 0 || (cap > 0 && (!out_models || !out_instances))) { g_err = "bad argument"; return MMP_E_ARG; }
  return registry_prune(f, self, now_ms, assume_gone_ms, missing_since, true, [&](PlaceCtx *c, int n_out) -> int32_t {
    std::vector<PrunedReg> regs((size_t)n_out);
    if (n_out) CK(cudaMemcpy(regs.data(), c->d_out.p, (size_t)n_out * sizeof(PrunedReg), cudaMemcpyDeviceToHost));
    std::sort(regs.begin(), regs.end(), [](const PrunedReg &a, const PrunedReg &b) { return a.model != b.model ? a.model < b.model : a.pos < b.pos; });
    for (int i = 0; i < std::min(n_out, cap); i++) { out_models[i] = regs[i].model; out_instances[i] = regs[i].inst; }
    return n_out;
  });
}


int32_t mmp_reaper_run(mmp_fleet *f, int32_t leader, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, uint64_t seed,
                       int32_t *pruned_models, int32_t *pruned_instances, int32_t pruned_cap, int32_t *repaired_models,
                       int32_t repaired_cap, mmp_reaper_load *loads, int32_t loads_cap, mmp_reaper_report *report) {
  NEED(f);
  if (leader < 0 || leader >= f->hs.cfg.max_instances || assume_gone_ms < 0 || !missing_since || !report || pruned_cap < 0 ||
      repaired_cap < 0 || loads_cap < 0 || (pruned_cap > 0 && (!pruned_models || !pruned_instances)) ||
      (repaired_cap > 0 && !repaired_models) || (loads_cap > 0 && !loads)) {
    g_err = "bad argument"; return MMP_E_ARG;
  }
  // The prune reads the live registry (as registry_prune does), the selection and the placement the epoch (as mmp_reaper_select
  // and mmp_place_batch do): holding both locks, the registry read is the one the epoch was built from.
  PodCall pc;
  int32_t rc = pc.open(f, "mmp_reaper_run", PodCall::PLACES);
  if (rc < 0) return rc;
  PlaceCtx *c = pc.c; const DeviceSnapshot &ds = *pc.ds; LiveState &lv = *pc.lv;
  const HostSnapshot &h = ds.host;
  const int32_t NM = ds.n_models, NI = f->hs.cfg.max_instances, np = (int)h.part_types.size();
  const int tc = h.tc_enabled ? 1 : 0, ns = tc ? np : 1;
  cudaStream_t st = c->stream;
  RpScratch &rs = c->rp;
  const size_t nmx = (size_t)std::max(NM, 1);
  const int32_t reg_cap = NM * HostState::EDGE_INL + lv.n_ovf;  // every registration
  // [the pruned and repaired model rows | pruned registrations | repaired models | loads (a run selects a model at most once)]
  mmp_model_row *view; PrunedReg *d_pruned; int *d_repaired; mmp_reaper_load *d_loads;
  rc = carve(c->d_task, [&](Carve &k) {
    view = k.take<mmp_model_row>(nmx); d_pruned = k.take<PrunedReg>(std::max(reg_cap, 1));
    d_repaired = k.take<int>(nmx); d_loads = k.take<mmp_reaper_load>(std::min(nmx, (size_t)loads_cap));
  });
  if (rc < 0) return rc;
  CK(c->d_n_open.ensure(16));
  // [missing_since (NI) | stats (np + 1) | the cluster's LRU, from Long.MAX_VALUE (ISST)]
  long long *d_miss, *d_min;
  StatsAcc *acc;
  rc = carve(c->d_trace, [&](Carve &k) { d_miss = k.take<long long>(NI); acc = k.take<StatsAcc>(np + 1); d_min = k.take<long long>(1); });
  if (rc < 0) return rc;
  int *d_cnt = c->d_n_open.as<int>();                         // [0] pruned registrations, [1] repaired models
  int *h_cnt = reinterpret_cast<int *>(c->mapped.get());      // ... read back with the selection count (pinned)
  static const long long lru_init = 0x7fffffffffffffffLL;
  CK(cudaMemcpyAsync(d_miss, missing_since, (size_t)NI * 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(d_cnt, 0, 8, st));
  CK(cudaMemsetAsync(acc, 0, (size_t)(np + 1) * sizeof(StatsAcc), st));
  CK(cudaMemcpyAsync(d_min, &lru_init, 8, cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(c->e0, st));
  if (NM) {
    k_registry_prune<<<(NM + 255) / 256, 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), lv.inst_meta.as<int2>(), NM, NI, leader,
                                                      now_ms, assume_gone_ms, d_miss, 1, nullptr, nullptr, d_pruned, reg_cap, d_cnt,
                                                      PruneView{view, d_repaired, d_cnt + 1});
    f->launches++;
    CK(cudaGetLastError());
  }
  CK(cudaMemcpyAsync(h_cnt, d_cnt, 8, cudaMemcpyDeviceToHost, st));
  k_missing_cleanup<<<(NI + 255) / 256, 256, 0, st>>>(d_miss, lv.inst_meta.as<int2>(), NI, now_ms, assume_gone_ms);
  f->launches++;
  if (h.n_ranks > 0) {
    k_stats<<<std::min(f->sm_count, (h.n_ranks + 255) / 256), 256, 0, st>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(),
                                                                           ds.part_of_rank.as<int32_t>(), h.n_ranks, f->hs.cfg.min_space_units,
                                                                           acc, d_min, np);
    f->launches++;
  }
  CK(cudaGetLastError());
  // the selection over the view: one run at now_ms, taken tags from a zeroed array (the pass reads the count back)
  int32_t n_sel = 0;
  if (NM) {
    CK(rs.taken.ensure(nmx * 4));
    CK(cudaMemsetAsync(rs.taken.p, 0, nmx * 4, st));
    int32_t gen = 0;
    rc = reaper_pass(f, ds, view, NM, tc, acc, d_min, std::vector<long long>{(long long)now_ms}, gen, rs, c->d_cub, st, &n_sel);
    if (rc < 0) return rc;
  }
  const int n_pruned = NM ? h_cnt[0] : 0, n_repaired = NM ? h_cnt[1] : 0;
  // the decisions, built on the device from the selections, placed as mmp_place_batch_device places a batch
  const int n_loads = std::min(n_sel, loads_cap);
  if (n_sel) {
    if ((rc = stage_fresh_self(c, nullptr, 1)) < 0) return rc;
    CK(c->d_in.ensure((size_t)n_sel * sizeof(mmp_decision_in)));
    CK(c->d_out.ensure((size_t)n_sel * sizeof(mmp_decision_out)));
    k_reaper_decisions<<<(n_sel + 255) / 256, 256, 0, st>>>(rs.sel.as<int2>(), n_sel, view, leader, c->d_in.as<mmp_decision_in>());
    f->launches++;
    CK(cudaGetLastError());
    CK(place_staged(f, c, ds.view, c->d_in.as<mmp_decision_in>(), n_sel, c->d_out.as<mmp_decision_out>(), now_ms, seed));
  }
  CK(cudaEventRecord(c->e1, st));
  if (n_loads) {
    k_reaper_loads<<<(n_loads + 255) / 256, 256, 0, st>>>(c->d_in.as<mmp_decision_in>(), c->d_out.as<mmp_decision_out>(), n_loads, d_loads);
    f->launches++;
    CK(cudaGetLastError());
  }
  // one copy back: the lists, the cleaned map, and the plan of the walk ([parts | space | plan | order], rp_plan_stage's layout)
  // with the candidate count, from which the partition a size estimate of 0 stopped at is named
  std::vector<PrunedReg> regs((size_t)n_pruned);
  std::vector<int32_t> rep((size_t)n_repaired);
  std::vector<mmp_reaper_load> ld((size_t)n_loads);
  std::vector<int64_t> miss((size_t)NI);
  const size_t parts_b = (size_t)ns * sizeof(RpPart), space_b = (size_t)ns * 8;
  std::vector<char> hb(parts_b + space_b + sizeof(RpPlan) + (size_t)ns * 4);
  int ncand = 0;
  if (n_pruned) CK(cudaMemcpyAsync(regs.data(), d_pruned, regs.size() * sizeof(PrunedReg), cudaMemcpyDeviceToHost, st));
  if (n_repaired) CK(cudaMemcpyAsync(rep.data(), d_repaired, rep.size() * 4, cudaMemcpyDeviceToHost, st));
  if (n_loads) CK(cudaMemcpyAsync(ld.data(), d_loads, ld.size() * sizeof(mmp_reaper_load), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(miss.data(), d_miss, (size_t)NI * 8, cudaMemcpyDeviceToHost, st));
  if (NM) {
    CK(cudaMemcpyAsync(hb.data(), rs.plan.p, hb.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&ncand, rs.idx.as<int>() + 2 * nmx, 4, cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));
  event_ms(c, f->t_reaper_run_ms);
  int stopped = -1;
  if (NM) {  // k_rp_walk's loop over the partitions: the first whose counts throw
    RpPlan plan;
    memcpy(&plan, hb.data() + parts_b + space_b, sizeof(RpPlan));
    for (int oi = 0; plan.go && ncand > 0 && oi < plan.n_order; oi++) {
      int s;
      RpPart p;
      unsigned long long space;
      memcpy(&s, hb.data() + parts_b + space_b + sizeof(RpPlan) + (size_t)oi * 4, 4);
      memcpy(&p, hb.data() + (size_t)s * sizeof(RpPart), sizeof(RpPart));
      memcpy(&space, hb.data() + parts_b + (size_t)s * 8, 8);
      int free_count, total;
      long long cutoff;
      if (!rp_counts(p, space, now_ms, free_count, total, cutoff)) { stopped = tc ? 1 + oi : 0; break; }
    }
  }
  std::sort(regs.begin(), regs.end(), [](const PrunedReg &a, const PrunedReg &b) { return a.model != b.model ? a.model < b.model : a.pos < b.pos; });
  std::sort(rep.begin(), rep.end());
  for (int i = 0; i < std::min(n_pruned, pruned_cap); i++) { pruned_models[i] = regs[i].model; pruned_instances[i] = regs[i].inst; }
  for (int i = 0; i < std::min(n_repaired, repaired_cap); i++) repaired_models[i] = rep[i];
  if (n_loads) memcpy(loads, ld.data(), ld.size() * sizeof(mmp_reaper_load));
  memcpy(missing_since, miss.data(), (size_t)NI * 8);
  *report = mmp_reaper_report{n_pruned, n_repaired, n_sel, stopped};
  return n_sel;
}

int32_t mmp_janitor_run(mmp_fleet *f, int32_t self, const mmp_janitor_entry *entries, int32_t n, const mmp_janitor_params *p,
                        mmp_janitor_edit *edits, int32_t cap, mmp_janitor_report *report) {
  NEED(f);
  if (self < 0 || self >= f->hs.cfg.max_instances || n < 0 || (n > 0 && !entries) || !p || !report || cap < 0 || (cap > 0 && !edits)) {
    g_err = "bad argument"; return MMP_E_ARG;
  }
  if (p->scale.now - p->scale.last_check_time <= 0 || p->scale.scale_up_rpm_threshold <= 0) {
    g_err = "now must be after last_check_time and the threshold positive"; return MMP_E_ARG;
  }
  int32_t rc = check_entries(f, entries, n);
  if (rc < 0) return rc;
  PodCall pc;
  if ((rc = pc.open(f, "mmp_janitor_run", PodCall::TIMES | PodCall::SLOTS)) < 0) return rc;
  PlaceCtx *c = pc.c; const DeviceSnapshot &ds = *pc.ds; LiveState &lv = *pc.lv;
  const int32_t NM = ds.n_models, np = (int)ds.host.part_types.size();
  cudaStream_t st = c->stream;
  // [entries | keys | sorted keys | values | sorted values | candidates | report | cnt[4] | edits]: the report, the counters
  // and the edits come back in one copy
  const size_t nx = (size_t)std::max(n, 1);
  JanitorBufs J{};
  mmp_janitor_entry *d_ent; unsigned long long *skeys; int *svals;
  rc = carve(c->d_task, [&](Carve &k) {
    J.entries = d_ent = k.take<mmp_janitor_entry>(nx); J.keys = k.take<unsigned long long>(nx); skeys = k.take<unsigned long long>(nx);
    J.vals = k.take<int>(nx); svals = k.take<int>(nx); J.cand = k.take<JanitorCand>(nx);
    J.report = k.take<mmp_janitor_report>(1); J.cnt = k.take<int>(4); J.edits = k.take<mmp_janitor_edit>(std::max(NM, 1));
  });
  if (rc < 0) return rc;
  J.slot = c->d_model_slot.as<int>();
  JanitorBufs Js = J;  // the same with the sorted keys and values
  Js.keys = skeys; Js.vals = svals;
  char *out = reinterpret_cast<char *>(J.report);
  const size_t o_cnt = reinterpret_cast<char *>(J.cnt) - out, hdr_b = reinterpret_cast<char *>(J.edits) - out;
  StatsAcc *acc;
  long long *d_min;
  if ((rc = carve(c->d_trace, [&](Carve &k) { acc = k.take<StatsAcc>(np + 1); d_min = k.take<long long>(1); })) < 0) return rc;
  static const long long lru_init = 0x7fffffffffffffffLL;
  CK(cudaMemsetAsync(acc, 0, (size_t)(np + 1) * sizeof(StatsAcc), st));
  CK(cudaMemcpyAsync(d_min, &lru_init, 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(J.cnt, 0, 16, st));
  if (n) {
    CK(cudaMemcpyAsync(d_ent, entries, (size_t)n * sizeof(mmp_janitor_entry), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(J.keys, 0xff, (size_t)n * 8, st));
  }
  CK(cudaEventRecord(c->e0, st));
  if ((rc = queue_janitor_pass(f, c, ds, lv, J, Js, n, self, *p, acc, d_min)) < 0) return rc;
  // one copy back: the report, the counters and the first edits
  const size_t first = janitor_first_edits(NM, n);
  std::vector<char> hb(hdr_b + first * sizeof(mmp_janitor_edit));
  CK(cudaMemcpyAsync(hb.data(), out, hb.size(), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  event_ms(c, f->t_janitor_ms);
  mmp_janitor_report r;
  int cnt[4];
  memcpy(&r, hb.data(), sizeof(r));
  memcpy(cnt, hb.data() + o_cnt, 16);
  if (cnt[JC_DUP]) { g_err = "two entries of one model"; return MMP_E_ARG; }
  if ((rc = janitor_edits_out(J, hb.data() + hdr_b, first, r.n_edits, edits, cap)) < 0) return rc;
  *report = r;
  return r.n_edits;
}

int32_t mmp_janitor_task(mmp_fleet *f, int32_t self, const mmp_janitor_task_entry *entries, int32_t n, const mmp_janitor_task_params *p,
                         mmp_janitor_cache_action *out, mmp_janitor_edit *edits, int32_t cap, mmp_janitor_task_report *report) {
  NEED(f);
  if (self < 0 || self >= f->hs.cfg.max_instances || n < 0 || n > (1 << 24) || (n > 0 && (!entries || !out)) || !p || !report || cap < 0 ||
      (cap > 0 && !edits)) {
    g_err = "bad argument"; return MMP_E_ARG;
  }
  const mmp_janitor_params &jp = p->janitor;
  if (jp.scale.now - jp.scale.last_check_time <= 0 || jp.scale.scale_up_rpm_threshold <= 0) {
    g_err = "now must be after last_check_time and the threshold positive"; return MMP_E_ARG;
  }
  int32_t rc = check_entries(f, entries, n);
  if (rc < 0) return rc;
  PodCall pc;
  if ((rc = pc.open(f, "mmp_janitor_task", PodCall::TIMES | PodCall::SLOTS)) < 0) return rc;
  PlaceCtx *c = pc.c; const DeviceSnapshot &ds = *pc.ds; LiveState &lv = *pc.lv;
  const int32_t NM = ds.n_models, np = (int)ds.host.part_types.size();
  cudaStream_t st = c->stream;
  // [task entries | the registry pass's entries | their records | keys | sorted keys | values | sorted values | candidates |
  //  header | cnt[4] | actions | edits]: the header, the counters, the actions and the edits come back in one copy
  const size_t nx = (size_t)std::max(n, 1);
  JanitorBufs J{};
  mmp_janitor_task_entry *d_te; mmp_janitor_entry *d_ent; JanitorOv *d_ov; unsigned long long *skeys; int *svals;
  JtHdr *hdr; mmp_janitor_cache_action *d_out;
  rc = carve(c->d_task, [&](Carve &k) {
    d_te = k.take<mmp_janitor_task_entry>(nx); J.entries = d_ent = k.take<mmp_janitor_entry>(nx); J.ov = d_ov = k.take<JanitorOv>(nx);
    J.keys = k.take<unsigned long long>(nx); skeys = k.take<unsigned long long>(nx);
    J.vals = k.take<int>(nx); svals = k.take<int>(nx); J.cand = k.take<JanitorCand>(nx);
    hdr = k.take<JtHdr>(1); J.cnt = k.take<int>(4); d_out = k.take<mmp_janitor_cache_action>(nx); J.edits = k.take<mmp_janitor_edit>(std::max(NM, 1));
  });
  if (rc < 0) return rc;
  J.slot = c->d_model_slot.as<int>();
  J.report = &hdr->rep.registry;
  J.halt = &hdr->halt;
  JanitorBufs Js = J;  // the same with the sorted keys and values
  Js.keys = skeys; Js.vals = svals;
  char *back = reinterpret_cast<char *>(hdr);
  const size_t o_cnt = reinterpret_cast<char *>(J.cnt) - back, o_out = reinterpret_cast<char *>(d_out) - back,
               hdr_b = reinterpret_cast<char *>(J.edits) - back;
  StatsAcc *acc;
  long long *d_min;
  if ((rc = carve(c->d_trace, [&](Carve &k) { acc = k.take<StatsAcc>(np + 1); d_min = k.take<long long>(1); })) < 0) return rc;
  static const long long lru_init = 0x7fffffffffffffffLL;
  CK(cudaMemsetAsync(acc, 0, (size_t)(np + 1) * sizeof(StatsAcc), st));
  CK(cudaMemcpyAsync(d_min, &lru_init, 8, cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(hdr, 0, sizeof(JtHdr) + 16, st));  // (and cnt)
  CK(cudaMemsetAsync(&hdr->stop, 0x7f, 4, st));
  if (n) {
    CK(cudaMemcpyAsync(d_te, entries, (size_t)n * sizeof(mmp_janitor_task_entry), cudaMemcpyHostToDevice, st));
    CK(cudaMemsetAsync(J.keys, 0xff, (size_t)n * 8, st));
  }
  // the window of MM:5933-5934 in Java long arithmetic
  const long long window = (long long)((uint64_t)p->janitor_freq_secs * 2000u + (uint64_t)p->load_timeout_ms);
  CK(cudaEventRecord(c->e0, st));
  if (n) {
    k_jt_plan<<<(n + 255) / 256, 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), NM, d_te, n, self, jp.scale.now, window,
                                               p->min_stale_age_ms, d_ent, d_ov, d_out, hdr);
    f->launches++;
  }
  k_jt_order<<<1, JT_ORDER_THREADS, 0, st>>>(d_te, n, lv.models.as<mmp_model_row>(), NM, d_out, hdr);
  f->launches++;
  CK(cudaGetLastError());
  if ((rc = queue_janitor_pass(f, c, ds, lv, J, Js, n, self, jp, acc, d_min)) < 0) return rc;
  const size_t first = janitor_first_edits(NM, n);
  std::vector<char> hb(hdr_b + first * sizeof(mmp_janitor_edit));
  CK(cudaMemcpyAsync(hb.data(), back, hb.size(), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  event_ms(c, f->t_janitor_task_ms);
  JtHdr H;
  int cnt[4];
  memcpy(&H, hb.data(), sizeof(H));
  memcpy(cnt, hb.data() + o_cnt, 16);
  if (cnt[JC_DUP]) { g_err = "two entries of one model"; return MMP_E_ARG; }
  const int32_t n_edits = H.rep.registry.n_edits;
  if ((rc = janitor_edits_out(J, hb.data() + hdr_b, first, n_edits, edits, cap)) < 0) return rc;
  if (n) memcpy(out, hb.data() + o_out, (size_t)n * sizeof(mmp_janitor_cache_action));
  *report = H.rep;
  return n_edits;
}


int32_t mmp_rate_run(mmp_fleet *f, int32_t self, const mmp_scale_in *entries, int32_t n, const mmp_rate_params *p,
                     const mmp_instance_row *fresh_self, uint64_t seed, mmp_scale_out *out, mmp_rate_load *loads, int32_t loads_cap,
                     mmp_rate_report *report) {
  NEED(f);
  if (self < 0 || self >= f->hs.cfg.max_instances || n < 0 || (n > 0 && (!entries || !out)) || !p || !report || loads_cap < 0 ||
      (loads_cap > 0 && !loads)) {
    g_err = "bad argument"; return MMP_E_ARG;
  }
  mmp_scale_params sp = p->scale;
  if (sp.now - sp.last_check_time <= 0 || sp.scale_up_rpm_threshold <= 0) {
    g_err = "now must be after last_check_time and the threshold positive"; return MMP_E_ARG;
  }
  sp.can_remove = 0;
  int32_t rc = check_entries(f, entries, n, [self](const mmp_scale_in &e) -> const char * {
    return e.instance != self ? "an entry of another instance than self" : nullptr;
  });
  if (rc < 0) return rc;
  FreshRow fr{};
  if ((rc = parse_fresh_self(fresh_self, fr)) < 0) return rc;
  PodCall pc;
  if ((rc = pc.open(f, "mmp_rate_run", PodCall::TIMES | PodCall::PLACES | PodCall::SLOTS)) < 0) return rc;
  PlaceCtx *c = pc.c; const DeviceSnapshot &ds = *pc.ds; LiveState &lv = *pc.lv;
  cudaStream_t st = c->stream;
  const int32_t NI = f->hs.cfg.max_instances, fresh_idx = fresh_self ? 0 : -1;
  // the gates of MM:5646-5670, in Java long arithmetic
  const int64_t delta = (int64_t)((uint64_t)sp.now - (uint64_t)sp.last_check_time);
  const bool too_soon = (int64_t)((uint64_t)delta * 5u) < (int64_t)((uint64_t)sp.rate_check_interval_ms * 3u);
  const int gate = too_soon ? MMP_RATE_TOO_SOON : ds.host.n_ranks < 2 ? MMP_RATE_FEW_INSTANCES : n == 0 ? MMP_RATE_NO_ENTRIES : MMP_RATE_RAN;
  // [header | entries | k_scale_eval's results | second copies | chains' decision 0 | chains | second copies' results | heavy set]
  const size_t nx = (size_t)std::max(n, 1);
  RateBufs B{};
  mmp_decision_out *sres;
  rc = carve(c->d_task, [&](Carve &k) {
    B.hdr = k.take<RateHdr>(1); B.entries = k.take<mmp_scale_in>(nx); B.sout = k.take<mmp_scale_out>(nx);
    B.sec = k.take<mmp_decision_in>(nx); B.c0 = k.take<mmp_decision_in>(nx); B.chains = k.take<RateChain>(nx);
    sres = k.take<mmp_decision_out>(nx); B.heavy = k.take<int32_t>(NI);
  });
  if (rc < 0) return rc;
  B.slot = c->d_model_slot.as<int>();
  RateHdr *h_hdr = reinterpret_cast<RateHdr *>(c->mapped.get());  // the one read-back before the placement (pinned)
  CK(cudaMemsetAsync(B.hdr, 0, sizeof(RateHdr), st));
  if (n) CK(cudaMemcpyAsync(const_cast<mmp_scale_in *>(B.entries), entries, (size_t)n * sizeof(mmp_scale_in), cudaMemcpyHostToDevice, st));
  if (gate != MMP_RATE_RAN) {  // nothing is evaluated; two entries of one model are still refused
    if (n) {
      k_slot_claim<<<(n + 255) / 256, 256, 0, st>>>(B.entries, n, B.slot, &B.hdr->dup);
      k_slot_release<<<(n + 255) / 256, 256, 0, st>>>(B.entries, n, B.slot);
      f->launches += 2;
      CK(cudaGetLastError());
      CK(cudaMemcpyAsync(h_hdr, B.hdr, sizeof(RateHdr), cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (h_hdr->dup) { g_err = "two entries of one model"; return MMP_E_ARG; }
    }
    for (int32_t r = 0; r < n; r++) out[r] = mmp_scale_out{0, 0, 0, 0, entries[r].i1, entries[r].i2, 0, 0};
    *report = mmp_rate_report{gate, 0, 0, 0, 0, 0, 0, 0};
    return 0;
  }
  if ((rc = stage_fresh_self(c, fresh_self ? &fr : nullptr, (size_t)n * MMP_MAX_EXTRA + 1)) < 0) return rc;
  B.extra = c->d_extra.as<int32_t>();
  CK(cudaEventRecord(c->e0, st));
  k_slot_claim<<<(n + 255) / 256, 256, 0, st>>>(B.entries, n, B.slot, &B.hdr->dup);
  f->launches++;
  if ((rc = queue_scale_eval(f, c, ds, lv, B.entries, n, sp, c->d_rate_rpm, const_cast<mmp_scale_out *>(B.sout), st)) < 0) return rc;
  k_slot_release<<<(n + 255) / 256, 256, 0, st>>>(B.entries, n, B.slot);
  k_rate_heavy<<<(NI + 255) / 256, 256, 0, st>>>(ds.rank_of.as<int32_t>(), ds.rows.as<RankRow>(), NI, self, sp.scale_up_rpm_threshold, B);
  const long long fail_since = (long long)((uint64_t)sp.now - (uint64_t)(p->load_failure_expiry_ms / 2));
  k_rate_plan<<<1, RATE_PLAN_THREADS, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), B, n, self, fail_since, fresh_idx);
  f->launches += 3;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(h_hdr, B.hdr, sizeof(RateHdr), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const RateHdr H = *h_hdr;
  if (H.dup) { g_err = "two entries of one model"; return MMP_E_ARG; }
  if (H.n_ids > (1LL << 24)) { g_err = "the call's decision ids do not fit in 24 bits (MMP_DF_OWN_ID)"; return MMP_E_ARG; }
  // the second copies under the epoch's tables, the chains round by round under the tables derived for the heavy set
  const int nq = H.n_chain, L = H.longest;
  SnapshotView vw = ds.view;
  vw.n_extra = 1 + MMP_MAX_EXTRA * nq;
  const int64_t now = sp.now;
  if (H.n_sec_place) CK(place_staged(f, c, vw, B.sec, n, sres, now, seed));
  if (nq) {
    CK(c->d_out.ensure((size_t)L * nq * sizeof(mmp_decision_out)));
    if (L > 1) CK(c->d_in.ensure((size_t)(L - 1) * nq * sizeof(mmp_decision_in)));
    SnapshotView xv = vw;
    if (H.n_heavy && (rc = derive_exclude_tables_dev(f, c, B.heavy, H.n_heavy, xv, st)) < 0) return rc;
    for (int j = 0; j < L; j++) {
      const mmp_decision_in *dj = j ? c->d_in.as<mmp_decision_in>() + (size_t)(j - 1) * nq : B.c0;
      if (j) {
        const mmp_decision_in *dp = j > 1 ? c->d_in.as<mmp_decision_in>() + (size_t)(j - 2) * nq : B.c0;
        k_rate_step<<<(nq + 255) / 256, 256, 0, st>>>(dp, c->d_out.as<mmp_decision_out>() + (size_t)(j - 1) * nq, B.chains, nq, j, self,
                                                      fresh_idx, B.extra, const_cast<mmp_decision_in *>(dj));
        f->launches++;
        CK(cudaGetLastError());
      }
      CK(place_staged(f, c, xv, dj, nq, c->d_out.as<mmp_decision_out>() + (size_t)j * nq, now, seed));
    }
  }
  CK(cudaEventRecord(c->e1, st));
  // one copy back: the per-entry results, the second copies, the chains and every round
  std::vector<mmp_decision_in> sec((size_t)n), dec((size_t)L * nq);
  std::vector<mmp_decision_out> sr((size_t)n), res((size_t)L * nq);
  std::vector<RateChain> chains((size_t)nq);
  CK(cudaMemcpyAsync(out, B.sout, (size_t)n * sizeof(mmp_scale_out), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(sec.data(), B.sec, (size_t)n * sizeof(mmp_decision_in), cudaMemcpyDeviceToHost, st));
  if (H.n_sec_place) CK(cudaMemcpyAsync(sr.data(), sres, (size_t)n * sizeof(mmp_decision_out), cudaMemcpyDeviceToHost, st));
  if (nq) {
    CK(cudaMemcpyAsync(chains.data(), B.chains, (size_t)nq * sizeof(RateChain), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(dec.data(), B.c0, (size_t)nq * sizeof(mmp_decision_in), cudaMemcpyDeviceToHost, st));
    if (L > 1) CK(cudaMemcpyAsync(dec.data() + nq, c->d_in.p, (size_t)(L - 1) * nq * sizeof(mmp_decision_in), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(res.data(), c->d_out.p, (size_t)L * nq * sizeof(mmp_decision_out), cudaMemcpyDeviceToHost, st));
  }
  CK(cudaStreamSynchronize(st));
  event_ms(c, f->t_rate_ms);
  // the loads in (entry, chain_pos) order; a chain whose last decision would continue and that has copies left is cut there
  std::vector<mmp_rate_load> ld;
  int n_cut = 0;
  for (int32_t r = 0, q = 0; r < n; r++) {
    if (sec[r].model >= 0) {
      ld.push_back(mmp_rate_load{r, sec[r].model, 0, self, sr[r].target, sr[r].n_candidates, sec[r].last_used, MMP_RL_SECOND_COPY, 0u});
      continue;
    }
    if (q >= nq || chains[q].entry != r) continue;
    const RateChain &ch = chains[q];
    for (int j = 0; j < L; j++) {
      const mmp_decision_in &d = dec[(size_t)j * nq + q];
      if (d.model < 0) break;
      const mmp_decision_out &o = res[(size_t)j * nq + q];
      ld.push_back(mmp_rate_load{r, d.model, j, d.self, o.target, o.n_candidates, d.last_used, 0u, 0u});
      if (j == MMP_RATE_CHAIN_MAX - 1 && ch.copies > MMP_RATE_CHAIN_MAX && o.target != MMP_TARGET_NONE && o.target != MMP_TARGET_INVALID) {
        ld.back().flags |= MMP_RL_CHAIN_CUT;
        ld.back().remaining = (uint32_t)(ch.copies - MMP_RATE_CHAIN_MAX);
        n_cut++;
      }
    }
    q++;
  }
  const int32_t n_loads = (int32_t)ld.size();
  if (loads_cap > 0 && n_loads) memcpy(loads, ld.data(), (size_t)std::min(n_loads, loads_cap) * sizeof(mmp_rate_load));
  *report = mmp_rate_report{MMP_RATE_RAN, H.n_second, H.n_scale_up, n_loads, H.n_heavy, n_cut, H.n_refused, 0};
  return n_loads;
}

int32_t mmp_shutdown_run(mmp_fleet *f, int32_t self, const mmp_shutdown_entry *entries, int32_t n, const mmp_shutdown_params *p,
                         const mmp_instance_row *fresh_self, uint64_t seed, mmp_shutdown_action *out, mmp_shutdown_report *report) {
  NEED(f);
  if (self < 0 || self >= f->hs.cfg.max_instances || n < 0 || n > (1 << 24) || (n > 0 && (!entries || !out)) || !p || !report) {
    g_err = "bad argument"; return MMP_E_ARG;  // (n <= 2^24: entry r draws with id r, MMP_DF_OWN_ID's 24 bits)
  }
  int32_t rc = check_entries(f, entries, n);
  if (rc < 0) return rc;
  FreshRow fr{};
  if ((rc = parse_fresh_self(fresh_self, fr)) < 0) return rc;
  PodCall pc;
  if ((rc = pc.open(f, "mmp_shutdown_run", PodCall::TIMES | PodCall::PLACES | PodCall::SLOTS)) < 0) return rc;
  PlaceCtx *c = pc.c; const DeviceSnapshot &ds = *pc.ds; LiveState &lv = *pc.lv;
  cudaStream_t st = c->stream;
  // [entries | decisions | results | header | actions]: the header and the actions come back in one copy
  const size_t nx = (size_t)std::max(n, 1);
  SdBufs B{};
  rc = carve(c->d_task, [&](Carve &k) {
    B.entries = k.take<mmp_shutdown_entry>(nx); B.dec = k.take<mmp_decision_in>(nx); B.res = k.take<mmp_decision_out>(nx);
    B.hdr = k.take<PackHdr<mmp_shutdown_report>>(1); B.out = k.take<mmp_shutdown_action>(nx);
  });
  if (rc < 0) return rc;
  B.slot = c->d_model_slot.as<int>();
  if ((rc = stage_fresh_self(c, fresh_self ? &fr : nullptr, 1)) < 0) return rc;
  B.extra = c->d_extra.as<int32_t>();
  CK(cudaMemsetAsync(B.hdr, 0, sizeof(*B.hdr), st));
  if (n) CK(cudaMemcpyAsync(const_cast<mmp_shutdown_entry *>(B.entries), entries, (size_t)n * sizeof(mmp_shutdown_entry), cudaMemcpyHostToDevice, st));
  const int64_t now = p->now;
  const long long cutoff = (long long)((uint64_t)now - (uint64_t)p->cutoff_age_ms);
  const long long fail_since = (long long)((uint64_t)now - (uint64_t)(p->load_failure_expiry_ms / 2));
  CK(cudaEventRecord(c->e0, st));
  // (launched at n == 0 too: block 0 writes found_other and extra[0])
  k_shutdown_plan<<<std::max((n + 255) / 256, 1), 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), ds.rank_of.as<int32_t>(),
                                                                ds.host.n_ranks, B, n, self, cutoff, fail_since, fresh_self ? 0 : -1);
  f->launches++;
  CK(cudaGetLastError());
  if (n) {
    SnapshotView vw = ds.view;
    vw.n_extra = 1;
    CK(place_staged(f, c, vw, B.dec, n, const_cast<mmp_decision_out *>(B.res), now, seed));
    k_shutdown_pack<<<(n + 255) / 256, 256, 0, st>>>(B, n, cutoff);
    f->launches++;
    CK(cudaGetLastError());
  }
  return pack_copy_back(c, B.hdr, n, f->t_shutdown_ms, out, report);
}

int32_t mmp_evict_run(mmp_fleet *f, int32_t self, const mmp_evict_entry *entries, int32_t n, const mmp_evict_params *p,
                      const mmp_instance_row *fresh_self, uint64_t seed, mmp_evict_action *out, mmp_evict_report *report) {
  NEED(f);
  if (self < 0 || self >= f->hs.cfg.max_instances || n < 0 || n > (1 << 24) || (n > 0 && (!entries || !out)) || !p || !report) {
    g_err = "bad argument"; return MMP_E_ARG;  // (n <= 2^24: entry r draws with id r, MMP_DF_OWN_ID's 24 bits)
  }
  int32_t rc = check_entries(f, entries, n);
  if (rc < 0) return rc;
  FreshRow fr{};
  if ((rc = parse_fresh_self(fresh_self, fr)) < 0) return rc;
  PodCall pc;
  if ((rc = pc.open(f, "mmp_evict_run", PodCall::TIMES | PodCall::PLACES | PodCall::SLOTS)) < 0) return rc;
  PlaceCtx *c = pc.c; const DeviceSnapshot &ds = *pc.ds; LiveState &lv = *pc.lv;
  cudaStream_t st = c->stream;
  // [entries | decisions | results | header | actions]: the header and the actions come back in one copy
  const size_t nx = (size_t)std::max(n, 1);
  EvBufs B{};
  rc = carve(c->d_task, [&](Carve &k) {
    B.entries = k.take<mmp_evict_entry>(nx); B.dec = k.take<mmp_decision_in>(nx); B.res = k.take<mmp_decision_out>(nx);
    B.hdr = k.take<PackHdr<mmp_evict_report>>(1); B.out = k.take<mmp_evict_action>(nx);
  });
  if (rc < 0) return rc;
  B.slot = c->d_model_slot.as<int>();
  if ((rc = stage_fresh_self(c, fresh_self ? &fr : nullptr, 1)) < 0) return rc;
  B.extra = c->d_extra.as<int32_t>();
  CK(cudaMemsetAsync(B.hdr, 0, sizeof(*B.hdr), st));
  if (n) CK(cudaMemcpyAsync(const_cast<mmp_evict_entry *>(B.entries), entries, (size_t)n * sizeof(mmp_evict_entry), cudaMemcpyHostToDevice, st));
  const int64_t now = p->now;
  const long long reload_age = (long long)(2u * (uint64_t)p->load_timeout_ms);
  const long long fail_since = (long long)((uint64_t)now - (uint64_t)(p->load_failure_expiry_ms / 2));
  CK(cudaEventRecord(c->e0, st));
  if (n) {  // (nothing at n == 0, the type-set stats included)
    TypeSetStats S;
    if ((rc = queue_type_stats(f, c, ds, lv, S, st)) < 0) return rc;
    k_evict_plan<<<(n + 255) / 256, 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), lv.model_lul.as<long long>(),
                                                  ds.rank_of.as<int32_t>(), S.types, lv.n_type_ids, B, n, self, now, reload_age, fail_since,
                                                  fresh_self ? 0 : -1);
    SnapshotView vw = ds.view;
    vw.n_extra = 1;
    CK(place_staged(f, c, vw, B.dec, n, const_cast<mmp_decision_out *>(B.res), now, seed));
    k_evict_pack<<<(n + 255) / 256, 256, 0, st>>>(B, n);
    f->launches += 2;
    CK(cudaGetLastError());
  }
  return pack_copy_back(c, B.hdr, n, f->t_evict_ms, out, report);
}

}  // extern "C"
