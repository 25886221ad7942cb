// churn_kernels.cuh — the closed loop of the placement / eviction path ON THE DEVICE (SURVEY.md §8a rows a11, a12; §8f-1,
// §8f-4): one call of mmp_churn_step = one republish window (2 s, MM:232) of the whole fleet:
//   reaper      (windows with REAPER events only) the reaper's selections, k_rp_* below; their count is read back once
//   classify    requests -> cache hits (runtimeCache.get on a registered copy) / cache misses (the first request of an unloaded
//               model in the window -> a getNext decision) / removals / the reaper's selections (decisions at the REAPER's
//               position); queued ensureLoadedElsewhere calls go first
//   place       the scoring kernel (k_place_lanes) over the window's decisions against the committed snapshot
//   route       every cache event to its instance: radix sort by (instance, position in the trace)
//   apply       k_lru_events: one warp per instance, events in order -- loadLocal's admission rules, the time-ordered
//               weighted LRU, the eviction listener (deregistration, reload-elsewhere rule MM:2915-2931)
//   registry    edge lists / copy counts / lastUsed of the models touched (MR:69, 239-246)
//   republish   getFreshInstanceRecord + publishInstanceRecord's significance thresholds (MM:5369-5470) per instance
//   commit      the device path of mmp_fleet_commit (commit_kernels.cuh): re-rank, rebuild tables and bitmap
// No host work between the phases (but the reaper's one read-back); the host reads the reports (decisions, evictions, rows)
// once at the end.
// Epoch semantics = oracle/mm_sim.inc, REAPER events = its step as tests/emul/reaper_sim.cpp extends it (the parity tests
// drive the same trace through both).  Included by mmplace.cu.
#pragma once

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

struct DecMeta { int event, weight, order, exclude; };
// The window's REAPER events for the classify kernels: ev_idx[0 .. n) their trace indices (ascending); event r selected
// models off[r] .. off[r + 1] of the selection list, and fpos (exclusive scan of the selections' first-decision flags, null
// when nothing was selected) says how many of them became decisions.
struct RpView { const int *ev_idx; int n; const int *off; const int *fpos; };
__device__ __forceinline__ int rp_decisions(const RpView &rp, int i) {
  if (!rp.fpos) return 0;
  int lo = 0, hi = rp.n;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (rp.ev_idx[mid] < i) lo = mid + 1; else hi = mid; }
  return rp.fpos[rp.off[lo + 1]] - rp.fpos[rp.off[lo]];
}

// phase A.1: the first cache miss of every unloaded model in the window (queued follow-ons count and come first)
__global__ void k_churn_first(const Follow *__restrict__ carry, int n_follow, const mmp_churn_event *__restrict__ ev, int n,
                              const mmp_model_row *__restrict__ models, int n_models, int *__restrict__ first_ev) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_follow + n) return;
  int model;
  if (q < n_follow) model = carry[q].model;
  else { const mmp_churn_event e = ev[q - n_follow]; if (e.type != 0) return; model = e.model; }
  if (model < 0 || model >= n_models) return;
  if (models[model].copy_count == 0) atomicMin(&first_ev[model], q);
}
// phase A.2: which items become decisions (every follow-on; the first miss of a model), and how many cache-event slots each
// item owns: one for a decision's load (phase C) or a cache hit, one per loaded copy for a REMOVE.  x = decision, y = slots.
// A REAPER item owns one decision and one slot per selection that is the first decision of its model in the window.
__global__ void k_churn_flag(const Follow *__restrict__ carry, int n_follow, const mmp_churn_event *__restrict__ ev, int n,
                             const mmp_model_row *__restrict__ models, int n_models, const int *__restrict__ first_ev,
                             int2 *__restrict__ is_dec, long long *__restrict__ used_t, int *__restrict__ counters, RpView rp) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_follow + n) return;
  int d = 0, slots = 0;
  if (q < n_follow) d = 1;
  else {
    const mmp_churn_event e = ev[q - n_follow];
    if (e.type == MMP_CHURN_REAPER) d = rp_decisions(rp, q - n_follow);
    else if (e.model >= 0 && e.model < n_models) {
      const int cc = models[e.model].copy_count;
      if (e.type == 0) {
        atomicMax(&used_t[e.model], (long long)e.t);  // MR.updateLastUsed at the end of the window
        if (cc > 0) slots = 1;
        else if (first_ev[e.model] == q) d = 1;
        else atomicAdd(&counters[3], 1);  // coalesced
      } else if (e.type == 1) slots = cc;
    }
  }
  is_dec[q] = make_int2(d, slots + d);
}
// phase A.3: decision records + the cache events of hits and removals, each in the slots the scan of k_churn_flag gave its
// item (pos.y); a slot whose copy names no instance keeps the key ~0 and sorts to the end.
__global__ void k_churn_emit(const Follow *__restrict__ carry, int n_follow, const mmp_churn_event *__restrict__ ev, int n,
                             const mmp_model_row *__restrict__ models, RegTables R, int n_models, int max_instances,
                             const int *__restrict__ first_ev, const int2 *__restrict__ is_dec, const int2 *__restrict__ dec_pos,
                             mmp_decision_in *__restrict__ dec_in, DecMeta *__restrict__ meta, int32_t *__restrict__ extra,
                             int *__restrict__ status, int *__restrict__ dec_of_model, LruEv *__restrict__ lev,
                             unsigned long long *__restrict__ keys, long long now0) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_follow + n) return;
  if (is_dec[q].x) {
    const int k = dec_pos[q].x;
    mmp_decision_in d;
    d.flags = 0; d.fresh = -1; d.extra_off = k; d.extra_n = 0;
    DecMeta m;
    int st = CH_INVALID;
    if (q < n_follow) {
      const Follow c = carry[q];
      d.model = c.model; d.self = c.exclude; d.last_used = c.last_used; d.extra_n = 1;
      extra[k] = c.exclude;
      m = DecMeta{-1 - q, c.weight, q, c.exclude};
      // ensureLoadedElsewhere: nothing to do when the model has a copy again, or was already queued in this window
      if (!(c.model >= 0 && c.model < n_models && models[c.model].copy_count == 0 && first_ev[c.model] == q)) { st = CH_SKIPPED; d.model = -1; }
      else dec_of_model[c.model] = k;
    } else {
      const mmp_churn_event e = ev[q - n_follow];
      if (e.type == MMP_CHURN_REAPER) return;  // (k_rp_emit writes its decisions)
      d.model = e.model; d.self = e.caller; d.last_used = e.t;
      extra[k] = -1;
      m = DecMeta{q - n_follow, models[e.model].size_units, q, -1};
      dec_of_model[e.model] = k;
    }
    dec_in[k] = d; meta[k] = m; status[k] = st;
    return;
  }
  if (q < n_follow) return;
  const mmp_churn_event e = ev[q - n_follow];
  if (e.model < 0 || e.model >= n_models) return;
  const int cc = models[e.model].copy_count;
  if (cc == 0 || e.type > 1) return;
  const size_t s0 = (size_t)dec_pos[q].y;
  const ModelRegs g = model_regs(R, e.model, (unsigned)cc);
  long long ts;
  if (e.type == 0) {  // cache hit on copy (u mod copies) in registration order
    const int inst = reg_at(R, g, (int)(e.u % (unsigned)cc), ts);
    keys[s0] = ~0ull;
    if (inst >= 0 && inst < max_instances) {
      lev[s0] = LruEv{LEV_TOUCH, e.model, 0, q, -1, 0, e.t, e.t};
      keys[s0] = ((unsigned long long)(unsigned)inst << 32) | (unsigned)q;
    }
  } else {
    for (int j = 0; j < cc; j++) {
      const int inst = reg_at(R, g, j, ts);
      keys[s0 + j] = ~0ull;
      if (inst < 0 || inst >= max_instances) continue;
      lev[s0 + j] = LruEv{LEV_REMOVE, e.model, 0, q, -1, 0, 0, e.t};
      keys[s0 + j] = ((unsigned long long)(unsigned)inst << 32) | (unsigned)q;
    }
  }
}
// phase C.1: a decision that found a target becomes a checked load on that instance; its clock is the clock of the request
// that caused it (queued follow-ons: the start of the window)
__device__ __forceinline__ void churn_route_one(int k, size_t slot, const mmp_decision_in *__restrict__ dec_in,
                                                const mmp_decision_out *__restrict__ dec_out, const DecMeta *__restrict__ meta,
                                                int max_instances, const mmp_churn_event *__restrict__ ev, long long now0,
                                                int *__restrict__ status, int *__restrict__ dec_target, LruEv *__restrict__ lev,
                                                unsigned long long *__restrict__ keys) {
  keys[slot] = ~0ull;
  dec_target[k] = -1;
  if (status[k] == CH_SKIPPED) return;
  const mmp_decision_out o = dec_out[k];
  const mmp_decision_in d = dec_in[k];
  if (o.target == MMP_TARGET_NONE) { status[k] = CH_NOWHERE; return; }
  const int tgt = o.target == MMP_TARGET_SELF ? d.self : o.target;
  if (tgt < 0 || tgt >= max_instances) { status[k] = CH_INVALID; return; }
  dec_target[k] = tgt;
  const DecMeta m = meta[k];
  lev[slot] = LruEv{LEV_LOAD, d.model, m.weight, m.order, k, 0, d.last_used, m.event >= 0 ? (long long)ev[m.event].t : now0};
  keys[slot] = ((unsigned long long)(unsigned)tgt << 32) | (unsigned)m.order;
}
__global__ void k_churn_route(const mmp_decision_in *__restrict__ dec_in, const mmp_decision_out *__restrict__ dec_out,
                              const DecMeta *__restrict__ meta, const int2 *__restrict__ is_dec, const int2 *__restrict__ dec_pos, int n_items,
                              int max_instances, const mmp_churn_event *__restrict__ ev, long long now0, int *__restrict__ status,
                              int *__restrict__ dec_target, LruEv *__restrict__ lev, unsigned long long *__restrict__ keys) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_items) return;
  if (!is_dec[q].x) return;
  const int k = dec_pos[q].x;
  const int e = meta[k].event;
  if (e >= 0 && ev[e].type == MMP_CHURN_REAPER) return;  // (k_rp_route routes its decisions)
  churn_route_one(k, (size_t)dec_pos[q].y, dec_in, dec_out, meta, max_instances, ev, now0, status, dec_target, lev, keys);
}
// per-instance ranges of the sorted event list
__global__ void k_churn_offsets(const unsigned long long *__restrict__ keys, int n_keys, int n_inst, int *__restrict__ off) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n_inst) return;
  const unsigned long long want = (unsigned long long)(unsigned)i << 32;  // first key of instance i (i == n_inst: one past the last)
  int lo = 0, hi = n_keys;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (keys[mid] < want) lo = mid + 1; else hi = mid; }
  off[i] = lo;  // (invalid keys are ~0: beyond every instance)
}
// the sort's input: value = slot; the slots past the last item's (n_used = pos.y + slots of the last item) hold no event
__global__ void k_churn_tail(unsigned long long *__restrict__ keys, int *__restrict__ vals, int n_keys, const int2 *__restrict__ is_dec,
                             const int2 *__restrict__ dec_pos, int n_items) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_keys) return;
  vals[i] = i;
  if (i >= dec_pos[n_items - 1].y + is_dec[n_items - 1].y) keys[i] = ~0ull;
}
// A model's registrations after the window: the surviving loaded copies in order, the window's accepted load, the failed
// loads.  emit(k, instance, ts) for each; returns {registrations, loaded}.  Each keeps the time it had (0 for the new load).
template <class Emit>
__device__ __forceinline__ int2 churn_regs_after(const RegTables &R, const ModelRegs &g, int cc, int nreg, unsigned rm, int add,
                                                 const unsigned char *ovf_dead, Emit emit) {
  int k = 0, loaded = 0;
  bool have = false;
  long long ts;
  for (int j = 0; j < cc; j++) {
    const int inst = reg_at(R, g, j, ts);
    if (inst < 0 || (j < 4 ? (rm >> j) & 1u : ovf_dead[g.ovf0 + j - 4])) continue;
    emit(k++, inst, ts); loaded++;
    if (inst == add) have = true;
  }
  if (add >= 0 && !have) { emit(k++, add, 0ll); loaded++; }
  for (int j = cc; j < nreg; j++) {
    const int inst = reg_at(R, g, j, ts);
    if (inst >= 0) emit(k++, inst, ts);
  }
  return make_int2(k, loaded);
}
// phase D: edge lists, copy counts, lastUsed.  One thread per model; only models touched in the window do any work.  A
// touched model with overflow registrations before or after the window keeps its marks for the re-lay below (k_ovf_relay)
// and raises counters[2].
__global__ void k_churn_registry(mmp_model_row *__restrict__ models, int4 *__restrict__ edges, int n_models, unsigned *__restrict__ rm_mask,
                                 int *__restrict__ add_inst, long long *__restrict__ used_t, int *__restrict__ counters) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  const unsigned rm = rm_mask[m];
  const int add = add_inst[m];
  const long long ut = used_t[m];
  if (rm == 0 && add < 0 && ut == 0) return;
  mmp_model_row r = models[m];
  if (ut > r.last_used) r.last_used = ut;  // MR:239-246
  if ((rm != 0 || add >= 0) && (r.reserved > 4u || (r.reserved == 4u && add >= 0))) atomicOr(&counters[2], 1);
  else if (rm != 0 || add >= 0) {
    int out[4] = {-1, -1, -1, -1};
    const RegTables R{edges, nullptr, nullptr, 0};
    const int2 kl = churn_regs_after(R, model_regs(R, m, 0u), r.copy_count, (int)r.reserved, rm, add, nullptr,
                                     [&](int k, int inst, long long) { out[k] = inst; });
    edges[m] = make_int4(out[0], out[1], out[2], out[3]);
    r.copy_count = (uint8_t)kl.y;
    r.reserved = (uint32_t)kl.x;
    rm_mask[m] = 0; add_inst[m] = -1;
  }
  used_t[m] = 0;
  models[m] = r;
}
// The re-lay of the overflow table, when counters[2] is up.  k_ovf_count: overflow registrations of every model after the
// window (a marked model: its new list; any other: as before); an exclusive scan gives each model its slice of the new table.
__global__ void k_ovf_count(RegTables R, const mmp_model_row *__restrict__ models, int n_models, const unsigned *__restrict__ rm_mask,
                            const int *__restrict__ add_inst, const unsigned char *__restrict__ ovf_dead, int *__restrict__ n_out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m > n_models) return;
  if (m == n_models) { n_out[m] = 0; return; }
  const mmp_model_row r = models[m];
  int k = (int)r.reserved;
  if (rm_mask[m] != 0 || add_inst[m] >= 0)
    k = churn_regs_after(R, model_regs(R, m, r.reserved), r.copy_count, (int)r.reserved, rm_mask[m], add_inst[m], ovf_dead,
                         [](int, int, long long) {}).x;
  n_out[m] = k > 4 ? k - 4 : 0;
}
// k_ovf_relay: every model writes its slice of the new table (sorted by model, then position, as the old one); a marked
// model also rewrites its inline edges, copy count and registration count, and clears its marks
__global__ void k_ovf_relay(RegTables R, mmp_model_row *models, int4 *edges, int n_models, unsigned *__restrict__ rm_mask,
                            int *__restrict__ add_inst, const unsigned char *__restrict__ ovf_dead, const int *__restrict__ off,
                            OvfEdge *__restrict__ out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  const unsigned rm = rm_mask[m];
  const int add = add_inst[m];
  mmp_model_row r = models[m];
  OvfEdge *o = out + off[m];
  if (rm == 0 && add < 0) {
    if (r.reserved <= 4u) return;
    const ModelRegs g = model_regs(R, m, r.reserved);
    for (int j = 4; j < (int)r.reserved; j++) o[j - 4] = R.ovf[g.ovf0 + j - 4];
    return;
  }
  int e[4] = {-1, -1, -1, -1};
  const int2 kl = churn_regs_after(R, model_regs(R, m, r.reserved), r.copy_count, (int)r.reserved, rm, add, ovf_dead,
                                   [&](int k, int inst, long long ts) { if (k < 4) e[k] = inst; else o[k - 4] = OvfEdge{m, inst, ts}; });
  edges[m] = make_int4(e[0], e[1], e[2], e[3]);
  r.copy_count = (uint8_t)kl.y;
  r.reserved = (uint32_t)kl.x;
  models[m] = r;
  rm_mask[m] = 0; add_inst[m] = -1;
}
__global__ void k_churn_collect_adds(const mmp_decision_in *__restrict__ dec_in, const int *__restrict__ status, const int *__restrict__ dec_target,
                                     int n_dec, int *__restrict__ add_inst, int *__restrict__ dec_of_model) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n_dec) return;
  const int m = dec_in[k].model;
  if (m < 0) return;
  if (status[k] == CH_ACCEPTED) add_inst[m] = dec_target[k];
  dec_of_model[m] = -1;          // scratch back to its idle state for the next window
}
__global__ void k_churn_reset_first(const Follow *__restrict__ carry, int n_follow, const mmp_churn_event *__restrict__ ev, int n, int n_models,
                                    int *__restrict__ first_ev) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n_follow + n) return;
  const int model = q < n_follow ? carry[q].model : ev[q - n_follow].model;
  if (model >= 0 && model < n_models) first_ev[model] = 0x7fffffff;
}

// publishInstanceRecord (MM:5390-5470) for every instance at the end of the window; literal thresholds MM:5443-5468
__device__ __forceinline__ long long llabs_w(long long x) { return x < 0 ? (long long)(0ull - (unsigned long long)x) : x; }
__device__ __forceinline__ bool loading_change(int cur, int l_threads, int now_) {  // MM:5536-5543
  if (now_ == cur) return false;
  if ((now_ == 0) != (cur == 0)) return true;
  if ((now_ <= l_threads) != (cur <= l_threads)) return true;
  const int d = (int)((unsigned)now_ - (unsigned)cur);
  return (d < 0 ? -d : d) >= 3;
}
__device__ __forceinline__ bool load_change(int cur, int rpms) {  // MM:5546-5550
  int diff = (int)((unsigned)cur - (unsigned)rpms);
  diff = diff < 0 ? -diff : diff;
  return diff >= 100 || (cur == 0 ? rpms != 0 : (int)((unsigned)100 * (unsigned)diff) / cur > 10);
}
__global__ void k_churn_republish(LruView v, mmp_instance_row *__restrict__ rows, const int2 *__restrict__ meta, int n_inst,
                                  long long *__restrict__ last_published, const unsigned char *__restrict__ force_publish, long long now1,
                                  long long min_space, int *__restrict__ counters) {
  const int lane = threadIdx.x & 31;
  const int inst = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (inst >= n_inst || inst >= v.n) return;
  if (!(meta[inst].y & 1)) return;
  long long t, s;
  const int o = lru_min_slot(v, inst, lane, false, 0, 0, &t, &s);
  if (lane != 0) return;
  const long long last_done = now1 - last_published[inst];
  const bool force = force_publish[inst] != 0;
  if (last_done < 2000 || (!force && last_done < 40000 - 1000)) return;  // MM:5397-5400
  const bool old = last_done > 4 * 40000;
  const long long oldest = o < 0 ? 0x7fffffffffffffffLL : t;
  const int count = v.count[inst];
  const long long cap = v.cap[inst], used = v.wsize[inst];
  mmp_instance_row cur = rows[inst];
  const long long cur_rem = cur.capacity - cur.used > 0 ? cur.capacity - cur.used : 0;
  const long long new_rem = cap - used > 0 ? cap - used : 0;
  bool publish;
  if (!old) {
    long long diff;
    const bool within =
        llabs_w(cur.capacity - cap) < cap / 50 && (diff = llabs_w(cur.lru_time - oldest)) < 20000 &&
        (cur.lru_time == 0x7fffffffffffffffLL || diff < (now1 - cur.lru_time) / 16) && (diff = (long long)abs(cur.count - count)) < 10 &&
        (cur.count == 0 ? count == 0 : (diff * 100) / cur.count < 15) &&
        (cur.used == 0 ? used == 0 : (llabs_w(cur.used - used) * 100) / cur.used < 20) && (cur_rem < min_space) == (new_rem < min_space) &&
        !loading_change(cur.l_in_prog, cur.l_threads, 0) && !load_change(cur.rpm, cur.rpm);
    publish = !within;
  } else {
    publish = !(cur.capacity == cap && cur.count == count && cur.lru_time == oldest && cur.used == used && cur.l_in_prog == 0);
  }
  if (!publish) return;
  cur.lru_time = oldest; cur.count = count; cur.capacity = cap; cur.used = used; cur.l_in_prog = 0;
  rows[inst] = cur;
  last_published[inst] = now1;
  atomicAdd(&counters[1], 1);
}
// typeSetStats (MM:1432-1438, TCM:230-233) -> "less than 95 % full and more than one instance" per type id (MM:2918-2920)
__global__ void k_churn_type_ok(const StatsAcc *__restrict__ acc, const int *__restrict__ type_part_off, const int *__restrict__ type_parts,
                                int n_type_ids, unsigned char *__restrict__ type_ok) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_type_ids) return;
  unsigned long long cap = 0, fr = 0;
  long long cnt = 0;
  const int a = type_part_off[t], b = type_part_off[t + 1];
  if (a == b) { cap = acc[0].cap; fr = acc[0].free; cnt = acc[0].count; }  // no subset: the cluster's stats
  else if (type_parts[a] < 0) { cap = 0; fr = 0; cnt = 0; }                // a subset without instances
  else for (int j = a; j < b; j++) { const StatsAcc s = acc[1 + type_parts[j]]; cap += s.cap; fr += s.free; cnt += s.count; }
  type_ok[t] = ((long long)cap > 0 && cnt > 1 && (long long)(20ull * fr) / (long long)cap >= 1) ? 1 : 0;
}

// ---------------------------------------------------------------------------------------------------------------
// The reaper's proactive loads (MMP_CHURN_REAPER; MM:6456-6494, 6574-6577, 6616-6747), on the step's stream against the
// window's snapshot: the stats of k_stats -> per-partition plan and PARTITION_STATS_COMP order (k_rp_plan) -> candidates
// (k_rp_flag, compaction) -> one radix sort by (lastUsed desc, model asc) -> spaceToFill per partition (k_rp_space) -> one
// block walks the sorted list per event and partition (k_rp_walk).  reaper_impl (scan_kernels.cuh) is the same arithmetic
// with its host parts; the parity tests hold the two equal.
// ---------------------------------------------------------------------------------------------------------------
// one slot per partition (the whole cluster when the fleet has no type constraints), as run_stats reports them
struct RpPart { long long cap, free, glru; int copies, count, size_est, pad; };
struct RpPlan { int go, n_order; long long global_lru; };
__device__ __forceinline__ long long rp_last_used(unsigned long long key) { return (long long)((~key) ^ 0x8000000000000000ull); }

__global__ void k_rp_plan(const StatsAcc *__restrict__ acc, const long long *__restrict__ min_lru, int n_slots, int tc, int def_size,
                          RpPart *__restrict__ parts, int *__restrict__ order, RpPlan *__restrict__ plan) {
  const long long mn = *min_lru;
  for (int s = threadIdx.x; s < n_slots; s += blockDim.x) {
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
    plan->n_order = n_in;
  }
}
__global__ void k_rp_flag(const mmp_model_row *__restrict__ models, int n_models, const RpPlan *__restrict__ plan, uint8_t *__restrict__ flag) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= n_models) return;
  const RpPlan p = *plan;
  flag[m] = p.go && reaper_candidate(models[m], p.global_lru) ? 1 : 0;
}
// sort keys of the compacted candidates (in model order); the positions past them sort last
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
// The selection of every REAPER event, one after the other, by one block: for each partition in order, the sorted candidates
// are walked in chunks of RP_WALK.  Per chunk: eligible = not taken by this run, type allowed in the partition (MM:6681-6683)
// and (free space or lastUsed > cutoff) (MM:6685-6688); of an equal-lastUsed run of eligible entries only the first counts
// (N12; a block-wide max scan finds each entry's previous eligible entry); the counted entries take ranks k by a block-wide
// sum scan, and the first totalProactiveLoadCount of them go through the emission rule (MM:6711-6719), which, the list
// being in descending lastUsed, emits a prefix of them.  The walk stops at the count, at the rule's break, or (full
// partition) at the first entry at or under the cutoff.  Emitted models are tagged taken and appended as (model, event).
constexpr int RP_WALK = 1024;
__global__ void __launch_bounds__(RP_WALK) k_rp_walk(const mmp_model_row *__restrict__ models, const unsigned long long *__restrict__ skey,
                                                      const int *__restrict__ sidx, const int *__restrict__ n_cand, const RpPlan *__restrict__ plan,
                                                      const RpPart *__restrict__ parts, const int *__restrict__ order,
                                                      const unsigned long long *__restrict__ space, int tc, const int *__restrict__ pt_off,
                                                      const int *__restrict__ pt_ids, const mmp_churn_event *__restrict__ ev,
                                                      const int *__restrict__ rp_ev, int n_rp, int gen0, int *__restrict__ taken,
                                                      int2 *__restrict__ sel, long long sel_cap, int *__restrict__ sel_off) {
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
    const long long t = ev[rp_ev[r]].t;
    for (int oi = 0; P.go && ncand > 0 && oi < P.n_order; oi++) {
      const int s = order[oi];
      const RpPart p = parts[s];
      int free_count = 0, total = 0;
      if (p.cap > 0 && p.free > 0) {  // MM:6621-6657
        if (p.size_est == 0) break;   // spaceToFill / sizeEstimate throws (MM:6651): the run ends here
        const long long fill = (long long)space[s] / 2;
        free_count = (int32_t)(fill / p.size_est);
        const long long d = (long long)(20ull * (unsigned long long)(long long)p.size_est);
        const int32_t cap_count = d == 0 ? 0 : (int32_t)(d == -1 ? -p.cap : p.cap / d);
        total = free_count > cap_count ? free_count : cap_count;
      }
      if (total <= 0) continue;
      const long long a3 = age_of(p.glru, t) / 3;
      const long long cutoff = p.glru == 0x7fffffffffffffffLL ? 0 : (long long)((unsigned long long)p.glru + (unsigned long long)(a3 > 1200000 ? a3 : 1200000));
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
        const bool emit = first && k < total && (k < free_count || !(rp_last_used(key) < cutoff));
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
// the window's items see the selections at their REAPER's position: first decisions (k_churn_first's rule), flags, records
__global__ void k_rp_first(const int2 *__restrict__ sel, int n_sel, const int *__restrict__ rp_ev, int n_follow, int *__restrict__ first_ev) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_sel) return;
  const int2 x = sel[s];
  atomicMin(&first_ev[x.x], n_follow + rp_ev[x.y]);
}
__global__ void k_rp_mark(const int2 *__restrict__ sel, int n_sel, const int *__restrict__ rp_ev, int n_follow, const int *__restrict__ first_ev,
                          int *__restrict__ flag, int *__restrict__ counters) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > n_sel) return;
  if (s == n_sel) { flag[s] = 0; return; }
  const int2 x = sel[s];
  const int f = first_ev[x.x] == n_follow + rp_ev[x.y];
  flag[s] = f;
  if (!f) atomicAdd(&counters[3], 1);  // coalesced
}
// decision k and event slot of selection s (which must be a first decision)
__device__ __forceinline__ int2 rp_dec_slot(const RpView &rp, int s, int r, const int2 *__restrict__ dec_pos, int n_follow) {
  const int2 p = dec_pos[n_follow + rp.ev_idx[r]];
  const int j = rp.fpos[s] - rp.fpos[rp.off[r]];
  return make_int2(p.x + j, p.y + j);
}
__global__ void k_rp_emit(const int2 *__restrict__ sel, int n_sel, const int *__restrict__ flag, RpView rp, int n_follow,
                          const mmp_churn_event *__restrict__ ev, const mmp_model_row *__restrict__ models, const int2 *__restrict__ dec_pos,
                          mmp_decision_in *__restrict__ dec_in, DecMeta *__restrict__ meta, int32_t *__restrict__ extra,
                          int *__restrict__ status, int *__restrict__ dec_of_model) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_sel || !flag[s]) return;
  const int2 x = sel[s];
  const int k = rp_dec_slot(rp, s, x.y, dec_pos, n_follow).x, e = rp.ev_idx[x.y];
  const mmp_model_row r = models[x.x];
  mmp_decision_in d;  // getNext(model, self = leader, lastUsed = the model's), UNBALANCED_KEY: no flags (MM:6727, 6940-6943)
  d.flags = 0; d.fresh = -1; d.extra_off = k; d.extra_n = 0;
  d.model = x.x; d.self = ev[e].caller; d.last_used = r.last_used;
  dec_in[k] = d;
  extra[k] = -1;
  meta[k] = DecMeta{e, r.size_units, n_follow + e, -1};
  status[k] = CH_INVALID;
  dec_of_model[x.x] = k;
}
__global__ void k_rp_route(const int2 *__restrict__ sel, int n_sel, const int *__restrict__ flag, RpView rp, int n_follow,
                           const int2 *__restrict__ dec_pos, const mmp_decision_in *__restrict__ dec_in,
                           const mmp_decision_out *__restrict__ dec_out, const DecMeta *__restrict__ meta, int max_instances,
                           const mmp_churn_event *__restrict__ ev, long long now0, int *__restrict__ status, int *__restrict__ dec_target,
                           LruEv *__restrict__ lev, unsigned long long *__restrict__ keys) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n_sel || !flag[s]) return;
  const int2 ks = rp_dec_slot(rp, s, sel[s].y, dec_pos, n_follow);
  churn_route_one(ks.x, (size_t)ks.y, dec_in, dec_out, meta, max_instances, ev, now0, status, dec_target, lev, keys);
}
__global__ void k_rp_reset(const int2 *__restrict__ sel, int n_sel, int *__restrict__ first_ev) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s < n_sel) first_ev[sel[s].x] = 0x7fffffff;
}

// ---------------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------------
static int32_t commit_locked(mmp_fleet *f, bool rows_on_device);  // mmplace.cu: mmp_fleet_commit without taking the ingest lock
static inline int32_t lv_n_types(mmp_fleet *f) { return f->live.n_type_ids; }

// rows: also take every present instance's row from lv.inst_rows (inside a window, after its republish; the caller makes sure
// no host row holds an update the device has not seen).  The copies go on the commit stream, behind the window's kernels.
static int32_t sync_host_from_device(mmp_fleet *f, bool rows) {
  HostState &hs = f->hs;
  cudaStream_t st = f->commit_stream;
  const int32_t nm = hs.n_models_used, NI = hs.cfg.max_instances;
  std::vector<OvfEdge> ovf((size_t)f->live.n_ovf);
  std::vector<mmp_instance_row> inst_rows(rows ? (size_t)NI : 0);
  if (nm) {
    CK(cudaMemcpyAsync(hs.models.data(), f->live.models.p, (size_t)nm * sizeof(mmp_model_row), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(hs.edge_inl.data(), f->live.edges.p, (size_t)nm * HostState::EDGE_INL * 4, cudaMemcpyDeviceToHost, st));
  }
  if (!ovf.empty()) CK(cudaMemcpyAsync(ovf.data(), f->live.ovf.p, ovf.size() * sizeof(OvfEdge), cudaMemcpyDeviceToHost, st));
  if (rows) CK(cudaMemcpyAsync(inst_rows.data(), f->live.inst_rows.p, (size_t)NI * sizeof(mmp_instance_row), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (rows)
    for (int32_t i = 0; i < NI; i++) if (hs.inst[i].present) hs.inst[i].row = inst_rows[i];
  // the overflow registrations as the loop left them: models that went back inline lose their entries
  hs.edge_ovf.clear(); hs.edge_ovf_ts.clear();
  for (const OvfEdge &e : ovf) { hs.edge_ovf[e.model].push_back(e.inst); hs.edge_ovf_ts[e.model].push_back(e.ts); }
  hs.ovf_dirty = true;
  f->device_ahead = false;
  return MMP_OK;
}
// Exclusive prefix sums of (decision, event slots) pairs
struct Int2Sum { __host__ __device__ int2 operator()(const int2 &a, const int2 &b) const { return make_int2(a.x + b.x, a.y + b.y); } };

// The registry phase's re-lay of the overflow table (lv.ovf / lv.n_ovf) after a window that touched a model with more than
// four registrations or pushed one past four: count, scan, write the new table beside the old one, swap.
static int32_t churn_relay_ovf(mmp_fleet *f, cudaStream_t st) {
  ChurnState &cs = f->churn;
  LiveState &lv = f->live;
  const int32_t NM = f->hs.n_models_used;
  CK(cs.ovf_count.ensure((size_t)(NM + 1) * 8));
  int *cnt = cs.ovf_count.as<int>(), *off = cnt + NM + 1;
  k_ovf_count<<<(NM + 1 + 255) / 256, 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), NM, cs.rm_mask.as<unsigned>(),
                                                   cs.add_inst.as<int>(), cs.ovf_dead.as<unsigned char>(), cnt);
  size_t tmp = 0;
  CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp, cnt, off, NM + 1, st));
  CK(cs.cub_tmp.ensure(tmp + 16));
  CK(cub::DeviceScan::ExclusiveSum(cs.cub_tmp.p, tmp, cnt, off, NM + 1, st));
  int total = 0;
  CK(cudaMemcpyAsync(&total, off + NM, 4, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  CK(cs.ovf_next.ensure((size_t)std::max(total, 1) * sizeof(OvfEdge)));
  k_ovf_relay<<<(NM + 255) / 256, 256, 0, st>>>(reg_tables(lv), lv.models.as<mmp_model_row>(), lv.edges.as<int4>(), NM, cs.rm_mask.as<unsigned>(),
                                               cs.add_inst.as<int>(), cs.ovf_dead.as<unsigned char>(), off, cs.ovf_next.as<OvfEdge>());
  f->launches += 4;
  CK(cudaGetLastError());
  std::swap(lv.ovf, cs.ovf_next);
  lv.n_ovf = total;
  return MMP_OK;
}

// The reaper pass of a window with REAPER events (rp_ev: their trace indices), after k_stats filled acc / min_lru: every
// event's selections in cs.rp_sel as (model, event) in emission order, cs.rp_ev = [rp_ev | selection offsets].  The total is
// read back (the window's one synchronisation for it: the decision buffers are sized from it); a second walk follows only
// when several events selected more models in all than the fleet has.
static int32_t churn_reaper_pass(mmp_fleet *f, const DeviceSnapshot &ds, const StatsAcc *acc, const long long *min_lru,
                                 const std::vector<int> &rp_ev, cudaStream_t st, int32_t *n_sel) {
  ChurnState &cs = f->churn;
  const HostSnapshot &h = ds.host;
  const int NM = f->hs.n_models_used, R = (int)rp_ev.size(), tc = h.tc_enabled ? 1 : 0;
  const int ns = tc ? (int)h.part_types.size() : 1;
  const size_t nmx = (size_t)std::max(NM, 1);
  // each partition's prohibited type ids of this epoch (reaper_impl's `excl`), sorted: [offsets (ns + 1) | ids]
  std::vector<int> pt((size_t)ns + 1, 0);
  for (int p = 0; tc && p < ns; p++) {
    std::vector<int> ids;
    for (int32_t tid : h.part_type_ids[p]) if (tid >= 0 && tid < (int32_t)h.type_slot.size()) ids.push_back(tid);
    std::sort(ids.begin(), ids.end());
    pt.insert(pt.end(), ids.begin(), ids.end());
    pt[p + 1] = pt[p] + (int)ids.size();
  }
  std::vector<int> evo(rp_ev);
  evo.resize((size_t)2 * R + 1, 0);
  CK(upload_vec(cs.rp_pt, pt, st));
  CK(upload_vec(cs.rp_ev, evo, st));
  CK(cs.rp_keys.ensure(nmx * 16)); CK(cs.rp_idx.ensure(nmx * 8 + 16)); CK(cs.rp_flag.ensure(nmx));
  CK(cs.rp_sel.ensure(nmx * sizeof(int2)));  // (one event selects each model at most once)
  const size_t parts_b = (size_t)ns * sizeof(RpPart), space_b = (size_t)ns * 8;
  CK(cs.rp_plan.ensure(parts_b + space_b + sizeof(RpPlan) + (size_t)ns * 4 + 16));
  const size_t taken_cap = cs.rp_taken.cap;
  CK(cs.rp_taken.ensure(nmx * 4));
  if (cs.rp_taken.cap != taken_cap || cs.rp_gen > INT32_MAX / 2) {  // tags start over on a zeroed array
    CK(cudaMemsetAsync(cs.rp_taken.p, 0, cs.rp_taken.cap, st));
    cs.rp_gen = 0;
  }
  RpPart *parts = cs.rp_plan.as<RpPart>();
  unsigned long long *space = reinterpret_cast<unsigned long long *>(cs.rp_plan.as<char>() + parts_b);
  RpPlan *plan = reinterpret_cast<RpPlan *>(cs.rp_plan.as<char>() + parts_b + space_b);
  int *order = reinterpret_cast<int *>(plan + 1);
  unsigned long long *keys = cs.rp_keys.as<unsigned long long>(), *skeys = keys + nmx;
  int *idx = cs.rp_idx.as<int>(), *sidx = idx + nmx, *d_n = sidx + nmx;
  CK(cudaMemsetAsync(space, 0, space_b, st));
  k_rp_plan<<<1, 256, 0, st>>>(acc, min_lru, ns, tc, f->hs.cfg.default_model_size_units, parts, order, plan);
  k_rp_flag<<<(int)((nmx + 255) / 256), 256, 0, st>>>(f->live.models.as<mmp_model_row>(), NM, plan, cs.rp_flag.as<uint8_t>());
  thrust::counting_iterator<int32_t> iota(0);
  size_t t1 = 0, t2 = 0;
  CK(cub::DeviceSelect::Flagged(nullptr, t1, iota, cs.rp_flag.as<uint8_t>(), idx, d_n, NM, st));
  CK(cub::DeviceRadixSort::SortPairs(nullptr, t2, keys, skeys, idx, sidx, NM, 0, 64, st));
  CK(cs.cub_tmp.ensure(std::max(t1, t2) + 16));
  CK(cub::DeviceSelect::Flagged(cs.cub_tmp.p, t1, iota, cs.rp_flag.as<uint8_t>(), idx, d_n, NM, st));
  k_rp_keys<<<(int)((nmx + 255) / 256), 256, 0, st>>>(f->live.models.as<mmp_model_row>(), idx, d_n, NM, keys);
  CK(cub::DeviceRadixSort::SortPairs(cs.cub_tmp.p, t2, keys, skeys, idx, sidx, NM, 0, 64, st));
  if (h.n_ranks > 0)
    k_rp_space<<<std::min(f->sm_count, (h.n_ranks + 255) / 256), 256, 0, st>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(),
                                                                            ds.lthreads_col.as<int32_t>(), ds.linprog_col.as<int32_t>(),
                                                                            ds.part_of_rank.as<int32_t>(), h.n_ranks, tc, ns, parts, space);
  f->launches += 6 + (h.n_ranks > 0);
  CK(cudaGetLastError());
  int *d_off = cs.rp_ev.as<int>() + R;
  for (int pass = 0;; pass++) {
    const long long sel_cap = (long long)(cs.rp_sel.cap / sizeof(int2));
    k_rp_walk<<<1, RP_WALK, 0, st>>>(f->live.models.as<mmp_model_row>(), skeys, sidx, d_n, plan, parts, order, space, tc,
                                     cs.rp_pt.as<int>(), cs.rp_pt.as<int>() + ns + 1, cs.ev.as<mmp_churn_event>(), cs.rp_ev.as<int>(), R,
                                     cs.rp_gen + 1, cs.rp_taken.as<int>(), cs.rp_sel.as<int2>(), sel_cap, d_off);
    f->launches++;
    CK(cudaGetLastError());
    cs.rp_gen += R;
    int total = 0;
    CK(cudaMemcpyAsync(&total, d_off + R, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (total <= sel_cap) { *n_sel = total; return MMP_OK; }
    if (pass) { g_err = "internal: the reaper's selections changed between two walks"; return MMP_E_STATE; }
    CK(cs.rp_sel.ensure((size_t)total * sizeof(int2)));
  }
}

extern "C" {

int32_t mmp_churn_init(mmp_fleet *f, const mmp_churn_config *cfg) {
  NEED(f);
  if (!cfg || cfg->slots_per_instance <= 0 || cfg->load_timeout_ms < 0) { g_err = "bad churn config"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  if (f->epoch == 0 || !f->live.valid) { g_err = "mmp_churn_init needs a committed snapshot"; return MMP_E_EPOCH; }
  if (f->hs.cfg.shard_count > 1) { g_err = "the closed loop runs on an unsharded fleet"; return MMP_E_STATE; }
  for (int32_t m = 0; m < f->hs.n_models_used; m++)
    if (f->hs.models[m].copy_count == 255 && f->hs.models[m].reserved > 255u) {
      g_err = "model " + std::to_string(m) + " holds more registrations than a copy count (255) can tell apart: its loaded copies are unknown";
      return MMP_E_STATE;
    }
  const int32_t NI = f->hs.cfg.max_instances, NM = f->hs.cfg.max_models;
  std::vector<int64_t> cap((size_t)NI, 0);
  for (int32_t i = 0; i < NI; i++) if (f->hs.inst[i].present) cap[i] = f->hs.inst[i].row.capacity;
  rc = mmp_lru_init(f, NI, cap.data(), cfg->slots_per_instance);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  ChurnState &cs = f->churn;
  cs.load_timeout_ms = cfg->load_timeout_ms;
  for (Event &e : cs.phase_ev) if (!e) CK(cudaEventCreate(e.put()));
  std::vector<long long> lp((size_t)NI, (long long)cfg->last_published_ms);
  CK(upload_vec(cs.last_published, lp, f->commit_stream));
  CK(cs.first_ev.ensure((size_t)NM * 4)); CK(cs.dec_of_model.ensure((size_t)NM * 4)); CK(cs.rm_mask.ensure((size_t)NM * 4));
  CK(cs.add_inst.ensure((size_t)NM * 4)); CK(cs.used_t.ensure((size_t)NM * 8)); CK(cs.force_publish.ensure((size_t)NI));
  CK(cs.counters.ensure(64));
  CK(cudaMemsetAsync(cs.first_ev.p, 0x7f, (size_t)NM * 4, f->commit_stream));  // 0x7f7f7f7f: larger than any item index
  CK(cudaMemsetAsync(cs.dec_of_model.p, 0xff, (size_t)NM * 4, f->commit_stream));
  CK(cudaMemsetAsync(cs.add_inst.p, 0xff, (size_t)NM * 4, f->commit_stream));
  CK(cudaMemsetAsync(cs.rm_mask.p, 0, (size_t)NM * 4, f->commit_stream));
  CK(cudaMemsetAsync(cs.used_t.p, 0, (size_t)NM * 8, f->commit_stream));
  CK(cudaStreamSynchronize(f->commit_stream));
  cs.n_carry = 0;
  cs.regs_from_host = true;
  cs.on = true;
  f->lru_loop = true;
  return MMP_OK;
}

int32_t mmp_churn_seed(mmp_fleet *f, int32_t n, const int32_t *instance, const int32_t *model, const int64_t *last_used,
                       const int32_t *weight, const int64_t *load_ts, int64_t now_ms) {
  NEED(f);
  if (n < 0 || (n > 0 && (!instance || !model || !last_used || !weight || !load_ts))) { g_err = "bad argument"; return MMP_E_ARG; }
  if (!f->churn.on) { g_err = "mmp_churn_init not called"; return MMP_E_STATE; }
  if (n == 0) return MMP_OK;
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  std::vector<int> off((size_t)f->lru_n + 1, 0), order((size_t)n);
  std::vector<LruEv> lev((size_t)n);
  for (int32_t i = 0; i < n; i++) {
    if (instance[i] < 0 || instance[i] >= f->lru_n || model[i] < 0 || model[i] >= f->hs.cfg.max_models || last_used[i] < 0 || load_ts[i] < 0) {
      g_err = "bad seed entry"; return MMP_E_ARG;
    }
    off[instance[i] + 1]++;
    lev[i] = LruEv{LEV_SEED, model[i], weight[i], i, -1, 0, last_used[i], load_ts[i]};
  }
  for (int i = 0; i < f->lru_n; i++) off[i + 1] += off[i];
  { std::vector<int> pos(off.begin(), off.end() - 1); for (int32_t i = 0; i < n; i++) order[pos[instance[i]]++] = i; }
  ChurnState &cs = f->churn;
  cudaStream_t st = f->commit_stream;
  CK(upload_vec(cs.lev, lev, st)); CK(upload_vec(cs.vals, order, st)); CK(upload_vec(cs.off, off, st));
  CK(cs.evict.ensure(sizeof(EvictRec) * 16));
  CK(cudaMemsetAsync(cs.counters.p, 0, 64, st));
  CK(cudaMemsetAsync(f->lru_pin.p, 0x80, (size_t)f->lru_n * 8, st));  // LRU_PIN_NONE: oldestTime() is the head (N14)
  ChurnHooks hk{};
  hk.min_space = f->hs.cfg.min_space_units; hk.min_churn_age = f->hs.cfg.min_churn_age_ms;
  const int grid = (f->lru_n + 3) / 4;
  size_t lsm = 0;
  const int lst = lru_stage_slots(f, &lsm);
  k_lru_events<false><<<grid, 128, lsm, st>>>(lru_view(f), cs.lev.as<LruEv>(), cs.vals.as<int>(), cs.off.as<int>(), now_ms, 0, hk, cs.evict.as<EvictRec>(),
                                      16, cs.counters.as<int>() + 4, cs.counters.as<int>() + 5, lst, OvfHooks{});
  f->launches++;
  CK(cudaGetLastError());
  int hdr[8];
  CK(cudaMemcpyAsync(hdr, cs.counters.p, sizeof(hdr), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (hdr[5]) { g_err = "LRU slot capacity exceeded (raise slots_per_instance)"; return MMP_E_NOMEM; }
  if (hdr[4]) { g_err = "the seed does not fit the caches (evictions while seeding)"; return MMP_E_ARG; }
  return MMP_OK;
}

int32_t mmp_churn_step(mmp_fleet *f, const mmp_churn_event *ev, int32_t n, int64_t now0, int64_t now1, uint64_t seed,
                       mmp_churn_decision *dec_out, int32_t dec_cap, int32_t *n_dec_out, mmp_churn_eviction *evict_out, int32_t evict_cap,
                       int32_t *n_evict_out, mmp_instance_row *rows_out, mmp_churn_report *report) {
  NEED(f);
  if (n < 0 || (n > 0 && !ev) || dec_cap < 0 || evict_cap < 0 || (dec_cap > 0 && !dec_out) || (evict_cap > 0 && !evict_out)) { g_err = "bad argument"; return MMP_E_ARG; }
  ChurnState &cs = f->churn;
  if (!cs.on) { g_err = "mmp_churn_init not called"; return MMP_E_STATE; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  if (f->hs.structural_dirty || !f->hs.dirty_inst.empty() || !f->hs.dirty_models.empty() || f->hs.all_models_dirty) {
    g_err = "uncommitted ingest: call mmp_fleet_commit before mmp_churn_step"; return MMP_E_STATE;
  }
  cudaStream_t st = f->commit_stream;
  CK(cs.type_ok.ensure((size_t)std::max(lv_n_types(f), 1)));
  const DeviceSnapshot &ds = f->snaps[f->cur];  // (placement calls of other threads share it; this thread is the only writer)
  LiveState &lv = f->live;
  const int32_t NI = f->hs.cfg.max_instances, NM = f->hs.n_models_used;
  const int32_t nF = cs.n_carry, Q = nF + n;
  CtxLease c(f);
  if (!c) { g_err = "cannot create CUDA stream"; return MMP_E_CUDA; }
  const Event *evs = cs.phase_ev;
  if (cs.regs_from_host) {  // (see ChurnState)
    cs.max_copies = 1; cs.deep_failed = false;
    for (int32_t m = 0; m < NM; m++) {
      const mmp_model_row &r = f->hs.models[m];
      cs.max_copies = std::max<int32_t>(cs.max_copies, r.copy_count);
      if (r.reserved >= 4u + r.copy_count) cs.deep_failed = true;
    }
    cs.regs_from_host = false;
  }
  // event slots: one per decision or cache hit, one per loaded copy of a REMOVE's model
  size_t n_remove = 0;
  std::vector<int> rp_ev;  // the REAPER events
  for (int32_t i = 0; i < n; i++) {
    n_remove += ev[i].type == 1;
    if (ev[i].type == MMP_CHURN_REAPER) rp_ev.push_back(i);
  }
  const int n_rp = (int)rp_ev.size();
  const size_t QQ = (size_t)std::max(Q, 1);
  // the window's marks may reach an overflow registration (a model with more than four), or its registry phase may push a
  // model with four failed loads past four: then the registry phase reads the mark flag back and re-lays lv.ovf
  const bool ovf_window = lv.n_ovf > 0 || cs.deep_failed;
  if (lv.n_ovf > 0) CK(cs.ovf_dead.ensure((size_t)lv.n_ovf));
  CK(cs.ev.ensure(QQ * sizeof(mmp_churn_event))); CK(cs.is_dec.ensure(QQ * 8 + 16)); CK(cs.dec_pos.ensure(QQ * 8 + 16));
  CK(cs.off.ensure((size_t)(NI + 2) * 4));
  CK(cs.stats_acc.ensure(((size_t)ds.host.part_types.size() + 2) * sizeof(StatsAcc) + 16));
  CK(cudaEventRecord(evs[0], st));
  if (n) CK(cudaMemcpyAsync(cs.ev.p, ev, (size_t)n * sizeof(mmp_churn_event), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(cs.counters.p, 0, 64, st));
  CK(cudaMemsetAsync(cs.force_publish.p, 0, (size_t)NI, st));
  if (lv.n_ovf > 0) CK(cudaMemsetAsync(cs.ovf_dead.p, 0, (size_t)lv.n_ovf, st));
  // ---- the rebalance rule's fullness test reads the stats of the window's snapshot (MM:2918-2920) ----
  int32_t n_sel = 0;  // the reaper's selections (one decision each at most)
  {
    const int np = (int)ds.host.part_types.size();
    const size_t bytes = (size_t)(np + 1) * sizeof(StatsAcc) + 8;
    CK(cudaMemsetAsync(cs.stats_acc.p, 0, bytes, st));
    long long *d_min = reinterpret_cast<long long *>(cs.stats_acc.as<char>() + (size_t)(np + 1) * sizeof(StatsAcc));
    if (n_rp) {  // the reaper reads the cluster's LRU too: start it at Long.MAX_VALUE (ISST)
      CK(cudaMemsetAsync(d_min, 0xff, 7, st));
      CK(cudaMemsetAsync(reinterpret_cast<char *>(d_min) + 7, 0x7f, 1, st));
    }
    if (ds.host.n_ranks > 0) {
      k_stats<<<std::min(f->sm_count, (ds.host.n_ranks + 255) / 256), 256, 0, st>>>(ds.rows.as<RankRow>(), ds.cap_col.as<int64_t>(),
                                                                                  ds.part_of_rank.as<int32_t>(), ds.host.n_ranks,
                                                                                  f->hs.cfg.min_space_units, cs.stats_acc.as<StatsAcc>(), d_min, np);
      f->launches++;
    }
    k_churn_type_ok<<<(lv.n_type_ids + 127) / 128, 128, 0, st>>>(cs.stats_acc.as<StatsAcc>(), lv.type_part_off.as<int>(), lv.type_parts.as<int>(),
                                                                lv.n_type_ids, cs.type_ok.as<unsigned char>());
    f->launches++;
    CK(cudaGetLastError());
    // ---- the reaper's proactive loads: selections of the window's REAPER events (then one read-back of their count) ----
    if (n_rp) {
      CK(cudaEventRecord(evs[7], st));
      rc = churn_reaper_pass(f, ds, cs.stats_acc.as<StatsAcc>(), d_min, rp_ev, st, &n_sel);
      if (rc < 0) return rc;
      CK(cudaEventRecord(evs[8], st));
    }
  }
  // decision records: one per item, one more per selection of the reaper (at most: the coalesced ones stay malformed)
  const size_t QD = QQ + (size_t)n_sel, NK = QD + n_remove * (size_t)(cs.max_copies - 1);
  if (NK > (size_t)INT32_MAX) { g_err = "too many cache events in one window"; return MMP_E_ARG; }
  CK(cs.dec_in.ensure(QD * sizeof(mmp_decision_in))); CK(cs.dec_out.ensure(QD * sizeof(mmp_decision_out)));
  CK(cs.dec_meta.ensure(QD * sizeof(DecMeta))); CK(cs.dec_target.ensure(QD * 4)); CK(cs.extra.ensure(QD * 4)); CK(cs.status.ensure(QD * 4));
  CK(cs.lev.ensure(NK * sizeof(LruEv))); CK(cs.keys.ensure(NK * 8)); CK(cs.vals.ensure(NK * 4)); CK(cs.keys2.ensure(NK * 8)); CK(cs.vals2.ensure(NK * 4));
  const int32_t ecap = (int32_t)std::min<size_t>(4 * QD + 65536, (size_t)1 << 26);
  CK(cs.evict.ensure((size_t)ecap * sizeof(EvictRec))); CK(cs.next_carry.ensure((size_t)ecap * sizeof(Follow)));
  const int qb = (Q + 255) / 256, qdb = (int)((QD + 255) / 256), sb = (n_sel + 255) / 256;
  const int QDi = Q + n_sel;  // (decisions placed / collected: == Q without REAPER events)
  const mmp_model_row *lmodels = lv.models.as<mmp_model_row>();
  const Follow *carry = cs.carry.as<Follow>();
  const RegTables R{lv.edges.as<int4>(), nullptr, lv.ovf.as<OvfEdge>(), lv.n_ovf};
  if (n_sel) CK(cs.rp_fpos.ensure((size_t)(n_sel + 1) * 8));
  const int2 *sel = cs.rp_sel.as<int2>();
  int *sel_flag = cs.rp_fpos.as<int>(), *sel_fpos = sel_flag + n_sel + 1;  // first-decision flags, their exclusive scan
  const RpView rp{cs.rp_ev.as<int>(), n_rp, cs.rp_ev.as<int>() + n_rp, n_sel ? sel_fpos : nullptr};
  bool relaid = false;
  if (Q > 0) {
    // ---- A: classify ----
    k_churn_first<<<qb, 256, 0, st>>>(carry, nF, cs.ev.as<mmp_churn_event>(), n, lmodels, NM, cs.first_ev.as<int>());
    if (n_sel) {  // the reaper's selections take part in the first-miss rule at their event's position
      k_rp_first<<<sb, 256, 0, st>>>(sel, n_sel, rp.ev_idx, nF, cs.first_ev.as<int>());
      k_rp_mark<<<(n_sel + 1 + 255) / 256, 256, 0, st>>>(sel, n_sel, rp.ev_idx, nF, cs.first_ev.as<int>(), sel_flag, cs.counters.as<int>());
      size_t t = 0;
      CK(cub::DeviceScan::ExclusiveSum(nullptr, t, sel_flag, sel_fpos, n_sel + 1, st));
      CK(cs.cub_tmp.ensure(t + 16));
      CK(cub::DeviceScan::ExclusiveSum(cs.cub_tmp.p, t, sel_flag, sel_fpos, n_sel + 1, st));
      f->launches += 3;
    }
    k_churn_flag<<<qb, 256, 0, st>>>(carry, nF, cs.ev.as<mmp_churn_event>(), n, lmodels, NM, cs.first_ev.as<int>(), cs.is_dec.as<int2>(),
                                    cs.used_t.as<long long>(), cs.counters.as<int>(), rp);
    size_t tmp = 0;
    CK(cub::DeviceScan::ExclusiveScan(nullptr, tmp, cs.is_dec.as<int2>(), cs.dec_pos.as<int2>(), Int2Sum(), make_int2(0, 0), Q, st));
    CK(cs.cub_tmp.ensure(tmp + 16));
    CK(cub::DeviceScan::ExclusiveScan(cs.cub_tmp.p, tmp, cs.is_dec.as<int2>(), cs.dec_pos.as<int2>(), Int2Sum(), make_int2(0, 0), Q, st));
    // decision records beyond the window's count stay malformed (model -1): the scoring kernel answers them INVALID
    CK(cudaMemsetAsync(cs.dec_in.p, 0xff, QD * sizeof(mmp_decision_in), st));
    CK(cudaMemsetAsync(cs.status.p, 0, QD * 4, st));
    k_churn_emit<<<qb, 256, 0, st>>>(carry, nF, cs.ev.as<mmp_churn_event>(), n, lmodels, R, NM, NI, cs.first_ev.as<int>(),
                                    cs.is_dec.as<int2>(), cs.dec_pos.as<int2>(), cs.dec_in.as<mmp_decision_in>(), cs.dec_meta.as<DecMeta>(),
                                    cs.extra.as<int32_t>(), cs.status.as<int>(), cs.dec_of_model.as<int>(), cs.lev.as<LruEv>(),
                                    cs.keys.as<unsigned long long>(), now0);
    f->launches += 5;
    if (n_sel) {
      k_rp_emit<<<sb, 256, 0, st>>>(sel, n_sel, sel_flag, rp, nF, cs.ev.as<mmp_churn_event>(), lmodels, cs.dec_pos.as<int2>(),
                                    cs.dec_in.as<mmp_decision_in>(), cs.dec_meta.as<DecMeta>(), cs.extra.as<int32_t>(), cs.status.as<int>(),
                                    cs.dec_of_model.as<int>());
      f->launches++;
    }
    CK(cudaGetLastError());
    CK(cudaEventRecord(evs[1], st));
    // ---- B: placement of the window's decisions against the committed snapshot (one clock for the batch: now0) ----
    SnapshotView vw = ds.view;
    vw.n_extra = QDi;
    CK(c->d_fresh.ensure(sizeof(FreshRow)));
    PlaceArgs a{vw, cs.dec_in.as<mmp_decision_in>(), QDi, c->d_fresh.as<FreshRow>(), 0, cs.extra.as<int32_t>(), cs.dec_out.as<mmp_decision_out>(),
                nullptr, nullptr, now0, seed, 0};
    CK(launch_place(f, a, st));
    CK(cudaEventRecord(evs[2], st));
    // ---- C: route every cache event to its instance ----
    k_churn_route<<<qb, 256, 0, st>>>(cs.dec_in.as<mmp_decision_in>(), cs.dec_out.as<mmp_decision_out>(), cs.dec_meta.as<DecMeta>(),
                                     cs.is_dec.as<int2>(), cs.dec_pos.as<int2>(), Q, NI, cs.ev.as<mmp_churn_event>(), now0, cs.status.as<int>(),
                                     cs.dec_target.as<int>(), cs.lev.as<LruEv>(), cs.keys.as<unsigned long long>());
    if (n_sel) {
      k_rp_route<<<sb, 256, 0, st>>>(sel, n_sel, sel_flag, rp, nF, cs.dec_pos.as<int2>(), cs.dec_in.as<mmp_decision_in>(),
                                     cs.dec_out.as<mmp_decision_out>(), cs.dec_meta.as<DecMeta>(), NI, cs.ev.as<mmp_churn_event>(), now0,
                                     cs.status.as<int>(), cs.dec_target.as<int>(), cs.lev.as<LruEv>(), cs.keys.as<unsigned long long>());
      f->launches++;
    }
    k_churn_tail<<<(int)((NK + 255) / 256), 256, 0, st>>>(cs.keys.as<unsigned long long>(), cs.vals.as<int>(), (int)NK, cs.is_dec.as<int2>(),
                                                          cs.dec_pos.as<int2>(), Q);
    tmp = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp, cs.keys.as<unsigned long long>(), cs.keys2.as<unsigned long long>(), cs.vals.as<int>(),
                                       cs.vals2.as<int>(), (int)NK, 0, 64, st));
    CK(cs.cub_tmp.ensure(tmp + 16));
    CK(cub::DeviceRadixSort::SortPairs(cs.cub_tmp.p, tmp, cs.keys.as<unsigned long long>(), cs.keys2.as<unsigned long long>(), cs.vals.as<int>(),
                                       cs.vals2.as<int>(), (int)NK, 0, 64, st));
    k_churn_offsets<<<(NI + 1 + 255) / 256, 256, 0, st>>>(cs.keys2.as<unsigned long long>(), (int)NK, NI, cs.off.as<int>());
    f->launches += 5;
    CK(cudaGetLastError());
    CK(cudaEventRecord(evs[3], st));
    // ---- apply: one warp per instance, its events in order ----
    ChurnHooks hk{};
    hk.enabled = 1;
    hk.min_space = f->hs.cfg.min_space_units; hk.min_churn_age = f->hs.cfg.min_churn_age_ms; hk.load_timeout = cs.load_timeout_ms;
    hk.status = cs.status.as<int>(); hk.dec_target = cs.dec_target.as<int>(); hk.dec_of_model = cs.dec_of_model.as<int>();
    hk.edges = R.edges; hk.models = lmodels; hk.rm_mask = cs.rm_mask.as<unsigned>();
    hk.type_ok = cs.type_ok.as<unsigned char>(); hk.n_type_ids = lv.n_type_ids;
    hk.next = cs.next_carry.as<Follow>(); hk.n_next = cs.counters.as<int>() + 6; hk.next_cap = ecap;
    hk.force_publish = cs.force_publish.as<unsigned char>();
    size_t lsm = 0;
    const int lst = lru_stage_slots(f, &lsm);
    // (a fleet without overflow registrations runs the listener over the four inline positions only)
    (lv.n_ovf > 0 ? k_lru_events<true> : k_lru_events<false>)<<<(f->lru_n + 3) / 4, 128, lsm, st>>>(
        lru_view(f), cs.lev.as<LruEv>(), cs.vals2.as<int>(), cs.off.as<int>(), now0, 1, hk,
                                                      cs.evict.as<EvictRec>(), ecap, cs.counters.as<int>() + 4, cs.counters.as<int>() + 5, lst,
                                                      OvfHooks{R.ovf, R.n_ovf, cs.ovf_dead.as<unsigned char>()});
    f->launches++;
    CK(cudaGetLastError());
    CK(cudaEventRecord(evs[4], st));
    // ---- D: registry ----
    k_churn_collect_adds<<<qdb, 256, 0, st>>>(cs.dec_in.as<mmp_decision_in>(), cs.status.as<int>(), cs.dec_target.as<int>(), QDi, cs.add_inst.as<int>(),
                                             cs.dec_of_model.as<int>());
    k_churn_reset_first<<<qb, 256, 0, st>>>(carry, nF, cs.ev.as<mmp_churn_event>(), n, NM, cs.first_ev.as<int>());
    if (n_sel) { k_rp_reset<<<sb, 256, 0, st>>>(sel, n_sel, cs.first_ev.as<int>()); f->launches++; }
    k_churn_registry<<<(NM + 255) / 256, 256, 0, st>>>(lv.models.as<mmp_model_row>(), lv.edges.as<int4>(), NM, cs.rm_mask.as<unsigned>(),
                                                      cs.add_inst.as<int>(), cs.used_t.as<long long>(), cs.counters.as<int>());
    f->launches += 3;
    CK(cudaGetLastError());
    if (ovf_window) {
      int marked = 0;
      CK(cudaMemcpyAsync(&marked, cs.counters.as<int>() + 2, 4, cudaMemcpyDeviceToHost, st));
      CK(cudaStreamSynchronize(st));
      if (marked) { rc = churn_relay_ovf(f, st); if (rc < 0) return rc; relaid = true; }
    }
  } else {
    for (int i = 1; i <= 4; i++) CK(cudaEventRecord(evs[i], st));
  }
  // ---- E: republish ----
  k_churn_republish<<<(f->lru_n + 3) / 4, 128, 0, st>>>(lru_view(f), lv.inst_rows.as<mmp_instance_row>(), lv.inst_meta.as<int2>(), NI,
                                                       cs.last_published.as<long long>(), cs.force_publish.as<unsigned char>(), now1,
                                                       f->hs.cfg.min_space_units, cs.counters.as<int>());
  f->launches++;
  CK(cudaGetLastError());
  CK(cudaEventRecord(evs[5], st));
  // ---- commit: the device path (re-rank, tables, bitmap from the device-resident edges); the host path, when the fleet
  // needs it, from the device's registry and instance rows ----
  f->device_ahead = true;
  rc = commit_locked(f, true);
  if (rc < 0) return rc;
  CK(cudaEventRecord(evs[6], st));
  // ---- reports ----
  int hdr[16];
  CK(cudaMemcpyAsync(hdr, cs.counters.p, 64, cudaMemcpyDeviceToHost, st));
  int2 last_flag = make_int2(0, 0), last_pos = make_int2(0, 0);
  if (Q > 0) {
    CK(cudaMemcpyAsync(&last_flag, cs.is_dec.as<int2>() + (Q - 1), 8, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(&last_pos, cs.dec_pos.as<int2>() + (Q - 1), 8, cudaMemcpyDeviceToHost, st));
  }
  std::vector<mmp_instance_row> rows((size_t)NI);
  CK(cudaMemcpyAsync(rows.data(), lv.inst_rows.p, (size_t)NI * sizeof(mmp_instance_row), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  if (hdr[5]) { g_err = "LRU slot capacity exceeded for some instance (raise slots_per_instance)"; return MMP_E_NOMEM; }
  if (hdr[2] && !relaid) { g_err = "internal: a window changed overflow registrations the step did not expect"; return MMP_E_STATE; }
  const int32_t n_dec = Q > 0 ? last_pos.x + last_flag.x : 0, n_evict = hdr[4], n_next = hdr[6];
  if (n_evict > ecap || n_next > ecap) { g_err = "eviction report overflow"; return MMP_E_NOMEM; }
  for (int32_t i = 0; i < NI; i++) if (f->hs.inst[i].present) f->hs.inst[i].row = rows[i];
  if (rows_out) memcpy(rows_out, rows.data(), (size_t)NI * sizeof(mmp_instance_row));
  if (n_dec_out) *n_dec_out = n_dec;
  if (n_evict_out) *n_evict_out = n_evict;
  {
    const int32_t nd = std::min(n_dec, dec_cap);
    std::vector<mmp_decision_in> din((size_t)nd);
    std::vector<mmp_decision_out> dout((size_t)nd);
    std::vector<int> stt((size_t)nd);
    std::vector<DecMeta> mt((size_t)nd);
    if (nd) {
      CK(cudaMemcpy(din.data(), cs.dec_in.p, (size_t)nd * sizeof(mmp_decision_in), cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(dout.data(), cs.dec_out.p, (size_t)nd * sizeof(mmp_decision_out), cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(stt.data(), cs.status.p, (size_t)nd * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(mt.data(), cs.dec_meta.p, (size_t)nd * sizeof(DecMeta), cudaMemcpyDeviceToHost));
    }
    for (int32_t k = 0; k < nd; k++) {
      const bool skipped = stt[k] == CH_SKIPPED;
      dec_out[k] = mmp_churn_decision{skipped ? -1 : din[k].model, din[k].self, skipped ? MMP_TARGET_NONE : dout[k].target,
                                      skipped ? 0 : dout[k].n_candidates, stt[k], mt[k].event};
    }
  }
  {
    std::vector<EvictRec> er((size_t)n_evict);
    if (n_evict) CK(cudaMemcpy(er.data(), cs.evict.p, (size_t)n_evict * sizeof(EvictRec), cudaMemcpyDeviceToHost));
    std::sort(er.begin(), er.end(), [](const EvictRec &a, const EvictRec &b) {
      return a.instance != b.instance ? a.instance < b.instance : (a.order != b.order ? a.order < b.order : a.seq < b.seq); });
    for (int32_t k = 0; k < n_evict && k < evict_cap; k++)
      evict_out[k] = mmp_churn_eviction{er[k].instance, er[k].model, er[k].last_used, er[k].weight, er[k].order, er[k].reload};
  }
  {  // the queued ensureLoadedElsewhere calls of the next window, in listener order (instance, trace position, eviction)
    std::vector<Follow> fo((size_t)n_next);
    if (n_next) CK(cudaMemcpy(fo.data(), cs.next_carry.p, (size_t)n_next * sizeof(Follow), cudaMemcpyDeviceToHost));
    std::sort(fo.begin(), fo.end(), [](const Follow &a, const Follow &b) {
      return a.inst != b.inst ? a.inst < b.inst : (a.order != b.order ? a.order < b.order : a.seq < b.seq); });
    CK(upload_vec(cs.carry, fo, st));
    CK(cudaStreamSynchronize(st));
    cs.n_carry = n_next;
  }
  float ms[7] = {0, 0, 0, 0, 0, 0, 0};
  for (int i = 0; i < 6; i++) cudaEventElapsedTime(&ms[i], evs[i], evs[i + 1]);
  cudaEventElapsedTime(&ms[6], evs[0], evs[6]);
  float ms_reaper = 0;  // (inside the classify interval: taken out of it)
  if (n_rp) { cudaEventElapsedTime(&ms_reaper, evs[7], evs[8]); ms[0] -= ms_reaper; }
  cs.t_classify = ms[0]; cs.t_place = ms[1]; cs.t_route = ms[2]; cs.t_apply = ms[3]; cs.t_registry = ms[4]; cs.t_commit = ms[5]; cs.t_total = ms[6];
  if (report) {
    report->n_published = hdr[1]; report->n_carry = n_next; report->n_coalesced = hdr[3]; report->n_lru_events = 0;
    report->ms_classify = ms[0]; report->ms_place = ms[1]; report->ms_route = ms[2]; report->ms_apply = ms[3]; report->ms_registry = ms[4];
    report->ms_commit = ms[5]; report->ms_total = ms[6]; report->ms_reaper = ms_reaper;
    int noff = 0;
    if (Q > 0 && cudaMemcpy(&noff, cs.off.as<int>() + NI, 4, cudaMemcpyDeviceToHost) == cudaSuccess) report->n_lru_events = noff;
  }
  return MMP_OK;
}

int32_t mmp_churn_model(mmp_fleet *f, int32_t model, mmp_model_row *row, int32_t *instances4) {
  NEED(f);
  if (model < 0 || model >= f->hs.n_models_used || !f->live.valid) { g_err = "bad model index"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  if (row) CK(cudaMemcpy(row, f->live.models.as<mmp_model_row>() + model, sizeof(mmp_model_row), cudaMemcpyDeviceToHost));
  if (instances4) CK(cudaMemcpy(instances4, f->live.edges.as<int32_t>() + (size_t)model * 4, 16, cudaMemcpyDeviceToHost));
  return MMP_OK;
}

int32_t mmp_churn_model_ids(mmp_fleet *f, int32_t model, mmp_model_row *row, int32_t *ids, int32_t cap) {
  NEED(f);
  if (model < 0 || model >= f->hs.n_models_used || !f->live.valid || cap < 0 || (cap > 0 && !ids)) { g_err = "bad model index or argument"; return MMP_E_ARG; }
  int32_t rc = set_device(f);
  if (rc < 0) return rc;
  std::lock_guard<std::mutex> g(f->ingest_mu);
  const LiveState &lv = f->live;
  mmp_model_row r;
  int4 e;
  CK(cudaMemcpy(&r, lv.models.as<mmp_model_row>() + model, sizeof(r), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&e, lv.edges.as<int4>() + model, sizeof(e), cudaMemcpyDeviceToHost));
  if (row) *row = r;
  const int32_t n = (int32_t)r.reserved, inl[4] = {e.x, e.y, e.z, e.w};
  for (int32_t j = 0; j < std::min(n, 4) && j < cap; j++) ids[j] = inl[j];
  if (n > 4 && cap > 4) {  // the model's slice of the overflow table: the entries from the first of its model on
    std::vector<OvfEdge> ovf((size_t)lv.n_ovf);
    if (lv.n_ovf) CK(cudaMemcpy(ovf.data(), lv.ovf.p, ovf.size() * sizeof(OvfEdge), cudaMemcpyDeviceToHost));
    const size_t q0 = std::lower_bound(ovf.begin(), ovf.end(), model, [](const OvfEdge &a, int32_t m) { return a.model < m; }) - ovf.begin();
    for (int32_t j = 4; j < n && j < cap; j++) {
      const size_t q = q0 + (size_t)(j - 4);
      ids[j] = q < ovf.size() && ovf[q].model == model ? ovf[q].inst : -1;
    }
  }
  return n;
}

}  // extern "C"
