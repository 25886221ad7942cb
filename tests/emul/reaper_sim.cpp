// reaper_sim.cpp — the CPU oracle (oracle/mm_oracle.cpp, compiled whole into this library) plus one more event type for its
// closed loop.  TEST INFRASTRUCTURE ONLY (tests/reaper_oracle.py builds and binds it).
//
//   orc_sim_step_reaper  orc_sim_step of oracle/mm_sim.inc, line for line, with a REAPER event (type 2; caller = the leader,
//                        t = its clock; model and u ignored): one run of the reaper's proactive loads (MM:6456-6494,
//                        6616-6747) through orc_reaper_select -- the whole cluster, or with type constraints every partition
//                        in getPartitionStats order sharing one `taken` set, all read from the epoch's start.  Every emitted
//                        model is a getNext decision (self = caller, lastUsed = the model's, no extra excludes) at the
//                        REAPER's position, loaded with last_used = the model's lastUsed on the clock t
//                        (ensureLoadedInternal(id, timestamp, 0, null, 0, false), MM:6727); a model already decided in the
//                        epoch is coalesced, as a later miss of a model it decided is.
//
// Divergences from the reference, all epoch batching (the device loop, mmp_churn_step, makes the same): every partition reads
// the epoch's snapshot (no sleep of 2 x INSTANCE_REC_PUBLISH_MIN_PERIOD_MS between partitions, MM:6481-6484); the prune half of
// pruneModelRegistry is a no-op (no instance leaves the table here); repairLastUsedTimeIfNeeded, vmodels and leaseless-record
// cleanup are out of scope; the leader is the event's caller; DISABLE_PROACTIVE_LOADING is a trace without REAPER events; a
// size estimate of 0 (MM:6651 throws) ends the run at that partition.  Everything but the REAPER branch is the oracle's own
// orc_sim_step; a trace without REAPER events gives what orc_sim_step gives.
#pragma GCC diagnostic ignored "-Wsubobject-linkage"  // (as mm_sim.inc: one translation unit)
#include "../../oracle/mm_oracle.cpp"

extern "C" {

int64_t orc_sim_step_reaper(orc_sim *s, const orc_sim_event_t *ev, int32_t n, int64_t now0, int64_t now1, uint64_t seed,
                            orc_sim_decision_t *dec_out, int32_t dec_cap, int32_t *n_dec_out, orc_sim_eviction_t *evict_out,
                            int32_t evict_cap, int32_t *n_evict_out, orc_inst_t *rows_out, int32_t *published_out) {
  if (!s || n < 0) return -1;
  Fleet &f = s->fleet->f;
  const int32_t NI = (int32_t)s->lru.size();
  static const std::string NOTYPE = "\x01<no-config>";
  struct Dec { int32_t model, self, extra; int64_t lastUsed, t; int32_t weight, event, target, ncand, status; int64_t order; };
  struct LEv { int64_t order; int32_t op, model, size, dec; int64_t lastUsed, t; };  // op: 1 TOUCH, 3 REMOVE, 10 LOAD
  std::vector<Dec> D;
  std::vector<std::vector<LEv>> lev((size_t)NI);
  std::unordered_map<int32_t, int32_t> decOfModel;
  // the type-set fullness test of the rebalance rule reads the stats of the epoch's snapshot (MM:2918-2920)
  std::vector<int8_t> rebalanceOk(s->typeNames.size() + 1, -1);
  auto rebalance_ok = [&](int32_t typeIdx) -> bool {
    int8_t &c = rebalanceOk[(typeIdx >= 0 && (size_t)typeIdx < s->typeNames.size()) ? (size_t)typeIdx : s->typeNames.size()];
    if (c < 0) {
      orc_stats_t st;
      orc_type_stats(s->fleet, (typeIdx >= 0 && (size_t)typeIdx < s->typeNames.size()) ? s->typeNames[typeIdx].c_str() : NOTYPE.c_str(), &st);
      c = (st.total_capacity > 0 && st.instance_count > 1 && jmul(20, st.total_free) / st.total_capacity >= 1) ? 1 : 0;
    }
    return c == 1;
  };
  // (evaluated lazily, but nothing below touches the fleet before phase E: it reads the snapshot of the start of the epoch)
  // ---- phase A: classify ----
  const int64_t nFollow = (int64_t)s->carry.size();
  for (int64_t k = 0; k < nFollow; k++) {
    const SimFollow &c = s->carry[(size_t)k];
    Dec d{c.model, c.exclude, c.exclude, c.lastUsed, now0, c.weight, (int32_t)(-1 - k), ORC_NONE, 0, SIM_SKIPPED, k};
    const SimModel &m = s->models[c.model];
    if (m.loaded.empty() && !decOfModel.count(c.model)) { d.status = SIM_INVALID; decOfModel[c.model] = (int32_t)D.size(); }
    D.push_back(d);
  }
  std::vector<std::pair<int32_t, int64_t>> used;  // (model, t) of every request: MR.updateLastUsed at the end of the epoch
  // one run of the reaper's proactive loads at t (MM:6456-6494): orc_reaper_select over the epoch's registry and fleet, for
  // the whole cluster or partition by partition in getPartitionStats order with one `taken` set; a size estimate of 0
  // (-4: the ArithmeticException of MM:6651) ends the run
  std::vector<orc_model_t> reg;
  std::vector<const char *> tnames;
  for (const std::string &t : s->typeNames) tnames.push_back(t.c_str());
  auto reaper_run = [&](int64_t t) {
    const int32_t nm = (int32_t)s->models.size();
    if (reg.empty())
      for (const SimModel &sm : s->models) reg.push_back(orc_model_t{sm.lastUsed, sm.typeIdx, (int32_t)sm.loaded.size(), (int32_t)sm.failed.size(), 0});
    std::vector<int32_t> parts{-1};
    if (f.haveTc) {
      const int32_t cap = (int32_t)f.tcm.ptsToInstanceSetStats.size();
      std::vector<orc_stats_t> ps((size_t)cap + 1);
      parts.assign((size_t)cap + 1, 0);
      parts.resize((size_t)orc_partition_stats(s->fleet, ps.data(), parts.data(), cap));
    }
    std::vector<uint8_t> taken((size_t)nm, 0);
    std::vector<int32_t> out((size_t)nm + 1), sel;
    for (int32_t p : parts) {
      const int64_t c = orc_reaper_select(s->fleet, nm, reg.data(), tnames.data(), (int32_t)tnames.size(), p, t, taken.data(), out.data(), nm);
      if (c < 0) break;
      sel.insert(sel.end(), out.begin(), out.begin() + c);
    }
    return sel;
  };
  for (int32_t i = 0; i < n; i++) {
    const orc_sim_event_t &e = ev[i];
    const int64_t order = nFollow + i;
    if (e.type == 2) {  // REAPER: its loads are decisions at its position, coalescing with the epoch's others like misses do
      for (int32_t model : reaper_run(e.t)) {
        if (decOfModel.count(model)) { s->coalesced++; continue; }
        const SimModel &m = s->models[model];
        decOfModel[model] = (int32_t)D.size();
        // getNext(model, self = leader, lastUsed = the model's) -> ensureLoadedInternal(id, lastUsed, 0, null, 0, false) MM:6727
        D.push_back(Dec{model, e.caller, -1, m.lastUsed, e.t, m.size, i, ORC_NONE, 0, SIM_INVALID, order});
      }
      continue;
    }
    if (e.model < 0 || (size_t)e.model >= s->models.size()) continue;
    SimModel &m = s->models[e.model];
    if (e.type == 0) {
      used.push_back({e.model, e.t});
      if (!m.loaded.empty()) {
        const int32_t inst = m.loaded[e.u % (uint32_t)m.loaded.size()];
        lev[inst].push_back(LEv{order, 1, e.model, 0, -1, e.t, e.t});
      } else if (!decOfModel.count(e.model)) {
        decOfModel[e.model] = (int32_t)D.size();
        D.push_back(Dec{e.model, e.caller, -1, e.t, e.t, m.size, i, ORC_NONE, 0, SIM_INVALID, order});
      } else s->coalesced++;
    } else if (e.type == 1) {
      for (int32_t inst : m.loaded) lev[inst].push_back(LEv{order, 3, e.model, 0, -1, 0, e.t});
    }
  }
  // ---- phase B: placement against the epoch snapshot (one clock for the batch: now0) ----
  int64_t did = 0;
  for (size_t k = 0; k < D.size(); k++) {
    Dec &d = D[k];
    const uint64_t my_id = (uint64_t)k;
    (void)did;
    if (d.status == SIM_SKIPPED) continue;
    const SimModel &m = s->models[d.model];
    if (d.self < 0 || (size_t)d.self >= f.byIdx.size() || !f.byIdx[d.self]) { d.status = SIM_INVALID; continue; }
    IR fresh = *f.byIdx[d.self];
    fresh.rpm = 0;  // N7
    std::vector<int32_t> ex(m.loaded);
    ex.insert(ex.end(), m.failed.begin(), m.failed.end());
    if (d.extra >= 0) ex.push_back(d.extra);
    ExcludeSet es{ex.data(), (int64_t)ex.size()};
    GetNextOut o;
    const std::string &type = (m.typeIdx >= 0 && (size_t)m.typeIdx < s->typeNames.size()) ? s->typeNames[m.typeIdx] : NOTYPE;
    getNext(f, type, d.self, fresh, false, d.lastUsed, es, now0, orc_hash64(seed, my_id), o);
    d.target = o.target; d.ncand = o.nCandidates;
    if (o.target == ORC_NONE) { d.status = SIM_NOWHERE; continue; }
    const int32_t tgt = o.target == ORC_SELF ? d.self : o.target;
    lev[tgt].push_back(LEv{d.order, 10, d.model, d.weight, (int32_t)k, d.lastUsed, d.t});
  }
  // ---- phase C: every instance applies its events in trace order ----
  std::vector<orc_sim_eviction_t> evs;
  std::vector<SimFollow> nextCarry;
  std::vector<std::pair<int32_t, int32_t>> dereg;  // (model, instance)
  std::vector<uint8_t> forcePublish((size_t)NI, 0);
  const int64_t minSpace = f.po.minSpaceUnits, minChurn = f.po.minChurnAgeMs;
  for (int32_t inst = 0; inst < NI; inst++) {
    auto &list = lev[inst];
    if (list.empty()) continue;
    std::stable_sort(list.begin(), list.end(), [](const LEv &a, const LEv &b) { return a.order < b.order; });
    Lru &l = *s->lru[inst];
    auto &lts = s->loadTs[inst];
    std::vector<orc_eviction_t> out;
    auto handle_evictions = [&](const LEv &e) {
      for (const orc_eviction_t &x : out) {
        auto it = lts.find(x.key);
        const bool inRegistry = it != lts.end();
        const bool attemptReload = inRegistry && jsub(e.t, it->second) > 2 * s->loadTimeoutMs;  // MM:2901
        if (inRegistry) lts.erase(it);
        dereg.push_back({x.key, inst});
        auto dk = decOfModel.find(x.key);
        if (dk != decOfModel.end()) {  // a load accepted earlier in this epoch on this instance does not survive it
          Dec &dd = D[dk->second];
          const int32_t t2 = dd.target == ORC_SELF ? dd.self : dd.target;
          if (t2 == inst && dd.status == SIM_ACCEPTED) dd.status = SIM_EVICTED_LATER;
        }
        bool reload = false;
        if (attemptReload && rebalance_ok(s->models[x.key].typeIdx)) {  // MM:2916-2922
          reload = true;
          nextCarry.push_back(SimFollow{x.key, inst, x.last_used, (int32_t)x.weight});
        }
        evs.push_back(orc_sim_eviction_t{inst, x.key, x.last_used, (int32_t)x.weight, (int32_t)e.order, reload ? 1 : 0});
        forcePublish[inst] = 1;
      }
      out.clear();
    };
    for (const LEv &e : list) {
      const int32_t ei = (int32_t)e.order;
      if (e.op == 1) l.apply(orc_lru_event_t{1, e.model, 0, e.lastUsed}, ei, e.t, out);
      else if (e.op == 3) {
        if (l.data.count(e.model)) forcePublish[inst] = 1;
        l.apply(orc_lru_event_t{3, e.model, 0, 0}, ei, e.t, out);
        if (lts.erase(e.model)) dereg.push_back({e.model, inst});
      } else {
        Dec &d = D[e.dec];
        // limit the rate of cache churn (MM:3872-3884)
        if (orc_churn_reject(l.capacity, l.weightedSize, l.oldestTime, minSpace, minChurn, e.t)) { d.status = SIM_CHURN; continue; }
        const bool exists = l.data.count(e.model) != 0;
        l.apply(orc_lru_event_t{0, e.model, 1 /* INSERTION_WEIGHT MM:5011 */, e.lastUsed}, ei, e.t, out);
        if (exists) { d.status = SIM_EXISTS; handle_evictions(e); continue; }
        forcePublish[inst] = 1;
        handle_evictions(e);
        if (!l.data.count(e.model)) { d.status = SIM_FALLTHRU; continue; }  // MM:5145-5148
        if (orc_early_reject(std::abs(e.size), l.capacity, l.weightedSize, l.oldestTime, e.lastUsed)) {  // MM:5185-5190
          l.apply(orc_lru_event_t{3, e.model, 0, 0}, ei, e.t, out);  // ce.remove()
          d.status = SIM_EARLY;
          continue;
        }
        lts[e.model] = e.t;                                                   // mr.getInstanceIds().put(instanceId, ce.loadTimestamp) MM:5203
        d.status = SIM_ACCEPTED;
        l.apply(orc_lru_event_t{2, e.model, e.size, 0}, ei, e.t, out);       // updateWeight(initialWeight) MM:2100
        handle_evictions(e);
        if (!l.data.count(e.model)) d.status = SIM_GROW_EVICTED;            // "check whether we were evicted when growing" MM:2102-2106
      }
    }
  }
  // ---- phase D: registry ----
  for (auto &p : dereg) {
    auto &v = s->models[p.first].loaded;
    auto it = std::find(v.begin(), v.end(), p.second);
    if (it != v.end()) v.erase(it);
  }
  for (Dec &d : D)
    if (d.status == SIM_ACCEPTED) {
      const int32_t tgt = d.target == ORC_SELF ? d.self : d.target;
      auto &v = s->models[d.model].loaded;
      if (std::find(v.begin(), v.end(), tgt) == v.end()) v.push_back(tgt);
    }
  for (auto &u : used) if (u.second > s->models[u.first].lastUsed) s->models[u.first].lastUsed = u.second;  // MR:239-246
  s->carry.swap(nextCarry);
  // ---- phase E: republish (publishInstanceRecord MM:5390-5470) at now1 ----
  int32_t nPub = 0;
  for (int32_t inst = 0; inst < NI; inst++) {
    if ((size_t)inst >= f.byIdx.size() || !f.byIdx[inst]) continue;
    const IR &cur = *f.byIdx[inst];
    const Lru &l = *s->lru[inst];
    const int64_t lastDone = jsub(now1, s->lastPublished[inst]);
    const bool force = forcePublish[inst] != 0;
    bool publish = !(lastDone < 2000 || (!force && lastDone < 40000 - 1000));  // MM:5397-5400
    if (publish) {
      const bool old = lastDone > 4 * 40000;
      int64_t oldest = l.deque.empty() ? -1 : l.deque.front().lastUsed;  // runtimeCache.oldestTime()
      if (oldest == -1) oldest = INT64_MAX;
      const int32_t count = (int32_t)l.data.size();
      publish = publishNeeded(f.po, cur, old, now1, oldest, count, l.capacity, l.weightedSize, cur.lThreads, 0, cur.rpm, cur.shuttingDown);
      if (publish) {
        auto rec = std::make_shared<IR>(cur);
        rec->lruTime = oldest; rec->count = count; rec->capacity = l.capacity; rec->used = l.weightedSize; rec->lInProg = 0;
        rec->prohibitedTypes = nullptr;
        f.instanceEvent(1, inst, f.keyByIdx[inst], rec, now1);
        s->lastPublished[inst] = now1;
        nPub++;
      }
    }
  }
  // ---- reports ----
  if (n_dec_out) *n_dec_out = (int32_t)D.size();
  for (size_t k = 0; k < D.size() && (int32_t)k < dec_cap; k++)
    dec_out[k] = orc_sim_decision_t{D[k].model, D[k].self, D[k].target, D[k].ncand, D[k].status, D[k].event};
  if (n_evict_out) *n_evict_out = (int32_t)evs.size();
  for (size_t k = 0; k < evs.size() && (int32_t)k < evict_cap; k++) evict_out[k] = evs[k];
  if (rows_out)
    for (int32_t inst = 0; inst < NI; inst++) {
      orc_inst_t r{};
      if ((size_t)inst < f.byIdx.size() && f.byIdx[inst]) {
        const IR &ir = *f.byIdx[inst];
        r.lru_time = ir.lruTime; r.capacity = ir.capacity; r.used = ir.used; r.start_time = ir.startTime; r.vers = ir.vers;
        r.count = ir.count; r.l_threads = ir.lThreads; r.l_in_prog = ir.lInProg; r.rpm = ir.rpm; r.shutting_down = ir.shuttingDown;
        r.active = (size_t)inst < f.siActive.size() ? f.siActive[inst] : 0;
      }
      rows_out[inst] = r;
    }
  if (published_out) *published_out = nPub;
  return (int64_t)s->carry.size();
}

}  // extern "C"
