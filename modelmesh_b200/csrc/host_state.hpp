// host_state.hpp — host side of libmmplace: ingest tables, PLACEMENT_ORDER ranking, type-constraint set algebra and
// the rank-space snapshot that is uploaded to HBM at mmp_fleet_commit.  Pure C++17 (no CUDA) so that the same code is
// compiled into libmmplace.so by nvcc and into the CPU-only test harness (tests/emul) by g++.
//
// Formulation (DESIGN.md §3): PLACEMENT_ORDER (MM:4646-4703) does not depend on the model being placed, so the
// "scoring" of instances is done once per snapshot epoch: every live instance gets a dense rank, and every per-type /
// per-snapshot instance set becomes a bitmask over ranks.  A placement decision is then bitmask algebra plus
// find-first-set (= argmin under PLACEMENT_ORDER) over one row of the model x instance exclusion bitmap.
//
// Reference citations: MM = ModelMesh.java, IR = InstanceRecord.java, TCM = TypeConstraintManager.java,
// UT = UpgradeTracker.java (kserve/modelmesh @ ea13cdc5).
#pragma once
#include <algorithm>
#include <cerrno>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/mmplace.h"
#include "place_core.cuh"

namespace mmp {

typedef std::u16string JStr;  // java.lang.String ordering = UTF-16 code units

inline JStr utf8_to_utf16(const char *s) {
  JStr out;
  if (!s) return out;
  const unsigned char *p = (const unsigned char *)s;
  while (*p) {
    uint32_t cp;
    int len = (*p < 0x80) ? 1 : ((*p >> 5) == 6) ? 2 : ((*p >> 4) == 14) ? 3 : ((*p >> 3) == 30) ? 4 : 0;
    bool ok = len > 0;
    for (int i = 1; ok && i < len; i++) ok = (p[i] & 0xC0) == 0x80;
    if (!ok) { out.push_back(0xFFFD); p++; continue; }
    switch (len) {
      case 1: cp = p[0]; break;
      case 2: cp = ((p[0] & 0x1Fu) << 6) | (p[1] & 0x3Fu); break;
      case 3: cp = ((p[0] & 0x0Fu) << 12) | ((p[1] & 0x3Fu) << 6) | (p[2] & 0x3Fu); break;
      default: cp = ((p[0] & 0x07u) << 18) | ((p[1] & 0x3Fu) << 12) | ((p[2] & 0x3Fu) << 6) | (p[3] & 0x3Fu); break;
    }
    p += len;
    if (cp >= 0x10000) { cp -= 0x10000; out.push_back((char16_t)(0xD800 + (cp >> 10))); out.push_back((char16_t)(0xDC00 + (cp & 0x3FF))); }
    else out.push_back((char16_t)cp);
  }
  return out;
}

struct HostInstance {
  bool present = false;
  mmp_instance_row row{};
  JStr id, loc, zone;
  bool has_loc = false, has_zone = false;
  std::vector<JStr> labels;  // sorted, as IR:90-91
};

struct TypeConfig {  // TCM.ConfigTypeConstraints (TCM:79-98), normalised: sorted, de-duplicated, disjoint
  std::vector<JStr> required, preferred;
};

// Dense ranks of a set of strings under String.compareTo; absent (null) values rank last (Ordering.nullsLast, MM:4644)
inline void dense_string_ranks(const std::vector<const JStr *> &vals, std::vector<uint32_t> &out) {
  size_t n = vals.size();
  std::vector<uint32_t> ord(n);
  for (size_t i = 0; i < n; i++) ord[i] = (uint32_t)i;
  auto less = [&](uint32_t a, uint32_t b) {
    const JStr *x = vals[a], *y = vals[b];
    if (!x || !y) return x && !y;  // non-null before null
    return *x < *y;                // u16string operator< compares code units lexicographically, then length
  };
  std::sort(ord.begin(), ord.end(), less);
  out.assign(n, 0);
  uint32_t r = 0;
  for (size_t i = 0; i < n; i++) {
    if (i > 0 && (less(ord[i - 1], ord[i]))) r++;
    out[ord[i]] = r;
  }
}

// Everything mmp_fleet_commit derives on the host; plain vectors, uploaded verbatim.
struct HostSnapshot {
  int32_t n_ranks = 0, row_words = 0, n_slots = 0, any_rs = 0, order_not_total = 0;
  int32_t tc_enabled = 0;
  std::vector<RankRow> rows;          // [n_ranks]
  std::vector<int32_t> rank_of;       // [max_instances]
  std::vector<uint32_t> cand;         // [n_slots][row_words]
  std::vector<uint32_t> candx;        // [n_slots][row_words] cand & ~rs
  std::vector<uint32_t> pref;         // [n_slots][row_words]
  std::vector<uint8_t> has_pref;      // [n_slots]
  std::vector<uint8_t> allowed_null;  // [n_slots] (introspection only)
  std::vector<uint16_t> type_slot;    // [n_type_ids] type id -> mask slot
  std::vector<uint16_t> type_slot_hp; // [n_type_ids] slot | has_pref << 15: what the decision context reads (one gather instead of two)
  std::vector<uint32_t> rs, full;     // [row_words]
  std::vector<WordSumI> csum;         // [row_words]
  std::vector<WordSumL> lsum;         // [row_words]
  std::vector<int32_t> count_col;     // [row_words*32] count by rank, 0 past the last rank
  // instance sharding (SURVEY.md §8e): the row words this process holds and the stride of a stored row
  int32_t word_lo = 0, word_hi = 0, excl_stride = 0;
  std::vector<int32_t> candx_before;  // [n_slots] members of candx at ranks below word_lo*32 (entries that beat this shard)
  // compressed word lists (LaneTables, place_core.cuh): per slot the row words of [word_lo, word_hi) in which the candidate
  // mask the lane routine reads (candx when a replicaset is flagged, else cand) has any bit, ascending
  std::vector<uint16_t> nzw;          // [n_slots][row_words]
  std::vector<int32_t> nz_n;          // [n_slots]
  std::vector<uint16_t> nzw_full;     // instance-sharded fleets: the same lists over the WHOLE row (the peer-access path decides whole rows)
  std::vector<int32_t> nz_n_full;
  std::vector<int32_t> part_of_rank;  // [n_ranks] partition (PTS) id, 0 when no type constraints
  std::vector<std::vector<std::string>> part_types;  // prohibited type names per partition id
  std::vector<std::vector<int32_t>> part_type_ids;   // the same as type ids of THIS epoch (readers never touch the ingest-side name table)
  // instance columns for the stats / reaper kernels, by rank
  std::vector<int64_t> cap_col;
  std::vector<int32_t> lthreads_col, linprog_col;
  // dense string ranks of the tie-break chain (MM:4697-4700), by rank: kept for the device-side re-ranking of later,
  // non-structural commits (strings do not change between structural commits)
  std::vector<uint32_t> tie_id, tie_loc, tie_zone, tie_lab;
};

// One registration past a model's four inline edges, as the device tables hold it: sorted by (model, registration position),
// so the registrations 4, 5, ... of model m are the entries from the first one whose model is m on.
struct OvfEdge { int32_t model, inst; int64_t ts; };

class HostState {
 public:
  mmp_config cfg{};
  std::vector<HostInstance> inst;
  bool tc_enabled = false;                       // typeConstraints != null (TCM.get returned non-null)
  std::map<std::string, TypeConfig> tc_config;   // type name -> constraints; every mmp_types_set_json is a fresh load (all types "new", TCM:639-650)
  std::unordered_map<std::string, int32_t> type_ids;  // interned model-type names; ids start at 1
  std::vector<std::string> type_names;           // [id]
  std::set<JStr> replaced_rs;                    // likelyReplacedReplicaSets keys (UT:71)
  // model registry columns (MR:61-114).  Edges = loaded ∪ failed instance indices; 4 inline per model + overflow map.
  static constexpr int EDGE_INL = 4;
  std::vector<mmp_model_row> models;
  std::vector<int32_t> edge_inl;
  // MR.instanceIds / failedIn VALUES (load-start / failure time of each inline edge, MR:69,73) and MR.lastUnloadTime ("lul",
  // MR:113): read by the scale-up / scale-down arithmetic (loadedSince MM:5858-5870, MM:6265-6272) and the registry prune sweep
  // (MM:6752-6784).  0 = unknown.  Allocated on first use.
  std::vector<int64_t> edge_ts, model_lul;
  bool times_dirty = false;
  std::unordered_map<int32_t, std::vector<int32_t>> edge_ovf;
  std::unordered_map<int32_t, std::vector<int64_t>> edge_ovf_ts;  // the times of the overflow edges: same keys, same order
  int32_t n_models_used = 0;
  std::string err;
  // Instance ids -> indices, maintained by upsert/remove.  Model records ingested as JSON name instances BY ID (MR:69,73);
  // the ids are kept and resolved against this table at every commit, so the two KV listeners may deliver in any order.
  std::unordered_map<JStr, int32_t> id_index;
  std::unordered_map<int32_t, std::vector<JStr>> json_ids;  // model -> loaded ∪ failed ids as the record named them
  std::unordered_map<int32_t, std::vector<int64_t>> json_ts; // their map values (load-start / failure times), same order
  uint64_t inst_gen = 1, json_resolved_gen = 0;             // id table generation / the one the JSON models were last resolved against
  // ---- what changed since the last commit (mmp_fleet_commit picks its path from these) ----
  // structural: the set of live instances, their strings / labels / siMap membership, the type configuration or the
  // replicaset list changed -> string ranks, type masks and partitions are rebuilt on the host (build_snapshot).
  // Otherwise only numeric columns and model records changed: they are scattered into the device-resident tables and
  // the snapshot is re-ranked and rebuilt ON THE DEVICE (commit_kernels.cuh).
  bool structural_dirty = true;
  std::vector<int32_t> dirty_inst, dirty_models;
  std::vector<uint8_t> inst_dirty_flag, model_dirty_flag;
  bool all_models_dirty = true, ovf_dirty = true;
  void mark_inst(int32_t idx) { if (!inst_dirty_flag[idx]) { inst_dirty_flag[idx] = 1; dirty_inst.push_back(idx); } }
  void mark_model(int32_t m) {
    if (all_models_dirty) return;
    if (!model_dirty_flag[m]) { model_dirty_flag[m] = 1; dirty_models.push_back(m); }
    if (dirty_models.size() > models.size() / 8 + 1024) all_models_dirty = true;
  }
  void clear_dirty() {
    structural_dirty = false; all_models_dirty = false; ovf_dirty = false;
    for (int32_t i : dirty_inst) inst_dirty_flag[i] = 0;
    for (int32_t m : dirty_models) model_dirty_flag[m] = 0;
    dirty_inst.clear(); dirty_models.clear();
  }

  void init(const mmp_config &c) {
    cfg = c;
    inst.assign((size_t)c.max_instances, HostInstance());
    type_names.assign(1, std::string());
    models.assign((size_t)c.max_models, mmp_model_row{});
    edge_inl.assign((size_t)c.max_models * EDGE_INL, -1);
    inst_dirty_flag.assign((size_t)c.max_instances, 0);
    model_dirty_flag.assign((size_t)c.max_models, 0);
  }

  int32_t upsert_instance(int32_t idx, const mmp_instance_row *row, const char *id, const char *loc, const char *zone,
                          const char *const *labels, int32_t n_labels) {
    if (idx < 0 || idx >= cfg.max_instances || !row || !id || n_labels < 0) { err = "bad instance index or null argument"; return MMP_E_ARG; }
    if (const char *m = validate_row(*row)) { err = m; return MMP_E_ARG; }
    HostInstance &h = inst[idx];
    JStr nid = utf8_to_utf16(id);
    {  // anything but a change of the numeric columns is structural
      std::vector<JStr> nl;
      for (int32_t i = 0; i < n_labels; i++) nl.push_back(utf8_to_utf16(labels[i]));
      std::sort(nl.begin(), nl.end());
      if (!h.present || h.id != nid || h.has_loc != (loc != nullptr) || h.loc != utf8_to_utf16(loc) || h.has_zone != (zone != nullptr) ||
          h.zone != utf8_to_utf16(zone) || h.labels != nl || h.row.active != row->active || h.row.shutting_down != row->shutting_down)
        structural_dirty = true;
      else mark_inst(idx);
    }
    if (!h.present || h.id != nid) {  // the id table changes: models held by id are re-resolved at the next commit
      if (h.present) { auto it = id_index.find(h.id); if (it != id_index.end() && it->second == idx) id_index.erase(it); }
      id_index[nid] = idx;
      inst_gen++;
    }
    h.present = true;
    h.row = *row;
    h.id = std::move(nid);
    h.has_loc = loc != nullptr; h.loc = utf8_to_utf16(loc);
    h.has_zone = zone != nullptr; h.zone = utf8_to_utf16(zone);
    h.labels.clear();
    for (int32_t i = 0; i < n_labels; i++) h.labels.push_back(utf8_to_utf16(labels[i]));
    std::sort(h.labels.begin(), h.labels.end());  // IR:90-91 Arrays.sort(labels)
    return MMP_OK;
  }
  int32_t update_instance(int32_t idx, const mmp_instance_row *row) {
    if (idx < 0 || idx >= cfg.max_instances || !row || !inst[idx].present) { err = "instance not present"; return MMP_E_ARG; }
    if (const char *m = validate_row(*row)) { err = m; return MMP_E_ARG; }
    if (inst[idx].row.active != row->active || inst[idx].row.shutting_down != row->shutting_down) structural_dirty = true;
    else mark_inst(idx);
    inst[idx].row = *row;
    return MMP_OK;
  }
  int32_t remove_instance(int32_t idx) {
    if (idx < 0 || idx >= cfg.max_instances) { err = "bad instance index"; return MMP_E_ARG; }
    if (inst[idx].present) {
      auto it = id_index.find(inst[idx].id);
      if (it != id_index.end() && it->second == idx) id_index.erase(it);
      inst_gen++;
      structural_dirty = true;
    }
    inst[idx] = HostInstance();
    return MMP_OK;
  }
  int32_t set_model_times(int32_t m, const int64_t *ts, int32_t n, int64_t last_unload_time) {
    if (m < 0 || m >= cfg.max_models || n < 0 || (n > 0 && !ts)) { err = "bad model index or null argument"; return MMP_E_ARG; }
    if (edge_ts.empty()) { edge_ts.assign((size_t)cfg.max_models * EDGE_INL, 0); model_lul.assign((size_t)cfg.max_models, 0); }
    for (int i = 0; i < EDGE_INL; i++) edge_ts[(size_t)m * EDGE_INL + i] = i < n ? ts[i] : 0;
    auto ov = edge_ovf_ts.find(m);  // times past the registration count are ignored
    if (ov != edge_ovf_ts.end())
      for (size_t k = 0; k < ov->second.size(); k++) ov->second[k] = (int64_t)k + EDGE_INL < n ? ts[k + EDGE_INL] : 0;
    model_lul[m] = last_unload_time;
    times_dirty = true;
    return MMP_OK;
  }
  int32_t set_replicasets(const char *const *prefixes, int32_t n) {
    if (n < 0 || (n > 0 && !prefixes)) { err = "bad replicaset list"; return MMP_E_ARG; }
    replaced_rs.clear();
    for (int32_t i = 0; i < n; i++) replaced_rs.insert(utf8_to_utf16(prefixes[i]));
    structural_dirty = true;
    return MMP_OK;
  }
  int32_t set_model(int32_t m, const mmp_model_row *row, const int32_t *ids, int32_t n_ids, bool from_json = false) {
    if (m < 0 || m >= cfg.max_models || !row || n_ids < 0 || (n_ids > 0 && !ids)) { err = "bad model index or null argument"; return MMP_E_ARG; }
    if (!from_json && !json_ids.empty()) { json_ids.erase(m); json_ts.erase(m); }  // an index-based upsert replaces a record held by id
    if (row->type_id >= type_names.size()) { err = "unknown type_id (use mmp_type_id)"; return MMP_E_ARG; }
    for (int32_t i = 0; i < n_ids; i++)
      if (ids[i] < 0 || ids[i] >= cfg.max_instances) { err = "model instance id out of range"; return MMP_E_ARG; }
    models[m] = *row;
    models[m].reserved = (uint32_t)n_ids;  // library-private: size of the exclusion row (instance-shard early-out)
    for (int i = 0; i < EDGE_INL; i++) edge_inl[(size_t)m * EDGE_INL + i] = i < n_ids ? ids[i] : -1;
    // an overflow position keeps its time until the next set_model_times, as an inline one does (new positions read 0)
    if (n_ids > EDGE_INL) { edge_ovf[m].assign(ids + EDGE_INL, ids + n_ids); edge_ovf_ts[m].resize((size_t)(n_ids - EDGE_INL), 0); ovf_dirty = true; }
    else if (!edge_ovf.empty() && edge_ovf.erase(m)) { edge_ovf_ts.erase(m); ovf_dirty = true; }
    mark_model(m);
    if (m + 1 > n_models_used) n_models_used = m + 1;
    return MMP_OK;
  }
  void ovf_table(std::vector<OvfEdge> &out) const {
    std::vector<int32_t> keys;
    size_t n = 0;
    for (auto &kv : edge_ovf) { keys.push_back(kv.first); n += kv.second.size(); }
    std::sort(keys.begin(), keys.end());
    out.clear();
    out.reserve(n);
    for (int32_t m : keys) {
      const std::vector<int32_t> &e = edge_ovf.at(m);
      const std::vector<int64_t> &t = edge_ovf_ts.at(m);
      for (size_t k = 0; k < e.size(); k++) out.push_back(OvfEdge{m, e[k], t[k]});
    }
  }
  // Words per bitmap row, rounded up to 32 words so that every row starts on a 128-byte line and is a whole number
  // of 16-byte TMA units (10 000 instances -> 320 words = 1 280 B).
  int32_t row_words() const { return ((cfg.max_instances + 31) / 32 + 31) / 32 * 32; }

  // Resolve the instance ids of JSON-ingested model records against the current id table (commit time; the reference tests
  // membership by id at decision time, MM:4735-4743).  An id that names no present instance cannot be a candidate either.
  void resolve_json_models() {
    if (json_ids.empty() || json_resolved_gen == inst_gen) return;
    std::vector<int32_t> ids;
    std::vector<int64_t> ts;
    for (auto &kv : json_ids) {
      ids.clear(); ts.clear();
      auto tv = json_ts.find(kv.first);
      for (size_t q = 0; q < kv.second.size(); q++) {
        auto it = id_index.find(kv.second[q]);
        if (it != id_index.end() && std::find(ids.begin(), ids.end(), it->second) == ids.end()) {
          ids.push_back(it->second);
          ts.push_back(tv != json_ts.end() && q < tv->second.size() ? tv->second[q] : 0);
        }
      }
      const mmp_model_row row = models[kv.first];
      set_model(kv.first, &row, ids.data(), (int32_t)ids.size(), true);
      if (!edge_ts.empty()) set_model_times(kv.first, ts.data(), (int32_t)ts.size(), model_lul[kv.first]);
    }
    json_resolved_gen = inst_gen;
  }

  int32_t set_types_json(const char *json);  // defined after TcJson
  int32_t upsert_instance_json(int32_t idx, const char *id, const char *json, int32_t active);  // defined after RecordJson
  int32_t set_model_json(int32_t m, const char *json, int32_t size_units);

  static const char *validate_row(const mmp_instance_row &r) {
    if (r.lru_time < 0) return "lru_time must be >= 0 (Long.MAX_VALUE when empty)";
    if (r.rpm < 0 || r.rpm > 500000000) return "rpm outside [0, 5e8]";
    if (r.count < 0 || r.count > 1000000000) return "count outside [0, 1e9]";
    if (r.capacity < 0 || r.used < 0) return "capacity/used must be >= 0";
    return nullptr;
  }
  // A caller's own instance record as the walk reads it (quirk N2): `out` is set when the row passes validate_row, whose
  // message is returned otherwise.  Free space below zero reads as zero.
  static const char *fresh_row(const mmp_instance_row &r, FreshRow &out) {
    if (const char *m = validate_row(r)) return m;
    out = FreshRow{r.lru_time, std::max<int64_t>(0, r.capacity - r.used), r.count, r.rpm};
    return nullptr;
  }

  int32_t intern_type(const std::string &name) {
    auto it = type_ids.find(name);
    if (it != type_ids.end()) return it->second;
    if (type_names.size() >= 65535) return -1;
    int32_t id = (int32_t)type_names.size();
    type_names.push_back(name);
    type_ids[name] = id;
    structural_dirty = true;  // the type-id -> mask-slot table grows
    return id;
  }

  // TCM.sortAndDeduplicate (TCM:100-113)
  static std::vector<JStr> sort_dedupe(std::vector<JStr> v, const std::vector<JStr> *exclude) {
    std::sort(v.begin(), v.end());
    v.erase(std::unique(v.begin(), v.end()), v.end());
    if (exclude) {
      std::vector<JStr> o;
      for (auto &l : v)
        if (!std::binary_search(exclude->begin(), exclude->end(), l)) o.push_back(l);
      return o;
    }
    return v;
  }

  // ---- PLACEMENT_ORDER as a comparator over numeric columns + dense string ranks: OrderKey / compare_keys live in
  // place_core.cuh (shared with the device-side ranking of the fast commit path) ----
  typedef mmp::OrderKey OrderKey;
  static int compare_keys(const OrderKey &a, const OrderKey &b, int64_t churn2) { return mmp::compare_keys(a, b, churn2); }

  template <class Cmp>
  static void merge_sort(std::vector<int32_t> &v, Cmp less) {  // tolerant of a non-transitive comparator (N1)
    std::vector<int32_t> tmp(v.size());
    for (size_t w = 1; w < v.size(); w *= 2) {
      for (size_t lo = 0; lo < v.size(); lo += 2 * w) {
        size_t mid = std::min(lo + w, v.size()), hi = std::min(lo + 2 * w, v.size());
        size_t i = lo, j = mid, k = lo;
        while (i < mid && j < hi) tmp[k++] = less(v[j], v[i]) ? v[j++] : v[i++];
        while (i < mid) tmp[k++] = v[i++];
        while (j < hi) tmp[k++] = v[j++];
      }
      v.swap(tmp);
    }
  }

  // Build the rank-space snapshot.  Returns nullptr on success or an error message.
  const char *build_snapshot(HostSnapshot &s) const {
    const int32_t NI = cfg.max_instances;
    const int32_t RW = row_words();
    s = HostSnapshot();
    s.row_words = RW;
    s.tc_enabled = tc_enabled ? 1 : 0;
    // --- live set (present and not shutting down: MM:1462-1464 treats a shutting-down record as deleted) ---
    std::vector<int32_t> live;
    for (int32_t i = 0; i < NI; i++)
      if (inst[i].present && !inst[i].row.shutting_down) live.push_back(i);
    const int32_t n = (int32_t)live.size();
    s.n_ranks = n;

    // --- dense string ranks for the tie-break chain (MM:4697-4700) ---
    std::vector<const JStr *> ids(n), locs(n), zones(n);
    for (int32_t k = 0; k < n; k++) {
      const HostInstance &h = inst[live[k]];
      ids[k] = &h.id;
      locs[k] = h.has_loc ? &h.loc : nullptr;
      zones[k] = h.has_zone ? &h.zone : nullptr;
    }
    std::vector<uint32_t> id_r, loc_r, zone_r, lab_r(n);
    dense_string_ranks(ids, id_r);
    dense_string_ranks(locs, loc_r);
    dense_string_ranks(zones, zone_r);
    {  // labels under Utils.STRING_ARRAY_COMP (Utils.java:25-36): length first, then element-wise
      std::vector<uint32_t> ord(n);
      for (int32_t k = 0; k < n; k++) ord[k] = k;
      auto cmp = [&](uint32_t a, uint32_t b) {
        const auto &x = inst[live[a]].labels, &y = inst[live[b]].labels;
        if (x.size() != y.size()) return x.size() < y.size();
        for (size_t i = 0; i < x.size(); i++)
          if (x[i] != y[i]) return x[i] < y[i];
        return false;
      };
      std::sort(ord.begin(), ord.end(), cmp);
      uint32_t r = 0;
      for (int32_t k = 0; k < n; k++) {
        if (k > 0 && cmp(ord[k - 1], ord[k])) r++;
        lab_r[ord[k]] = r;
      }
    }
    std::vector<OrderKey> keys(n);
    bool any_saturated = false, mixed_vers = false;
    const int64_t churn2 = (int64_t)((uint64_t)cfg.min_churn_age_ms * 2u);
    for (int32_t k = 0; k < n; k++) {
      const mmp_instance_row &r = inst[live[k]].row;
      OrderKey &o = keys[k];
      o.vers = r.vers;
      o.rem = std::max<int64_t>(0, r.capacity - r.used);  // IR:203-205
      o.lru = r.lru_time;
      o.cap = r.capacity;
      o.count = r.count;
      o.free_threads = (int32_t)((uint32_t)r.l_threads - (uint32_t)r.l_in_prog);
      o.lip = r.l_in_prog;
      o.rpm = r.rpm;
      o.id_rank = id_r[k]; o.loc_rank = loc_r[k]; o.zone_rank = zone_r[k]; o.labels_rank = lab_r[k];
      o.full = o.rem < cfg.min_space_units;  // MM:4640-4642
      o.shutting_down = false;
      if (o.full && !(o.lru > churn2)) any_saturated = true;
      if (r.vers != inst[live[0]].row.vers) mixed_vers = true;
    }
    s.order_not_total = (any_saturated && mixed_vers) ? 1 : 0;  // N1: comparator may be non-transitive
    std::vector<int32_t> ord(n);
    for (int32_t k = 0; k < n; k++) ord[k] = k;
    merge_sort(ord, [&](int32_t a, int32_t b) { return compare_keys(keys[a], keys[b], churn2) < 0; });

    s.rows.resize(n);
    s.tie_id.resize(n); s.tie_loc.resize(n); s.tie_zone.resize(n); s.tie_lab.resize(n);
    s.rank_of.assign(NI, -1);
    s.cap_col.resize(n); s.lthreads_col.resize(n); s.linprog_col.resize(n);
    s.rs.assign(RW, 0); s.full.assign(RW, 0);
    s.csum.assign(RW, WordSumI{INT32_MAX, INT32_MIN});
    s.lsum.assign(RW, WordSumL{INT64_MAX, INT64_MIN});
    s.count_col.assign((size_t)RW * 32, 0);
    shard_words(RW, cfg.shard_rank, cfg.shard_count, s.word_lo, s.word_hi, s.excl_stride);
    s.any_rs = replaced_rs.empty() ? 0 : 1;
    for (int32_t r = 0; r < n; r++) {
      int32_t k = ord[r];
      int32_t idx = live[k];
      const HostInstance &h = inst[idx];
      RankRow &row = s.rows[r];
      row.lru = keys[k].lru; row.rem = keys[k].rem; row.count = h.row.count; row.rpm = h.row.rpm; row.idx = idx;
      row.flags = keys[k].full ? 1u : 0u;
      s.rank_of[idx] = r;
      s.tie_id[r] = keys[k].id_rank; s.tie_loc[r] = keys[k].loc_rank; s.tie_zone[r] = keys[k].zone_rank; s.tie_lab[r] = keys[k].labels_rank;
      s.cap_col[r] = h.row.capacity; s.lthreads_col[r] = h.row.l_threads; s.linprog_col[r] = h.row.l_in_prog;
      if (keys[k].full) s.full[r >> 5] |= 1u << (r & 31);
      // MM:4769-4770: iid.length() >= 7 and first six chars name a likely-replaced replicaset
      if (!replaced_rs.empty() && h.id.size() >= 7 && replaced_rs.count(h.id.substr(0, 6))) s.rs[r >> 5] |= 1u << (r & 31);
      s.count_col[r] = row.count;
      WordSumI &ci = s.csum[r >> 5];
      ci.lo = std::min(ci.lo, row.count); ci.hi = std::max(ci.hi, row.count);
      WordSumL &li = s.lsum[r >> 5];
      li.lo = std::min(li.lo, row.lru); li.hi = std::max(li.hi, row.lru);
    }

    // --- type-constraint set algebra (converged state of TCM.refreshPerTypeInstanceSets, TCM:680-747) ---
    build_type_masks(s, live);
    s.candx = s.cand;
    for (int32_t sl = 0; sl < s.n_slots; sl++)
      for (int32_t w = 0; w < RW; w++) s.candx[(size_t)sl * RW + w] &= ~s.rs[w];
    if (s.n_slots > 0x7fff) return "more than 32767 distinct type-constraint masks";
    s.type_slot_hp.resize(s.type_slot.size());
    for (size_t t = 0; t < s.type_slot.size(); t++)
      s.type_slot_hp[t] = (uint16_t)(s.type_slot[t] | (s.has_pref[s.type_slot[t]] ? 0x8000u : 0u));
    slot_word_lists(s, s.word_lo, s.word_hi, s.nzw, s.nz_n);
    if (cfg.shard_count > 1) slot_word_lists(s, 0, RW, s.nzw_full, s.nz_n_full);
    s.part_type_ids.assign(s.part_types.size(), {});
    for (size_t p = 0; p < s.part_types.size(); p++)
      for (const std::string &t : s.part_types[p]) {
        auto it = type_ids.find(t);
        if (it != type_ids.end()) s.part_type_ids[p].push_back(it->second);
      }
    s.candx_before.assign((size_t)s.n_slots, 0);
    for (int32_t sl = 0; sl < s.n_slots; sl++)
      for (int32_t w = 0; w < s.word_lo; w++) s.candx_before[sl] += __builtin_popcount(s.candx[(size_t)sl * RW + w]);
    return nullptr;
  }

  // Compressed word lists of s's candidate masks (the host side of k_slot_lists): per slot the row words of [lo, hi) in which
  // the mask the lane routine reads (candx when a replicaset is flagged, else cand) has any bit, ascending, then 0xffff
  static void slot_word_lists(const HostSnapshot &s, int32_t lo, int32_t hi, std::vector<uint16_t> &nzw, std::vector<int32_t> &nz_n) {
    const int32_t RW = s.row_words;
    nzw.assign((size_t)s.n_slots * RW, 0xffff);
    nz_n.assign((size_t)s.n_slots, 0);
    for (int32_t sl = 0; sl < s.n_slots; sl++) {
      const uint32_t *cx = (s.any_rs ? s.candx.data() : s.cand.data()) + (size_t)sl * RW;
      int32_t k = 0, skip = 0;
      for (int32_t w = lo; w < hi; w++)
        if (cx[w]) { nzw[(size_t)sl * RW + k++] = (uint16_t)w; if (w < lo + MMP_LANE_WIN) skip++; }
      nz_n[sl] = k | (skip << 24);  // (place_core.cuh nz_count / nz_skipped)
    }
  }

  // Contiguous rank ranges per instance shard, in whole 16-byte granules (TMA bulk copies): shard k of n holds row words
  // [lo, hi); a stored row is `stride` words (hi - lo rounded up to 4, at least 4).
  static void shard_words(int32_t row_words, int32_t rank, int32_t count, int32_t &lo, int32_t &hi, int32_t &stride) {
    if (count <= 1) { lo = 0; hi = row_words; stride = row_words; return; }
    const int32_t block = ((row_words + count - 1) / count + 3) / 4 * 4;
    lo = std::min(row_words, rank * block);
    hi = std::min(row_words, lo + block);
    stride = block;  // the same for every shard (a short or empty last shard is zero-padded): the row gather is a plain all-gather
  }

 private:
  // instanceMatches TCM:478-486 over sorted label vectors
  static bool instance_matches(const std::vector<JStr> &inst_labels, const std::vector<JStr> &type_labels, bool match_all) {
    if (inst_labels.empty() || type_labels.empty()) return false;
    for (auto &l : type_labels) {
      bool has = std::binary_search(inst_labels.begin(), inst_labels.end(), l);
      if (match_all && !has) return false;
      if (!match_all && has) return true;
    }
    return match_all;
  }

  struct Resolved {  // per configured type name, over ranks
    bool allowed_null = true, pref_null = true, cfg_pref_null = true;
    std::vector<uint8_t> allowed, pref, cfg_pref;
  };

  // inferPreferredInstances TCM:727-747
  static bool infer_preferred(const std::vector<int32_t> &scores, const std::vector<uint8_t> *include, std::vector<uint8_t> &out) {
    int32_t mn = INT32_MAX, mx = 0;
    out.assign(scores.size(), 0);
    for (size_t r = 0; r < scores.size(); r++) {
      if (include && !(*include)[r]) continue;
      int32_t sc = scores[r];
      if (sc < mn) mn = sc;
      if (sc >= mx) {
        if (sc > mx) { std::fill(out.begin(), out.end(), 0); mx = sc; }
        out[r] = 1;
      }
    }
    return mn < mx;  // false => null
  }

  void build_type_masks(HostSnapshot &s, const std::vector<int32_t> & /*live*/) const {
    const int32_t n = s.n_ranks, RW = s.row_words;
    const size_t n_type_ids = type_names.size();
    s.type_slot.assign(n_type_ids, 0);
    s.part_of_rank.assign(n, 0);
    s.part_types.clear();

    // active (siMap) mask applies to every slot (MM:4765)
    std::vector<uint32_t> active(RW, 0);
    for (int32_t r = 0; r < n; r++)
      if (inst[s.rows[r].idx].row.active) active[r >> 5] |= 1u << (r & 31);

    auto add_slot = [&](const std::vector<uint8_t> *allowed, const std::vector<uint8_t> *pref) -> uint16_t {
      std::vector<uint32_t> c(RW, 0), p(RW, 0);
      for (int32_t r = 0; r < n; r++) {
        if (!allowed || (*allowed)[r]) c[r >> 5] |= 1u << (r & 31);
        if (pref && (*pref)[r]) p[r >> 5] |= 1u << (r & 31);
      }
      for (int32_t w = 0; w < RW; w++) c[w] &= active[w];
      // de-duplicate identical slots
      for (int32_t sl = 0; sl < s.n_slots; sl++) {
        if (s.has_pref[sl] == (pref ? 1 : 0) && s.allowed_null[sl] == (allowed ? 0 : 1) &&
            !memcmp(&s.cand[(size_t)sl * RW], c.data(), RW * 4) && !memcmp(&s.pref[(size_t)sl * RW], p.data(), RW * 4))
          return (uint16_t)sl;
      }
      s.cand.insert(s.cand.end(), c.begin(), c.end());
      s.pref.insert(s.pref.end(), p.begin(), p.end());
      s.has_pref.push_back(pref ? 1 : 0);
      s.allowed_null.push_back(allowed ? 0 : 1);
      return (uint16_t)(s.n_slots++);
    };

    if (!tc_enabled) {
      uint16_t sl = add_slot(nullptr, nullptr);  // constrainTo == null, prefer == null (MM:4789, 4817)
      for (size_t t = 0; t < n_type_ids; t++) s.type_slot[t] = sl;
      s.part_types.push_back({});
      return;
    }
    // per configured type: allowed / configured-preferred sets via updateInstance semantics (TCM:455-468)
    std::map<std::string, Resolved> res;
    for (auto &e : tc_config) {
      Resolved R;
      const TypeConfig &tc = e.second;
      R.allowed_null = tc.required.empty();
      R.allowed.assign(n, 0); R.cfg_pref.assign(n, 0);
      bool any_pref = false;
      for (int32_t r = 0; r < n; r++) {
        const auto &labels = inst[s.rows[r].idx].labels;
        if (!R.allowed_null && instance_matches(labels, tc.required, true)) R.allowed[r] = 1;
        if (instance_matches(labels, tc.preferred, false)) { R.cfg_pref[r] = 1; any_pref = true; }
      }
      R.cfg_pref_null = !any_pref;
      res[e.first] = std::move(R);
    }
    // prohibited type sets (TCM:557-579): types whose required labels the instance does not satisfy
    std::map<std::vector<std::string>, int32_t> pts_ids;
    std::vector<int32_t> scores(n, 0);
    for (int32_t r = 0; r < n; r++) {
      std::vector<std::string> pts;
      for (auto &e : res)
        if (!e.second.allowed_null && !e.second.allowed[r]) pts.push_back(e.first);  // std::map iterates sorted
      auto it = pts_ids.find(pts);
      int32_t id;
      if (it == pts_ids.end()) { id = (int32_t)s.part_types.size(); pts_ids[pts] = id; s.part_types.push_back(pts); }
      else id = it->second;
      s.part_of_rank[r] = id;
      scores[r] = (int32_t)pts.size() * 4;  // TCM:686-688
    }
    if (s.part_types.empty()) s.part_types.push_back({});
    for (auto &e : res)
      if (!e.second.cfg_pref_null)
        for (int32_t r = 0; r < n; r++)
          if (e.second.cfg_pref[r]) scores[r] -= 1;  // TCM:689-698
    std::vector<uint8_t> def_pref;
    bool def_pref_nonnull = infer_preferred(scores, nullptr, def_pref);
    for (auto &e : res) {  // TCM:706-722
      Resolved &R = e.second;
      if (R.allowed_null) {
        R.pref_null = !def_pref_nonnull; R.pref = def_pref;  // N11
      } else {
        bool allowed_empty = true;
        for (int32_t r = 0; r < n; r++) if (R.allowed[r]) { allowed_empty = false; break; }
        if (!R.cfg_pref_null || allowed_empty) { R.pref_null = R.cfg_pref_null; R.pref = R.cfg_pref; }
        else { R.pref_null = !infer_preferred(scores, &R.allowed, R.pref); }
      }
    }
    // slots: id 0 and every interned name resolve through getTypeConstraints (TCM:258-262): own entry, else "_default"
    auto slot_for = [&](const std::string &name, bool named) -> uint16_t {
      const Resolved *R = nullptr;
      if (named) { auto it = res.find(name); if (it != res.end()) R = &it->second; }
      if (!R) { auto it = res.find("_default"); if (it != res.end()) R = &it->second; }
      if (R) return add_slot(R->allowed_null ? nullptr : &R->allowed, R->pref_null ? nullptr : &R->pref);
      return add_slot(nullptr, def_pref_nonnull ? &def_pref : nullptr);  // TCM:250: defaultPreferredInstances
    };
    s.type_slot[0] = slot_for(std::string(), false);
    for (size_t t = 1; t < n_type_ids; t++) s.type_slot[t] = slot_for(type_names[t], true);
  }
};

// ---- minimal JSON reader for the MM_TYPE_CONSTRAINTS document (object of objects of string arrays) ----
class TcJson {
 public:
  explicit TcJson(const char *s) : p_(s) {}
  // returns false on malformed input; unknown properties are ignored like jackson's FAIL_ON_UNKNOWN_PROPERTIES=false (TCM:72)
  bool parse(std::map<std::string, TypeConfig> &out, std::string &err) {
    ws();
    if (!eat('{')) { err = "expected '{'"; return false; }
    ws();
    if (eat('}')) return tail(err);
    for (;;) {
      std::string name;
      ws();
      if (!str(name)) { err = "expected type name"; return false; }
      ws();
      if (!eat(':')) { err = "expected ':'"; return false; }
      std::vector<JStr> req, pref;
      if (!type_obj(req, pref, err)) return false;
      TypeConfig tc;
      tc.required = HostState::sort_dedupe(req, nullptr);
      tc.preferred = HostState::sort_dedupe(pref, &tc.required);
      out[name] = tc;  // duplicate keys: last wins, as jackson
      ws();
      if (eat(',')) continue;
      if (eat('}')) return tail(err);
      err = "expected ',' or '}'";
      return false;
    }
  }

 protected:
  const char *p_;
  void ws() { while (*p_ == ' ' || *p_ == '\t' || *p_ == '\n' || *p_ == '\r') p_++; }
  bool eat(char c) { if (*p_ == c) { p_++; return true; } return false; }
  bool tail(std::string &err) { ws(); if (*p_) { err = "trailing characters"; return false; } return true; }
  static void put_utf8(std::string &o, uint32_t cp) {
    if (cp < 0x80) o.push_back((char)cp);
    else if (cp < 0x800) { o.push_back((char)(0xC0 | (cp >> 6))); o.push_back((char)(0x80 | (cp & 0x3F))); }
    else if (cp < 0x10000) { o.push_back((char)(0xE0 | (cp >> 12))); o.push_back((char)(0x80 | ((cp >> 6) & 0x3F))); o.push_back((char)(0x80 | (cp & 0x3F))); }
    else { o.push_back((char)(0xF0 | (cp >> 18))); o.push_back((char)(0x80 | ((cp >> 12) & 0x3F))); o.push_back((char)(0x80 | ((cp >> 6) & 0x3F))); o.push_back((char)(0x80 | (cp & 0x3F))); }
  }
  bool hex4(uint32_t &v) {
    v = 0;
    for (int i = 0; i < 4; i++) {
      char c = *p_++;
      v <<= 4;
      if (c >= '0' && c <= '9') v |= c - '0'; else if (c >= 'a' && c <= 'f') v |= c - 'a' + 10; else if (c >= 'A' && c <= 'F') v |= c - 'A' + 10; else return false;
    }
    return true;
  }
  bool str(std::string &o) {
    if (!eat('"')) return false;
    while (*p_ && *p_ != '"') {
      if (*p_ == '\\') {
        p_++;
        char c = *p_++;
        switch (c) {
          case '"': o.push_back('"'); break; case '\\': o.push_back('\\'); break; case '/': o.push_back('/'); break;
          case 'b': o.push_back('\b'); break; case 'f': o.push_back('\f'); break; case 'n': o.push_back('\n'); break;
          case 'r': o.push_back('\r'); break; case 't': o.push_back('\t'); break;
          case 'u': {
            uint32_t v;
            if (!hex4(v)) return false;
            if (v >= 0xD800 && v < 0xDC00 && p_[0] == '\\' && p_[1] == 'u') {
              p_ += 2; uint32_t lo; if (!hex4(lo)) return false;
              v = 0x10000 + ((v - 0xD800) << 10) + (lo - 0xDC00);
            }
            put_utf8(o, v);
            break;
          }
          default: return false;
        }
      } else o.push_back(*p_++);
    }
    return eat('"');
  }
  bool skip_value() {  // skip any JSON value (for unknown properties)
    ws();
    if (*p_ == '"') { std::string d; return str(d); }
    if (*p_ == '{' || *p_ == '[') {
      char open = *p_, close = open == '{' ? '}' : ']';
      p_++; ws();
      if (eat(close)) return true;
      for (;;) {
        if (open == '{') { std::string k; ws(); if (!str(k)) return false; ws(); if (!eat(':')) return false; }
        if (!skip_value()) return false;
        ws();
        if (eat(',')) continue;
        return eat(close);
      }
    }
    const char *q = p_;
    while (*p_ && *p_ != ',' && *p_ != '}' && *p_ != ']' && *p_ != ' ' && *p_ != '\n' && *p_ != '\t' && *p_ != '\r') p_++;
    return p_ != q;
  }
  bool str_array(std::vector<JStr> &out) {
    ws();
    if (!strncmp(p_, "null", 4)) { p_ += 4; return true; }
    if (!eat('[')) return false;
    ws();
    if (eat(']')) return true;
    for (;;) {
      std::string s8;
      ws();
      if (!str(s8)) return false;
      out.push_back(utf8_to_utf16(s8.c_str()));
      ws();
      if (eat(',')) continue;
      return eat(']');
    }
  }
  bool type_obj(std::vector<JStr> &req, std::vector<JStr> &pref, std::string &err) {
    ws();
    if (!eat('{')) { err = "expected '{' for type constraints"; return false; }
    ws();
    if (eat('}')) return true;
    for (;;) {
      std::string k;
      ws();
      if (!str(k)) { err = "expected property name"; return false; }
      ws();
      if (!eat(':')) { err = "expected ':'"; return false; }
      bool ok;
      if (k == "required") { req.clear(); ok = str_array(req); }
      else if (k == "preferred") { pref.clear(); ok = str_array(pref); }
      else ok = skip_value();
      if (!ok) { err = "bad value for property " + k; return false; }
      ws();
      if (eat(',')) continue;
      if (eat('}')) return true;
      err = "expected ',' or '}' in type constraints";
      return false;
    }
  }
};

// ---- KV-record codecs (SURVEY.md §8f-1): the registry keeps InstanceRecord / ModelRecord as jackson JSON; a host that
// watches the KV store can hand the bytes over as they are.  Unknown properties are ignored, absent ones keep the
// defaults of the record's jackson constructor (IR:76-78, MR:117-125). ----
class RecordJson : public TcJson {
 public:
  explicit RecordJson(const char *s) : TcJson(s) {}
  // InstanceRecord wire format (IR:37-69): lruTime count cap used lThreads lInProg rpm shutdown startTime vers loc zone labels
  bool instance(mmp_instance_row &row, std::string &loc, bool &has_loc, std::string &zone, bool &has_zone,
                std::vector<std::string> &labels, std::string &err) {
    memset(&row, 0, sizeof(row));
    has_loc = has_zone = false;
    labels.clear();
    return object([&](const std::string &k) -> bool {
      int64_t v = 0;
      if (k == "lruTime") { if (!integer(v)) return false; row.lru_time = v; }
      else if (k == "count") { if (!integer(v)) return false; row.count = (int32_t)v; }
      else if (k == "cap") { if (!integer(v)) return false; row.capacity = v; }
      else if (k == "used") { if (!integer(v)) return false; row.used = v; }
      else if (k == "lThreads") { if (!integer(v)) return false; row.l_threads = (int32_t)v; }
      else if (k == "lInProg") { if (!integer(v)) return false; row.l_in_prog = (int32_t)v; }
      else if (k == "rpm") { if (!integer(v)) return false; row.rpm = (int32_t)v; }
      else if (k == "shutdown") { bool b; if (!boolean(b)) return false; row.shutting_down = b ? 1 : 0; }
      else if (k == "startTime") { if (!integer(v)) return false; row.start_time = v; }
      else if (k == "vers") { if (!integer(v)) return false; row.vers = v; }
      else if (k == "loc") return nullable_string(loc, has_loc);
      else if (k == "zone") return nullable_string(zone, has_zone);
      else if (k == "labels") return string_list(labels);
      else return skip();
      return true;
    }, err);
  }
  // ModelRecord wire format (MR:61-114): type, instanceIds {iid: loadStart}, failedIn {iid: failTime}, lu; the rest is ignored
  bool model(std::string &type, std::vector<std::string> &loaded, std::vector<std::string> &failed, int64_t &last_used,
             std::string &err, std::vector<int64_t> *loaded_ts = nullptr, std::vector<int64_t> *failed_ts = nullptr,
             int64_t *last_unload = nullptr) {
    type.clear(); loaded.clear(); failed.clear(); last_used = 0;
    if (last_unload) *last_unload = 0;
    return object([&](const std::string &k) -> bool {
      bool has;
      if (k == "type") return nullable_string(type, has);
      if (k == "instanceIds") return key_list(loaded, loaded_ts);
      if (k == "failedIn") return key_list(failed, failed_ts);
      if (k == "lu") return integer(last_used);
      if (k == "lul" && last_unload) return integer(*last_unload);
      return skip();
    }, err);
  }

 private:
  template <class F> bool object(F &&field, std::string &err) {
    ws();
    if (!eat('{')) { err = "expected '{'"; return false; }
    ws();
    if (eat('}')) return tail(err);
    for (;;) {
      std::string k;
      ws();
      if (!str(k)) { err = "expected property name"; return false; }
      ws();
      if (!eat(':')) { err = "expected ':'"; return false; }
      ws();
      if (!field(k)) { err = "bad value for property " + k; return false; }
      ws();
      if (eat(',')) continue;
      if (eat('}')) return tail(err);
      err = "expected ',' or '}'";
      return false;
    }
  }
  bool skip() { return skip_value(); }
  bool integer(int64_t &v) {
    ws();
    char *end = nullptr;
    errno = 0;
    long long x = strtoll(p_, &end, 10);
    if (end == p_ || errno == ERANGE) return false;
    if (*end == '.' || *end == 'e' || *end == 'E') return false;  // jackson would coerce; the records never hold fractions
    p_ = end; v = (int64_t)x;
    return true;
  }
  bool boolean(bool &b) {
    ws();
    if (!strncmp(p_, "true", 4)) { p_ += 4; b = true; return true; }
    if (!strncmp(p_, "false", 5)) { p_ += 5; b = false; return true; }
    return false;
  }
  bool nullable_string(std::string &s, bool &has) {
    ws();
    if (!strncmp(p_, "null", 4)) { p_ += 4; has = false; s.clear(); return true; }
    s.clear(); has = true;
    return str(s);
  }
  bool string_list(std::vector<std::string> &out) {
    ws();
    if (!strncmp(p_, "null", 4)) { p_ += 4; return true; }
    if (!eat('[')) return false;
    ws();
    if (eat(']')) return true;
    for (;;) {
      std::string s8;
      ws();
      if (!str(s8)) return false;
      out.push_back(s8);
      ws();
      if (eat(',')) continue;
      return eat(']');
    }
  }
  bool key_list(std::vector<std::string> &keys, std::vector<int64_t> *vals = nullptr) {  // {"iid": 123, ...} -> the keys (and values)
    ws();
    if (!strncmp(p_, "null", 4)) { p_ += 4; return true; }
    if (!eat('{')) return false;
    ws();
    if (eat('}')) return true;
    for (;;) {
      std::string k;
      ws();
      if (!str(k)) return false;
      ws();
      if (!eat(':')) return false;
      ws();
      int64_t v = 0;
      const char *save = p_;
      if (!(vals && integer(v))) { p_ = save; v = 0; if (!skip_value()) return false; }
      if (vals) vals->push_back(v);
      keys.push_back(k);
      ws();
      if (eat(',')) continue;
      return eat('}');
    }
  }
};

inline int32_t HostState::upsert_instance_json(int32_t idx, const char *id, const char *json, int32_t active) {
  if (!json || !id) { err = "null argument"; return MMP_E_ARG; }
  mmp_instance_row row;
  std::string loc, zone, e;
  bool has_loc, has_zone;
  std::vector<std::string> labels;
  if (!RecordJson(json).instance(row, loc, has_loc, zone, has_zone, labels, e)) { err = "instance record json: " + e; return MMP_E_ARG; }
  row.active = active ? 1 : 0;
  std::vector<const char *> lp;
  for (auto &l : labels) lp.push_back(l.c_str());
  return upsert_instance(idx, &row, id, has_loc ? loc.c_str() : nullptr, has_zone ? zone.c_str() : nullptr, lp.data(), (int32_t)lp.size());
}

inline int32_t HostState::set_model_json(int32_t m, const char *json, int32_t size_units) {
  if (!json) { err = "null argument"; return MMP_E_ARG; }
  std::string type, e;
  std::vector<std::string> loaded, failed;
  int64_t lu = 0;
  std::vector<int64_t> lts, fts;
  int64_t lul = 0;
  if (!RecordJson(json).model(type, loaded, failed, lu, e, &lts, &fts, &lul)) { err = "model record json: " + e; return MMP_E_ARG; }
  // the ids are kept as the record names them and resolved against the id table now AND at every commit after the table
  // changed (resolve_json_models), so a model record may arrive before the records of the instances it names
  std::vector<JStr> raw;
  std::vector<int32_t> ids;
  std::vector<int64_t> ts, raw_ts;
  {
    size_t li = 0;
    for (const auto *lst : {&loaded, &failed}) {
      const std::vector<int64_t> &tv = lst == &loaded ? lts : fts;
      for (size_t q = 0; q < lst->size(); q++, li++) {
        JStr j = utf8_to_utf16((*lst)[q].c_str());
        if (std::find(raw.begin(), raw.end(), j) != raw.end()) continue;
        auto it = id_index.find(j);
        if (it != id_index.end() && std::find(ids.begin(), ids.end(), it->second) == ids.end()) { ids.push_back(it->second); ts.push_back(q < tv.size() ? tv[q] : 0); }
        raw.push_back(std::move(j));
        raw_ts.push_back(q < tv.size() ? tv[q] : 0);
      }
    }
  }
  mmp_model_row row{};
  row.last_used = lu;
  row.size_units = size_units;
  // a record without "type" is built by the jackson constructor with DEFAULT_TYPE (MR:117-130)
  const int32_t tid = intern_type(type.empty() ? std::string("NLCLASSIFIER") : type);
  if (tid < 0) { err = "more than 65534 model types"; return MMP_E_ARG; }
  row.type_id = (uint16_t)tid;
  row.copy_count = (uint8_t)std::min<size_t>(255, loaded.size());
  row.fail_count = (uint8_t)std::min<size_t>(255, failed.size());
  const int32_t rc = set_model(m, &row, ids.data(), (int32_t)ids.size(), true);
  if (rc == MMP_OK) {
    if (raw.empty()) { json_ids.erase(m); json_ts.erase(m); } else { json_ids[m] = std::move(raw); json_ts[m] = std::move(raw_ts); }
    bool any_time = lul != 0;
    for (int64_t t : ts) any_time = any_time || t != 0;
    if (any_time || !edge_ts.empty()) set_model_times(m, ts.data(), (int32_t)ts.size(), lul);
  }
  return rc;
}

inline int32_t HostState::set_types_json(const char *json) {
  if (!json || !*json) { tc_enabled = false; tc_config.clear(); structural_dirty = true; return MMP_OK; }
  std::map<std::string, TypeConfig> cfgmap;
  std::string e;
  if (!TcJson(json).parse(cfgmap, e)) { err = "type constraints json: " + e; return MMP_E_ARG; }
  tc_enabled = true;
  structural_dirty = true;
  tc_config.swap(cfgmap);
  for (auto &t : tc_config) intern_type(t.first);
  return MMP_OK;
}

}  // namespace mmp
