// tests/emul/emul.cpp — CPU-ONLY TEST HARNESS.  Not part of the product and never loaded by modelmesh_b200/.
//
// It compiles the product's host-side snapshot builder (csrc/host_state.hpp) and the rank-space decision routine
// (csrc/place_core.cuh, single-lane Coop1 shape) with g++ and exposes them under the same mmp_* entry points as
// libmmplace.so, so that the `-m "not gpu"` tests can check the bitmask formulation, the PLACEMENT_ORDER ranking, the
// type-constraint masks and the JSON reader against the oracle on a box with no GPU.  The CUDA library differs from
// this harness only in the cooperative shape (Coop32: shuffles/ballots, vector loads) and in where the arrays live.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../modelmesh_b200/csrc/host_state.hpp"

using namespace mmp;

struct mmp_fleet {
  HostState hs;
  HostSnapshot snap;
  std::vector<uint32_t> excl;
  std::vector<mmp_model_row> models;
  int32_t epoch = 0;
  int64_t launches = 0;
  uint64_t id_base = 0;      // mmp_fleet_set_id_base
  uint64_t *keys = nullptr;  // harness-only: per-decision instance-shard keys of the next batch (mmp_emul_set_keys)
};
static thread_local std::string g_err;
static int g_window = 32;  // fast-path window width under test (32: warp tile, 16: half-warp tile); 1: lane-per-decision shape
static int g_lane_budget = 48;  // CoopLane walk budget (row words) when g_window == 1
static int g_lane_global = 1;  // decide_stream: steps beyond the window may read the row itself (the kernel's second chance: L2)
static int g_lane_window = MMP_LANE_WIN;  // decide_stream: row words available to a lane (LANE_WIN of k_place_lanes: the window copied out of the landing stage)
static long g_bails = 0, g_lane_decisions = 0;

extern "C" {

int32_t mmp_abi_version(void) { return MMP_ABI_VERSION; }
void mmp_emul_set_window(int w) { g_window = (w == 16 || w == 8 || w == 1 || w == 2) ? w : 32; }  // harness-only entry points
void mmp_emul_set_lane_budget(int words) { g_lane_budget = words; }
void mmp_emul_set_lane_window(int words) { g_lane_window = words; }
void mmp_emul_set_lane_global(int on) { g_lane_global = on; }
void mmp_emul_set_keys(mmp_fleet *f, uint64_t *keys) { f->keys = keys; }
void mmp_emul_key_decode(uint64_t k, int32_t *target, int32_t *n_candidates, int32_t *open) {
  shard_key_decode(k, *target, *n_candidates);
  *open = shard_key_open(k) ? 1 : 0;
}
long mmp_emul_lane_bails(long *decisions) { long b = g_bails; if (decisions) *decisions = g_lane_decisions; g_bails = g_lane_decisions = 0; return b; }
const char *mmp_last_error(mmp_fleet *) { return g_err.c_str(); }

int32_t mmp_fleet_create(const mmp_config *cfg, mmp_fleet **out) {
  if (!cfg || !out || cfg->max_instances <= 0 || cfg->max_instances > 65536 || cfg->max_models <= 0) { g_err = "bad config"; return MMP_E_ARG; }
  if (cfg->shard_count < 1 || cfg->shard_rank < 0 || cfg->shard_rank >= cfg->shard_count) { g_err = "bad shard_rank/shard_count"; return MMP_E_ARG; }
  auto *f = new mmp_fleet();
  f->hs.init(*cfg);
  *out = f;
  return MMP_OK;
}
void mmp_fleet_destroy(mmp_fleet *f) { delete f; }

#define FWD(call) do { int32_t rc_ = (call); if (rc_ < 0) g_err = f->hs.err; return rc_; } while (0)
int32_t mmp_instance_upsert(mmp_fleet *f, int32_t idx, const mmp_instance_row *row, const char *id, const char *loc,
                            const char *zone, const char *const *labels, int32_t n_labels) {
  FWD(f->hs.upsert_instance(idx, row, id, loc, zone, labels, n_labels));
}
int32_t mmp_instance_update(mmp_fleet *f, int32_t idx, const mmp_instance_row *row) { FWD(f->hs.update_instance(idx, row)); }
int32_t mmp_instance_upsert_json(mmp_fleet *f, int32_t idx, const char *id, const char *json, int32_t active) { FWD(f->hs.upsert_instance_json(idx, id, json, active)); }
int32_t mmp_model_upsert_json(mmp_fleet *f, int32_t m, const char *json, int32_t size_units) { FWD(f->hs.set_model_json(m, json, size_units)); }
int32_t mmp_instance_remove(mmp_fleet *f, int32_t idx) { FWD(f->hs.remove_instance(idx)); }
int32_t mmp_types_set_json(mmp_fleet *f, const char *json) { FWD(f->hs.set_types_json(json)); }
int32_t mmp_type_id(mmp_fleet *f, const char *name) {
  if (!name) return MMP_E_ARG;
  int32_t id = f->hs.intern_type(name);
  if (id < 0) { g_err = "too many types"; return MMP_E_ARG; }
  return id;
}
int32_t mmp_replicasets_set(mmp_fleet *f, const char *const *p, int32_t n) { FWD(f->hs.set_replicasets(p, n)); }
int32_t mmp_model_upsert(mmp_fleet *f, int32_t m, const mmp_model_row *row, const int32_t *ids, int32_t n) { FWD(f->hs.set_model(m, row, ids, n)); }
int32_t mmp_models_bulk(mmp_fleet *f, int32_t first, int32_t n, const mmp_model_row *rows, const int64_t *off, const int32_t *e) {
  for (int32_t i = 0; i < n; i++) {
    int32_t rc = f->hs.set_model(first + i, &rows[i], e + off[i], (int32_t)(off[i + 1] - off[i]));
    if (rc < 0) { g_err = f->hs.err; return rc; }
  }
  return MMP_OK;
}

int32_t mmp_fleet_commit(mmp_fleet *f) {
  f->hs.resolve_json_models();
  if (const char *m = f->hs.build_snapshot(f->snap)) { g_err = m; return MMP_E_ARG; }
  const int RW = f->snap.row_words;
  const int32_t nm = f->hs.n_models_used;
  f->models.assign(f->hs.models.begin(), f->hs.models.begin() + nm);
  const int32_t WS = f->snap.word_lo, WE = f->snap.word_hi, ST = f->snap.excl_stride;
  (void)RW;
  f->excl.assign((size_t)nm * ST, 0u);
  auto setbit = [&](int32_t m, int32_t inst) {
    int32_t r = f->snap.rank_of[inst];
    if (r >= 0 && (r >> 5) >= WS && (r >> 5) < WE) f->excl[(size_t)m * ST + ((r >> 5) - WS)] |= 1u << (r & 31);
  };
  for (int32_t m = 0; m < nm; m++)
    for (int i = 0; i < HostState::EDGE_INL; i++) {
      int32_t e = f->hs.edge_inl[(size_t)m * HostState::EDGE_INL + i];
      if (e >= 0) setbit(m, e);
    }
  for (auto &kv : f->hs.edge_ovf)
    for (int32_t e : kv.second) setbit(kv.first, e);
  return ++f->epoch;
}

static SnapshotView make_view(mmp_fleet *f) {
  SnapshotView v{};
  const HostSnapshot &s = f->snap;
  v.n_ranks = s.n_ranks; v.row_words = s.row_words; v.n_models = (int32_t)f->models.size(); v.max_instances = f->hs.cfg.max_instances;
  v.any_rs = s.any_rs; v.n_type_ids = (int32_t)s.type_slot.size(); v.min_space = f->hs.cfg.min_space_units;
  v.word_lo = s.word_lo; v.word_hi = s.word_hi; v.excl_stride = s.excl_stride; v.n_slots = s.n_slots;
  v.count_col = s.count_col.data(); v.cand_before = s.candx_before.data();
  v.excl = f->excl.data(); v.cand = s.cand.data(); v.candx = s.candx.data(); v.pref = s.pref.data(); v.has_pref = s.has_pref.data();
  v.type_slot = s.type_slot_hp.data(); v.full = s.full.data(); v.rows = s.rows.data();
  v.rank_of = s.rank_of.data(); v.csum = s.csum.data(); v.lsum = s.lsum.data(); v.models = f->models.data();
  v.nzw = s.nzw.data(); v.nz_n = s.nz_n.data();
  return v;
}

int32_t mmp_place_batch_trace(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                              const int32_t *extra, int32_t n_extra, mmp_decision_out *out, mmp_decision_trace *trace,
                              uint32_t *cand_mask, int64_t now_ms, uint64_t seed) {
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  SnapshotView v = make_view(f);
  v.n_extra = n_extra;
  std::vector<FreshRow> fr((size_t)(n_fresh > 0 ? n_fresh : 0));
  for (int32_t i = 0; i < n_fresh; i++)
    if (const char *m = HostState::fresh_row(fresh[i], fr[i])) { g_err = m; return MMP_E_ARG; }
  Coop1 co;
  CoopHost<16> co16;
  CoopHost<8> co8;
  const int win = g_window;
  for (int32_t i = 0; i < n; i++) {
    DecideOut o;
    DecisionCtx cx;
    prepare_ctx(v, in[i], fr.data(), n_fresh, extra, cx);
    const uint32_t *erow = v.excl + (size_t)(cx.slot >= 0 ? in[i].model : 0) * v.excl_stride;
    const bool sharded = v.word_lo != 0 || v.word_hi != v.row_words;
    bool done = false;
    if (sharded && !cand_mask && cx.slot >= 0 && shard_cannot_win(v, cx, f->models[in[i].model].reserved)) {
      // a lower shard holds an entry: this shard publishes "none" without looking at its row (as k_place_lanes does)
      o = DecideOut(); o.target = MMP_TARGET_NONE; o.first_rank = -1; o.best = -1; o.best_rank = -1; o.cut_rank = (int32_t)NONE_RANK;
      done = true;
    } else
    if (win == 2 && !cand_mask) {  // the lockstep lane routine of k_place_lanes (one decision per lane), general routine when it declines
      uint32_t self_eword = 0;
      if (cx.self_rank >= 0 && (cx.self_rank >> 5) >= v.word_lo && (cx.self_rank >> 5) < v.word_hi) self_eword = erow[(cx.self_rank >> 5) - v.word_lo];
      // the lane sees a COPY of exactly the window (as k_place_lanes gives it): the first ww words of the stored row; an
      // over-read is a heap overflow under ASAN
      LaneTables T = lane_tables_global(v, cx.slot >= 0 ? ctx_slot(cx) : 0);
      const uint32_t ww = (uint32_t)std::min<int64_t>(g_lane_window, (int64_t)(v.word_hi - v.word_lo));
      std::vector<uint32_t> window(erow, erow + ww);
      T.nz_skip = 0;  // list entries inside THIS window (k_place_lanes uses the count stored for its MMP_LANE_WIN words)
      while (T.nz_skip < T.nz_n && (uint32_t)T.nzw[T.nz_skip] < (uint32_t)v.word_lo + ww) T.nz_skip++;
      done = decide_stream(v, T, T, cx, true, window.data(), ww, RowPtr{g_lane_global ? erow : nullptr, (uint32_t)v.word_lo}, self_eword, now_ms, seed,
                           pick_id(in[i], f->id_base + (uint64_t)i), SoloVote(), o, g_lane_budget);
      g_lane_decisions++;
      if (!done) g_bails++;
    } else if (sharded) {
      // instance-sharded harness: only the general routine knows about rank ranges (decide_fast assumes whole rows)
    } else if (win == 1 && !cand_mask) {  // the lane-per-decision shape of k_place_lanes: budgeted walk, cooperative redo when it bails
      CoopLane cl(g_lane_budget);
      decide_ctx<CoopLane>(v, cx, erow, extra, now_ms, seed, pick_id(in[i], f->id_base + (uint64_t)i), cl, o, nullptr);
      g_lane_decisions++;
      done = !(o.flags & MMP_TF_BAIL);
      if (!done) g_bails++;
    } else if (!cand_mask) done = win == 16 ? decide_fast<true>(v, cx, erow, now_ms, seed, pick_id(in[i], f->id_base + (uint64_t)i), co16, o)
                         : win == 8 ? decide_fast<true>(v, cx, erow, now_ms, seed, pick_id(in[i], f->id_base + (uint64_t)i), co8, o)
                                    : decide_fast<true>(v, cx, erow, now_ms, seed, pick_id(in[i], f->id_base + (uint64_t)i), co, o);
    if (!done)
      decide_ctx<Coop1>(v, cx, erow, extra, now_ms, seed, pick_id(in[i], f->id_base + (uint64_t)i), co, o,
                        cand_mask ? cand_mask + (size_t)i * 2 * v.row_words : nullptr);
    out[i].target = o.target; out[i].n_candidates = o.n_candidates;
    if (f->keys) f->keys[i] = shard_key(o, f->hs.cfg.shard_rank);
    if (trace) {
      trace[i].best = o.best; trace[i].n_remaining = o.n_remaining; trace[i].pick_index = o.pick_index; trace[i].flags = o.flags;
      trace[i].cut_rank = o.cut_rank; trace[i].best_rank = o.best_rank; trace[i].reserved[0] = trace[i].reserved[1] = 0;
    }
  }
  f->launches++;
  return MMP_OK;
}
int32_t mmp_place_batch(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                        const int32_t *extra, int32_t n_extra, mmp_decision_out *out, int64_t now_ms, uint64_t seed) {
  return mmp_place_batch_trace(f, in, n, fresh, n_fresh, extra, n_extra, out, nullptr, nullptr, now_ms, seed);
}

int32_t mmp_place_sweep(mmp_fleet *f, int32_t first_model, int32_t n, const int32_t *self, int32_t self_stride,
                        const uint32_t *favour_bits, mmp_decision_out *out, int64_t now_ms, uint64_t seed) {
  if (n < 0 || first_model < 0 || (n > 0 && (!self || !out)) || (self_stride != 0 && self_stride != 1)) { g_err = "bad argument"; return MMP_E_ARG; }
  if ((int64_t)first_model + n > (int64_t)f->models.size()) { g_err = "sweep runs past the registry"; return MMP_E_ARG; }
  std::vector<mmp_decision_in> d((size_t)n);
  for (int32_t i = 0; i < n; i++) {
    d[i].model = first_model + i; d[i].self = self[(size_t)i * self_stride]; d[i].last_used = 0;
    d[i].flags = MMP_DF_MODEL_LAST_USED | ((favour_bits && ((favour_bits[i >> 5] >> (i & 31)) & 1u)) ? MMP_DF_FAVOUR_SELF : 0u);
    d[i].fresh = -1; d[i].extra_off = 0; d[i].extra_n = 0;
  }
  return mmp_place_batch(f, d.data(), n, nullptr, 0, nullptr, 0, out, now_ms, seed);
}

int32_t mmp_row_words(mmp_fleet *f) { return f->hs.row_words(); }
int32_t mmp_live_instances(mmp_fleet *f) { return f->snap.n_ranks; }
int32_t mmp_cluster_order(mmp_fleet *f, int32_t *out_idx, int32_t cap) {
  for (int32_t r = 0; r < f->snap.n_ranks && r < cap; r++) out_idx[r] = f->snap.rows[r].idx;
  return f->snap.n_ranks;
}
int32_t mmp_type_sets(mmp_fleet *f, int32_t type_id, int32_t n_idx, uint8_t *allowed, int32_t *allowed_null, uint8_t *preferred,
                      int32_t *preferred_null) {
  const HostSnapshot &s = f->snap;
  if (type_id < 0 || type_id > 65535) { g_err = "bad type id"; return MMP_E_ARG; }
  // a name interned after this snapshot was committed had no configuration in it: it resolves like id 0
  int sl = s.type_slot[type_id < (int32_t)s.type_slot.size() ? type_id : 0];
  *allowed_null = s.allowed_null[sl]; *preferred_null = !s.has_pref[sl];
  for (int32_t i = 0; i < n_idx; i++) {
    int32_t r = i < (int32_t)s.rank_of.size() ? s.rank_of[i] : -1;
    // NB the candidate mask also folds in the siMap "active" bit (MM:4765)
    allowed[i] = (r >= 0 && !s.allowed_null[sl]) ? (s.cand[(size_t)sl * s.row_words + (r >> 5)] >> (r & 31)) & 1u : 0;
    preferred[i] = (r >= 0) ? (s.pref[(size_t)sl * s.row_words + (r >> 5)] >> (r & 31)) & 1u : 0;
  }
  return MMP_OK;
}
int32_t mmp_instance_partition(mmp_fleet *f, int32_t idx) {
  if (idx < 0 || idx >= (int32_t)f->snap.rank_of.size() || f->snap.rank_of[idx] < 0) return -1;
  return f->snap.part_of_rank[f->snap.rank_of[idx]];
}
int64_t mmp_kernel_launches(mmp_fleet *f) { return f->launches; }
int32_t mmp_fleet_set_id_base(mmp_fleet *f, uint64_t b) { f->id_base = b; return MMP_OK; }

}  // extern "C"
