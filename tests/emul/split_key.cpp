// tests/emul/split_key.cpp — CPU-ONLY TEST HARNESS for the per-model entry k_place_split reads.  Not part of the product.
//
// The split_place harness (included whole: the tests/emul fleet, the excluded-rank lists, the slot summaries) plus one
// entry point that answers every decision of a batch twice: by split_answer on the model's SplitKey, built here with
// make_split_key as k_build_bitmap / k_build_bitmap_ovf build it, and by the rule the kernel applied before it read the
// entry, restated below on the model row (CtxA) and the model's excluded ranks (RowRanks).  The two must agree.
#include "split_place.cpp"

namespace {
// k_build_bitmap / k_build_bitmap_ovf: every model's SplitKey from its row, the ranks of its inline edges and the type
// slots, SPLIT_KEY_OVF for a model with overflow pairs
std::vector<SplitKey> build_split_keys(const mmp_fleet *f, const SnapshotView &v) {
  const int32_t nm = (int32_t)f->models.size();
  std::vector<SplitKey> k((size_t)std::max(nm, 1));
  for (int32_t m = 0; m < nm; m++) {
    int32_t rs[4] = {-1, -1, -1, -1};
    for (int i = 0; i < HostState::EDGE_INL; i++) {
      const int32_t e = f->hs.edge_inl[(size_t)m * HostState::EDGE_INL + i];
      if (e >= 0) rs[i] = f->snap.rank_of[e];
    }
    k[(size_t)m] = make_split_key(f->models[(size_t)m], rs, v.type_slot, v.n_type_ids);
  }
  for (auto &kv : f->hs.edge_ovf)
    if (!kv.second.empty() && kv.first < nm) k[(size_t)kv.first].slot |= SPLIT_KEY_OVF;
  return k;
}
// what k_place_split does with a decision: its validity from the record, then rank_of[self] and its model's SplitKey
bool split_answer_keyed(const SnapshotView &v, const mmp_decision_in &d, const FreshRow *fresh, int32_t n_fresh, const SlotSummary *sums,
                        const int32_t *members, int64_t now_ms, uint64_t seed, uint64_t decision_id, mmp_decision_out &r, SplitKey &k) {
  const int32_t ok = decision_ok(v, d);
  k.last_used = 0; k.min_rank = INT32_MAX; k.slot = 0;
  if (ok && !request_model(d)) k = load_split_key(v.split_key + d.model);
  const int32_t self_rank = ok ? v.rank_of[d.self] : -1;
  return split_answer(v, d, ok, self_rank, k, fresh, n_fresh, sums, members, now_ms, seed, decision_id, r);
}
// The rule k_place_split applied before it read SplitKey, restated from the model row (CtxA) and its excluded ranks
// (RowRanks): the reference the keyed rule is compared against
bool split_answer_rows(const SnapshotView &s, const mmp_decision_in &d, const CtxA &a, const RowRanks &row, const FreshRow *fresh,
                       int32_t n_fresh, const SlotSummary *sums, const int32_t *members, int64_t now, uint64_t seed,
                       uint64_t decision_id, mmp_decision_out &out) {
  if (!a.ok || request_model(d) || d.extra_n != 0 || row.overflow()) return false;
  FreshRow fr;
  if (d.fresh >= 0 && d.fresh < n_fresh) fr = fresh[d.fresh];
  else if (a.self_rank >= 0) { const RankRow sr = load_row(s.rows + a.self_rank); fr.lru = sr.lru; fr.rem = sr.rem; fr.count = sr.count; fr.rpm = 0; }
  else return false;
  const int slot = (int)slot_key(s, a.mr.type_id);
  const SlotSummary &sm = sums[slot];
  int cs;
  if (sm.best_full) {
    const int64_t a10 = age_of(sm.best_lru, now) / 10, df = jsub(fr.lru, sm.best_lru);
    cs = df > 45000 && df > a10;
  } else cs = fr.rem < s.min_space || fr.rem < (sm.best_rem >> 2);
  const int32_t reach = sm.reach[cs];
  if (reach < 0 || (a.self_rank >= 0 && a.self_rank < reach)) return false;
  for (int j = 0; j < 4; j++) if (row.r[j] >= 0 && row.r[j] < reach) return false;
  const int32_t n_in = sm.n_in[cs];
  const int64_t last_used = (d.flags & MMP_DF_MODEL_LAST_USED) ? a.mr.last_used : d.last_used;
  const PickOut pk = pick_survivor(n_in, false, sm.best_rpm, fr.rpm, sm.best_rpm, last_used, now, seed, decision_id);
  if (pk.kind == PICK_SELF) return false;
  const int32_t cidx = pk.kind == PICK_BEST ? sm.best_idx : members[((size_t)slot * 2 + (size_t)cs) * SPLIT_CAP + pk.kth];
  out.target = target_of(cidx, d);
  out.n_candidates = 1 + n_in;
  return true;
}
}  // namespace

extern "C" {
// The keyed rule (split_answer on SplitKey) against the rule it replaced (split_answer_rows on the model row and its
// excluded ranks), decision by decision; request-model decisions take the fleet's zero row, as on an unsharded fleet.
// counts (5 entries): decisions, answered by the row rule, answered by the keyed rule, decisions whose verdicts differ,
// answered decisions whose outputs differ.
int32_t mmp_emul_split_key_rule(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                                int32_t n_extra, int64_t now_ms, uint64_t seed, int64_t *counts) {
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  SnapshotView v = make_view(f);
  const std::vector<uint32_t> zero((size_t)v.excl_stride, 0u);
  v.zero_row = zero.data();
  const std::vector<int32_t> ranks = build_excl_ranks(f);
  v.excl_ranks = ranks.data();
  const std::vector<SplitKey> keys = build_split_keys(f, v);
  v.split_key = keys.data();
  v.n_extra = n_extra;
  std::vector<FreshRow> fr((size_t)(n_fresh > 0 ? n_fresh : 0));
  for (int32_t i = 0; i < n_fresh; i++)
    if (const char *m = HostState::fresh_row(fresh[i], fr[i])) { g_err = m; return MMP_E_ARG; }
  std::vector<SlotSummary> sums;
  std::vector<int32_t> members;
  build_summaries(v, now_ms, sums, members);
  for (int j = 0; j < 5; j++) counts[j] = 0;
  for (int32_t i = 0; i < n; i++) {
    const mmp_decision_in &d = in[i];
    const uint64_t id = pick_id(d, f->id_base + (uint64_t)i);
    const int32_t m = excl_row_id(v, d.model, d.flags);
    RowRanks row;
    row.r[0] = row.r[1] = row.r[2] = row.r[3] = -1;
    if (m != ZERO_ROW) row = load_ranks(v.excl_ranks + (size_t)m * 4);
    CtxA a;
    prepare_ctx_a(v, d, a);
    mmp_decision_out ra{-9, -9}, rb{-9, -9};
    SplitKey k;
    const bool fa = split_answer_rows(v, d, a, row, fr.data(), n_fresh, sums.data(), members.data(), now_ms, seed, id, ra);
    const bool fb = split_answer_keyed(v, d, fr.data(), n_fresh, sums.data(), members.data(), now_ms, seed, id, rb, k);
    counts[0]++; counts[1] += fa; counts[2] += fb; counts[3] += fa != fb;
    counts[4] += fa && fb && (ra.target != rb.target || ra.n_candidates != rb.n_candidates);
  }
  return MMP_OK;
}
}  // extern "C"
