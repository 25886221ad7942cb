// tests/emul/split_widen.cpp — CPU-ONLY TEST HARNESS for the widened fast-path rule of k_place_split.  Not part of the product.
//
// The split_place harness (included whole: the tests/emul fleet, the excluded-rank lists, the slot summaries, the walk)
// plus one entry point that answers every decision of a batch twice: by the rule before the keys covered every edge (the
// RowRanks overload of split_answer: inline ranks only, a model with overflow ids declined, any self below the reach
// walked), and by split_answer on the SplitKey the commit builds now -- every live edge, inline and overflow, counted when
// it is a member of its slot's cand, SPLIT_KEY_ALL_EDGES set -- with self's candidate bit gathered as k_place_split
// gathers it.  Every widened answer must equal the walk, and every decision the old rule answered must still be answered.
#include "split_place.cpp"

namespace {
// k_build_bitmap / k_build_bitmap_ovf with the snapshot's cand masks: every model's SplitKey, overflow edges folded in
std::vector<SplitKey> build_wide_keys(const mmp_fleet *f, const SnapshotView &v) {
  const int32_t nm = (int32_t)f->models.size();
  std::vector<SplitKey> k((size_t)std::max(nm, 1));
  for (int32_t m = 0; m < nm; m++) {
    int32_t rs[4] = {-1, -1, -1, -1};
    for (int i = 0; i < HostState::EDGE_INL; i++) {
      const int32_t e = f->hs.edge_inl[(size_t)m * HostState::EDGE_INL + i];
      if (e >= 0) rs[i] = f->snap.rank_of[e];
    }
    k[(size_t)m] = make_split_key(f->models[(size_t)m], rs, v.type_slot, v.n_type_ids, v.cand, v.row_words);
  }
  for (auto &kv : f->hs.edge_ovf) {
    if (kv.second.empty() || kv.first >= nm) continue;
    SplitKey &key = k[(size_t)kv.first];
    key.slot |= SPLIT_KEY_OVF;
    const uint32_t *cm = v.cand + (size_t)(key.slot & SPLIT_KEY_SLOT) * (size_t)v.row_words;
    for (int32_t e : kv.second) {
      const int32_t r = f->snap.rank_of[e];
      if (r >= 0 && mask_bit(cm, r) && r < key.min_rank) key.min_rank = r;
    }
  }
  return k;
}
}  // namespace

extern "C" {
// the type slot of model m's summary (slot_key of its type id), -1 for no such model
int32_t mmp_emul_model_slot(mmp_fleet *f, int32_t m) {
  if (f->epoch == 0 || m < 0 || m >= (int32_t)f->models.size()) return -1;
  return (int32_t)slot_key(make_view(f), f->models[(size_t)m].type_id);
}

// verdict (n entries): bit 0 the old rule answered, bit 1 the widened rule answered, bit 2 the widened answer differs from
// the walk.  out: the walked results.  counts (5 entries): decisions, answered by the old rule, answered by the widened
// rule, widened answers that differ from the walk, decisions the old rule answered and the widened rule did not.
int32_t mmp_emul_split_widen(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                             const int32_t *extra, int32_t n_extra, mmp_decision_out *out, int64_t now_ms, uint64_t seed,
                             int8_t *verdict, int64_t *counts) {
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  int32_t rc = mmp_emul_place_ranks(f, in, n, fresh, n_fresh, extra, n_extra, MMP_LANE_WIN, 192, out, now_ms, seed, nullptr);
  if (rc < 0) return rc;
  SnapshotView v = make_view(f);
  const std::vector<uint32_t> zero((size_t)v.excl_stride, 0u);
  v.zero_row = zero.data();
  const std::vector<int32_t> ranks = build_excl_ranks(f);
  v.excl_ranks = ranks.data();
  const std::vector<SplitKey> keys = build_wide_keys(f, v);
  v.split_key = keys.data();
  v.n_extra = n_extra;
  std::vector<FreshRow> fr((size_t)(n_fresh > 0 ? n_fresh : 0));
  for (int32_t i = 0; i < n_fresh; i++)
    if (const char *m = HostState::fresh_row(fresh[i], fr[i])) { g_err = m; return MMP_E_ARG; }
  std::vector<SlotSummary> sums;
  std::vector<int32_t> members;
  build_summaries(v, now_ms, sums, members);
  const uint32_t *cx = v.any_rs ? v.candx : v.cand;
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
    const bool fa = split_answer(v, d, a, row, fr.data(), n_fresh, sums.data(), members.data(), now_ms, seed, id, ra);
    // what k_place_split reads: the record's validity, rank_of[self], the model's key, self's word of its slot's mask
    const int32_t ok = decision_ok(v, d);
    SplitKey k;
    k.last_used = 0; k.min_rank = INT32_MAX; k.slot = 0;
    if (ok && !request_model(d)) k = load_split_key(v.split_key + d.model);
    const int32_t self_rank = ok ? v.rank_of[d.self] : -1;
    bool self_cand = true;
    if (ok && !request_model(d) && self_rank >= 0) self_cand = mask_bit(cx + (size_t)(k.slot & SPLIT_KEY_SLOT) * (size_t)v.row_words, self_rank);
    const bool fb = ok && split_answer(v, d, ok, self_rank, k, fr.data(), n_fresh, sums.data(), members.data(), now_ms, seed, id, rb, self_cand);
    const bool bad = fb && (rb.target != out[i].target || rb.n_candidates != out[i].n_candidates);
    verdict[i] = (int8_t)((fa ? 1 : 0) | (fb ? 2 : 0) | (bad ? 4 : 0));
    counts[0]++; counts[1] += fa; counts[2] += fb; counts[3] += bad; counts[4] += fa && !fb;
  }
  return MMP_OK;
}
}  // extern "C"
