// tests/emul/row_ranks.cpp — CPU-ONLY TEST HARNESS for k_place_direct's row access.  Not part of the product.
//
// The tests/emul harness (included whole: same mmp_* entry points, same fleet) plus one entry point that resolves a batch
// the way k_place_direct does: the model's excluded ranks (SnapshotView::excl_ranks, built here as k_build_bitmap /
// k_build_bitmap_ovf build them on the device) stand in for its bitmap row -- the lane's window, self's row word and every
// word a walk reads beyond the window come from RowRanks -- a model with overflow ids is declined, and whatever the lane
// routine declines is resolved by the general routine from the bitmap row (decide_warp).  Every decision the ranks walk
// resolves is also walked through the bitmap row (RowPtr) and must agree with it field for field.
#include "emul.cpp"

namespace {
// k_build_bitmap / k_build_bitmap_ovf: entry j = rank of inline edge j (-1: no edge, or not live), EXCL_RANKS_OVF in
// entry 0 of a model with overflow pairs
std::vector<int32_t> build_excl_ranks(const mmp_fleet *f) {
  const int32_t nm = (int32_t)f->models.size();
  std::vector<int32_t> r((size_t)std::max(nm, 1) * 4, -1);
  for (int32_t m = 0; m < nm; m++)
    for (int i = 0; i < HostState::EDGE_INL; i++) {
      const int32_t e = f->hs.edge_inl[(size_t)m * HostState::EDGE_INL + i];
      if (e >= 0) r[(size_t)m * 4 + i] = f->snap.rank_of[e];
    }
  for (auto &kv : f->hs.edge_ovf)
    if (!kv.second.empty() && kv.first < nm) r[(size_t)kv.first * 4] = EXCL_RANKS_OVF;
  return r;
}
bool same(const DecideOut &a, const DecideOut &b) {
  return a.target == b.target && a.n_candidates == b.n_candidates && a.best == b.best && a.n_remaining == b.n_remaining &&
         a.pick_index == b.pick_index && a.flags == b.flags && a.cut_rank == b.cut_rank && a.best_rank == b.best_rank &&
         a.first_rank == b.first_rank;
}
}  // namespace

extern "C" {
// counts (optional, 4 entries): decisions whose ranks walk differs from the bitmap-row walk, overflow models declined,
// decisions the ranks walk resolved, decisions it declined for other reasons
int32_t mmp_emul_place_ranks(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                             const int32_t *extra, int32_t n_extra, int32_t window, int32_t budget, mmp_decision_out *out,
                             int64_t now_ms, uint64_t seed, int64_t *counts) {
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  SnapshotView v = make_view(f);
  if (v.word_lo != 0 || v.word_hi != v.row_words) { g_err = "excluded-rank lists exist for unsharded fleets only"; return MMP_E_ARG; }
  if (window < 0 || window > MMP_LANE_WIN) { g_err = "window out of range"; return MMP_E_ARG; }
  const std::vector<int32_t> ranks = build_excl_ranks(f);
  v.excl_ranks = ranks.data();
  v.n_extra = n_extra;
  std::vector<FreshRow> fr((size_t)(n_fresh > 0 ? n_fresh : 0));
  for (int32_t i = 0; i < n_fresh; i++)
    if (const char *m = HostState::fresh_row(fresh[i], fr[i])) { g_err = m; return MMP_E_ARG; }
  int64_t mismatch = 0, ovf = 0, resolved = 0, declined = 0;
  const uint32_t ww = (uint32_t)std::min<int64_t>(window, v.row_words);
  Coop1 co;
  for (int32_t i = 0; i < n; i++) {
    DecisionCtx cx;
    prepare_ctx(v, in[i], fr.data(), n_fresh, extra, cx);
    const int32_t m = (in[i].model >= 0 && in[i].model < v.n_models) ? in[i].model : 0;  // (as the kernel)
    const uint32_t *erow = v.excl + (size_t)m * v.excl_stride;
    const uint64_t id = pick_id(in[i], f->id_base + (uint64_t)i);
    const RowRanks rr = load_ranks(v.excl_ranks + (size_t)m * 4);
    DecideOut o;
    bool done = false;
    if (rr.overflow()) ovf++;
    else {
      LaneTables T = lane_tables_global(v, cx.slot >= 0 ? ctx_slot(cx) : 0);
      T.nz_skip = 0;  // list entries inside this window
      while (T.nz_skip < T.nz_n && (uint32_t)T.nzw[T.nz_skip] < ww) T.nz_skip++;
      std::vector<uint32_t> win_r(ww), win_p(erow, erow + ww);
      for (uint32_t k = 0; k < ww; k++) win_r[k] = rr.word(k);
      const uint32_t self_w = cx.self_rank >= 0 ? (uint32_t)cx.self_rank >> 5 : 0u;
      done = decide_stream(v, T, T, cx, true, win_r.data(), ww, rr, cx.self_rank >= 0 ? rr.word(self_w) : 0u, now_ms, seed, id,
                           SoloVote(), o, budget);
      DecideOut op;
      const bool done_p = decide_stream(v, T, T, cx, true, win_p.data(), ww, RowPtr{erow, 0u}, cx.self_rank >= 0 ? erow[self_w] : 0u,
                                        now_ms, seed, id, SoloVote(), op, budget);
      if (done != done_p || (done && !same(o, op))) mismatch++;
      if (done) resolved++;
      else declined++;
    }
    if (!done && !decide_fast<false>(v, cx, erow, now_ms, seed, id, co, o))  // decide_warp
      decide_ctx<Coop1>(v, cx, erow, extra, now_ms, seed, id, co, o, nullptr);
    out[i].target = o.target; out[i].n_candidates = o.n_candidates;
  }
  if (counts) { counts[0] = mismatch; counts[1] = ovf; counts[2] = resolved; counts[3] = declined; }
  f->launches++;
  return MMP_OK;
}
}  // extern "C"
