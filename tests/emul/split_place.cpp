// tests/emul/split_place.cpp — CPU-ONLY TEST HARNESS for the two-pass placement path.  Not part of the product.
//
// The row_ranks harness (included whole: the tests/emul fleet, the excluded-rank lists) plus one entry point that does
// what k_slot_summary and k_place_split do -- the slot summaries of the snapshot for both values of c_self, then the
// summary's answer for every decision it takes -- and resolves every decision the way k_place_direct does as well
// (mmp_emul_place_ranks' routine).  Every answer the summary gives must equal that walk.
#include "row_ranks.cpp"

extern "C" {
// counts (4 entries): decisions the summary answered, of those the ones whose walk differs, slots summarised for
// c_self = 0 and for c_self = 1.  out: the walked results (the summary's where it answered and agreed).
int32_t mmp_emul_place_split(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                             const int32_t *extra, int32_t n_extra, mmp_decision_out *out, int64_t now_ms, uint64_t seed, int64_t *counts) {
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  int32_t rc = mmp_emul_place_ranks(f, in, n, fresh, n_fresh, extra, n_extra, MMP_LANE_WIN, 192, out, now_ms, seed, nullptr);
  if (rc < 0) return rc;
  SnapshotView v = make_view(f);
  const std::vector<int32_t> ranks = build_excl_ranks(f);
  v.excl_ranks = ranks.data();
  v.n_extra = n_extra;
  std::vector<FreshRow> fr((size_t)(n_fresh > 0 ? n_fresh : 0));
  for (int32_t i = 0; i < n_fresh; i++)
    if (const char *m = HostState::fresh_row(fresh[i], fr[i])) { g_err = m; return MMP_E_ARG; }
  const int ns = v.n_slots > 0 ? v.n_slots : 1;
  std::vector<SlotSummary> sums((size_t)ns);
  std::vector<int32_t> members((size_t)ns * 2 * SPLIT_CAP, -1);
  const uint32_t ww = (uint32_t)std::min<int64_t>(MMP_LANE_WIN, v.row_words);
  std::vector<uint32_t> ewin(ww, 0u);
  int64_t summarised[2] = {0, 0};
  for (int sl = 0; sl < v.n_slots; sl++) {
    LaneTables T = lane_tables_global(v, sl);
    T.nz_skip = 0;  // list entries inside this window
    while (T.nz_skip < T.nz_n && (uint32_t)T.nzw[T.nz_skip] < ww) T.nz_skip++;
    for (int cs = 0; cs < 2; cs++) {
      slot_summary(v, T, sl, true, cs, ewin.data(), ww, now_ms, SoloVote(), nullptr, sums[sl], members.data() + ((size_t)sl * 2 + cs) * SPLIT_CAP);
      if (sums[sl].reach[cs] >= 0) summarised[cs]++;
    }
  }
  int64_t fast = 0, mismatch = 0;
  for (int32_t i = 0; i < n; i++) {
    const mmp_decision_in &d = in[i];
    const int32_t m = excl_row_id(v, d.model, d.flags);
    RowRanks row;
    row.r[0] = row.r[1] = row.r[2] = row.r[3] = -1;
    if (m != ZERO_ROW) row = load_ranks(v.excl_ranks + (size_t)m * 4);
    CtxA a;
    prepare_ctx_a(v, d, a);
    mmp_decision_out r;
    if (!split_answer(v, d, a, row, fr.data(), n_fresh, sums.data(), members.data(), now_ms, seed, pick_id(d, f->id_base + (uint64_t)i), r)) continue;
    fast++;
    if (r.target != out[i].target || r.n_candidates != out[i].n_candidates) mismatch++;
  }
  counts[0] = fast; counts[1] = mismatch; counts[2] = summarised[0]; counts[3] = summarised[1];
  return MMP_OK;
}
}  // extern "C"
