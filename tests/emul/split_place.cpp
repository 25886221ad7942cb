// tests/emul/split_place.cpp — CPU-ONLY TEST HARNESS for the two-pass placement path.  Not part of the product.
//
// The row_ranks harness (included whole: the tests/emul fleet, the excluded-rank lists) plus one entry point that does
// what k_slot_summary and k_place_split do -- the slot summaries of the snapshot for both values of c_self, then the
// summary's answer for every decision it takes -- and resolves every decision the way k_place_direct does as well
// (mmp_emul_place_ranks' routine).  Every answer the summary gives must equal that walk.
#include "row_ranks.cpp"

namespace {
// what k_slot_summary computes: the summary of every type slot for both values of c_self, and its shortlist members
void build_summaries(const SnapshotView &v, int64_t now_ms, std::vector<SlotSummary> &sums, std::vector<int32_t> &members) {
  const int ns = v.n_slots > 0 ? v.n_slots : 1;
  sums.assign((size_t)ns, SlotSummary());
  members.assign((size_t)ns * 2 * SPLIT_CAP, -1);
  const uint32_t ww = (uint32_t)std::min<int64_t>(MMP_LANE_WIN, v.row_words);
  std::vector<uint32_t> ewin(ww, 0u);
  for (int sl = 0; sl < v.n_slots; sl++) {
    LaneTables T = lane_tables_global(v, sl);
    T.nz_skip = 0;  // list entries inside this window
    while (T.nz_skip < T.nz_n && (uint32_t)T.nzw[T.nz_skip] < ww) T.nz_skip++;
    for (int cs = 0; cs < 2; cs++)
      slot_summary(v, T, sl, true, cs, ewin.data(), ww, now_ms, SoloVote(), nullptr, sums[sl], members.data() + ((size_t)sl * 2 + cs) * SPLIT_CAP);
  }
}
}  // namespace

extern "C" {
// The slot summaries of the committed snapshot (n_slots of them, SlotSummary layout) and their members ([slot][c_self]
// [SPLIT_CAP] instance indices, -1 past the end); sums / members may hold cap slots.  Returns the number of slots.
int32_t mmp_emul_slot_summaries(mmp_fleet *f, int64_t now_ms, SlotSummary *sums, int32_t *members, int32_t cap) {
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  SnapshotView v = make_view(f);
  const std::vector<int32_t> ranks = build_excl_ranks(f);
  v.excl_ranks = ranks.data();
  std::vector<SlotSummary> s;
  std::vector<int32_t> m;
  build_summaries(v, now_ms, s, m);
  for (int sl = 0; sl < v.n_slots && sl < cap; sl++) {
    sums[sl] = s[sl];
    std::copy(m.begin() + (size_t)sl * 2 * SPLIT_CAP, m.begin() + (size_t)(sl + 1) * 2 * SPLIT_CAP, members + (size_t)sl * 2 * SPLIT_CAP);
  }
  return v.n_slots;
}

// counts (6 entries): decisions the summary answered, of those the ones whose walk differs, slots summarised for
// c_self = 0 and for c_self = 1, summaries (slot, c_self) whose best and shortlist members run on more than one instance
// version (a rolling upgrade), decisions answered in a slot with such a summary.  out: the walked results (the summary's
// where it answered and agreed).
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
  std::vector<SlotSummary> sums;
  std::vector<int32_t> members;
  build_summaries(v, now_ms, sums, members);
  int64_t summarised[2] = {0, 0}, crossing = 0;
  std::vector<char> slot_crosses((size_t)ns, 0);
  for (int sl = 0; sl < v.n_slots; sl++) {
    for (int cs = 0; cs < 2; cs++) {
      const int32_t *mem = members.data() + ((size_t)sl * 2 + cs) * SPLIT_CAP;
      if (sums[sl].reach[cs] < 0) continue;
      summarised[cs]++;
      const int32_t vers = f->hs.inst[sums[sl].best_idx].row.vers;
      bool mixed = false;
      for (int32_t k = 0; k < sums[sl].n_in[cs] && k < SPLIT_CAP; k++) mixed |= f->hs.inst[mem[k]].row.vers != vers;
      crossing += mixed;
      slot_crosses[sl] |= mixed;
    }
  }
  int64_t fast = 0, mismatch = 0, fast_crossing = 0;
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
    fast_crossing += slot_crosses[(size_t)slot_key(v, a.mr.type_id)];
    if (r.target != out[i].target || r.n_candidates != out[i].n_candidates) mismatch++;
  }
  counts[0] = fast; counts[1] = mismatch; counts[2] = summarised[0]; counts[3] = summarised[1];
  counts[4] = crossing; counts[5] = fast_crossing;
  return MMP_OK;
}
}  // extern "C"
