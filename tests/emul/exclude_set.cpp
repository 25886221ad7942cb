// tests/emul/exclude_set.cpp — CPU-ONLY TEST HARNESS for call-wide exclude sets (mmp_place_batch_excluding).  Not part of
// the product.
//
// request_model.cpp (and through it row_ranks.cpp and the tests/emul harness) plus one entry point that derives the call's
// slot tables on the host as k_exclude_slots and k_slot_lists derive them on the device -- the set's ranks cleared from
// cand / candx / pref, the compressed word lists rebuilt by HostState::slot_word_lists -- and resolves the batch on a view
// of them in the three shapes of mmp_emul_place_request (tile routine with traces and masks; the lane routine on a window
// copied from the row; k_place_direct's window rebuilt from the ranks).  Everything per rank or per row is the snapshot's.
#include "request_model.cpp"

extern "C" {
int32_t mmp_emul_place_excluding(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                                 const int32_t *extra, int32_t n_extra, const int32_t *exclude, int32_t n_exclude, int32_t shape,
                                 int32_t window, int32_t budget, mmp_decision_out *out, mmp_decision_trace *trace, uint32_t *cand_mask,
                                 int64_t now_ms, uint64_t seed) {
  if (n_exclude < 0 || (n_exclude > 0 && !exclude)) { g_err = "bad exclude set"; return MMP_E_ARG; }
  for (int32_t k = 0; k < n_exclude; k++)
    if (exclude[k] < 0 || exclude[k] >= f->hs.cfg.max_instances) { g_err = "exclude set: instance index outside [0, max_instances)"; return MMP_E_ARG; }
  if (n_exclude > 0 && f->hs.cfg.shard_count > 1) { g_err = "an exclude set is not available on an instance-sharded fleet"; return MMP_E_STATE; }
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  HostSnapshot &s = f->snap;
  const int32_t RW = s.row_words;
  std::vector<uint32_t> x((size_t)RW, 0u);
  for (int32_t k = 0; k < n_exclude; k++) {
    const int32_t r = s.rank_of[exclude[k]];
    if (r >= 0) x[r >> 5] |= 1u << (r & 31);
  }
  HostSnapshot d;  // the derived tables (only what slot_word_lists reads besides them)
  d.row_words = RW; d.n_slots = s.n_slots; d.any_rs = s.any_rs;
  d.cand = s.cand; d.candx = s.candx; d.pref = s.pref;
  for (size_t i = 0; i < d.cand.size(); i++) {
    const uint32_t keep = ~x[i % RW];
    d.cand[i] &= keep; d.candx[i] &= keep; d.pref[i] &= keep;
  }
  HostState::slot_word_lists(d, s.word_lo, s.word_hi, d.nzw, d.nz_n);
  // the snapshot's tables out, the call's in, for the length of the call
  auto flip = [&] { std::swap(s.cand, d.cand); std::swap(s.candx, d.candx); std::swap(s.pref, d.pref); std::swap(s.nzw, d.nzw); std::swap(s.nz_n, d.nz_n); };
  if (n_exclude > 0) flip();
  const int32_t rc = mmp_emul_place_request(f, in, n, fresh, n_fresh, extra, n_extra, shape, window, budget, out, trace, cand_mask, now_ms, seed);
  if (n_exclude > 0) flip();
  return rc;
}
}  // extern "C"
