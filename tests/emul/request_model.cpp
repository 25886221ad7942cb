// tests/emul/request_model.cpp — CPU-ONLY TEST HARNESS for MMP_DF_REQUEST_MODEL decisions.  Not part of the product.
//
// The tests/emul harness (with row_ranks.cpp's excluded-rank lists) plus one entry point that resolves a batch the way
// each kernel family reads a decision's exclusion row -- through the shared helpers of place_core.cuh (excl_row_id /
// excl_row: the model's stored row, or the fleet's all-zero row for a request-model decision):
//   shape 0  the tile kernels (k_place, traced calls): the 32-word fast path unless masks are asked for, then the general
//            routine; trace and candidate masks as mmp_place_batch_trace writes them
//   shape 1  the lane routine on a copy of the row's first `window` words, the rest of the row through RowPtr
//            (k_place_lanes, k_place_small, k_place_server), the warp routine for whatever it declines (decide_warp)
//   shape 2  k_place_direct: the window rebuilt from the model's excluded ranks (none for a request-model decision),
//            overflow models declined, the warp routine on the row for whatever the lane declines
// As in the library, only an unsharded fleet has the zero row; on an instance-sharded one the general routine runs alone
// and the shard keys are written (mmp_emul_set_keys).
#include "row_ranks.cpp"

extern "C" {
int32_t mmp_emul_place_request(mmp_fleet *f, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                               const int32_t *extra, int32_t n_extra, int32_t shape, int32_t window, int32_t budget, mmp_decision_out *out,
                               mmp_decision_trace *trace, uint32_t *cand_mask, int64_t now_ms, uint64_t seed) {
  if (f->epoch == 0) { g_err = "no committed snapshot"; return MMP_E_EPOCH; }
  SnapshotView v = make_view(f);
  const bool sharded = v.word_lo != 0 || v.word_hi != v.row_words;
  if (shape < 0 || shape > 2 || window < 0 || window > MMP_LANE_WIN || (sharded && shape != 0)) { g_err = "bad shape"; return MMP_E_ARG; }
  const std::vector<uint32_t> zero((size_t)v.excl_stride, 0u);
  v.zero_row = sharded ? nullptr : zero.data();
  const std::vector<int32_t> ranks = sharded ? std::vector<int32_t>() : build_excl_ranks(f);
  v.excl_ranks = sharded ? nullptr : ranks.data();
  v.n_extra = n_extra;
  std::vector<FreshRow> fr((size_t)(n_fresh > 0 ? n_fresh : 0));
  for (int32_t i = 0; i < n_fresh; i++)
    if (const char *m = HostState::fresh_row(fresh[i], fr[i])) { g_err = m; return MMP_E_ARG; }
  const uint32_t ww = (uint32_t)std::min<int64_t>(window, v.row_words);
  Coop1 co;
  for (int32_t i = 0; i < n; i++) {
    DecisionCtx cx;
    prepare_ctx(v, in[i], fr.data(), n_fresh, extra, cx);
    const int32_t m = excl_row_id(v, in[i].model, in[i].flags);
    const uint32_t *erow = excl_row(v, m);
    const uint64_t id = pick_id(in[i], f->id_base + (uint64_t)i);
    DecideOut o;
    o.first_rank = -1; o.flags = 0;
    bool done = false;
    if (shape == 0) {
      if (!cand_mask && !sharded) done = decide_fast<true>(v, cx, erow, now_ms, seed, id, co, o);
    } else {
      RowRanks rr;
      rr.r[0] = rr.r[1] = rr.r[2] = rr.r[3] = -1;
      if (shape == 2 && m != ZERO_ROW) rr = load_ranks(v.excl_ranks + (size_t)m * 4);
      if (!rr.overflow()) {
        LaneTables T = lane_tables_global(v, cx.slot >= 0 ? ctx_slot(cx) : 0);
        T.nz_skip = 0;  // list entries inside this window
        while (T.nz_skip < T.nz_n && (uint32_t)T.nzw[T.nz_skip] < ww) T.nz_skip++;
        const uint32_t self_w = cx.self_rank >= 0 ? (uint32_t)cx.self_rank >> 5 : 0u;
        std::vector<uint32_t> win(ww);
        if (shape == 1) {
          for (uint32_t k = 0; k < ww; k++) win[k] = erow[k];
          done = decide_stream(v, T, T, cx, true, win.data(), ww, RowPtr{erow, 0u}, cx.self_rank >= 0 ? erow[self_w] : 0u, now_ms, seed, id,
                               SoloVote(), o, budget);
        } else {
          for (uint32_t k = 0; k < ww; k++) win[k] = rr.word(k);
          done = decide_stream(v, T, T, cx, true, win.data(), ww, rr, cx.self_rank >= 0 ? rr.word(self_w) : 0u, now_ms, seed, id,
                               SoloVote(), o, budget);
        }
      }
      if (!done) done = decide_fast<false>(v, cx, erow, now_ms, seed, id, co, o);  // decide_warp
    }
    if (!done)
      decide_ctx<Coop1>(v, cx, erow, extra, now_ms, seed, id, co, o, cand_mask ? cand_mask + (size_t)i * 2 * v.row_words : nullptr);
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
}  // extern "C"
