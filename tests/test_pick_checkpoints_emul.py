"""CPU checks of the hash-indexed pick (phase C) of decide_stream, the lane routine of k_place_direct and the other lane
kernels.  Phase C does not walk the shortlist from its start: it starts from the last window step before the pick at
which phase B recorded its count of shortlist members, then walks on as before (beyond the window too).  A self candidate
that the rpm filter drops was counted by phase B, so the checkpoints past self's word count one member fewer for phase C.

Every decision is answered twice through the tests/emul harness: by the lane routine (window `window`, budget `budget`)
and by the general routine, which also returns its survivor mask.  Both must equal the oracle, field for field; the
survivor masks classify the picks, and the fleets are chosen so that each case where a checkpoint matters occurs.
"""
import numpy as np

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import compare_decisions, oracle_from_synth, solver_from_synth

NONE_RANK = 0xFFFFFFFF
TF_FAST = 256

# (config, models, instances, fleet seed, window words, budget): window 0 has no checkpoints (phase C walks from the
# shortlist's start), budget 1 000 lets the long C5 walks run to their end
CASES = [("C3", 2000, 1300, 33, 12, 192), ("C5", 1500, 500, 5, 12, 192), ("MIX", 500, 300, 14, 3, 64),
         ("MIX", 500, 700, 41, 1, 64), ("MIX", 600, 160, 8, 5, 64), ("C5", 900, 10000, 5, 0, 1000),
         ("C5", 900, 5000, 6, 12, 192)]


def _classify(fl, solver, sd, seed, window, seen):
    """Count, per case, the decisions whose pick the lane routine made in phase C."""
    fresh = sd.fresh if len(sd.fresh) else None
    extra = sd.extra if len(sd.extra) else None
    out, tr, cm = solver.place_batch(sd.dec, fl.now_ms, seed, fresh=fresh, extra=extra, trace=True, masks=True)
    out2, tr2, _ = solver.place_batch(sd.dec, fl.now_ms, seed, fresh=fresh, extra=extra, trace=True)
    order = solver.cluster_order()
    rank_of = np.full(max(int(order.max()) + 1, fl.n_instances), -1, dtype=np.int64)
    rank_of[order] = np.arange(len(order))
    for i in range(len(sd.dec)):
        f = int(tr2["flags"][i])
        if not f & TF_FAST or f & L.TF_FAVOUR_EXIT or tr2["n_remaining"][i] <= 1:
            continue
        self_idx = int(sd.dec["self"][i])
        self_rank = int(rank_of[self_idx]) if 0 <= self_idx < len(rank_of) else -1
        t = int(out2["target"][i])
        rank = self_rank if t == L.TARGET_SELF else int(rank_of[t])
        if rank < 0 or rank == int(tr2["best_rank"][i]):
            continue
        if not f & L.TF_KEEP_OTHERS:
            seen["pick is self (!keep_others)"] += 1
            continue
        w, b = rank >> 5, rank & 31
        surv = int(cm[i, 1, w]) & ~(1 << (int(tr2["best_rank"][i]) & 31) if (int(tr2["best_rank"][i]) >> 5) == w else int(cm[i, 1, w]))
        where = "window" if w < window else "beyond the window"
        if surv & ((1 << b) - 1) == 0:
            seen[f"first member of a word {where}"] += 1
        if surv >> (b + 1) == 0:
            seen[f"last member of a word {where}"] += 1
        cut = int(tr2["cut_rank"][i]) & 0xFFFFFFFF
        if cut != NONE_RANK and (cut >> 5) == w:
            seen["pick in the cut word"] += 1
        cut_r = cut if cut != NONE_RANK else 1 << 40
        if not f & L.TF_KEEP_SELF and int(tr2["best_rank"][i]) < self_rank < cut_r and t != L.TARGET_SELF:
            sw = self_rank >> 5
            seen["drop_self, self's word " + ("before" if sw < w else ("=" if sw == w else "after")) + " the pick's"] += 1


def test_phase_c_picks_equal_the_general_routine_and_the_oracle(emul_lib, oracle_lib):
    import collections
    seen = collections.Counter()
    emul_lib.mmp_emul_set_window(2)
    emul_lib.mmp_emul_set_lane_global(1)
    try:
        for config, nm, ni, fseed, window, budget in CASES:
            emul_lib.mmp_emul_set_lane_window(window)
            emul_lib.mmp_emul_set_lane_budget(budget)
            fl = make_fleet(config, nm, ni, fseed)
            o = oracle_from_synth(fl)
            s = solver_from_synth(fl, emul_lib)
            for k, sd in enumerate((make_decisions(fl, 900, fseed, sweep=True, plain=True), make_decisions(fl, 900, fseed + 1))):
                for pick_seed in (fseed + 3 * k, fseed + 3 * k + 1):  # another seed: other picks on the same shortlists
                    compare_decisions(fl, sd, o, s, seed=pick_seed, full_lists=False)
                    _classify(fl, s, sd, pick_seed, window, seen)
    finally:
        emul_lib.mmp_emul_set_window(32)
        emul_lib.mmp_emul_set_lane_window(12)
        emul_lib.mmp_emul_set_lane_budget(48)
    want = ["first member of a word window", "last member of a word window", "first member of a word beyond the window",
            "last member of a word beyond the window", "pick in the cut word", "drop_self, self's word before the pick's",
            "drop_self, self's word = the pick's", "drop_self, self's word after the pick's", "pick is self (!keep_others)"]
    missing = [c for c in want if seen[c] == 0]
    assert not missing, (missing, dict(seen))
