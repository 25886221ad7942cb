"""The per-slot summaries of the two-pass placement path where k_slot_summary's reads change sides.  It copies the first
12 row words (ranks 0-383) of the rank tables and of the first 64 type slots' masks into shared memory: a rank or word
past the window is read from global memory, and so are the masks of slot 64 on, whatever the rank.  The fleet here has
more than 64 type slots (so a second block of the kernel fills its own copy), and summaries whose best, shortlist
members and reach lie on either side of rank 384, in slots on either side of 64."""
import ctypes as C
import itertools

import numpy as np
import pytest

from helpers import oracle_from_synth, oracle_inputs_fast, solver_from_synth
from modelmesh_b200.synth import make_decisions, make_fleet
from split_place import split_lib  # noqa: F401  (split_lib: module fixture)

WIN_RANKS = 12 * 32  # MMP_LANE_WIN row words
WIN_SLOTS = 64       # LANE_SLOTS
SLOT_SUMMARY = np.dtype([("best_rem", "<i8"), ("best_lru", "<i8"), ("best_idx", "<i4"), ("best_rpm", "<i4"), ("best_full", "<i4"),
                         ("reach", "<i4", (2,)), ("n_in", "<i4", (2,)), ("pad", "<i4")])


def _many_slot_fleet():
    """C3's instances (8 labels, 1-3 per instance) under 96 types that ask for label pairs, required and preferred:
    74 distinct type slots, pairs of required labels sparse enough that some shortlists run past rank 384."""
    nm, seed = 20_000, 61
    fl = make_fleet("C3", nm, 3000, seed)
    labs = [f"lbl-{k:02d}" for k in range(8)]
    pairs = list(itertools.combinations(labs, 2))
    cfg = {}
    for k in range(96):
        a, b = pairs[k % len(pairs)]
        if k % 3 == 0:
            ent = {"required": [a, b]}
        elif k % 3 == 1:
            ent = {"required": [labs[k % 8]], "preferred": [a, b] if (k // 8) % 2 else [b]}
        elif k < 56:
            ent = {"required": [a], "preferred": [b]}
        elif k < 84:
            ent = {"preferred": [a, b]}
        else:
            ent = {"required": [b, a], "preferred": [labs[k % 8]]}
        cfg[f"type-{k:02d}"] = ent
    fl.type_config = cfg
    fl.type_names = list(cfg) + ["untyped"]
    fl.model_type = np.random.default_rng(seed).integers(0, len(fl.type_names), nm).astype(np.int32)
    return fl


def test_fleet_has_summaries_on_both_sides_of_the_window(split_lib, oracle_lib):  # noqa: F811
    """What the GPU test below relies on, from the CPU harness's summaries (the routine k_slot_summary runs)."""
    fl = _many_slot_fleet()
    s = solver_from_synth(fl, split_lib)
    cap = 256
    sums = np.zeros(cap, dtype=SLOT_SUMMARY)
    members = np.full((cap, 2, 256), -1, dtype=np.int32)
    try:
        split_lib.mmp_emul_slot_summaries.restype = C.c_int32
        n = s._ck(split_lib.mmp_emul_slot_summaries(s.h, C.c_int64(fl.now_ms), sums.ctypes.data_as(C.c_void_p),
                                                    members.ctypes.data_as(C.c_void_p), cap))
    finally:
        s.close()
    assert WIN_SLOTS < n <= cap
    order = oracle_from_synth(fl).cluster_order()
    rank = np.empty(fl.n_instances, dtype=np.int64)
    rank[order] = np.arange(len(order))
    reach = sums["reach"][:n, 0].astype(np.int64)
    assert (reach >= 0).all()
    best = rank[sums["best_idx"][:n]]
    last = np.array([rank[members[sl, 0, sums["n_in"][sl, 0] - 1]] if sums["n_in"][sl, 0] > 0 else best[sl] for sl in range(n)])
    for lo, hi in ((0, WIN_SLOTS), (WIN_SLOTS, n)):
        assert (reach[lo:hi] <= WIN_RANKS).any() and (reach[lo:hi] > WIN_RANKS).any(), (lo, reach[lo:hi])
        assert (last[lo:hi] >= WIN_RANKS).any(), (lo, last[lo:hi])
    assert ((best[:WIN_SLOTS] < WIN_RANKS) & (last[:WIN_SLOTS] >= WIN_RANKS)).any()  # a listing that crosses rank 384
    assert (best[WIN_SLOTS:] >= WIN_RANKS).any()  # a best row read from global memory


@pytest.mark.gpu
def test_split_equals_walk_and_oracle_across_the_window(product_lib, oracle_lib):
    """A plain sweep (most decisions answered from the summaries) and a mixed batch, placed with the two passes forced
    on and off: both equal each other and the oracle, byte for byte."""
    fl = _many_slot_fleet()
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    try:
        for what, sd, seed in (("sweep", make_decisions(fl, 40_000, 61, sweep=True, plain=True), 61),
                               ("mixed", make_decisions(fl, 30_000, 62), 63)):
            kw = dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
            got = {}
            for split in (1, 0):
                s._ck(product_lib.mmp_tune(s.h, b"split", split))
                try:
                    got[split] = s.place_batch(sd.dec, fl.now_ms, seed, **kw)
                finally:
                    s._ck(product_lib.mmp_tune(s.h, b"split", 2))
            assert got[1].tobytes() == got[0].tobytes(), (what, int(np.sum(got[1] != got[0])))
            od, off, idx = oracle_inputs_fast(fl, sd)
            want = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=kw["fresh"])
            bad = np.nonzero((got[1]["target"] != want["target"]) | (got[1]["n_candidates"] != want["n_candidates"]))[0]
            assert len(bad) == 0, (what, len(bad), bad[:5])
    finally:
        s.close()
