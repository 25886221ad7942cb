"""CPU checks of every placement routine at the decision arithmetic's edges (tests/decision_edges.py): the caller-record
cut, the count cut, the full best's distance test, non-simple case (b) and the rpm filter's bands, each with values on
both sides of its threshold.  The routines are place_core.cuh's, compiled by g++ in the tests/emul harnesses: the window
fast path (32- and 16-word windows), the general routine (traced with masks), the budgeted lane walk and the lockstep
lane routine, and the two-pass path's slot summaries and the answers they give."""
import ctypes as C

import numpy as np
import pytest

from modelmesh_b200 import _lib as L

from decision_edges import _jdiv, all_cases, check_built
from helpers import compare_decisions, oracle_from_synth, oracle_inputs, solver_from_synth
from split_place import place_split, split_lib  # noqa: F401  (module fixture)

CASES = all_cases()
FAMILIES = sorted({c.family for c in CASES})


@pytest.fixture(scope="module")
def built(emul_lib, oracle_lib):
    """per case: the oracle, the emul solver and the oracle's answers with candidate lists"""
    out = {}
    for c in CASES:
        o = oracle_from_synth(c.fl)
        od, off, idx = oracle_inputs(c.fl, c.sd)
        ores = o.get_next_batch(od, c.fl.type_names, off, idx, c.fl.now_ms, 5, fresh=c.sd.fresh if len(c.sd.fresh) else None)
        out[c.id] = (o, solver_from_synth(c.fl, emul_lib), ores)
    yield out
    for _, s, _ in out.values():
        s.close()


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_fleet_is_built_as_intended(built, case):
    """ranks as intended, the designed shortlist lengths, and different answers on the two sides of every threshold"""
    o, s, ores = built[case.id]
    assert np.array_equal(s.cluster_order(), case.order)
    check_built(case, o, ores)


def _families(built, emul_lib, window, seed):
    """every case through compare_decisions with the harness window `window`; per family: decisions, fast-path answers
    and the trace flags seen"""
    emul_lib.mmp_emul_set_window(window)
    stats = {f: [0, 0, 0] for f in FAMILIES}
    try:
        for c in CASES:
            o, s, _ = built[c.id]
            _, _, tr = compare_decisions(c.fl, c.sd, o, s, seed=seed, full_lists=window in (32, 16))
            st = stats[c.family]
            st[0] += len(c.sd.dec)
            st[1] += int(round(compare_decisions.fast_fraction * len(c.sd.dec)))
            st[2] |= int(np.bitwise_or.reduce(tr["flags"]))
    finally:
        emul_lib.mmp_emul_set_window(32)
    return stats


@pytest.mark.parametrize("window", [32, 16])
def test_window_fast_path_and_general_routine(built, emul_lib, window):
    """traced with masks (the general routine, full shortlists and survivors), traced without masks and untraced (the
    one-window fast path, the general routine where it declines)"""
    stats = _families(built, emul_lib, window, 7)
    fast = {f: st[1] / st[0] for f, st in stats.items()}
    assert 0 < fast["count-cut"] < 1, fast        # the cut past the window leaves the fast path
    assert fast["caller-cut"] > 0 and fast["rpm"] > 0 and fast["pref-a"] > 0, fast
    assert fast["full-best"] == 0 and fast["pref-b"] == 0, fast  # a full best: the general routine
    assert stats["full-best"][2] & L.TF_BEST_FULL and stats["pref-b"][2] & L.TF_BEST_FULL
    assert stats["pref-b"][2] & L.TF_PREF_B


@pytest.mark.parametrize("budget", [1, 48])
@pytest.mark.parametrize("shape", [1, 2])
def test_lane_routines(built, emul_lib, shape, budget):
    """1: the general routine as a budgeted single-lane walk; 2: the lockstep lane routine of k_place_direct /
    k_place_lanes; the cooperative redo where either declines"""
    emul_lib.mmp_emul_lane_bails.restype = C.c_long
    emul_lib.mmp_emul_set_lane_budget(budget)
    try:
        emul_lib.mmp_emul_lane_bails(None)
        _families(built, emul_lib, shape, 11)
        n = C.c_long()
        bails = emul_lib.mmp_emul_lane_bails(C.byref(n))
        assert n.value > 0
        assert bails < n.value
    finally:
        emul_lib.mmp_emul_set_lane_budget(48)


def test_two_pass_answers(built, split_lib):  # noqa: F811
    """k_place_split's answers: every answer from a summary equals the walk and the oracle, and the families built for it
    are answered from summaries"""
    for c in CASES:
        o, _, ores = built[c.id]
        s = solver_from_synth(c.fl, split_lib)
        try:
            out, counts = place_split(split_lib, s, c.sd, c.fl.now_ms, 5)
        finally:
            s.close()
        assert counts[1] == 0, (c.id, counts)
        assert np.array_equal(out["target"], ores["target"]) and np.array_equal(out["n_candidates"], ores["n_candidates"]), c.id
        if c.summarised:
            assert counts[0] > 0, (c.id, counts)


SLOT_SUMMARY = np.dtype([("best_rem", "<i8"), ("best_lru", "<i8"), ("best_idx", "<i4"), ("best_rpm", "<i4"), ("best_full", "<i4"),
                         ("reach", "<i4", (2,)), ("n_in", "<i4", (2,)), ("pad", "<i4")])


def _wrap(x):  # Java long arithmetic
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


@pytest.mark.parametrize("case", [c for c in CASES if c.summarised], ids=[c.id for c in CASES if c.summarised])
def test_slot_summaries_equal_the_oracle(built, split_lib, case):  # noqa: F811
    """k_slot_summary itself, for both values of c_self: its shortlist equals the oracle's for a caller whose record makes
    c_self come out that way.  With a full best the c_self = 1 summary is walked with a record whose lruTime is forced past
    the distance test (r0.lru + max(age/10, 45 000) + 1, a wrapping add); at a best lruTime of Long.MAX_VALUE the sum wraps
    to a negative lruTime.  No caller can publish one (lruTime >= 0), so no decision reads that summary, but the oracle
    can be asked what such a caller gets: one candidate."""
    o, _, _ = built[case.id]
    s = solver_from_synth(case.fl, split_lib)
    try:
        split_lib.mmp_emul_slot_summaries.restype = C.c_int32
        sums = np.zeros(4, dtype=SLOT_SUMMARY)
        members = np.full((4, 2, 256), -1, dtype=np.int32)
        n_slots = s._ck(split_lib.mmp_emul_slot_summaries(s.h, C.c_int64(case.fl.now_ms), sums.ctypes.data_as(C.c_void_p),
                                                          members.ctypes.data_as(C.c_void_p), 4))
    finally:
        s.close()
    assert n_slots == 1  # (an unconstrained fleet: every type shares one slot)
    sm = sums[0]
    fresh = np.zeros(2, dtype=L.INSTANCE_ROW)
    fresh["capacity"] = 4_000_000
    if sm["best_full"]:
        a10 = _jdiv(0 if sm["best_lru"] == 0 else case.fl.now_ms - int(sm["best_lru"]), 10)
        fresh["lru_time"] = [int(sm["best_lru"]), _wrap(int(sm["best_lru"]) + max(a10, 45_000) + 1)]
        fresh["used"] = 4_000_000
    else:
        fresh["used"] = [0, 4_000_000]
    if case.id == "full-best:long-max":
        assert fresh["lru_time"][1] < 0  # the wrapped record
    sd = type(case.sd)(case.sd.dec[:2].copy(), fresh, case.sd.extra)
    sd.dec["model"] = 0
    sd.dec["self"] = case.ghost
    sd.dec["fresh"] = [0, 1]
    sd.dec["flags"] = 0
    od, off, idx = oracle_inputs(case.fl, sd)
    want, coff, cidx, _, _ = o.get_next_batch(od, case.fl.type_names, off, idx, case.fl.now_ms, 5, fresh=fresh, want_candidates=True)
    for cs in (0, 1):
        assert sm["reach"][cs] >= 0, (case.id, cs, sm)
        assert want["best"][cs] == sm["best_idx"]
        n = int(sm["n_in"][cs])
        assert want["n_candidates"][cs] == 1 + n, (case.id, cs, sm, want[cs])
        assert [int(x) for x in cidx[coff[cs]:coff[cs + 1]] if x != sm["best_idx"]] == [int(x) for x in members[0, cs, :n]], (case.id, cs)
    if sm["best_full"]:
        assert want["n_candidates"][1] == 1
