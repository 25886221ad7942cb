"""CPU checks of the rank-space formulation (product host code + single-lane decision routine) against the oracle.

These do not touch a GPU: they exercise csrc/host_state.hpp and csrc/place_core.cuh through the tests/emul harness.
Parity of everything here is "unpinned by reference tests" beyond the golden scenarios (see test_oracle_golden.py).
"""
import numpy as np
import pytest

from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import compare_decisions, oracle_from_synth, solver_from_synth
from test_rolling_upgrade_gpu import fleet_for


@pytest.mark.parametrize("config,nm,ni,seed", [
    ("C1", 200, 16, 1), ("C2", 3000, 200, 2), ("C2", 2000, 1000, 12), ("C3", 4000, 700, 3), ("C5", 4000, 500, 5),
    ("C3", 1500, 1300, 33), ("C5", 1000, 33, 55),
])
def test_decisions_match_oracle(emul_lib, oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, emul_lib)
    assert np.array_equal(s.cluster_order(), o.cluster_order())
    sd = make_decisions(fl, 3000, seed)
    compare_decisions(fl, sd, o, s, seed=seed * 7919)
    sd = make_decisions(fl, 1000, seed + 1, sweep=True, plain=True)
    compare_decisions(fl, sd, o, s, seed=seed)


@pytest.mark.parametrize("seed", range(40))
def test_mixed_regimes_match_oracle(emul_lib, oracle_lib, seed):
    """Regime-randomised fleets (synth._make_mix) that reach the rare branches: filter retry, non-simple (a)/(b),
    long full-case shortlists, equal keys down to the string tie-breaks."""
    ni = [33, 64, 97, 160, 300][seed % 5]
    fl = make_fleet("MIX", 600, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, emul_lib)
    assert np.array_equal(s.cluster_order(), o.cluster_order())
    sd = make_decisions(fl, 1500, seed)
    compare_decisions(fl, sd, o, s, seed=seed + 99)


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 2000, 1000, 12), ("C3", 4000, 700, 3), ("C5", 3000, 500, 5), ("MIX", 600, 160, 8),
                                               ("MIX", 600, 300, 14), ("C3", 1500, 1300, 33), ("C3/half", 4000, 700, 3),
                                               ("MIX/saturated", 600, 300, 14)])
def test_half_warp_window_matches_oracle(emul_lib, oracle_lib, config, nm, ni, seed):
    """The fast path with 16-word windows (the half-warp tile of the GPU kernel: two decisions per warp)."""
    emul_lib.mmp_emul_set_window(16)
    try:
        fl = fleet_for(config, nm, ni, seed)
        o = oracle_from_synth(fl)
        s = solver_from_synth(fl, emul_lib)
        sd = make_decisions(fl, 2500, seed)
        compare_decisions(fl, sd, o, s, seed=seed * 31)
        sd = make_decisions(fl, 1500, seed + 1, sweep=True, plain=True)
        compare_decisions(fl, sd, o, s, seed=seed)
    finally:
        emul_lib.mmp_emul_set_window(32)


@pytest.mark.parametrize("budget", [1, 48])
@pytest.mark.parametrize("shape", [1, 2])
@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 2000, 1000, 12), ("C3", 4000, 700, 3), ("C5", 3000, 500, 5), ("MIX", 600, 160, 8),
                                               ("MIX", 600, 300, 14), ("MIX", 600, 97, 21), ("C3", 1500, 1300, 33),
                                               ("C3/half", 4000, 700, 3), ("MIX/saturated", 600, 300, 14)])
def test_lane_shape_matches_oracle(emul_lib, oracle_lib, config, nm, ni, seed, budget, shape):
    """The lane-per-decision shapes: 1 = the general routine as a budgeted single-lane walk (CoopLane), 2 = the lockstep
    streaming routine k_place_lanes runs (decide_stream); both with the cooperative redo when the lane declines.
    budget=1 forces most decisions through the redo path; 48 is of the order of the kernel's setting (LANE_BUDGET)."""
    import ctypes as C
    emul_lib.mmp_emul_lane_bails.restype = C.c_long
    emul_lib.mmp_emul_set_window(shape)
    emul_lib.mmp_emul_set_lane_budget(budget)
    try:
        fl = fleet_for(config, nm, ni, seed)
        o = oracle_from_synth(fl)
        s = solver_from_synth(fl, emul_lib)
        emul_lib.mmp_emul_lane_bails(None)
        sd = make_decisions(fl, 2500, seed)
        compare_decisions(fl, sd, o, s, seed=seed * 31)
        sd = make_decisions(fl, 1500, seed + 1, sweep=True, plain=True)
        compare_decisions(fl, sd, o, s, seed=seed)
        n = C.c_long()
        bails = emul_lib.mmp_emul_lane_bails(C.byref(n))
        assert n.value > 0
        if budget == 1 and ni >= 300 and config != "C2":  # (every C2 walk ends inside its first row word)
            assert bails > 0  # the redo path was exercised
    finally:
        emul_lib.mmp_emul_set_window(32)
        emul_lib.mmp_emul_set_lane_budget(48)


@pytest.mark.parametrize("seed", range(40, 70))
def test_stream_routine_mixed_regimes(emul_lib, oracle_lib, seed):
    """decide_stream (the lockstep lane routine) on regime-randomised fleets, with a budget small enough that both its
    own answers and its hand-offs to the general routine occur."""
    emul_lib.mmp_emul_set_window(2)
    emul_lib.mmp_emul_set_lane_budget([3, 8, 48][seed % 3])
    try:
        ni = [33, 64, 97, 160, 300, 700][seed % 6]
        fl = make_fleet("MIX", 500, ni, seed)
        o = oracle_from_synth(fl)
        s = solver_from_synth(fl, emul_lib)
        sd = make_decisions(fl, 1200, seed)
        compare_decisions(fl, sd, o, s, seed=seed + 5, full_lists=False)
    finally:
        emul_lib.mmp_emul_set_window(32)
        emul_lib.mmp_emul_set_lane_budget(48)


def test_slices_with_id_base_equal_the_batch(emul_lib, oracle_lib):
    """A registry shard places a slice of a larger batch: with mmp_fleet_set_id_base(lo) the hash-indexed pick (N4) of
    decision lo + i is the one the whole batch gives it."""
    fl = make_fleet("C3", 3000, 700, 3)
    s = solver_from_synth(fl, emul_lib)
    for shape in (32, 2):
        emul_lib.mmp_emul_set_window(shape)
        try:
            sd = make_decisions(fl, 3000, 4, sweep=True, plain=True)
            whole = s.place_batch(sd.dec, fl.now_ms, 5)
            parts = []
            cuts = [0, 1, 33, 1000, 3000]
            for lo, hi in zip(cuts[:-1], cuts[1:]):
                s._ck(emul_lib.mmp_fleet_set_id_base(s.h, lo))
                parts.append(s.place_batch(sd.dec[lo:hi], fl.now_ms, 5))
            s._ck(emul_lib.mmp_fleet_set_id_base(s.h, 0))
            assert np.array_equal(np.concatenate(parts), whole)
            assert len(np.unique(whole["target"])) > 3
        finally:
            emul_lib.mmp_emul_set_window(32)


def test_registry_sweep_equals_the_batch_of_records(emul_lib, oracle_lib):
    """mmp_place_sweep (model first + i for self[i], lastUsed from the model row, favourSelf bits) = mmp_place_batch on
    the equivalent records; with one self for the whole sweep it is the leader's reaper batch (MM:6616-6735)."""
    from modelmesh_b200._lib import DF_FAVOUR_SELF
    fl = make_fleet("C3", 3000, 700, 3)
    s = solver_from_synth(fl, emul_lib)
    sd = make_decisions(fl, 3000, 4, sweep=True, plain=True)
    whole = s.place_batch(sd.dec, fl.now_ms, 5)
    fav = (sd.dec["flags"] & DF_FAVOUR_SELF) != 0
    assert np.array_equal(s.place_sweep(0, 3000, sd.dec["self"], fl.now_ms, 5, favour=fav), whole)
    # a slice of the registry, numbered like the whole sweep
    s._ck(emul_lib.mmp_fleet_set_id_base(s.h, 1000))
    assert np.array_equal(s.place_sweep(1000, 777, sd.dec["self"][1000:1777], fl.now_ms, 5, favour=fav[1000:1777]), whole[1000:1777])
    s._ck(emul_lib.mmp_fleet_set_id_base(s.h, 0))
    # one caller for the whole sweep
    leader = int(sd.dec["self"][0])
    d2 = sd.dec.copy()
    d2["self"] = leader
    d2["flags"] &= ~np.uint32(DF_FAVOUR_SELF)
    assert np.array_equal(s.place_sweep(0, 3000, leader, fl.now_ms, 5), s.place_batch(d2, fl.now_ms, 5))


@pytest.mark.parametrize("second_chance", [0, 1])
@pytest.mark.parametrize("window", [1, 2, 5, 10])
@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 2000, 1300, 33), ("C5", 1500, 500, 5), ("MIX", 500, 300, 14), ("MIX", 500, 700, 41),
                                               ("C3/three", 2000, 1300, 33), ("MIX/saturated", 500, 700, 41)])
def test_stream_routine_window_widths(emul_lib, oracle_lib, config, nm, ni, seed, window, second_chance):
    """decide_stream sees a window of the decision's exclusion row: its first `window` words (the kernels copy MMP_LANE_WIN = 12);
    beyond it a walk steps through the type slot's compressed word list.  second_chance = 0: a walk that leaves the window must be
    declined, never answered from partial information; 1: it goes on reading the row itself (the kernel reads it from L2)."""
    import ctypes as C
    emul_lib.mmp_emul_lane_bails.restype = C.c_long
    emul_lib.mmp_emul_set_window(2)
    emul_lib.mmp_emul_set_lane_window(window)
    emul_lib.mmp_emul_set_lane_global(second_chance)
    emul_lib.mmp_emul_set_lane_budget(64)
    try:
        fl = fleet_for(config, nm, ni, seed)
        o = oracle_from_synth(fl)
        s = solver_from_synth(fl, emul_lib)
        emul_lib.mmp_emul_lane_bails(None)
        sd = make_decisions(fl, 2000, seed)
        compare_decisions(fl, sd, o, s, seed=seed * 13, full_lists=False)
        sd = make_decisions(fl, 1500, seed + 1, sweep=True, plain=True)
        compare_decisions(fl, sd, o, s, seed=seed, full_lists=False)
        n = C.c_long()
        bails = emul_lib.mmp_emul_lane_bails(C.byref(n))
        assert n.value > 0
        if window == 1 and ni >= 300 and not second_chance:
            assert bails > 0
    finally:
        emul_lib.mmp_emul_set_window(32)
        emul_lib.mmp_emul_set_lane_global(1)
        emul_lib.mmp_emul_set_lane_window(12)
        emul_lib.mmp_emul_set_lane_budget(48)


@pytest.mark.parametrize("window,budget", [(12, 192), (0, 1000), (3, 400)])
@pytest.mark.parametrize("config,nm,ni,seed", [("C5", 900, 10000, 5), ("C5", 900, 5000, 6), ("C3", 900, 10000, 3)])
def test_long_walks_match_oracle(emul_lib, oracle_lib, config, nm, ni, seed, window, budget):
    """Rows of 160-320 words with the budgets the kernels run with: walks of a hundred and more steps beyond the window go
    through the chunk machinery of decide_stream (8 list entries gathered at a time; a chunk none of whose steps can stop the
    walk is taken at once), a full best instance is handled by the lane routine (simple case).  window 0 = k_place_small."""
    import ctypes as C
    emul_lib.mmp_emul_lane_bails.restype = C.c_long
    emul_lib.mmp_emul_set_window(2)
    emul_lib.mmp_emul_set_lane_window(window)
    emul_lib.mmp_emul_set_lane_global(1)
    emul_lib.mmp_emul_set_lane_budget(budget)
    try:
        fl = make_fleet(config, nm, ni, seed)
        o = oracle_from_synth(fl)
        s = solver_from_synth(fl, emul_lib)
        emul_lib.mmp_emul_lane_bails(None)
        for plain in (True, False):
            sd = make_decisions(fl, 900, seed, sweep=plain, plain=plain)
            compare_decisions(fl, sd, o, s, seed=seed + 5, full_lists=False)
        n = C.c_long()
        bails = emul_lib.mmp_emul_lane_bails(C.byref(n))
        assert n.value > 0 and bails < n.value // 4  # the lane routine itself answers (almost) all of them
    finally:
        emul_lib.mmp_emul_set_window(32)
        emul_lib.mmp_emul_set_lane_window(12)
        emul_lib.mmp_emul_set_lane_budget(48)
