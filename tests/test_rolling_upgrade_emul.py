"""CPU checks of placement on fleets in a rolling upgrade (test_rolling_upgrade_gpu.upgrade): the product's host code and
the decision routine (tests/emul) against the oracle, and the two-pass path's slot summaries across the version boundary."""
import numpy as np
import pytest

from helpers import compare_decisions, oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200._lib import DF_FAVOUR_SELF
from modelmesh_b200.synth import make_decisions, make_fleet
from split_place import oracle_same, place_split, split_lib  # noqa: F401 (split_lib: fixture)
from upgrade import PATTERNS, check_total_order, full_best_then_room, upgrade, versions

# fleets whose slot summaries reach past the newer pods (long shortlists: C5's near-full fleet, MIX's low counts, a saturated
# front); elsewhere a summary's best and shortlist lie among the newer pods
CROSSING = {("C5", "half"), ("C5", "three"), ("C5", "saturated"), ("MIX", "half"), ("MIX", "three"), ("MIX", "saturated"), ("C3", "saturated")}
CONFIGS = [("C3", 3000, 1300, 33), ("C5", 1500, 500, 5), ("MIX", 800, 300, 14), ("MIX", 800, 700, 41), ("C2", 2000, 400, 2)]


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("config,nm,ni,seed", CONFIGS)
def test_upgrade_decisions_match_oracle(emul_lib, oracle_lib, config, nm, ni, seed, pattern):
    """Cluster order, then traced decisions with both candidate planes and the untraced batch of a mixed batch and a sweep;
    the saturated pattern reaches a full best with instances with room after it, the replicaset roll the filter retry."""
    fl = upgrade(make_fleet(config, nm, ni, seed), pattern, seed)
    o = oracle_from_synth(fl)
    check_total_order(fl, o, seed)
    assert len(versions(fl)) == (3 if pattern == "three" else 2)
    s = solver_from_synth(fl, emul_lib)
    assert np.array_equal(s.cluster_order(), o.cluster_order())
    _, out, tr = compare_decisions(fl, make_decisions(fl, 2000, seed), o, s, seed=seed * 7919)
    _, out_w, tr_w = compare_decisions(fl, make_decisions(fl, 1500, seed + 1, sweep=True, plain=True), o, s, seed=seed)
    if pattern == "saturated":
        assert full_best_then_room(fl, tr, out) + full_best_then_room(fl, tr_w, out_w) > (20 if config != "MIX" else 0)
    if pattern == "rsroll" and config == "C3":
        assert np.count_nonzero(tr["flags"] & L.TF_RS_RETRY) + np.count_nonzero(tr_w["flags"] & L.TF_RS_RETRY) > 20
    s.close()


@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("config,nm,ni,seed", CONFIGS)
def test_upgrade_split_summaries(split_lib, oracle_lib, config, nm, ni, seed, pattern):
    """The slot summaries of the two-pass path on upgrade fleets: every answer from a summary equals the walk and the
    oracle, and where a pattern moves a share of the fleet some summaries and the decisions they answer span versions."""
    fl = upgrade(make_fleet(config, nm, ni, seed), pattern, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, split_lib)
    sweep = make_decisions(fl, 3000, seed, sweep=True, plain=True)
    fav = make_decisions(fl, 2000, seed + 3, sweep=True, plain=True)
    fav.dec["flags"] |= DF_FAVOUR_SELF
    total = np.zeros(6, dtype=np.int64)
    for k, sd in enumerate((sweep, fav, make_decisions(fl, 2000, seed + 1))):
        out, counts = place_split(split_lib, s, sd, fl.now_ms, seed + k)
        assert counts[1] == 0, (config, pattern, k, counts)
        oracle_same(o, fl, sd, out, seed + k)
        total += counts
    assert total[0] > 0
    if (config, pattern) in CROSSING:
        assert total[4] > 0 and total[5] > 0, total
    s.close()
