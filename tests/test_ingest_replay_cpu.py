"""Replayed ingest streams (tests/replay.py) on the CPU harness, against the oracle rebuilt from scratch at every commit.

The harness compiles the library's host-side ingest (host_state.hpp) and rebuilds its snapshot from those tables at every
commit, so this checks the host bookkeeping of an evolving fleet: instances removed, re-added under new pod ids and at
never-used indices; models entering and leaving the overflow map; the id table and JSON model records resolved by pod id
after a pod re-registers at another index; type-config and replicaset changes; registry rows past the old end that were
never upserted."""
import numpy as np
import pytest

from modelmesh_b200.synth import make_fleet
from replay import NUMERIC, SCHEDULE, STRUCTURAL, Replay, check_against_oracle, describe, run_window


@pytest.mark.parametrize("config,nm,ni,seed,n_windows", [("C3", 2500, 1200, 3, 10), ("C5", 2000, 600, 5, 8), ("MIX", 1500, 300, 14, 12),
                                                         ("MIX", 1500, 160, 41, 8)])
def test_replayed_stream_matches_oracle(emul_lib, oracle_lib, config, nm, ni, seed, n_windows):
    rp = Replay(make_fleet(config, nm, ni, seed), emul_lib, seed)
    n0 = rp.n_used
    check_against_oracle(rp, seed, 300, 1500)
    for w in range(n_windows):
        run_window(rp, w)
        check_against_oracle(rp, seed * 100 + w, 300, 1500)
    kinds = [k for k, _, _, _ in rp.windows]
    assert kinds.count(NUMERIC) >= 4 and kinds.count(STRUCTURAL) >= 4, describe(rp)
    # the stream did what it is for: the registry grew with gaps, instances came and went, JSON records are held by id
    assert rp.n_used > n0 and (~rp.present[:rp.n_ever]).any() and rp.n_ever > ni and rp.json_ids, describe(rp)
    assert any(len(e) > 4 for e in rp.current_edges()), describe(rp)
    print(f"{config} {ni}x{nm}: {rp.n_compared} decisions compared over {len(rp.windows)} windows: {describe(rp)}")


def test_schedule_covers_both_paths_and_every_event():
    kinds = [k for k, _ in SCHEDULE]
    assert kinds.count(NUMERIC) == kinds.count(STRUCTURAL)
    events = {e for k, spec in SCHEDULE if k == STRUCTURAL for e in spec}
    assert events == {"remove", "reuse", "add", "reregister", "toggle", "relabel", "types", "replicasets"}
    assert any(spec == "all_dirty" for k, spec in SCHEDULE if k == NUMERIC)
    assert any(isinstance(spec, dict) and spec.get("overflow") is False for _, spec in SCHEDULE)
    assert any(isinstance(spec, dict) and spec.get("n_growth") for _, spec in SCHEDULE)
