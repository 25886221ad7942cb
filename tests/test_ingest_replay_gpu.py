"""Replayed ingest streams (tests/replay.py) on the CUDA library.

A fleet reaches every epoch through a chain of ingest calls and commits.  Numeric instance updates and model-record
edits take the device path of a commit (only the dirty rows are scattered into the device-resident tables, then the
bitmap and excl_ranks are rebuilt from them); everything else takes the host path.  After every commit of every stream
the fleet is compared with the oracle rebuilt from scratch (cluster order, traced decisions with candidate masks,
untraced batches through k_place_direct, a slot-sorted batch of 8 192+ decisions, a sweep of the whole registry) and
with a fresh fleet loaded with one commit (byte-identical batches and sweeps, partition stats, reaper selections,
registry prune)."""
import numpy as np
import pytest

from helpers import compare_decisions
from modelmesh_b200.synth import LONG_MAX, make_fleet
from replay import (NUMERIC, STRUCTURAL, Replay, assert_same_results, check_against_oracle, check_against_scratch,
                    check_sorted_batch, describe, oracle_batch, run_window)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("config,nm,ni,seed,n_windows", [("C3", 3000, 2000, 3, 10), ("C5", 2500, 1500, 5, 10), ("MIX", 2000, 400, 14, 12),
                                                         ("C3", 2500, 10240, 7, 5)])
def test_replayed_stream_matches_oracle_and_scratch(product_lib, oracle_lib, config, nm, ni, seed, n_windows):
    rp = Replay(make_fleet(config, nm, ni, seed), product_lib, seed)
    n0 = rp.n_used
    for w in range(n_windows):
        run_window(rp, w)
        check_against_oracle(rp, seed * 100 + w, 500, 3000)
        check_sorted_batch(rp, seed * 100 + w)
        check_against_scratch(rp, seed * 100 + w)
    paths = [(k, p) for k, p, _, _ in rp.windows]
    assert (NUMERIC, 2) in paths and (STRUCTURAL, 1) in paths, describe(rp)  # each window took the path its kind implies
    assert rp.n_used > n0 and (~rp.present[:rp.n_ever]).any() and rp.json_ids, describe(rp)
    print(f"{config} {ni}x{nm}: {rp.n_compared} decisions compared over {len(rp.windows)} windows: {describe(rp)}")


def test_registry_growth_on_the_device_path(product_lib, oracle_lib):
    """Models upserted well past n_models_used in a window that commits on the device path: the rows in between were never
    upserted, so they must read as the host holds them (a zero row, no edges) -- nothing excluded, no copies.  Instance 0
    is live and the emptiest instance, the best answer for every one of those rows: a row whose edges read as instance 0
    would exclude it."""
    fl = make_fleet("C2", 1500, 600, 23)
    fl.inst_rows[0]["used"], fl.inst_rows[0]["count"], fl.inst_rows[0]["lru_time"] = 0, 0, LONG_MAX
    fl.inst_rows[0]["shutting_down"], fl.inst_rows[0]["active"] = 0, 1
    rp = Replay(fl, product_lib, 23, max_models=8000)
    assert rp.f.commit_info()[0] == 1
    # one pod leaves (host path): the copies it held are what the registry prune below finds
    held = np.bincount(fl.edge_inst, minlength=fl.n_instances)
    held[0] = 0
    rp.remove(int(np.argmax(held)))
    rp.commit(STRUCTURAL, 0, ["remove"])
    n0 = rp.n_used
    grown = (n0 + 150, n0 + 1100, n0 + 1101, n0 + 3000, n0 + 6200)
    for m in grown:
        rp.upsert_model(m, [int(x) for x in rp.rng.choice(np.arange(1, 600), size=3, replace=False)])
    rp.update_numeric(5)
    rp.commit(NUMERIC, len(grown))  # asserts the device path
    gaps = np.asarray([m for m in range(n0, rp.n_used) if m not in grown])
    assert len(gaps) > 6000 and not rp.mrow[gaps].tobytes().strip(b"\0")
    v, o = rp.view(), rp.oracle()
    # a sweep of the whole registry, against the oracle and against a fresh fleet
    rng = np.random.default_rng(1)
    live = rp._live()
    self_idx = live[rng.integers(1, len(live), size=rp.n_used)].astype(np.int32)
    fav = rng.uniform(size=rp.n_used) < 0.3
    got = rp.f.place_sweep(0, rp.n_used, self_idx, rp.now, 7, favour=fav)
    want = oracle_batch(v, rp.sweep_decisions(self_idx, fav), o, 7)
    assert_same_results(got, want, "sweep")
    # the never-upserted rows: no exclusions, so instance 0 is the best instance of each of their decisions
    sd = rp.decisions(3000, 5, plain=True, models=gaps[rng.integers(0, len(gaps), size=3000)])
    sd.dec["self"] = live[rng.integers(1, len(live), size=3000)]
    ores, out, tr = compare_decisions(v, sd, o, rp.f, seed=11)
    assert (ores["best"] == 0).all() and (tr["best"] == 0).all()
    assert_same_results(rp.f.place_batch(sd.dec, rp.now, 11), ores, "gap batch")
    # reaper and registry prune read the registry rows themselves: a leftover that is not zero shows here
    assert check_against_scratch(rp, 13) > 0  # models pruned of the pod that left, the same in both fleets
    o.close()
