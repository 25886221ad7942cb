"""The oracle's end-of-window republish (publishNeeded and phase E of oracle/mm_sim.inc, and phase E's copy in
tests/emul/reaper_sim.cpp) against publishInstanceRecord restated from the Java text (tests/publish_rule.py), at every
threshold (tests/publish_edges.py) and on random pods."""
import numpy as np
import pytest

import publish_edges as pe
from churn_harness import build_oracle
from oracle import binding as ob
from reaper_oracle import _reaper_oracle_so, reaper_oracle, with_reaper  # noqa: F401

PAIRS = pe.all_pairs()
SEED = 11


def oracle_run(pods, last_done, force, reaper=False):
    """one window of the oracle's loop over a fleet of `pods`, checked pod by pod against publish_rule; returns
    (bool[n] published, the run, the oracle's decisions, evictions)"""
    r = pe.build_run(pods, last_done, force)
    fl = r.w.fleet
    o, sim = build_oracle(r.w, r.last_published)
    if reaper:
        sim = with_reaper(sim, fl.n_models)
    for i in r.updates:  # the published capacity differs from the cache's
        o.instance_event(ob.UPDATED, i, r.rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i], pe.NOW0)
    dec, evi, rows, npub, _ = sim.step(r.events, pe.NOW0, pe.NOW1, SEED)
    caches = [pe.cache_of(sim, i, p.cap) for i, p in enumerate(pods)]
    forced = set(r.forced)
    pub, want = pe.expected(r.rows, [r.last_published] * len(pods), forced, caches)
    pe.same_rows(rows, want, (last_done, force))
    assert npub == int(pub.sum()), (last_done, force, npub, int(pub.sum()))
    # the fleet is the one it was built to be: caches as designed, every force source fired
    for i, p in enumerate(pods):
        if p.event is None:
            assert caches[i] == pe.designed_cache(p), (i, caches[i], pe.designed_cache(p))
        elif p.event == "evict":
            assert i in set(int(x) for x in evi["instance"]), i
        elif p.event == "load":
            k = np.nonzero((dec["self"] == i) & (dec["status"] == ob.SIM_ACCEPTED))[0]  # target: i or ORC_SELF (-2)
            assert len(k) == 1 and int(dec["target"][k[0]]) in (i, -2), (i, dec[k])
        elif p.event == "remove":
            assert caches[i][2] == len(p.entries) - 1, (i, caches[i])
        else:
            assert caches[i] == pe.designed_cache(p), (i, caches[i])
    return pub, r, dec, evi


@pytest.fixture(scope="module")
def pair_runs(oracle_lib):
    pods = pe.pods_of(PAIRS)
    return {run: oracle_run(pods, *run)[0] for run in pe.RUNS}


def test_pairs_match_the_restatement(pair_runs):
    """every pod of every pair on every lastDone x force fleet: rows and n_published as publish_rule (inside oracle_run)"""
    assert set(pair_runs) == set(pe.RUNS)
    assert any(p.any() for p in pair_runs.values()) and not all(p.all() for p in pair_runs.values())


@pytest.mark.parametrize("k", range(len(PAIRS)), ids=[p.name for p in PAIRS])
def test_pair_sides_differ(pair_runs, k):
    pe.check_pairs([PAIRS[k]], {run: pub[2 * k:2 * k + 2] for run, pub in pair_runs.items()})


def test_gates_close_everything(pair_runs):
    """lastDone 1999 publishes nothing even when forced; 38999 without force nothing"""
    assert not pair_runs[(1_999, True)].any() and not pair_runs[(1_999, False)].any()
    forced_only = [i for i, p in enumerate(pe.pods_of(PAIRS)) if p.event in ("evict", "load", "remove")]
    assert set(np.nonzero(pair_runs[(38_999, False)])[0]) <= set(forced_only)


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_random_pods_match_the_restatement(oracle_lib, seed):
    """600 random pods per seed, each a few units around every threshold, a random half of them forced"""
    rng = np.random.default_rng(100 + seed)
    pods = pe.random_pods(600, seed)
    last_done = int(rng.choice(list(pe.LAST_DONE) + [int(rng.integers(2_000, 170_000))]))
    force = set(int(i) for i in np.nonzero(rng.random(len(pods)) < 0.5)[0])
    pub, *_ = oracle_run(pods, last_done, force)
    if last_done >= 2_000:
        assert 0 < pub.sum() < len(pods), (last_done, int(pub.sum()))


@pytest.mark.usefixtures("reaper_oracle")
@pytest.mark.parametrize("run", [(2_000, False), (39_000, False), (160_000, True), (160_001, False)])
def test_reaper_sim_phase_e_matches_the_restatement(run, pair_runs):
    """the copy of phase E in tests/emul/reaper_sim.cpp (orc_sim_step_reaper, a trace without REAPER events): every pair
    pod as publish_rule, and the same answers as the oracle's own loop"""
    pub, *_ = oracle_run(pe.pods_of(PAIRS), *run, reaper=True)
    assert np.array_equal(pub, pair_runs[run])
