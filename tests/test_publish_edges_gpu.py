"""The device's end-of-window republish (k_churn_republish, phase E of mmp_churn_step) at every threshold of
publishInstanceRecord (MM:5390-5470): the pairs of tests/publish_edges.py stepped through the device loop and the oracle's
(churn_harness.compare_window), each pod's new record as tests/publish_rule.py restates it from the Java text, then a
second window and a placement batch that read what was published.  Also the kernel's shapes: one warp per pod, four pods
per block, the oldest entry by a warp reduction over the slots."""
import numpy as np
import pytest

import publish_edges as pe
from churn_harness import build, compare_window
from helpers import same_answers
from modelmesh_b200 import _lib as L
from oracle import binding as ob

pytestmark = pytest.mark.gpu

PAIRS = pe.all_pairs()
FREE = pe.event_free(PAIRS)
SEED = 11
KEEP = ("rpm", "l_threads", "vers", "start_time")


def _caches(sim, s, pods):
    """each pod's cache after the window, the same on both sides"""
    oldest_p, weighted_p, count_p = s.lru_state()
    out = []
    for i, p in enumerate(pods):
        c = pe.cache_of(sim, i, p.cap)
        assert (int(oldest_p[i]), int(weighted_p[i]), int(count_p[i])) == ((-1 if c[3] is None else c[3]), c[1], c[2]), (i, c)
        out.append(c)
    return out


def _check(before, rows_p, pub, want, n_published, what, present=None):
    """rows of the pods in the table as publish_rule; the changed rows exactly the published ones that changed; fields a
    republish does not write untouched; n_published as publish_rule"""
    keep = np.ones(len(want), dtype=bool) if present is None else present
    idx = np.nonzero(keep)[0]
    pe.same_rows(rows_p[idx], [want[i] for i in idx], what)
    changed = {int(i) for i in idx if any(int(rows_p[i][k]) != int(before[i][k]) for k in pe.publish_rule.FIELDS)}
    assert changed == {int(i) for i in idx if pub[i] and any(want[i][k] != int(before[i][k]) for k in pe.publish_rule.FIELDS)}, what
    for k in KEEP:
        assert np.array_equal(rows_p[k][idx], before[k][idx]), (what, k)
    assert n_published == int(pub.sum()), (what, n_published, int(pub.sum()))


def device_run(product_lib, pods, last_done, force, slots=128, removed=()):
    """one window of both loops over a fleet of `pods`, checked against publish_rule; returns (bool[n] published, rows
    afterwards, the run, oracle fleet, oracle loop, device fleet)"""
    r = pe.build_run(pods, last_done, force, removed=removed)
    fl = r.w.fleet
    o, sim, s = build(product_lib, r.w, slots, r.last_published)
    present = np.ones(len(pods), dtype=bool)
    for i in r.updates:  # the published capacity differs from the cache's (mmp_churn_init sized it from the row)
        s.instance_update(i, r.rows[i])
        o.instance_event(ob.UPDATED, i, r.rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i], pe.NOW0)
    for i in removed:
        s.instance_remove(i)
        o.instance_event(ob.DELETED, i, None, fl.inst_ids[i], now_ms=pe.NOW0)
        present[i] = False
    if r.updates or len(removed):
        s.commit()
    what = (last_done, "forced" if force is True else "", len(pods), slots)
    if len(removed):  # the rows of a pod out of the table are not compared: the oracle reports none
        _, _, rows_o, npub_o, _ = sim.step(r.events, pe.NOW0, pe.NOW1, SEED)
        _, _, rows_p, rep = s.churn_step(r.events, pe.NOW0, pe.NOW1, SEED)
        for k in pe.publish_rule.FIELDS:
            assert np.array_equal(rows_p[k][present], rows_o[k][present]), (what, k)
        assert rep.n_published == npub_o, (what, rep.n_published, npub_o)
        assert np.array_equal(s.cluster_order(), o.cluster_order()), what
    else:
        out = {}
        _, _, rep = compare_window(0, o, sim, s, r.events, pe.NOW0, pe.NOW1, SEED, out=out)
        rows_p = out["rows_p"]
    caches = _caches(sim, s, pods)
    pub, want = pe.expected(r.rows, [r.last_published] * len(pods), r.forced, caches, present)
    _check(r.rows, rows_p, pub, want, rep.n_published, what, present)
    assert not pub[~present].any()
    return pub, rows_p[:len(pods)].copy(), r, o, sim, s


def second_window(r, o, sim, s, pub1, rows1):
    """2 s later, a REMOVE of the newest entry of every third event-free pod: a pod that just published republishes only
    if that forces it (its lastPublished moved to NOW1), every pod as publish_rule"""
    now0, now1 = pe.NOW1, pe.NOW1 + 2_000
    forced = [i for i, p in enumerate(r.pods) if p.event is None and p.entries and i % 3 == 0]
    ev = np.zeros(len(forced), dtype=L.CHURN_EVENT)
    for k, i in enumerate(forced):
        j = max(range(len(r.pods[i].entries)), key=lambda x: r.pods[i].entries[x][0])
        ev[k]["type"], ev[k]["model"], ev[k]["caller"], ev[k]["t"] = 1, r.entry_models[i][j], i, now0 + 10 + k
    out = {}
    _, _, rep = compare_window(1, o, sim, s, ev, now0, now1, SEED + 1, out=out)
    caches = _caches(sim, s, r.pods)
    last = [pe.NOW1 if pub1[i] else r.last_published for i in range(len(r.pods))]
    pub2, want = pe.expected(rows1, last, set(forced), caches, now=now1)
    _check(rows1, out["rows_p"], pub2, want, rep.n_published, "second window")
    assert set(np.nonzero(pub2 & pub1)[0]) <= set(forced)
    return pub2


def placement_after(r, o, s, now):
    """a batch placed on the spare models reads the republished records: device and oracle agree"""
    n = 96
    dec = np.zeros(n, dtype=L.DECISION_IN)
    dec["model"] = r.spare[np.arange(n) % len(r.spare)]
    dec["self"] = np.arange(n) % len(r.pods)
    dec["last_used"] = now - (np.arange(n) * 997_331) % (12 * pe.HOUR)
    dec["fresh"] = -1
    od = np.zeros(n, dtype=ob.DECISION)
    od["type_idx"], od["self"], od["fresh_idx"], od["last_used"] = 0, dec["self"], -1, dec["last_used"]
    od["decision_id"] = np.arange(n, dtype=np.uint64)
    want = o.get_next_batch(od, r.w.fleet.type_names, np.zeros(n + 1, dtype=np.int64), np.zeros(0, dtype=np.int32), now, 5)
    got = s.place_batch(dec, now, 5)
    same_answers(got, want, "placement after the republish")
    assert np.count_nonzero(want["target"] != -1) > n // 2  # placed (an instance or ORC_SELF)


@pytest.fixture(scope="module")
def pair_runs(product_lib, oracle_lib):
    pods = pe.pods_of(PAIRS)
    out = {}
    for run in pe.RUNS:
        pub, rows1, r, o, sim, s = device_run(product_lib, pods, *run)
        pub2 = second_window(r, o, sim, s, pub, rows1)
        if run in ((39_000, False), (160_001, True)):
            placement_after(r, o, s, pe.NOW1 + 2_000)
        out[run] = (pub, pub2)
    return out


def test_pairs_on_the_device(pair_runs):
    assert set(pair_runs) == set(pe.RUNS)
    assert any(p[1].any() & p[0].any() for p in pair_runs.values())


@pytest.mark.parametrize("k", range(len(PAIRS)), ids=[p.name for p in PAIRS])
def test_pair_sides_differ_on_the_device(pair_runs, k):
    pe.check_pairs([PAIRS[k]], {run: pub[0][2 * k:2 * k + 2] for run, pub in pair_runs.items()})


@pytest.mark.parametrize("slots", [1, 31, 32, 33, 65])
def test_slot_counts(product_lib, oracle_lib, slots):
    """caches holding exactly slots_per_instance entries, seeded newest first so that the oldest sits in the last slot,
    published 19999 and 20000 ms off it; then the pairs that fit"""
    full = pe.ents(slots)[::-1]
    t0 = full[-1][0]
    pods = [pe.pod(full, lru_time=t0 - 19_999), pe.pod(full, lru_time=t0 - 20_000), pe.pod(full, count=slots + 1),
            pe.pod(full, l_in_prog=1)]
    fit = [p for p in FREE if max(len(p.a.entries), len(p.b.entries)) <= slots]
    pub, *_ = device_run(product_lib, pods + pe.pods_of(fit), 39_000, False, slots=slots)
    assert list(pub[:2]) == [False, True] and pub[3], pub[:4]
    pe.check_pairs(fit, {(39_000, False): pub[len(pods):]})


@pytest.mark.parametrize("n", [1, 3, 4, 5, 129])
def test_pod_counts(product_lib, oracle_lib, n):
    """fleets of n pods, every pod forced: the last block of four partial (n = 129: one pod in it)"""
    free = pe.pods_of(FREE)
    pods = [free[k % len(free)] for k in range(n)]
    pub, *_ = device_run(product_lib, pods, 39_000, True)
    if n >= 5:
        assert 0 < pub.sum() < n


def test_removed_pod_is_not_republished(product_lib, oracle_lib):
    """pods that left the table: neither loop republishes them, though their caches say to"""
    pods = pe.pods_of(FREE)[:24]
    r0, *_ = device_run(product_lib, pods, 160_001, False)
    gone = [i for i in np.nonzero(r0)[0][:3]]
    assert len(gone) == 3
    pub, *_ = device_run(product_lib, pods, 160_001, False, removed=gone)
    assert not pub[gone].any() and pub.sum() == r0.sum() - 3
