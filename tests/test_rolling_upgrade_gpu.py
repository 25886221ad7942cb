"""Fleets in a rolling upgrade, on the CUDA library against the oracle.

During an upgrade some pods run a newer instance version.  With realistic lruTimes the version clause of PLACEMENT_ORDER
(MM:4663-4665, quirk N1) puts every newer-version instance ahead of every older one, full or not, so the order changes
shape: the full instances no longer form one suffix, counts and lruTimes restart at the version boundary, and a full best
can be followed by non-full candidates.  A commit whose live set holds more than one version leaves the device path for
the host's merge sort (path 1); the closed loop must then build that commit from the device's instance rows and registry.

upgrade() and fleet_for() build the fleets; the CPU side of these tests is test_rolling_upgrade_emul.py."""
import dataclasses

import numpy as np
import pytest

from exclude_set import oracle_excluding
from helpers import compare_decisions, oracle_from_synth, oracle_inputs_fast, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import LONG_MAX, SynthFleet, make_churn, make_decisions, make_fleet
from oracle import binding as ob
from replay import STRUCTURAL, Replay, check_against_oracle, check_against_scratch, check_sorted_batch, describe

pytestmark = pytest.mark.gpu

PATTERNS = ("canary", "half", "rsroll", "saturated", "three")
NEW_RS = "mmupgr"  # the replicaset prefix of the pods an rsroll upgrade brings up


# ---------------------------------------------------------------------------------------------------------------
# upgrade fleets
# ---------------------------------------------------------------------------------------------------------------
def upgrade(fl: SynthFleet, pattern: str, seed: int) -> SynthFleet:
    """fl with some of its pods moved to newer versions:
      canary     one to three live pods on vers + 1
      half       about half of the pods, drawn at random
      rsroll     up to a tenth of the pods, drawn among those without labels, on vers + 1 under the new replicaset
                 prefix NEW_RS; every old prefix is listed as likely-replaced (UpgradeTracker, MM:4769-4770): a type that
                 requires a label has every candidate flagged, and the candx filter is retried across the boundary
      saturated  about a third of the pods on vers + 1, every one of them full with an lruTime hours old: the best is
                 full and non-full older pods follow it
      three      three versions (about 50 / 30 / 20 %)
    Every full instance keeps an lruTime above 2 * minChurnAgeMs, so the comparator stays a strict total order."""
    rng = np.random.default_rng(seed ^ 0x5EED)
    rows = fl.inst_rows.copy()
    ni = len(rows)
    v0 = int(rows["vers"][0])
    assert (rows["vers"] == v0).all()
    ids, replaced = list(fl.inst_ids), list(fl.replaced_replicasets)
    live = np.nonzero(rows["shutting_down"] == 0)[0]
    if pattern == "canary":
        rows["vers"][rng.choice(live, size=int(rng.integers(1, 4)), replace=False)] = v0 + 1
    elif pattern == "half":
        rows["vers"][rng.uniform(size=ni) < 0.5] = v0 + 1
    elif pattern == "rsroll":
        pool = [int(i) for i in live if not fl.inst_labels[i]] or list(live)
        new = rng.choice(pool, size=max(1, min(len(pool), ni // 10)), replace=False)
        rows["vers"][new] = v0 + 1
        for i in new:
            ids[i] = f"{NEW_RS}-{i:05x}"
        replaced = sorted({ids[i][:6] for i in range(ni) if len(ids[i]) >= 7 and not ids[i].startswith(NEW_RS)})
    elif pattern == "saturated":
        new = np.nonzero(rng.uniform(size=ni) < 0.33)[0]
        rows["vers"][new] = v0 + 1
        rows["used"][new] = rows["capacity"][new] - rng.integers(0, fl.min_space_units, size=len(new))
        rows["lru_time"][new] = fl.now_ms - rng.integers(3_600_000, 12 * 3_600_000, size=len(new))
    elif pattern == "three":
        u = rng.uniform(size=ni)
        rows["vers"] = v0 + (u < 0.5) + (u < 0.2)
    else:
        raise ValueError(pattern)
    return dataclasses.replace(fl, inst_rows=rows, inst_ids=ids, replaced_replicasets=replaced)


def fleet_for(config: str, nm: int, ni: int, seed: int) -> SynthFleet:
    """make_fleet(config) or, for "BASE/pattern", make_fleet(BASE) in that rolling upgrade"""
    base, _, pattern = config.partition("/")
    fl = make_fleet(base, nm, ni, seed)
    return upgrade(fl, pattern, seed) if pattern else fl


def check_total_order(fl: SynthFleet, o: ob.OracleFleet, seed: int, n: int = 3000):
    """No full live instance at or below 2 * minChurnAgeMs (N1's non-transitive corner), and the oracle's comparator
    is antisymmetric and transitive on sampled triples of live instances."""
    r = fl.inst_rows
    live = np.nonzero(r["shutting_down"] == 0)[0]
    full = (np.maximum(0, r["capacity"] - r["used"]) < fl.min_space_units)[live]
    assert not (full & (r["lru_time"][live] <= 2 * fl.min_churn_age_ms)).any()
    rng = np.random.default_rng(seed)
    for a, b, c in live[rng.integers(0, len(live), size=(n, 3))]:
        a, b, c = int(a), int(b), int(c)
        if len({a, b, c}) < 3:
            continue
        ab, bc, ac = o.compare(a, b), o.compare(b, c), o.compare(a, c)
        assert np.sign(ab) == -np.sign(o.compare(b, a)) != 0, (a, b)
        if ab < 0 and bc < 0:
            assert ac < 0, (a, b, c)
        if ab > 0 and bc > 0:
            assert ac > 0, (a, b, c)


def versions(fl: SynthFleet) -> np.ndarray:
    return np.unique(fl.inst_rows["vers"][fl.inst_rows["shutting_down"] == 0])


def full_best_then_room(fl: SynthFleet, tr: np.ndarray, out: np.ndarray) -> int:
    """decisions whose best is full and whose answer is an instance with room: non-full candidates after a full best"""
    r = fl.inst_rows
    t = out["target"]
    ok = (t >= 0) & ((tr["flags"] & L.TF_BEST_FULL) != 0)
    room = np.zeros(len(t), dtype=bool)
    room[ok] = (r["capacity"][t[ok]] - r["used"][t[ok]]) >= fl.min_space_units
    return int(np.count_nonzero(room))


def _kw(sd):
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


def _oracle(fl, sd, o, seed, candidates=False):
    od, off, idx = oracle_inputs_fast(fl, sd)
    return o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None,
                            want_candidates=candidates)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


# ---------------------------------------------------------------------------------------------------------------
# placement
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pattern", PATTERNS)
@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 4000, 3000, 3), ("C5", 3000, 2000, 5), ("MIX", 1500, 700, 14), ("C2", 3000, 1000, 2)])
def test_upgrade_decisions_match_oracle(product_lib, oracle_lib, monkeypatch, config, nm, ni, seed, pattern):
    """Traced decisions with both candidate planes, the traced fast path and the untraced batch (helpers.compare_decisions),
    then k_place_lanes on a second fleet, on every upgrade pattern."""
    fl = upgrade(make_fleet(config, nm, ni, seed), pattern, seed)
    o = oracle_from_synth(fl)
    check_total_order(fl, o, seed)
    assert len(versions(fl)) == (3 if pattern == "three" else 2)
    s = solver_from_synth(fl, product_lib)
    assert np.array_equal(s.cluster_order(), o.cluster_order())
    assert s.commit_info()[0] == 1
    sd = make_decisions(fl, 3000, seed)
    ores, out, tr = compare_decisions(fl, sd, o, s, seed=seed * 7919)
    sw = make_decisions(fl, 2000, seed + 1, sweep=True, plain=True)
    _, out_w, tr_w = compare_decisions(fl, sw, o, s, seed=seed)
    s.close()
    if pattern == "saturated":  # the full newer pods come first: their best is full, the answer often an older pod with room
        assert full_best_then_room(fl, tr, out) + full_best_then_room(fl, tr_w, out_w) > 0
    if pattern == "rsroll" and config in ("C3", "C5"):  # types whose allowed pods are all flagged: the filter is retried
        assert np.count_nonzero(tr["flags"] & L.TF_RS_RETRY) + np.count_nonzero(tr_w["flags"] & L.TF_RS_RETRY) > 20
    monkeypatch.setenv("MMP_KERNEL", "lanes")
    s = solver_from_synth(fl, product_lib)
    compare_decisions(fl, sd, o, s, seed=seed * 17, full_lists=False)
    compare_decisions(fl, sw, o, s, seed=seed, full_lists=False)
    s.close()


@pytest.mark.parametrize("pattern", PATTERNS)
def test_upgrade_batches_split_sorted_sweep_and_latency(product_lib, oracle_lib, pattern):
    """A 10 000-instance fleet in each upgrade pattern: k_place_direct sweeps and mixed batches of 20-40 k decisions with
    the two-pass path forced on and off (byte-identical, and equal to the oracle), batches around 8 192 decisions with
    sort_slots 0 and 1, mmp_place_sweep against mmp_place_batch, and the four one-decision launch paths against the batch."""
    fl = upgrade(make_fleet("C3", 20_000, 10_000, 3), pattern, 3)
    o = oracle_from_synth(fl)
    check_total_order(fl, o, 3)
    s = solver_from_synth(fl, product_lib)
    lib = product_lib
    vers = fl.inst_rows["vers"]
    crossing = 0
    for k, sd in enumerate((make_decisions(fl, 40_000, 3, sweep=True, plain=True), make_decisions(fl, 30_000, 4))):
        got = {}
        for split in (1, 0):
            s._ck(lib.mmp_tune(s.h, b"split", split))
            got[split] = s.place_batch(sd.dec, fl.now_ms, 7 + k, **_kw(sd))
        s._ck(lib.mmp_tune(s.h, b"split", 2))
        assert got[1].tobytes() == got[0].tobytes(), (pattern, k, int(np.sum(got[1] != got[0])))
        want, coff, cidx, _, _ = _oracle(fl, sd, o, 7 + k, candidates=True)
        _same(got[1], want, (pattern, "split", k))
        # decisions whose best and shortlist hold more than one version
        owner = np.repeat(np.arange(len(sd.dec)), np.diff(coff))
        lo, hi = np.full(len(sd.dec), LONG_MAX), np.full(len(sd.dec), -1)
        np.minimum.at(lo, owner, vers[cidx])
        np.maximum.at(hi, owner, vers[cidx])
        crossing += int(np.count_nonzero((hi >= 0) & (lo != hi)))
    if pattern == "saturated":  # (elsewhere a shortlist on this fleet lies among the newer pods)
        assert crossing > 100, crossing
    for n in (8192 - 1, 8192 + 77):
        sd = make_decisions(fl, n, 11 + n)
        want = _oracle(fl, sd, o, 5)
        for sort in (0, 1):
            s._ck(lib.mmp_tune(s.h, b"sort_slots", sort))
            _same(s.place_batch(sd.dec, fl.now_ms, 5, **_kw(sd)), want, (pattern, "sort_slots", sort, n))
        s._ck(lib.mmp_tune(s.h, b"sort_slots", 2))
    sd = make_decisions(fl, 20_000, 12, sweep=True, plain=True)
    whole = s.place_batch(sd.dec, fl.now_ms, 5)
    fav = (sd.dec["flags"] & L.DF_FAVOUR_SELF) != 0
    assert np.array_equal(s.place_sweep(0, 20_000, sd.dec["self"], fl.now_ms, 5, favour=fav), whole)
    _same(whole, _oracle(fl, sd, o, 5), (pattern, "sweep"))
    sd = make_decisions(fl, 400, 13)
    whole = s.place_batch(sd.dec, fl.now_ms, 11, **_kw(sd))
    for mode in (3, 2, 1, 0):
        s._ck(lib.mmp_tune(s.h, b"one_mode", mode))
        for lo, cnt in ((0, 1), (5, 7), (40, 32), (100, 33)):
            s._ck(lib.mmp_fleet_set_id_base(s.h, lo))
            assert np.array_equal(s.place_batch(sd.dec[lo:lo + cnt], fl.now_ms, 11, **_kw(sd)), whole[lo:lo + cnt]), (pattern, mode, lo)
        s._ck(lib.mmp_fleet_set_id_base(s.h, 0))
    s._ck(lib.mmp_tune(s.h, b"one_mode", 3))
    s.close()


@pytest.mark.parametrize("pattern", ["canary", "rsroll", "saturated", "three"])
def test_exclude_set_moves_best_across_the_boundary(product_lib, oracle_lib, pattern):
    """mmp_place_batch_excluding with a set of every newest-version pod: every answer is an older pod, and each one
    equals the oracle's with the set added to every decision's exclusions."""
    fl = upgrade(make_fleet("C3", 6000, 4000, 9), pattern, 9)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    vers = fl.inst_rows["vers"]
    newest = np.nonzero(vers == vers.max())[0].astype(np.int32)
    for split in (1, 0):
        for sd in (make_decisions(fl, 8192 + 77, 9, sweep=True, plain=True), make_decisions(fl, 3000, 10)):
            s._ck(product_lib.mmp_tune(s.h, b"split", split))
            plain = s.place_batch(sd.dec, fl.now_ms, 5, **_kw(sd))
            got = s.place_batch(sd.dec, fl.now_ms, 5, exclude=newest, **_kw(sd))
            s._ck(product_lib.mmp_tune(s.h, b"split", 2))
            _same(got, oracle_excluding(o, fl, sd, newest, 5), (pattern, split, "exclude"))
            t, t0 = got["target"], plain["target"]
            assert (vers[t[t >= 0]] < vers.max()).all()
            assert np.count_nonzero((t0 >= 0) & (vers[np.maximum(t0, 0)] == vers.max())) > 10  # without the set, best was newer
    s.close()


# ---------------------------------------------------------------------------------------------------------------
# commit paths across an upgrade
# ---------------------------------------------------------------------------------------------------------------
def _bump(rp: Replay, idx, vers: int):
    """mmp_instance_update with a new version and nothing else changed (the same pod, restarted on a new image)"""
    for i in np.atleast_1d(idx):
        r = rp.rows[int(i)].copy()
        r["vers"] = vers
        rp.f.instance_update(int(i), r)
        rp.rows[int(i)] = r


def _check(rp: Replay, seed: int):
    check_against_oracle(rp, seed, 400, 3000)
    check_sorted_batch(rp, seed)
    check_against_scratch(rp, seed)


def test_commit_paths_across_an_upgrade(product_lib, oracle_lib):
    """A replayed stream through a whole upgrade; Replay.commit asserts the path of every commit (mmp_commit_info): the
    device path (2) for numeric windows while the live set holds one version, the host path (1) otherwise."""
    fl = make_fleet("C3", 3000, 2000, 3)
    rp = Replay(fl, product_lib, 3)
    v0 = int(fl.inst_rows["vers"][0])
    paths = []
    # 1. a uniform fleet: numeric windows on the device
    paths.append(rp.numeric_window(n_inst=40, n_models=80)); _check(rp, 1)
    # 2. one pod restarts on the new version (same id, numeric update): the device path finds two versions, falls back
    _bump(rp, rp._live()[7], v0 + 1)
    paths.append(rp.numeric_window(n_inst=40, n_models=80)); _check(rp, 2)
    # 3. new-version pods of a new replicaset join at new indices, the old replicasets are marked likely-replaced
    for k in range(3):
        src = int(rp._live()[k])
        row = rp._arrived(rp.rows[src])
        row["vers"] = v0 + 1
        rp._upsert_instance(rp.n_ever, row, f"{NEW_RS}-u{k:04x}", rp.locs[src], rp.zones[src], rp.labels[src])
    rp.set_replicasets(sorted({p for p in rp.rs_prefixes if p != NEW_RS}))
    paths.append(rp.commit(STRUCTURAL, 0, ["upgrade"])); _check(rp, 3)
    # 4. numeric windows while versions are mixed
    for w in range(2):
        paths.append(rp.numeric_window(n_inst=40, n_models=80, n_json=3)); _check(rp, 4 + w)
    # 5. the last old pods are bumped: back on the device path
    live = rp._live()
    _bump(rp, live[rp.rows["vers"][live] == v0], v0 + 1)
    paths.append(rp.numeric_window(n_inst=20, n_models=40)); _check(rp, 6)
    paths.append(rp.numeric_window(n_inst=20, n_models=40)); _check(rp, 7)
    # an odd version held only by a shutting-down pod does not force the host path
    i = int(rp._live()[11])
    rp.toggle(i, "shutting_down")
    paths.append(rp.commit(STRUCTURAL, 0, ["toggle"])); _check(rp, 8)
    _bump(rp, i, v0 + 5)
    paths.append(rp.numeric_window(n_inst=20, n_models=40)); _check(rp, 9)
    assert paths == [2, 1, 1, 1, 1, 2, 2, 1, 2], describe(rp)


# ---------------------------------------------------------------------------------------------------------------
# the closed loop
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_types,fill,seed", [(False, 0.90, 4), (True, 0.90, 5), (False, 0.97, 6), (True, 0.97, 7)])
def test_closed_loop_on_an_upgrade_fleet(product_lib, oracle_lib, with_types, fill, seed):
    """12 windows of the closed loop with about half of the pods on vers + 1, event for event against the oracle's loop;
    every window's commit takes the host path (the live set holds two versions)."""
    from test_churn_gpu import run_small_closed_loop
    w = make_churn(20_000, 200, seed, fill=fill, with_types=with_types)
    w = dataclasses.replace(w, fleet=upgrade(w.fleet, "half", seed))
    assert len(versions(w.fleet)) == 2
    run_small_closed_loop(product_lib, with_types, fill, seed, slots=256, w=w, path=1)


def test_closed_loop_commit_host_only(product_lib, oracle_lib):
    """The closed loop on a uniform fleet with every commit on the host path (mmp_tune "commit_host_only"): equal to
    the oracle window by window, and byte for byte to a twin fleet whose commits take the device path."""
    from test_churn_gpu import _build, _compare_window
    w = make_churn(20_000, 200, 4, fill=0.90)
    fl = w.fleet
    o, sim, s = _build(product_lib, w, slots=256)
    _, _, twin = _build(product_lib, w, slots=256)
    s._ck(product_lib.mmp_tune(s.h, b"commit_host_only", 1))
    steps = []  # what s.churn_step returned, window by window
    step = s.churn_step
    s.churn_step = lambda *a, **k: steps.append(step(*a, **k)) or steps[-1]
    pub = 0
    for ep in range(12):
        ev = w.events(ep, 2000, 4)
        now0 = fl.now_ms + ep * w.window_ms
        _, _, rep = _compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, 400 + ep, path=1)
        got, want = steps[-1], twin.churn_step(ev, now0, now0 + w.window_ms, 400 + ep)
        assert twin.commit_info()[0] == 2
        for k in range(3):  # decisions, evictions, published rows, field by field (an eviction record has 4 bytes of padding)
            assert len(got[k]) == len(want[k]), (ep, k)
            for name in got[k].dtype.names:
                assert got[k][name].tobytes() == want[k][name].tobytes(), (ep, k, name)
        assert (got[3].n_published, got[3].n_carry) == (want[3].n_published, want[3].n_carry), ep
        assert np.array_equal(s.cluster_order(), twin.cluster_order()), ep
        pub += rep.n_published
    assert pub > 50
    for m in range(0, fl.n_models, 37):
        assert s.churn_model(m)[0].tobytes() == twin.churn_model(m)[0].tobytes(), m
