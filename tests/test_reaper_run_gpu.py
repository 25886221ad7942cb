"""mmp_reaper_run, one run of the leader's reaper task in one call, against the oracle composition of the reference's loop
(tests/reaper_run_oracle.py): pruned pairs, repaired ids, loads (model, target, n_candidates, last_used), the report and the
`missings` map after its cleanup, exactly --
  * on the closed loop's reaper workloads (free / cutoff / full fill, with and without type constraints, equal-lastUsed runs,
    0 / 1 / 2 failed loads, a partition whose count is 0, no candidates, a size estimate of 0 first and in a later partition),
    where nothing prunes or repairs: there the loads are also mmp_reaper_select over the partitions followed by
    mmp_place_batch of the same records with the same seed;
  * with pods removed from the table and committed (the structural path): the only copy, one of two copies, or one of two
    failed loads on a gone pod; registration times on both sides of assume_gone_ms; missing_since absent, recent and old; the
    leader gone from its own table; models at lastUsed = Long.MAX_VALUE, loaded and not; caps below every total;
  * on fleets whose pruned registrations sit past the fourth position, and on a replayed ingest stream after a device-path
    and after a host-path commit;
  * argument errors and MMP_E_EPOCH."""
import ctypes as C

import numpy as np
import pytest

import reaper_run_oracle as rro
from helpers import oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import load_into_fleet, make_churn, make_churn_overflow, make_fleet
from oracle import binding as ob
from replay import Replay, run_window
from test_churn_reaper_gpu import _with_failed, _workload, device_selection

pytestmark = pytest.mark.gpu

GONE_MS = 600_000   # ASSUME_INSTANCE_GONE_AFTER_MS


def _times(fl, rng, recent=0.3):
    """a load / failure time for every registration: `recent` of them within assume_gone_ms, the others 10 min - 4 h old"""
    n = len(fl.edge_inst)
    return np.where(rng.uniform(size=n) < recent, fl.now_ms - rng.integers(0, GONE_MS, size=n),
                    fl.now_ms - rng.integers(GONE_MS, 4 * rro.HOUR, size=n)).astype(np.int64)


def _build(product_lib, fl, ts, gone=()):
    s = solver_from_synth(fl, product_lib)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if a < b:
            s.model_times(m, ts[a:b])
    for i in gone:
        s.instance_remove(int(i))
    s.commit()
    # the oracle's table as the commit holds it: every instance but the gone ones, as ADDED events, one converged refresh
    o = ob.OracleFleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units)
    o.types_set(fl.type_config)
    out = set(int(i) for i in gone)
    for i in range(fl.n_instances):
        if i not in out:
            o.instance_event(ob.ADDED, i, fl.inst_rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i], fl.now_ms)
    if fl.type_config is not None:
        o.tc_converge()
    o.set_replaced_replicasets(fl.replaced_replicasets)
    # a pruned registration names an instance outside the table: no rank, so the committed exclusion rows are those of the
    # pruned records.  That needs every ranked instance to be in the table.
    assert not set(int(i) for i in s.cluster_order()) & set(int(i) for i in gone)
    return s, o


def _loads(a):
    return [(int(x["model"]), int(x["target"]), int(x["n_candidates"]), int(x["last_used"])) for x in a]


def _check(s, o, fl, ts, leader, now, missing, in_table, seed, live_leader=True):
    mp, mo = missing.copy(), missing.copy()
    (pm, pi), rep, loads, r = s.reaper_run(leader, now, GONE_MS, mp, seed, pruned_cap=len(fl.edge_inst) + 1)
    want = rro.reaper_run(o, fl, ts, leader, now, GONE_MS, mo, in_table, seed)
    assert list(zip(pm.tolist(), pi.tolist())) == want["pairs"]
    assert rep.tolist() == want["repaired"]
    got = _loads(loads)
    if live_leader:
        assert got == want["loads"], (len(got), len(want["loads"]), next((k, a, b) for k, (a, b) in enumerate(zip(got, want["loads"])) if a != b))
    else:  # the leader is not live in the epoch: malformed decisions (mmp_place_batch's answer for such a self)
        assert [(m, lu) for m, _, _, lu in got] == [(m, lu) for m, _, _, lu in want["loads"]]
        assert all(t == L.TARGET_INVALID for _, t, _, _ in got)
    assert (r.n_pruned, r.n_repaired, r.n_loads, r.stopped_partition) == (len(want["pairs"]), len(want["repaired"]), len(want["loads"]), want["stopped"])
    assert np.array_equal(mp, mo)
    timing = C.c_double()
    s._ck(s.lib.mmp_last_timing(s.h, b"reaper_run", C.byref(timing)))
    assert timing.value > 0
    return want, r


def _late_zero(seed):
    """type constraints; the second partition in PARTITION_STATS_COMP order publishes no use (size estimate 0: more than 10
    copies, used = 0) on caches small enough that its free space stays below the first partition's"""
    w = make_churn(20_000, 200, seed, fill=0.5, with_types=True)
    fl = w.fleet
    o = oracle_from_synth(fl)
    stats, ids = o.partition_stats()
    part = np.asarray([o.instance_partition(i) for i in range(fl.n_instances)])
    p1 = part == ids[1]
    free0 = int(stats[0]["total_free"])
    fl.inst_rows["used"][p1] = 0
    fl.inst_rows["capacity"][p1] = max(2 * fl.min_space_units, free0 // (4 * int(p1.sum())))
    return w


@pytest.mark.parametrize("case,seed", [("free", 3), ("free_tc", 4), ("cutoff", 5), ("cutoff_tc", 6), ("full", 7), ("ties", 8),
                                       ("none", 9), ("zero", 10), ("part0_tc", 11), ("late0_tc", 12)])
def test_reaper_run_without_prune(product_lib, oracle_lib, case, seed):
    w = _late_zero(seed) if case == "late0_tc" else _workload(case, seed)
    fl = w.fleet
    ts = np.full(len(fl.edge_inst), fl.now_ms - rro.HOUR, dtype=np.int64)
    s, o = _build(product_lib, fl, ts)
    now, leader = fl.now_ms + 500, 17
    missing = np.zeros(fl.n_instances, dtype=np.int64)
    want, r = _check(s, o, fl, ts, leader, now, missing, np.ones(fl.n_instances, dtype=bool), seed)
    assert r.n_pruned == 0 and r.n_repaired == 0
    # the composed route: mmp_reaper_select over the partitions, then mmp_place_batch of the same records, same seed
    sel = device_selection(s, now)
    dec = np.zeros(len(sel), dtype=L.DECISION_IN)
    dec["model"], dec["self"], dec["last_used"], dec["fresh"] = sel, leader, fl.model_last_used[sel], -1
    (_, _), _, loads, _ = s.reaper_run(leader, now, GONE_MS, missing.copy(), seed)
    assert loads["model"].tolist() == sel
    if sel:
        out = s.place_batch(dec, now, seed)
        assert loads["target"].tobytes() == out["target"].tobytes() and loads["n_candidates"].tobytes() == out["n_candidates"].tobytes()
    if case in ("free", "free_tc", "cutoff", "cutoff_tc", "ties", "part0_tc", "late0_tc"):
        assert len(sel) > 10, (case, len(sel))
    if case in ("none", "zero"):
        assert not sel
    assert r.stopped_partition == {"zero": 0, "late0_tc": 2}.get(case, -1), (case, r.stopped_partition)
    s.close()
    o.close()


@pytest.mark.parametrize("with_types,leader_gone,seed", [(False, False, 21), (True, False, 22), (False, True, 23)])
def test_reaper_run_with_pods_gone(product_lib, oracle_lib, with_types, leader_gone, seed):
    w = make_churn(20_000, 200, seed, fill=0.5, with_types=with_types)
    twice = [int(m) for m in w.unloaded_models[:300]]
    w = _with_failed(w, {m: 2 for m in twice})   # two failed loads, on instances 0 and 1
    fl = w.fleet
    rng = np.random.default_rng(seed)
    fl.model_last_used[twice] = fl.now_ms - rng.integers(0, 1000, size=len(twice))  # the most recent: selected once candidates
    maxed = np.concatenate([rng.choice(w.unloaded_models[300:], 20, replace=False), rng.choice(w.loaded_models, 20, replace=False)])
    fl.model_last_used[maxed] = rro.LONG_MAX
    ts = _times(fl, rng)
    gone = np.concatenate([[0], rng.choice(np.arange(2, fl.n_instances), size=9, replace=False)])
    s, o = _build(product_lib, fl, ts, gone)
    in_table = ~np.isin(np.arange(fl.n_instances), gone)
    leader = int(gone[-1]) if leader_gone else int(np.nonzero(in_table)[0][5])
    now = fl.now_ms
    missing = np.zeros(fl.n_instances, dtype=np.int64)
    missing[gone[:7]] = now - 660_000                  # first seen missing 11 minutes ago: pruned
    missing[gone[7]] = now - 60_000                    # one minute ago: kept, not pruned yet
    missing[np.nonzero(in_table)[0][:4]] = now - rng.integers(1, 900_000, size=4)  # instances back in the table: cleared
    want, r = _check(s, o, fl, ts, leader, now, missing, in_table, seed, live_leader=not leader_gone)
    pr = want["pruned"]
    loaded_models = set(m for m, _, _, _ in want["loads"])
    sole = [m for m in range(fl.n_models) if fl.n_loaded[m] == 1 and pr.n_loaded[m] == 0]
    assert sole and set(sole) & loaded_models                      # only copy gone: a candidate, placed in this run
    assert any(fl.n_loaded[m] == 2 and pr.n_loaded[m] == 1 and m not in loaded_models for m in range(fl.n_models))
    assert set(m for m in twice if pr.n_failed[m] == 1) & loaded_models   # one of two failed loads gone
    assert r.n_repaired == 40 and set(want["repaired"]) == set(int(m) for m in maxed)
    assert set(m for m, _, _, lu in want["loads"] if lu == now - rro.REPAIR_AGE_MS) & set(int(m) for m in maxed)
    if leader_gone:
        assert r.n_pruned > 0 and not any(i == leader for _, i in want["pairs"])
    # caps below every total: the first entries, the same totals and map
    caps = (max(1, r.n_pruned // 3), max(1, r.n_repaired // 3), max(1, r.n_loads // 3))
    mc = missing.copy()
    (pm, pi), rep, loads, rc = s.reaper_run(leader, now, GONE_MS, mc, seed, *caps)
    assert (rc.n_pruned, rc.n_repaired, rc.n_loads, rc.stopped_partition) == (r.n_pruned, r.n_repaired, r.n_loads, r.stopped_partition)
    assert list(zip(pm.tolist(), pi.tolist())) == want["pairs"][:caps[0]] and rep.tolist() == want["repaired"][:caps[1]]
    assert _loads(loads) == _loads(s.reaper_run(leader, now, GONE_MS, missing.copy(), seed)[2])[:caps[2]]
    mo = missing.copy()
    rro.reaper_run(o, fl, ts, leader, now, GONE_MS, mo, in_table, seed)
    assert np.array_equal(mc, mo)
    s.close()
    o.close()


def test_reaper_run_overflow_registrations(product_lib, oracle_lib):
    w = make_churn_overflow(make_churn(20_000, 200, 25, fill=0.6), 0.05, 25)
    fl = w.fleet
    rng = np.random.default_rng(25)
    ts = _times(fl, rng)
    at_ovf = np.concatenate([fl.edge_inst[fl.edge_off[m] + 4:fl.edge_off[m + 1]] for m in range(fl.n_models)])
    gone = np.argsort(-np.bincount(at_ovf, minlength=fl.n_instances), kind="stable")[:8]
    s, o = _build(product_lib, fl, ts, gone)
    in_table = ~np.isin(np.arange(fl.n_instances), gone)
    missing = np.zeros(fl.n_instances, dtype=np.int64)
    missing[gone] = fl.now_ms - 660_000
    leader = int(np.nonzero(in_table)[0][0])
    want, r = _check(s, o, fl, ts, leader, fl.now_ms, missing, in_table, 25)
    pos = [int(np.nonzero(fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]] == i)[0][0]) for m, i in want["pairs"]]
    assert r.n_pruned > 0 and max(pos) >= 4 and r.n_loads > 0
    s.close()
    o.close()


def test_reaper_run_replayed_stream(product_lib, oracle_lib):
    """after a device-path commit and after a host-path commit of a replayed ingest stream (no registration times: they read
    0, so every registration outside the table is old enough)"""
    rp = Replay(make_fleet("C3", 3000, 600, 3), product_lib, 3)
    seen = set()
    for w in range(12):
        run_window(rp, w)
        path = rp.windows[-1][1]
        if path in seen:
            continue
        seen.add(path)
        v, o = rp.view(), rp.oracle()
        in_table = rp.present.copy()
        missing = np.where(in_table, 0, rp.now - 660_000).astype(np.int64)
        missing[np.nonzero(in_table)[0][:3]] = rp.now - 30_000
        _check(rp.f, o, v, np.zeros(len(v.edge_inst), dtype=np.int64), int(rp._live()[0]), rp.now, missing, in_table, 100 + w)
        o.close()
        if seen == {1, 2}:
            break
    assert seen == {1, 2}, seen


def test_reaper_run_errors(product_lib):
    fl = make_fleet("C3", 200, 40, 5)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    missing = np.zeros(fl.n_instances, dtype=np.int64)
    with pytest.raises(MmpError) as e:
        s.reaper_run(0, fl.now_ms, GONE_MS, missing, 1)
    assert e.value.code == L.E_EPOCH
    load_into_fleet(fl, s)
    for leader in (-1, fl.n_instances):
        with pytest.raises(MmpError) as e:
            s.reaper_run(leader, fl.now_ms, GONE_MS, missing, 1)
        assert e.value.code == L.E_ARG
    with pytest.raises(MmpError) as e:
        s.reaper_run(0, fl.now_ms, -1, missing, 1)
    assert e.value.code == L.E_ARG
    rep = L.ReaperReport()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    buf = np.zeros(16, dtype=np.int32)
    loads = np.zeros(4, dtype=L.REAPER_LOAD)
    for args in ((vp(buf), vp(buf), -1, vp(buf), 4, vp(loads), 4), (None, vp(buf), 4, vp(buf), 4, vp(loads), 4),
                 (vp(buf), vp(buf), 4, None, 4, vp(loads), 4), (vp(buf), vp(buf), 4, vp(buf), 4, None, 4)):
        before = missing.copy()
        assert s.lib.mmp_reaper_run(s.h, 0, fl.now_ms, GONE_MS, vp(missing), 1, *args, C.byref(rep)) == L.E_ARG
        assert np.array_equal(before, missing)
    assert s.lib.mmp_reaper_run(s.h, 0, fl.now_ms, GONE_MS, None, 1, None, None, 0, None, 0, None, 0, C.byref(rep)) == L.E_ARG
    assert s.lib.mmp_reaper_run(s.h, 0, fl.now_ms, GONE_MS, vp(missing), 1, None, None, 0, None, 0, None, 0, None) == L.E_ARG
    # zero caps and NULL outputs: the totals only
    n = s.lib.mmp_reaper_run(s.h, 0, fl.now_ms, GONE_MS, vp(missing), 1, None, None, 0, None, 0, None, 0, C.byref(rep))
    assert n == rep.n_loads >= 0
    s.close()
