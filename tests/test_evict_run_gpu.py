"""mmp_evict_run, one pod's eviction listener over a burst of evictions in one call, against its restatement from the Java
text (tests/evict_run_oracle.py): out and report, exactly --
  * on C2, C3, C5, MIX and a C3 fleet in a rolling upgrade (half the pods on a newer version, the old replicasets
    likely-replaced), for the pod with the most registrations evicting every model it is registered on (a quarter of its
    loaded models with no other copy, some of them with three recent failure records elsewhere), its registrations at,
    just past and well past 2 x loadTimeoutMs, load / failure times that match the entry or not, failed entries, lastUsed 0,
    older or newer than the record's, and models it does not hold; with and without a fresh row; then with every instance 2 %
    from full, where the rebalance gate closes;
  * against the composed route: the same classification on the host and mmp_place_batch of the same records (MMP_DF_OWN_ID,
    extra {self}), byte for byte;
  * on a replayed ingest stream, after device-path and host-path commits;
  * a pod out of the table, with and without a fresh row;
  * every argument error, MMP_E_EPOCH and MMP_E_STATE."""
import ctypes as C

import numpy as np
import pytest

import evict_run_oracle as ero
from common import EXPIRY, HOUR, vp
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import load_into_fleet, make_fleet
from pod_tasks import (TASK_FLEETS, TimedReplay, busiest_pod, composed_evict, evict_params, held_models, report_dict, set_regs,
                       task_fleet, timed_solver)
from replay import run_window

pytestmark = pytest.mark.gpu
WORKLOAD_TIMEOUT = 120_000   # load_timeout_ms of these workloads (the hand-built cases take pod_tasks.HAND_TIMEOUT, 60 000)


def _workload(config, nm, ni, seed):
    """(fleet, times, lastUnloadTime, pod): a quarter of the pod's loaded models (at most 40) left with the pod as their only
    copy; the pod added as one more loaded copy of 40 other models, as a failed load of 20 and as the only copy of 12; three
    recent failure records on every fourth model of which the pod is the only copy; the pod's own registrations at the reload
    edges"""
    fl = task_fleet(config, nm, ni, seed)
    rng = np.random.default_rng(seed)
    S = busiest_pod(fl)
    held = held_models(fl, S)
    loaded = [m for m in held if S in set(int(i) for i in fl.edge_inst[fl.edge_off[m]:fl.edge_off[m] + fl.n_loaded[m]])]
    free = rng.permutation([m for m in range(nm) if m not in set(held)])
    others = [i for i in range(ni) if i != S]
    regs = lambda m: ([int(i) for i in fl.edge_inst[fl.edge_off[m]:fl.edge_off[m] + fl.n_loaded[m]] if i != S],
                      [int(i) for i in fl.edge_inst[fl.edge_off[m] + fl.n_loaded[m]:fl.edge_off[m + 1]] if i != S])
    changes = {}
    only = [int(m) for m in rng.choice(loaded, min(40, max(1, len(loaded) // 4)), replace=False)] + [int(m) for m in free[60:72]]
    for m in free[:40]:
        x, y = regs(m)
        changes[int(m)] = (x + [S], y)
    for m in free[40:60]:
        x, y = regs(m)
        changes[int(m)] = (x, y + [S])
    failing = only[::4]
    for m in only:
        _, y = regs(m)
        if m in failing:
            y += [int(i) for i in rng.choice(others, 8, replace=False) if i not in y][:3]
        changes[m] = ([S], y)
    set_regs(fl, changes)
    n, now = len(fl.edge_inst), fl.now_ms
    ts = np.where(rng.uniform(size=n) < 0.3, now - rng.integers(0, EXPIRY, size=n), now - rng.integers(EXPIRY, 4 * HOUR, size=n)).astype(np.int64)
    for m in failing:
        ts[int(fl.edge_off[m + 1]) - 3:int(fl.edge_off[m + 1])] = now - rng.integers(0, EXPIRY // 2, size=3)
    mine = np.nonzero(fl.edge_inst == S)[0]
    edge = rng.choice(mine, min(len(mine), 12), replace=False)
    ts[edge[0::2]] = now - 2 * WORKLOAD_TIMEOUT
    ts[edge[1::2]] = now - 2 * WORKLOAD_TIMEOUT - 1
    lul = np.where(rng.uniform(size=nm) < 0.3, now - rng.integers(0, 200_000, size=nm), 0).astype(np.int64)
    return fl, ts, lul, S


def _entries(fl, ts, S, rng, n_unreg=30):
    """the evictions of a burst in listener order: every model the pod is registered on, and models it does not hold"""
    now = fl.now_ms
    models = held_models(fl, S)
    rest = [m for m in range(fl.n_models) if m not in set(models)]
    models += [int(m) for m in rng.choice(rest, n_unreg, replace=False)]
    e = np.zeros(len(models), dtype=L.EVICT_ENTRY)
    for r, m in enumerate(models):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        pos = [j for j in range(b - a) if fl.edge_inst[a + j] == S]
        lt = next((int(ts[a + j]) for j in pos if j < k), int(rng.integers(1, now)))
        ft = next((int(ts[a + j]) for j in pos if j >= k), 0)
        e[r]["model"] = m
        e[r]["load_ts"] = lt if rng.uniform() < 0.85 else lt + 1
        e[r]["load_complete_ts"] = ft if rng.uniform() < 0.85 else ft + 1
        u = rng.uniform()
        e[r]["last_used"] = 0 if u < 0.1 else (now - int(rng.integers(2 * HOUR, 8 * HOUR)) if u < 0.3 else now - int(rng.integers(1, HOUR)))
        e[r]["flags"] = L.EV_ENTRY_FAILED if rng.uniform() < 0.1 else 0
    return e[rng.permutation(len(e))]


def _check(s, o, fl, ts, lul, S, ents, p, seed, fresh=None):
    out, r = s.evict_run(S, ents, p, seed, fresh_self=fresh)
    want, wr = ero.evict_run(o, fl, ts, lul, S, ents, p, seed, fresh_self=fresh)
    bad = np.nonzero(out != want)[0]
    assert len(bad) == 0, (len(bad), out[bad[:3]], want[bad[:3]])
    assert report_dict(r) == wr
    return out, wr


@pytest.mark.parametrize("config,nm,ni,seed", TASK_FLEETS)
def test_evict_run_matches_the_restatement(product_lib, oracle_lib, config, nm, ni, seed):
    fl, ts, lul, S = _workload(config, nm, ni, seed)
    ents = _entries(fl, ts, S, np.random.default_rng(seed))
    s, o = timed_solver(product_lib, fl, ts, lul), oracle_from_synth(fl)
    fresh = fl.inst_rows[S].copy()
    fresh["used"] = fresh["used"] + fresh["capacity"] // 100
    p = evict_params(fl.now_ms, WORKLOAD_TIMEOUT)
    seen = {k: 0 for k in ero.REPORT_KEYS}
    out = np.zeros(len(ents), dtype=L.EVICT_ACTION)
    for fr in (None, fresh):
        got, wr = _check(s, o, fl, ts, lul, S, ents, p, 100 + seed, fresh=fr)
        assert composed_evict(s, S, ents, got, p, 100 + seed, fr) == wr["n_placed"]
        for k in seen:
            seen[k] += wr[k]
        t = C.c_double()
        s._ck(s.lib.mmp_last_timing(s.h, b"evict_run", C.byref(t)))
        assert t.value > 0
        again, _ = s.evict_run(S, ents, p, 100 + seed, fresh_self=fr, out=out)   # into a caller-allocated array
        assert again is out and out.tobytes() == got.tobytes()
    assert seen["n_unregister"] > 0 and seen["n_drop_failure"] > 0 and seen["n_reload"] > 0, seen
    # (C5 is 99 % full as made: there every reload stops at the gate)
    assert seen["n_cluster_full"] == seen["n_reload"] or all(seen[k] > 0 for k in ("n_loaded_elsewhere", "n_refused", "n_placed")), seen
    # every instance 2 % from full: no type set passes the rebalance gate
    o.close()
    fl.inst_rows["used"] = fl.inst_rows["capacity"] - fl.inst_rows["capacity"] // 50
    for i in range(ni):
        s.instance_update(i, fl.inst_rows[i])
    s.commit()
    o = oracle_from_synth(fl)
    _, wr = _check(s, o, fl, ts, lul, S, ents, p, 100 + seed)
    assert wr["n_cluster_full"] == wr["n_reload"] > 0 and wr["n_placed"] == 0
    s.close()
    o.close()


def test_evict_run_replayed_stream(product_lib, oracle_lib):
    """after device-path and host-path commits of a replayed ingest stream whose upserts come with registration times"""
    rp = TimedReplay(make_fleet("C3", 3000, 600, 3), product_lib, 3)
    paths = set()
    for w in range(8):
        run_window(rp, w)
        paths.add(rp.windows[-1][1])
        v, o = rp.view(), rp.oracle()
        ts, lul = rp.view_times(v)
        S = busiest_pod(v, ranked=o.cluster_order())   # (the stream takes pods out: the pod places from its published row)
        ents = _entries(v, ts, S, np.random.default_rng(w), n_unreg=10)
        _, wr = _check(rp.f, o, v, ts, lul, S, ents, evict_params(rp.now, WORKLOAD_TIMEOUT), 7)
        assert wr["n_unregister"] > 0 and wr["n_reload"] > 0
        o.close()
    assert paths == {1, 2}, paths


def test_evict_run_pod_out_of_the_table(product_lib, oracle_lib):
    """a pod that is shutting down (out of the epoch): the same edits; its reloads place through its fresh row, and without
    one are answered MMP_TARGET_INVALID"""
    fl, ts, lul, S = _workload("C3", 4000, 600, 3)
    ents = _entries(fl, ts, S, np.random.default_rng(4))
    s = timed_solver(product_lib, fl, ts, lul)
    fl.inst_rows["shutting_down"][S] = 1
    s.instance_update(S, fl.inst_rows[S])
    s.commit()
    o = oracle_from_synth(fl)
    assert S not in set(int(i) for i in o.cluster_order())
    fresh = fl.inst_rows[S].copy()
    fresh["shutting_down"] = 0
    p = evict_params(fl.now_ms, WORKLOAD_TIMEOUT)
    with_row, wr = _check(s, o, fl, ts, lul, S, ents, p, 9, fresh=fresh)
    without, wr2 = _check(s, o, fl, ts, lul, S, ents, p, 9)
    placed = (without["what"] & L.EV_PLACED) != 0
    assert placed.any() and wr2["n_placed"] == wr["n_placed"] and wr2["n_none"] == 0
    assert (without["target"][placed] == L.TARGET_INVALID).all() and (with_row["target"][placed] != L.TARGET_INVALID).all()
    for k in ("model", "what", "last_used", "last_unload_time"):
        assert (without[k] == with_row[k]).all(), k
    s.close()
    o.close()


def test_evict_run_errors(product_lib):
    fl = make_fleet("C3", 200, 40, 5)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    p = evict_params(fl.now_ms, WORKLOAD_TIMEOUT)
    ents = np.zeros(2, dtype=L.EVICT_ENTRY)
    ents["model"], ents["last_used"] = [3, 4], fl.now_ms - 1
    with pytest.raises(MmpError) as e:
        s.evict_run(0, ents, p, 1)
    assert e.value.code == L.E_EPOCH
    load_into_fleet(fl, s)
    s.commit()
    with pytest.raises(MmpError) as e:   # no registration times
        s.evict_run(0, ents, p, 1)
    assert e.value.code == L.E_STATE
    for m in range(fl.n_models):
        s.model_times(m, np.full(int(fl.edge_off[m + 1] - fl.edge_off[m]), fl.now_ms - HOUR, dtype=np.int64), 0)
    s.commit()
    s.evict_run(0, ents, p, 1)
    out = np.zeros(2, dtype=L.EVICT_ACTION)
    rep = L.EvictReport()
    bad_row = fl.inst_rows[0:1].copy()
    bad_row["used"] = -1
    call = lambda sf, e, n, pp, fr, o_, r_: s.lib.mmp_evict_run(s.h, sf, e, n, pp, fr, 1, o_, r_)
    args = lambda **k: {**dict(sf=0, e=vp(ents), n=2, pp=vp(p), fr=None, o_=vp(out), r_=C.byref(rep)), **k}
    before = out.copy()
    for self_idx in (-1, fl.n_instances):
        assert call(**args(sf=self_idx)) == L.E_ARG
    for bad in ([3, 3], [-1, 4], [3, fl.n_models]):
        b = ents.copy()
        b["model"] = bad
        assert call(**args(e=vp(b))) == L.E_ARG
    assert call(**args(n=-1)) == L.E_ARG
    assert call(**args(n=(1 << 24) + 1)) == L.E_ARG
    assert call(**args(pp=None)) == L.E_ARG
    assert call(**args(r_=None)) == L.E_ARG
    assert call(**args(o_=None)) == L.E_ARG
    assert call(**args(e=None)) == L.E_ARG
    assert call(**args(fr=vp(bad_row))) == L.E_ARG
    assert out.tobytes() == before.tobytes()
    assert call(**args(n=0, e=None, o_=None)) == 0 and rep.n_unregister == 0
    # the slot array is left clean after a refused duplicate: the next call sees the entries again
    b = ents.copy()
    b["model"] = [3, 3]
    assert call(**args(e=vp(b))) == L.E_ARG
    assert call(**args()) == 2
    s.close()
