"""mmp_rate_run, one pod's rate-tracking task in one call, against its composition from the oracle
(tests/rate_run_oracle.py): out, loads and report, exactly --
  * on C2, C3, C5 and MIX fleets with registration times, for the pod with the most registrations holding entries of the
    models it holds, of models it does not hold and of models with three recent failure records, at thresholds 2 000, 300
    and 5 (at 5 chains run past the cut), with and without a fresh row for the pod;
  * with heavy sets that are empty (C2: every published rpm 0), of at most 16, and of more than 1 000 members;
  * with caps below the load count, and on a replayed ingest stream after a device-path and after a host-path commit;
  * every argument error, MMP_E_EPOCH and MMP_E_STATE.
Cross-checks (pod_tasks.cross_check_rate): out is mmp_scale_eval's (can_remove = 0) field by field; round-0 scale-up loads are
mmp_place_batch_excluding's under the heavy set with the same MMP_DF_OWN_ID ids; second copies are mmp_place_batch's with extra
{self}."""
import ctypes as C

import numpy as np
import pytest

import rate_run_oracle as rro
from common import EXPIRY, HOUR, vp
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import load_into_fleet, make_fleet
from pod_tasks import IT, TimedReplay, busiest_pod, cross_check_rate, held_models, rate_params, same_out, set_regs, timed_solver
from replay import run_window

pytestmark = pytest.mark.gpu
# each fleet with what it is there to cover over its three thresholds (checked, so that a changed fleet does not stop covering it)
FLEETS = [("C2", 3000, 400, 2, "no-heavy cut refused"), ("C3", 4000, 600, 3, "small-heavy cut refused"), ("C5", 3000, 500, 5, "second"),
          ("MIX", 1500, 320, 14, "small-heavy cut refused"), ("C3", 3000, 4000, 31, "large-heavy refused")]


def _workload(config, nm, ni, seed):
    """(fleet, times, pod): published rpm spread so that the heavy set grows as the threshold drops (C2: all 0), and three
    recent failure records on 10 of the pod's models"""
    fl = make_fleet(config, nm, ni, seed)
    rng = np.random.default_rng(seed)
    u = rng.uniform(size=ni)
    rpm = np.where(u < 0.7, rng.integers(0, 21, size=ni), np.where(u < 0.9, rng.integers(21, 1500, size=ni), rng.integers(1500, 10_000, size=ni)))
    fl.inst_rows["rpm"] = 0 if config == "C2" else rpm
    S = busiest_pod(fl)
    fl.inst_rows["rpm"][S] = min(int(fl.inst_rows["rpm"][S]), 20)
    held = held_models(fl, S)
    changes = {}
    others = [i for i in range(ni) if i != S]
    for m in rng.choice(held, min(10, len(held)), replace=False):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        regs = list(fl.edge_inst[a:b])
        extra = [i for i in rng.choice(others, 8, replace=False) if i not in regs][:3]
        changes[int(m)] = (list(fl.edge_inst[a:a + k]), list(fl.edge_inst[a + k:b]) + extra)
    set_regs(fl, changes)
    n = len(fl.edge_inst)
    ts = np.where(rng.uniform(size=n) < 0.3, fl.now_ms - rng.integers(0, EXPIRY, size=n),
                  fl.now_ms - rng.integers(EXPIRY, 4 * HOUR, size=n)).astype(np.int64)
    for m in changes:   # the three added failures are recent
        ts[int(fl.edge_off[m + 1]) - 3:int(fl.edge_off[m + 1])] = fl.now_ms - rng.integers(0, EXPIRY // 2, size=3)
    return fl, ts, S


def _entries(fl, S, rng, n_unreg=30):
    """the pod's cache: every model it holds or has failed on, and models it does not hold, counts from idle to far past
    the threshold, usage iterations in and out of the second-copy window"""
    mine = held_models(fl, S)
    rest = [m for m in range(fl.n_models) if m not in set(mine)]
    models = mine + [int(m) for m in rng.choice(rest, n_unreg, replace=False)]
    e = np.zeros(len(models), dtype=L.SCALE_IN)
    e["instance"], e["model"] = S, models
    u = rng.uniform(size=len(models))
    e["count"] = np.where(u < 0.5, rng.integers(0, 20, size=len(models)),
                          np.where(u < 0.9, rng.integers(20, 2000, size=len(models)), rng.integers(5000, 20_000, size=len(models))))
    e["last_used"] = fl.now_ms - rng.integers(0, HOUR, size=len(models))
    e["i1"] = IT - rng.integers(0, 400, size=len(models))
    e["i2"] = np.minimum(IT, e["i1"] + rng.integers(0, 300, size=len(models)))
    return e[rng.permutation(len(e))]


def _check(s, o, fl, ts, S, ents, p, seed, fresh=None, cap=None):
    out, loads, r = s.rate_run(S, ents, p, seed, fresh_self=fresh, loads_cap=cap)
    wout, wloads, wr = rro.rate_run(o, fl, ts, S, ents, p, seed, fresh_self=fresh)
    assert same_out(out, wout), next((k for k in out.dtype.names if not np.array_equal(out[k], wout[k])))
    got = [tuple(int(x) for x in ld) for ld in loads]
    assert got == wloads[:len(got)] and len(got) == (len(wloads) if cap is None else min(cap, len(wloads))), \
        next(((a, b) for a, b in zip(got, wloads) if a != b), (len(got), len(wloads)))
    assert {k: getattr(r, k) for k in wr} == wr
    return out, wloads, wr


@pytest.mark.parametrize("config,nm,ni,seed,covers", FLEETS)
def test_rate_run_matches_the_composition(product_lib, oracle_lib, config, nm, ni, seed, covers):
    fl, ts, S = _workload(config, nm, ni, seed)
    rng = np.random.default_rng(seed)
    ents = _entries(fl, S, rng)
    s, o = timed_solver(product_lib, fl, ts), oracle_from_synth(fl)
    fresh = fl.inst_rows[S].copy()
    fresh["used"] = fresh["used"] + fresh["capacity"] // 100
    seen = dict(second=0, up=0, cut=0, refused=0, heavy=set())
    for thr in (2000, 300, 5):
        p = rate_params(fl.now_ms, thr)
        for fr in (None, fresh):
            out, loads, rep = _check(s, o, fl, ts, S, ents, p, 100 + thr, fresh=fr)
            heavy = rro.heavy_set(o, fl, S, thr)
            cross_check_rate(s, fl, ts, S, ents, p, 100 + thr, out, loads, heavy, fr)
            seen["second"] += rep["n_second"]
            seen["up"] += rep["n_scale_up"]
            seen["cut"] += rep["n_chains_cut"]
            seen["refused"] += rep["n_refused_failures"]
            seen["heavy"].add(len(heavy))
            if rep["n_loads"] > 3:   # a cap below the load count: the first loads, the same report
                _check(s, o, fl, ts, S, ents, p, 100 + thr, fresh=fr, cap=rep["n_loads"] // 3)
        t = C.c_double()
        s._ck(s.lib.mmp_last_timing(s.h, b"rate_run", C.byref(t)))
        assert t.value > 0
    checks = {"no-heavy": seen["heavy"] == {0}, "small-heavy": 0 < min(seen["heavy"]) <= 16, "large-heavy": max(seen["heavy"]) > 1000,
              "cut": seen["cut"] > 0, "refused": seen["refused"] > 0, "second": seen["second"] > 0}
    assert all(checks[c] for c in covers.split()), (checks, seen)
    s.close()
    o.close()


def test_rate_run_replayed_stream(product_lib, oracle_lib):
    """after a device-path commit and after a host-path commit of a replayed ingest stream whose upserts come with
    registration times"""
    rp = TimedReplay(make_fleet("C3", 3000, 600, 3), product_lib, 3)
    seen = set()
    for w in range(12):
        run_window(rp, w)
        path = rp.windows[-1][1]
        if path in seen:
            continue
        seen.add(path)
        v, o = rp.view(), rp.oracle()
        ts, _ = rp.view_times(v)
        S = busiest_pod(v)
        ents = _entries(v, S, np.random.default_rng(w), n_unreg=10)
        ents["count"] = np.maximum(ents["count"], 200)
        _, loads, _ = _check(rp.f, o, v, ts, S, ents, rate_params(rp.now, 300), 7)
        assert loads
        o.close()
        if seen == {1, 2}:
            break
    assert seen == {1, 2}, seen


def test_rate_run_gates(product_lib, oracle_lib):
    fl, ts, S = _workload("C3", 1000, 200, 4)
    ents = _entries(fl, S, np.random.default_rng(4), n_unreg=5)
    s, o = timed_solver(product_lib, fl, ts), oracle_from_synth(fl)
    for delta, gate in ((5999, L.RATE_TOO_SOON), (6000, L.RATE_RAN)):
        _, _, r = _check(s, o, fl, ts, S, ents, rate_params(fl.now_ms, 300, delta=delta), 1)
        assert r["gate"] == gate
    _, _, r = _check(s, o, fl, ts, S, ents[:0], rate_params(fl.now_ms, 300), 1)
    assert r["gate"] == L.RATE_NO_ENTRIES
    # a gated call still refuses two entries of one model
    dup = np.concatenate([ents[:2], ents[:1]])
    with pytest.raises(MmpError) as e:
        s.rate_run(S, dup, rate_params(fl.now_ms, 300, delta=10), 1)
    assert e.value.code == L.E_ARG
    s.close()
    o.close()
    one = make_fleet("C3", 10, 1, 4)
    s = Fleet(one.min_space_units, one.min_churn_age_ms, one.default_model_size_units, 1, one.n_models, lib=product_lib)
    load_into_fleet(one, s)
    for m in range(one.n_models):
        s.model_times(m, np.full(int(one.edge_off[m + 1] - one.edge_off[m]), one.now_ms - HOUR, dtype=np.int64), 0)
    s.commit()
    e1 = np.zeros(1, dtype=L.SCALE_IN)
    e1["instance"], e1["model"], e1["count"], e1["i1"], e1["i2"] = 0, 0, 5000, 7, 9
    out, loads, r = s.rate_run(0, e1, rate_params(one.now_ms, 300), 1)
    assert r.gate == L.RATE_FEW_INSTANCES and len(loads) == 0 and out["action"][0] == 0 and (out["i1"][0], out["i2"][0]) == (7, 9)
    s.close()


def test_rate_run_errors(product_lib):
    fl = make_fleet("C3", 200, 40, 5)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    p = rate_params(fl.now_ms, 1000)
    ents = np.zeros(2, dtype=L.SCALE_IN)
    ents["instance"], ents["model"] = 0, [3, 4]
    with pytest.raises(MmpError) as e:
        s.rate_run(0, ents, p, 1)
    assert e.value.code == L.E_EPOCH
    load_into_fleet(fl, s)
    s.commit()
    with pytest.raises(MmpError) as e:   # no registration times
        s.rate_run(0, ents, p, 1)
    assert e.value.code == L.E_STATE
    for m in range(fl.n_models):
        s.model_times(m, np.full(int(fl.edge_off[m + 1] - fl.edge_off[m]), fl.now_ms - HOUR, dtype=np.int64), 0)
    s.commit()
    s.rate_run(0, ents, p, 1)
    out = np.zeros(2, dtype=L.SCALE_OUT)
    loads = np.zeros(4, dtype=L.RATE_LOAD)
    rep = L.RateReport()
    call = lambda sf, e, n, pp, o_, l_, cap, r_: s.lib.mmp_rate_run(s.h, sf, e, n, pp, None, 1, o_, l_, cap, r_)
    args = lambda **k: {**dict(sf=0, e=vp(ents), n=2, pp=vp(p), o_=vp(out), l_=vp(loads), cap=4, r_=C.byref(rep)), **k}
    for self_idx in (-1, fl.n_instances):
        assert call(**args(sf=self_idx)) == L.E_ARG
    for field, bad in (("model", [3, 3]), ("model", [-1, 4]), ("model", [3, fl.n_models]), ("instance", [0, 1])):
        b = ents.copy()
        b[field] = bad
        before = out.copy()
        assert call(**args(e=vp(b))) == L.E_ARG
        assert same_out(out, before)
    assert call(**args(n=-1)) == L.E_ARG
    assert call(**args(pp=None)) == L.E_ARG
    assert call(**args(r_=None)) == L.E_ARG
    assert call(**args(o_=None)) == L.E_ARG
    assert call(**args(l_=None)) == L.E_ARG
    for k, v in (("last_check_time", fl.now_ms), ("scale_up_rpm_threshold", 0)):
        b = p.copy()
        b["scale"][k] = v
        assert call(**args(pp=vp(b))) == L.E_ARG
    # zero cap and NULL loads: the totals only
    assert call(**args(l_=None, cap=0)) == rep.n_loads >= 0
    s.close()
