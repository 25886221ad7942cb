"""mmp_janitor_run, the registry loop of one pod's janitor task in one call, against the plain restatement of the reference's
loop (tests/janitor_run_oracle.py): edits (model, what, last_used, last_unload_time) and the report, exactly --
  * on C2, C3 and MIX fleets 2 % from full with registration times, for a pod holding stale registrations, failed entries,
    expired and fresh failure records, unregistered entries, equal-lastUsed candidates, Long.MAX_VALUE lastUsed values and
    loadTimestamps that do not match, with and without MMP_SCALE_NO_LOCAL_STATS, with a budget that binds and one that does not
    (where it does not, the SCALE_DOWN set is mmp_scale_eval's remove on the candidates whose load_ts matches);
  * with self's registration past the fourth (the sixth of seven), a saturated copy count (UNDECIDED), self not in the table,
    and a cap below the edit count;
  * on a replayed ingest stream after a device-path and after a host-path commit;
  * every argument error, MMP_E_EPOCH and MMP_E_STATE."""
import ctypes as C

import numpy as np
import pytest

import janitor_run_oracle as jro
from common import HOUR, vp
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import load_into_fleet, make_fleet
from pod_tasks import TimedReplay, busiest_pod, janitor_entries, janitor_params, janitor_workload, report_dict, timed_solver
from replay import run_window

pytestmark = pytest.mark.gpu


def _check(s, o, fl, ts, lul, S, ents, p, cap=None):
    edits, r = s.janitor_run(S, ents, p, cap)
    want, wr = jro.janitor_run(o, fl, ts, lul, S, ents, p)
    got = [(int(e["model"]), int(e["what"]), int(e["last_used"]), int(e["last_unload_time"])) for e in edits]
    assert got == want[:len(got)] and len(got) == min(len(want), len(got) if cap is None else cap), \
        next(((a, b) for a, b in zip(got, want) if a != b), (len(got), len(want)))
    assert report_dict(r) == wr
    t = C.c_double()
    s._ck(s.lib.mmp_last_timing(s.h, b"janitor_run", C.byref(t)))
    assert t.value > 0
    return want, wr


def _scale_down_set(s, fl, ts, S, ents, p):
    """mmp_scale_eval(can_remove = 1).remove over the entries that are candidates and whose load_ts matches"""
    rec = []
    for e in ents:
        m = int(e["model"])
        a, k = int(fl.edge_off[m]), int(fl.n_loaded[m])
        regs = list(fl.edge_inst[a:a + k])
        if S not in regs or e["flags"] or e["last_used"] <= 0 or int(ts[a + regs.index(S)]) != int(e["load_ts"]):
            continue
        x = np.zeros(1, dtype=L.SCALE_IN)[0]
        x["instance"], x["model"], x["count"], x["last_used"], x["last_heavy"] = S, m, e["count"], e["last_used"], e["last_heavy"]
        x["weight"], x["flags"] = e["weight"], int(p["flags"][0]) & 1
        rec.append(x)
    rec = np.array(rec, dtype=L.SCALE_IN)
    sp = p["scale"].copy()
    sp["can_remove"] = 1
    out = np.zeros(len(rec), dtype=L.SCALE_OUT)
    s._ck(s.lib.mmp_scale_eval(s.h, vp(rec), len(rec), vp(sp), vp(out)))
    # the TreeSet keeps the first model of an equal-lastUsed run (N15)
    first = {}
    for x in sorted(rec, key=lambda x: (int(x["last_used"]), int(x["model"]))):
        first.setdefault(int(x["last_used"]), int(x["model"]))
    keep = set(first.values())
    return sorted(int(x["model"]) for x, o in zip(rec, out) if o["remove"] and int(x["model"]) in keep)


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 3000, 400, 2), ("C3", 6000, 400, 3), ("MIX", 1500, 320, 14), ("MIX", 1500, 400, 41)])
def test_janitor_run_matches_the_loop(product_lib, oracle_lib, config, nm, ni, seed):
    fl, ts, lul, S = janitor_workload(config, nm, ni, seed, wide=True, saturated=True)
    rng = np.random.default_rng(seed)
    ents = janitor_entries(fl, ts, S, rng)
    s, o = timed_solver(product_lib, fl, ts, lul), oracle_from_synth(fl)
    seen = 0
    for cap_units, flags in ((2_000, 0), (1 << 40, 0), (2_000, 1)):
        p = janitor_params(fl.now_ms, cap_units, flags)
        p["scale"]["second_copy_remove_max_age_ms"] = 36 * HOUR
        want, wr = _check(s, o, fl, ts, lul, S, ents, p)
        whats = [w for _, w, _, _ in want]
        assert any(w & L.JE_UNDECIDED for w in whats) and any(w & L.JE_UNREGISTER for w in whats)
        assert any(w & L.JE_DROP_FAILURE for w in whats) and any(w & L.JE_REMOVE_LOCAL for w in whats)
        seen += wr["n_removed"]
        if cap_units == 1 << 40:  # the budget does not bind
            assert [m for m, w, _, _ in want if w & L.JE_SCALE_DOWN] == _scale_down_set(s, fl, ts, S, ents, p)
        if flags and fl.type_config is not None:
            assert wr["n_removed"] == 0   # EMPTY_STATS (N13)
        # a cap below the edit count: the first edits in model order, the same report
        if len(want) > 3:
            _check(s, o, fl, ts, lul, S, ents, p, cap=len(want) // 3)
    assert seen > 0 or config == "C2"   # (the C2 pod drops no copy; the other fleets cover SCALE_DOWN)
    sixth = [m for m in range(nm) if fl.n_loaded[m] == 7 and fl.edge_inst[fl.edge_off[m] + 5] == S]
    assert len(sixth) == 20
    s.close()
    o.close()


def test_janitor_run_self_not_live(product_lib, oracle_lib):
    fl, ts, lul, S = janitor_workload("C3", 3000, 300, 5)
    ents = janitor_entries(fl, ts, S, np.random.default_rng(5))
    s = timed_solver(product_lib, fl, ts, lul, gone=[S])
    o = oracle_from_synth(fl, bulk=False, gone=[S])
    assert S not in set(int(i) for i in s.cluster_order())
    want, wr = _check(s, o, fl, ts, lul, S, ents, janitor_params(fl.now_ms, 1 << 40))
    assert wr["n_referencing"] > 0 and len(want) > 0
    s.close()
    o.close()


def test_janitor_run_replayed_stream(product_lib, oracle_lib):
    """after a device-path commit and after a host-path commit of a replayed ingest stream whose upserts come with registration
    times (TimedReplay; JSON records carry none: their times read 0)"""
    rp = TimedReplay(make_fleet("C3", 3000, 600, 3), product_lib, 3)
    seen = set()
    for w in range(12):
        run_window(rp, w)
        path = rp.windows[-1][1]
        if path in seen:
            continue
        seen.add(path)
        v, o = rp.view(), rp.oracle()
        ts, lul = rp.view_times(v)
        S = busiest_pod(v)
        ents = janitor_entries(v, ts, S, np.random.default_rng(w), n_unreg=10)
        want, _ = _check(rp.f, o, v, ts, lul, S, ents, janitor_params(rp.now, 1 << 40))
        assert want
        o.close()
        if seen == {1, 2}:
            break
    assert seen == {1, 2}, seen


def test_janitor_run_errors(product_lib):
    fl = make_fleet("C3", 200, 40, 5)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    p = janitor_params(fl.now_ms, 1000)
    ents = np.zeros(2, dtype=L.JANITOR_ENTRY)
    ents["model"] = [3, 4]
    with pytest.raises(MmpError) as e:
        s.janitor_run(0, ents, p)
    assert e.value.code == L.E_EPOCH
    load_into_fleet(fl, s)
    s.commit()
    with pytest.raises(MmpError) as e:   # no registration times
        s.janitor_run(0, ents, p)
    assert e.value.code == L.E_STATE
    for m in range(fl.n_models):
        s.model_times(m, np.full(int(fl.edge_off[m + 1] - fl.edge_off[m]), fl.now_ms - HOUR, dtype=np.int64), 0)
    s.commit()
    s.janitor_run(0, ents, p)
    edits = np.zeros(4, dtype=L.JANITOR_EDIT)
    rep = L.JanitorReport()
    for self_idx in (-1, fl.n_instances):
        assert s.lib.mmp_janitor_run(s.h, self_idx, vp(ents), 2, vp(p), vp(edits), 4, C.byref(rep)) == L.E_ARG
    for bad in ([3, 3], [-1, 4], [3, fl.n_models]):
        b = ents.copy()
        b["model"] = bad
        before = edits.copy()
        assert s.lib.mmp_janitor_run(s.h, 0, vp(b), 2, vp(p), vp(edits), 4, C.byref(rep)) == L.E_ARG
        assert edits.tobytes() == before.tobytes()
    assert s.lib.mmp_janitor_run(s.h, 0, vp(ents), -1, vp(p), vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert s.lib.mmp_janitor_run(s.h, 0, vp(ents), 2, None, vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert s.lib.mmp_janitor_run(s.h, 0, vp(ents), 2, vp(p), vp(edits), 4, None) == L.E_ARG
    assert s.lib.mmp_janitor_run(s.h, 0, vp(ents), 2, vp(p), None, 4, C.byref(rep)) == L.E_ARG
    for k, v in (("last_check_time", fl.now_ms), ("scale_up_rpm_threshold", 0)):
        b = p.copy()
        b["scale"][k] = v
        assert s.lib.mmp_janitor_run(s.h, 0, vp(ents), 2, vp(b), vp(edits), 4, C.byref(rep)) == L.E_ARG
    # zero cap and NULL edits: the totals only
    assert s.lib.mmp_janitor_run(s.h, 0, vp(ents), 2, vp(p), None, 0, C.byref(rep)) == rep.n_edits >= 0
    s.close()
