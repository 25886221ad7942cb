"""mmp_janitor_task, one pod's whole janitor task in one call, against the plain restatement (tests/janitor_task_oracle.py):
the actions per entry, the edits and the report, exactly --
  * on C2, C3 and MIX fleets with registration times, for a cache in most-recently-used order with undone and uncached
    entries, out-of-order times, recent entries, stale records, mismatched registrations (re-registered or removed), every
    removal reason, and with and without a Long.MAX_VALUE entry (the stop);
  * on a replayed ingest stream after a device-path and after a host-path commit;
  * on every hand-built case of tests/test_janitor_task_oracle.py;
  * at the block edges of k_jt_plan (256 entries a block) and k_jt_order (512 a tile): n = 1, and one under, at and over each;
  * with a cache pass that writes nothing, edits and registry report equal to mmp_janitor_run's, byte for byte;
  * every argument error, MMP_E_EPOCH and MMP_E_STATE."""
import ctypes as C

import numpy as np
import pytest

import janitor_task_oracle as jto
from helpers import oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import load_into_fleet, make_fleet
from replay import run_window
from test_janitor_run_gpu import _build, _entries, _workload
from test_janitor_run_oracle import HOUR, LONG_MAX
from test_janitor_task_oracle import CASES, MIN_STALE, WINDOW, params
from test_registry_overflow_gpu import _TimedReplay

pytestmark = pytest.mark.gpu
vp = lambda a: a.ctypes.data_as(C.c_void_p)
REPORT_FIELDS = ["n_not_done", "n_not_cached", "n_out_of_order", "n_stop", "n_repair", "n_not_reached", "n_stale_update", "n_remove",
                 "n_reregister", "n_undecided", "stopped_at", "registry_ran", "cache_changed"]
REGISTRY_FIELDS = ["n_referencing", "n_edits", "n_candidates", "n_removed", "weight_removed"]


def _report(r):
    d = {k: getattr(r, k) for k in REPORT_FIELDS}
    d["registry"] = {k: getattr(r.registry, k) for k in REGISTRY_FIELDS}
    return d


def _check(s, o, fl, ts, lul, S, ents, p, cap=None):
    out, edits, r = s.janitor_task(S, ents, p, cap)
    want_out, want_edits, want_rep = jto.janitor_task(o, fl, ts, lul, S, ents, p)
    got_out = [(int(a["model"]), int(a["what"]), int(a["last_used"]), int(a["replaced_ts"])) for a in out]
    assert got_out == want_out, next(((k, a, b) for k, (a, b) in enumerate(zip(got_out, want_out)) if a != b), None)
    got = [(int(e["model"]), int(e["what"]), int(e["last_used"]), int(e["last_unload_time"])) for e in edits]
    n = len(want_edits) if cap is None else min(cap, len(want_edits))
    assert got == want_edits[:n], next(((a, b) for a, b in zip(got, want_edits) if a != b), (len(got), len(want_edits)))
    assert _report(r) == want_rep
    t = C.c_double()
    s._ck(s.lib.mmp_last_timing(s.h, b"janitor_task", C.byref(t)))
    assert t.value > 0
    return want_out, want_edits, want_rep


def _task_entries(fl, ts, S, rng, with_stop, n_unreg=40):
    """test_janitor_run_gpu's cache, in most-recently-used order with a few neighbours swapped (out of order), as task entries:
    some undone, some out of LOADING..ACTIVE or unloaded recently, some recent; failed ones carry their failure time or not;
    Long.MAX_VALUE entries only with_stop"""
    base = _entries(fl, ts, S, rng, n_unreg)
    te = np.zeros(len(base), dtype=L.JANITOR_TASK_ENTRY)
    te["e"] = base
    e = te["e"]
    now = fl.now_ms
    if not with_stop:
        e["last_used"] = np.where(e["last_used"] == LONG_MAX, now - 5 * HOUR, e["last_used"])
    u = rng.uniform(size=len(te))
    e["last_used"] = np.where(u < 0.08, now - rng.integers(1, WINDOW + 2, size=len(te)), e["last_used"])   # recent
    e["last_used"] = np.where((u > 0.98) & (e["last_used"] != LONG_MAX), rng.choice([0, -1], size=len(te)), e["last_used"])
    flags = e["flags"].copy()
    flags |= np.where(rng.uniform(size=len(te)) < 0.05, L.JANITOR_NOT_DONE, 0).astype(np.uint32)
    flags |= np.where(rng.uniform(size=len(te)) < 0.15, L.JANITOR_NOT_LIVE, 0).astype(np.uint32)
    flags |= np.where(rng.uniform(size=len(te)) < 0.05, L.JANITOR_UNLOAD_RECENT, 0).astype(np.uint32)
    flags |= np.where(flags & L.JANITOR_FAILED, L.JANITOR_NOT_LIVE, 0).astype(np.uint32)
    e["flags"] = flags
    te["e"] = e
    # a failed entry's load_complete_ts: its failure record's time (matched) or not
    for k in range(len(te)):
        m = int(te["e"]["model"][k])
        a, nl, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        f = [q for q in range(a + nl, b) if fl.edge_inst[q] == S]
        te["load_complete_ts"][k] = int(ts[f[0]]) + (0 if rng.uniform() < 0.6 else 1) if f else 7
    order = np.argsort(-te["e"]["last_used"], kind="stable")
    for k in range(0, len(order) - 1, 17):   # out-of-order neighbours
        order[k], order[k + 1] = order[k + 1], order[k]
    te = te[order]
    te = np.ascontiguousarray(te)
    if with_stop:   # the Long.MAX_VALUE entries go in the middle, the first of them done
        k = len(te) // 2
        te["e"]["last_used"][k] = LONG_MAX
        te["e"]["flags"][k] &= np.uint32(~L.JANITOR_NOT_DONE & 0xffffffff)
        mx = np.nonzero(te["e"]["last_used"] == LONG_MAX)[0]
        rest = np.nonzero(te["e"]["last_used"] != LONG_MAX)[0]
        te = np.ascontiguousarray(np.concatenate([te[rest[:k]], te[mx], te[rest[k:]]]))
    return te


def _tparams(now, cap_units=2_000, flags=0, min_stale=MIN_STALE):
    return params(now, cap_units, flags, min_stale=min_stale)


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 3000, 400, 2), ("C3", 6000, 400, 3), ("MIX", 1500, 320, 14), ("MIX", 1500, 400, 41)])
def test_janitor_task_matches_the_restatement(product_lib, oracle_lib, config, nm, ni, seed):
    fl, ts, lul, S = _workload(config, nm, ni, seed, wide=True, saturated=True)
    s, o = _build(product_lib, fl, ts, lul), oracle_from_synth(fl)
    seen = 0
    for with_stop in (False, True):
        ents = _task_entries(fl, ts, S, np.random.default_rng(seed + with_stop), with_stop)
        for cap_units, flags, min_stale in ((2_000, 0, MIN_STALE), (1 << 40, 0, HOUR), (2_000, 1, MIN_STALE)):
            out, edits, rep = _check(s, o, fl, ts, lul, S, ents, _tparams(fl.now_ms, cap_units, flags, min_stale))
            for _, w, _, _ in out:
                seen |= w
            assert rep["registry_ran"] == (not with_stop)
            if edits and not with_stop:
                _check(s, o, fl, ts, lul, S, ents, _tparams(fl.now_ms, cap_units, flags, min_stale), cap=max(1, len(edits) // 3))
    assert seen & (L.JC_REREGISTER | L.JC_REMOVE | L.JC_STALE_UPDATE | L.JC_STOP | L.JC_NOT_REACHED | L.JC_OUT_OF_ORDER | L.JC_NOT_DONE) == \
        (L.JC_REREGISTER | L.JC_REMOVE | L.JC_STALE_UPDATE | L.JC_STOP | L.JC_NOT_REACHED | L.JC_OUT_OF_ORDER | L.JC_NOT_DONE), bin(seen)
    s.close()
    o.close()


def test_janitor_task_replayed_stream(product_lib, oracle_lib):
    rp = _TimedReplay(make_fleet("C3", 3000, 600, 3), product_lib, 3)
    seen = set()
    for w in range(12):
        run_window(rp, w)
        path = rp.windows[-1][1]
        if path in seen:
            continue
        seen.add(path)
        v, o = rp.view(), rp.oracle()
        ts = np.zeros(len(v.edge_inst), dtype=np.int64)
        lul = np.zeros(v.n_models, dtype=np.int64)
        for m, (t, u) in rp.times.items():
            a, b = int(v.edge_off[m]), int(v.edge_off[m + 1])
            k = min(len(t), b - a)
            ts[a:a + k] = t[:k]
            lul[m] = u
        S = int(np.argmax(np.bincount(v.edge_inst, minlength=v.n_instances)))
        ents = _task_entries(v, ts, S, np.random.default_rng(w), False, n_unreg=10)
        _, edits, _ = _check(rp.f, o, v, ts, lul, S, ents, _tparams(rp.now, 1 << 40))
        assert edits
        o.close()
        if seen == {1, 2}:
            break
    assert seen == {1, 2}, seen


@pytest.mark.parametrize("name", sorted(CASES))
def test_janitor_task_hand_cases(product_lib, oracle_lib, name):
    c = CASES[name]()
    s = solver_from_synth(c.fl, product_lib, max_models=c.max_models)
    for m in range(c.fl.n_models):
        s.model_times(m, c.ts[c.fl.edge_off[m]:c.fl.edge_off[m + 1]], int(c.lul[m]))
    s.commit()
    o = oracle_from_synth(c.fl)
    _check(s, o, c.fl, c.ts, c.lul, c.S, c.entries, c.params)
    s.close()
    o.close()


@pytest.fixture(scope="module")
def edge_fleet(product_lib):
    fl, ts, lul, S = _workload("C3", 3200, 400, 9)
    return fl, ts, lul, S, _build(product_lib, fl, ts, lul)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025])
def test_janitor_task_block_edges(edge_fleet, oracle_lib, n):
    """n entries of models the pod holds or not, their times falling with a few rising (out of order across tile edges), one
    undone and one uncached entry at each tile's end; then the same with a Long.MAX_VALUE entry in the last tile"""
    fl, ts, lul, S, s = edge_fleet
    rng = np.random.default_rng(n)
    te = np.zeros(n, dtype=L.JANITOR_TASK_ENTRY)
    te["e"]["model"] = rng.choice(fl.n_models, n, replace=False)
    lu = fl.now_ms - np.sort(rng.integers(1, 40 * HOUR, size=n))
    lu[rng.uniform(size=n) < 0.05] += HOUR
    te["e"]["last_used"] = lu
    te["e"]["weight"] = 10
    for k in range(n):
        m = int(te["e"]["model"][k])
        a, nl = int(fl.edge_off[m]), int(fl.n_loaded[m])
        hit = [q for q in range(a, a + nl) if fl.edge_inst[q] == S]
        te["e"]["load_ts"][k] = int(ts[hit[0]]) if hit and rng.uniform() < 0.7 else 5
    te["e"]["flags"][rng.uniform(size=n) < 0.3] = L.JANITOR_NOT_LIVE
    te["e"]["flags"][255::256] |= np.uint32(L.JANITOR_NOT_DONE)
    te["e"]["last_used"][511::512] = -1
    o = oracle_from_synth(fl)
    p = _tparams(fl.now_ms, 1 << 40)
    out, _, rep = _check(s, o, fl, ts, lul, S, te, p)
    assert rep["registry_ran"] == 1
    stop = n - 1 if n < 3 else n - 2
    te2 = te.copy()
    te2["e"]["last_used"][stop] = LONG_MAX
    te2["e"]["flags"][stop] = 0
    _, edits, rep = _check(s, o, fl, ts, lul, S, te2, p)
    assert rep["stopped_at"] == stop and len(edits) == 0
    o.close()


def test_janitor_task_without_writes_is_janitor_run(product_lib, oracle_lib):
    """entries the cache pass writes nothing for (recent, with records that are not stale; undone ones) give mmp_janitor_run's
    edits and registry report on the same entries, byte for byte"""
    fl, ts, lul, S = _workload("C3", 6000, 400, 3, wide=True, saturated=True)
    s = _build(product_lib, fl, ts, lul)
    base = _entries(fl, ts, S, np.random.default_rng(3))
    base["last_used"] = np.where(base["last_used"] == LONG_MAX, fl.now_ms - 1000, base["last_used"])
    te = np.zeros(len(base), dtype=L.JANITOR_TASK_ENTRY)
    te["e"] = base
    recent = te["e"]["last_used"] > fl.now_ms - WINDOW
    te["e"]["flags"][~recent] |= np.uint32(L.JANITOR_NOT_DONE)
    te = np.ascontiguousarray(te[np.argsort(-te["e"]["last_used"], kind="stable")])
    for cap_units in (2_000, 1 << 40):
        p = _tparams(fl.now_ms, cap_units, min_stale=1 << 62)
        out, edits, r = s.janitor_task(S, te, p)
        assert not any(int(w) & (L.JC_STALE_UPDATE | L.JC_REMOVE | L.JC_REREGISTER | L.JC_STOP) for w in out["what"])
        run_ents = np.ascontiguousarray(te["e"])
        jp = np.array([p[0]["janitor"]], dtype=L.JANITOR_PARAMS)
        e2, r2 = s.janitor_run(S, run_ents, jp)
        assert edits.tobytes() == e2.tobytes() and bytes(r.registry) == bytes(r2) and r2.n_edits > 0
    s.close()


def test_janitor_task_errors(product_lib):
    fl = make_fleet("C3", 200, 40, 5)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    p = _tparams(fl.now_ms, 1000)
    ents = np.zeros(2, dtype=L.JANITOR_TASK_ENTRY)
    ents["e"]["model"] = [3, 4]
    with pytest.raises(MmpError) as e:
        s.janitor_task(0, ents, p)
    assert e.value.code == L.E_EPOCH
    load_into_fleet(fl, s)
    s.commit()
    with pytest.raises(MmpError) as e:   # no registration times
        s.janitor_task(0, ents, p)
    assert e.value.code == L.E_STATE
    for m in range(fl.n_models):
        s.model_times(m, np.full(int(fl.edge_off[m + 1] - fl.edge_off[m]), fl.now_ms - HOUR, dtype=np.int64), 0)
    s.commit()
    s.janitor_task(0, ents, p)
    out = np.full(2, 0x5a, dtype=L.JANITOR_CACHE_ACTION)
    edits = np.zeros(4, dtype=L.JANITOR_EDIT)
    rep = L.JanitorTaskReport()
    call = lambda self_idx, e, n, pp, o, ed, cap, r: s.lib.mmp_janitor_task(s.h, self_idx, e, n, pp, o, ed, cap, r)
    for self_idx in (-1, fl.n_instances):
        assert call(self_idx, vp(ents), 2, vp(p), vp(out), vp(edits), 4, C.byref(rep)) == L.E_ARG
    for bad in ([3, 3], [-1, 4], [3, fl.n_models]):
        b = ents.copy()
        b["e"]["model"] = bad
        before = (out.tobytes(), edits.tobytes())
        assert call(0, vp(b), 2, vp(p), vp(out), vp(edits), 4, C.byref(rep)) == L.E_ARG
        assert (out.tobytes(), edits.tobytes()) == before
    assert call(0, vp(ents), -1, vp(p), vp(out), vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert call(0, vp(ents), (1 << 24) + 1, vp(p), vp(out), vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert call(0, vp(ents), 2, None, vp(out), vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert call(0, vp(ents), 2, vp(p), vp(out), vp(edits), 4, None) == L.E_ARG
    assert call(0, vp(ents), 2, vp(p), None, vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert call(0, None, 2, vp(p), vp(out), vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert call(0, vp(ents), 2, vp(p), vp(out), None, 4, C.byref(rep)) == L.E_ARG
    for k, v in (("last_check_time", fl.now_ms), ("scale_up_rpm_threshold", 0)):
        b = p.copy()
        b["janitor"]["scale"][k] = v
        assert call(0, vp(ents), 2, vp(b), vp(out), vp(edits), 4, C.byref(rep)) == L.E_ARG
    assert out.tobytes() == np.full(2, 0x5a, dtype=L.JANITOR_CACHE_ACTION).tobytes()
    # zero cap and NULL edits: the totals only; n = 0: no entries, the registry pass on an empty cache
    assert call(0, vp(ents), 2, vp(p), vp(out), None, 0, C.byref(rep)) == rep.registry.n_edits >= 0
    assert call(0, None, 0, vp(p), None, None, 0, C.byref(rep)) == rep.registry.n_edits >= 0
    assert rep.registry_ran == 1 and rep.stopped_at == -1
    s.close()
