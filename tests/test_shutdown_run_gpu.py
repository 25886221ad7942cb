"""mmp_shutdown_run, one pod's pre-shutdown migration in one call, against its restatement from the Java text
(tests/shutdown_run_oracle.py): out and report, exactly --
  * on C2, C3, C5, MIX and a C3 fleet in a rolling upgrade (half the pods on a newer version, the old replicasets
    likely-replaced), for the pod with the most registrations holding entries of the models it holds (three recent failure
    records on a quarter of them, at most ten), of models it has only failed on and of models it does not hold, lru_t
    values recent, stale, at the cutoff and 0 with every kind of last_used, and gone, failed and aborted entries; with and
    without a fresh row;
  * against the composed route: the same classification on the host and mmp_place_batch of the same records (MMP_DF_OWN_ID,
    extra {self}), byte for byte;
  * before and after the pod's own shutting-down record is committed, with the same fresh row: the same output;
  * on a replayed ingest stream, after every commit;
  * every argument error, MMP_E_EPOCH and MMP_E_STATE."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

import shutdown_run_oracle as sro
from helpers import oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import load_into_fleet, make_fleet
from replay import run_window
from test_janitor_run_gpu import _set_regs
from test_registry_overflow_gpu import _TimedReplay
from test_rolling_upgrade_gpu import upgrade
from test_shutdown_run_oracle import EXPIRY, HOUR, params

pytestmark = pytest.mark.gpu
vp = lambda a: a.ctypes.data_as(C.c_void_p)
FLEETS = [("C2", 3000, 400, 2), ("C3", 4000, 600, 3), ("C5", 3000, 500, 5), ("MIX", 1500, 320, 14), ("C3/upgrade", 4000, 600, 21)]


def _fleet(config, nm, ni, seed):
    base, _, upg = config.partition("/")
    fl = make_fleet(base, nm, ni, seed)
    if upg:
        fl = upgrade(fl, "half", seed)
        fl = dataclasses.replace(fl, replaced_replicasets=sorted({i[:6] for i in fl.inst_ids if len(i) >= 7}))
        assert fl.replaced_replicasets and len(set(fl.inst_rows["vers"])) == 2
    return fl


def _workload(config, nm, ni, seed):
    """(fleet, times, pod): three recent failure records on a quarter of the pod's models, at most 10"""
    fl = _fleet(config, nm, ni, seed)
    rng = np.random.default_rng(seed)
    S = int(np.argmax(np.bincount(fl.edge_inst, minlength=ni)))
    held = sorted(set(int(m) for m in np.searchsorted(fl.edge_off, np.nonzero(fl.edge_inst == S)[0], side="right") - 1))
    others = [i for i in range(ni) if i != S]
    changes = {}
    for m in rng.choice(held, min(10, max(1, len(held) // 4)), replace=False):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        regs = list(fl.edge_inst[a:b])
        extra = [i for i in rng.choice(others, 8, replace=False) if i not in regs][:3]
        changes[int(m)] = (list(fl.edge_inst[a:a + k]), list(fl.edge_inst[a + k:b]) + extra)
    _set_regs(fl, changes)
    n = len(fl.edge_inst)
    ts = np.where(rng.uniform(size=n) < 0.3, fl.now_ms - rng.integers(0, EXPIRY, size=n),
                  fl.now_ms - rng.integers(EXPIRY, 4 * HOUR, size=n)).astype(np.int64)
    for m in changes:
        ts[int(fl.edge_off[m + 1]) - 3:int(fl.edge_off[m + 1])] = fl.now_ms - rng.integers(0, EXPIRY // 2, size=3)
    return fl, ts, S


def _entries(fl, S, rng, n_unreg=30):
    """the pod's cache: every model it is registered on (loaded or failed) and models it does not hold, in descending lru_t
    order as descendingLruMap returns them"""
    mine = sorted(set(int(m) for m in np.searchsorted(fl.edge_off, np.nonzero(fl.edge_inst == S)[0], side="right") - 1))
    rest = [m for m in range(fl.n_models) if m not in set(mine)]
    models = mine + [int(m) for m in rng.choice(rest, n_unreg, replace=False)]
    n, now, cut = len(models), fl.now_ms, fl.now_ms - HOUR
    e = np.zeros(n, dtype=L.SHUTDOWN_ENTRY)
    e["model"] = models
    u = rng.uniform(size=n)
    e["lru_t"] = np.where(u < 0.5, now - rng.integers(0, HOUR, size=n),
                          np.where(u < 0.75, now - rng.integers(HOUR + 1, 6 * HOUR, size=n), np.where(u < 0.85, cut, 0)))
    v = rng.uniform(size=n)
    e["last_used"] = np.where(v < 0.3, -1, np.where(v < 0.4, 0, np.where(v < 0.55, cut, now - rng.integers(1, 3 * HOUR, size=n))))
    w = rng.uniform(size=n)
    e["flags"] = np.where(w < 0.05, L.SD_ENTRY_GONE, np.where(w < 0.1, L.SD_ENTRY_FAILED, np.where(w < 0.2, L.SD_ENTRY_ABORTED, 0)))
    return e[np.argsort(-e["lru_t"], kind="stable")]


def _build(lib, fl, ts):
    s = solver_from_synth(fl, lib)
    for m in range(fl.n_models):
        s.model_times(m, ts[fl.edge_off[m]:fl.edge_off[m + 1]], 0)
    s.commit()
    return s


def _rep(r):
    return {k: getattr(r, k) for k, _ in L.ShutdownReport._fields_ if k != "reserved"}


def _check(s, o, fl, ts, S, ents, p, seed, fresh=None):
    out, r = s.shutdown_run(S, ents, p, seed, fresh_self=fresh)
    want, wr = sro.shutdown_run(o, fl, ts, S, ents, p, seed, fresh_self=fresh)
    bad = np.nonzero(out != want)[0]
    assert len(bad) == 0, (len(bad), out[bad[:3]], want[bad[:3]])
    assert _rep(r) == wr
    return out, wr


def _composed(s, S, ents, out, p, seed, fresh):
    """the placed entries as mmp_place_batch records with the same ids: the answers must be out's, byte for byte"""
    rows = np.nonzero(out["what"] & L.SD_PLACED)[0]
    if not len(rows):
        return 0
    d = np.zeros(len(rows), dtype=L.DECISION_IN)
    d["model"], d["self"], d["last_used"] = ents["model"][rows], S, out["last_used"][rows]
    d["flags"] = L.DF_FAVOUR_SELF | L.DF_OWN_ID | (rows.astype(np.uint32) << 8)
    d["fresh"], d["extra_off"], d["extra_n"] = -1 if fresh is None else 0, 0, 1
    kw = dict(fresh=None if fresh is None else np.asarray(fresh, dtype=L.INSTANCE_ROW).reshape(1))
    res = s.place_batch(d, int(p["now"][0]), seed, extra=np.array([S], dtype=np.int32), **kw)
    assert res.tobytes() == out[["target", "n_candidates"]][rows].astype(res.dtype).tobytes()
    return len(rows)


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_shutdown_run_matches_the_restatement(product_lib, oracle_lib, config, nm, ni, seed):
    fl, ts, S = _workload(config, nm, ni, seed)
    ents = _entries(fl, S, np.random.default_rng(seed))
    s, o = _build(product_lib, fl, ts), oracle_from_synth(fl)
    fresh = fl.inst_rows[S].copy()
    fresh["used"] = fresh["used"] + fresh["capacity"] // 100
    p = params(fl.now_ms)
    seen = {k: 0 for k in ("n_registered", "will_be_skipped", "n_placed", "n_refused", "n_wait", "not_registered")}
    for fr in (None, fresh):
        out, wr = _check(s, o, fl, ts, S, ents, p, 100 + seed, fresh=fr)
        assert _composed(s, S, ents, out, p, 100 + seed, fr) == wr["n_placed"]
        for k in seen:
            seen[k] += wr[k] if k in wr else int(np.count_nonzero(out["what"] & L.SD_NOT_REGISTERED))
        t = C.c_double()
        s._ck(s.lib.mmp_last_timing(s.h, b"shutdown_run", C.byref(t)))
        assert t.value > 0
    assert all(v > 0 for v in seen.values()), seen
    # the pod's own shutting-down record committed: the same answers for the same fresh row
    before, rb = s.shutdown_run(S, ents, p, 7, fresh_self=fresh)
    row = fl.inst_rows[S].copy()
    row["shutting_down"] = 1
    s.instance_update(S, row)
    s.commit()
    after, ra = s.shutdown_run(S, ents, p, 7, fresh_self=fresh)
    assert after.tobytes() == before.tobytes() and _rep(ra) == _rep(rb)
    s.close()
    o.close()


def test_shutdown_run_replayed_stream(product_lib, oracle_lib):
    """after every commit of a replayed ingest stream whose upserts come with registration times, device and host paths"""
    rp = _TimedReplay(make_fleet("C3", 3000, 600, 3), product_lib, 3)
    paths = set()
    for w in range(8):
        run_window(rp, w)
        paths.add(rp.windows[-1][1])
        v, o = rp.view(), rp.oracle()
        ts = np.zeros(len(v.edge_inst), dtype=np.int64)
        for m, (t, _) in rp.times.items():
            a, b = int(v.edge_off[m]), int(v.edge_off[m + 1])
            k = min(len(t), b - a)
            ts[a:a + k] = t[:k]
        co = o.cluster_order()
        cnt = np.bincount(v.edge_inst, minlength=max(v.n_instances, int(co.max()) + 1))
        ranked = np.zeros(len(cnt), dtype=bool)
        ranked[co] = True
        S = int(np.argmax(np.where(ranked, cnt, -1)))   # (the stream takes pods out: the pod places from its published row)
        ents = _entries(v, S, np.random.default_rng(w), n_unreg=10)
        _, wr = _check(rp.f, o, v, ts, S, ents, params(rp.now), 7)
        assert wr["n_placed"] > 0
        o.close()
    assert paths == {1, 2}, paths


def test_shutdown_run_only_instance(product_lib):
    one = make_fleet("C3", 10, 1, 4)
    s = Fleet(one.min_space_units, one.min_churn_age_ms, one.default_model_size_units, 1, one.n_models, lib=product_lib)
    load_into_fleet(one, s)
    for m in range(one.n_models):
        s.model_times(m, np.full(int(one.edge_off[m + 1] - one.edge_off[m]), one.now_ms - HOUR, dtype=np.int64), 0)
    s.commit()
    e = np.zeros(3, dtype=L.SHUTDOWN_ENTRY)
    e["model"], e["lru_t"] = [0, 1, 2], one.now_ms - 1
    out, r = s.shutdown_run(0, e, params(one.now_ms), 1)
    assert r.found_other == 0 and r.n_registered == 0 and r.n_placed == 0
    assert list(out["what"]) == [0, 0, 0] and list(out["target"]) == [L.TARGET_INVALID] * 3 and list(out["model"]) == [0, 1, 2]
    s.close()


def test_shutdown_run_errors(product_lib):
    fl = make_fleet("C3", 200, 40, 5)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    p = params(fl.now_ms)
    ents = np.zeros(2, dtype=L.SHUTDOWN_ENTRY)
    ents["model"], ents["lru_t"] = [3, 4], fl.now_ms - 1
    with pytest.raises(MmpError) as e:
        s.shutdown_run(0, ents, p, 1)
    assert e.value.code == L.E_EPOCH
    load_into_fleet(fl, s)
    s.commit()
    with pytest.raises(MmpError) as e:   # no registration times
        s.shutdown_run(0, ents, p, 1)
    assert e.value.code == L.E_STATE
    for m in range(fl.n_models):
        s.model_times(m, np.full(int(fl.edge_off[m + 1] - fl.edge_off[m]), fl.now_ms - HOUR, dtype=np.int64), 0)
    s.commit()
    s.shutdown_run(0, ents, p, 1)
    out = np.zeros(2, dtype=L.SHUTDOWN_ACTION)
    rep = L.ShutdownReport()
    bad_row = fl.inst_rows[0:1].copy()
    bad_row["used"] = -1
    call = lambda sf, e, n, pp, fr, o_, r_: s.lib.mmp_shutdown_run(s.h, sf, e, n, pp, fr, 1, o_, r_)
    args = lambda **k: {**dict(sf=0, e=vp(ents), n=2, pp=vp(p), fr=None, o_=vp(out), r_=C.byref(rep)), **k}
    before = out.copy()
    for self_idx in (-1, fl.n_instances):
        assert call(**args(sf=self_idx)) == L.E_ARG
    for bad in ([3, 3], [-1, 4], [3, fl.n_models]):
        b = ents.copy()
        b["model"] = bad
        assert call(**args(e=vp(b))) == L.E_ARG
    assert call(**args(n=-1)) == L.E_ARG
    assert call(**args(pp=None)) == L.E_ARG
    assert call(**args(r_=None)) == L.E_ARG
    assert call(**args(o_=None)) == L.E_ARG
    assert call(**args(e=None)) == L.E_ARG
    assert call(**args(fr=vp(bad_row))) == L.E_ARG
    assert out.tobytes() == before.tobytes()
    assert call(**args(n=0, e=None, o_=None)) == 0 and rep.found_other == 1
    s.close()
