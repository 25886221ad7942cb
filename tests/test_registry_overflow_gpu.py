"""The registry-side batch scans over EVERY registration of a model, not only the four inline edges:
  mmp_scale_eval          rateTrackingTask's loop body and the janitor's removeModelCopies for models with any number of
                          loaded copies and failed loads, against orc_rate_task_eval / orc_janitor_eval
  mmp_registry_prune_ids  pruneMissingInstances over every registration, against orc_prune_missing
  mmp_registry_prune      the four-registration view, against the oracle run on each model's first four registrations
Times reach positions past the fourth through mmp_model_times and through mmp_model_upsert_json alike, and survive the
incremental commits of a replayed ingest stream (tests/replay.py) as a fleet rebuilt from scratch holds them."""
import ctypes as C
import json

import numpy as np
import pytest

from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet
from modelmesh_b200.synth import load_into_fleet, make_fleet
from oracle import binding as ob
from replay import Replay, run_window

pytestmark = pytest.mark.gpu

HOUR = 3_600_000
GONE_MS = 600_000   # ASSUME_INSTANCE_GONE_AFTER_MS
PARAM_SETS = ((2000, 1, 6 * HOUR), (300, 1, 1000), (5, 0, 6 * HOUR))
vp = lambda a: a.ctypes.data_as(C.c_void_p)


def _overflow_heavy(nm: int, ni: int, seed: int):
    """C3 instances with about a quarter of the models holding 5-40 registrations, loaded and failed mixed (a quarter of those
    with one copy and 4-39 failed loads), the cluster 2 % from full (the janitor's scale-down needs <= 5 % free), and one last
    model with a saturated copy count: 280 copies + 20 failed loads."""
    fl = make_fleet("C3", nm, ni, seed)
    rng = np.random.default_rng(seed)
    heavy = rng.uniform(size=nm) < 0.25
    deg = np.where(heavy, rng.integers(5, 41, size=nm), rng.integers(0, 5, size=nm))
    nl = np.where(heavy & (rng.uniform(size=nm) < 0.25), 1, rng.integers(0, deg + 1))
    nl = np.where(heavy & (nl == 0), 2, nl)
    deg[-1], nl[-1] = 300, 280
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(deg, out=fl.edge_off[1:])
    fl.edge_inst = np.concatenate([rng.choice(ni, size=int(d), replace=False) for d in deg]).astype(np.int32)
    fl.n_loaded, fl.n_failed = nl.astype(np.int32), (deg - nl).astype(np.int32)
    fl.inst_rows["used"] = fl.inst_rows["capacity"] - fl.inst_rows["capacity"] // 50
    return fl


def _fleet(config: str, nm: int, ni: int, seed: int):
    return _overflow_heavy(nm, ni, seed) if config == "HEAVY" else make_fleet(config, nm, ni, seed)


def _times(fl, rng):
    """A load / failure time for every registration and a lastUnloadTime per model.  Half of the models have only old times
    (1-4 h), the others a mix with 30 % within the last two minutes, at every position."""
    n, nm = len(fl.edge_inst), fl.n_models
    old = np.repeat(rng.uniform(size=nm) < 0.5, np.diff(fl.edge_off))
    ts = fl.now_ms - rng.integers(HOUR, 4 * HOUR, size=n)
    mixed = np.where(rng.uniform(size=n) < 0.3, fl.now_ms - rng.integers(0, 120_000, size=n), fl.now_ms - rng.integers(0, 4 * HOUR, size=n))
    ts = np.where(old, ts, mixed).astype(np.int64)
    lul = np.where(rng.uniform(size=nm) < 0.3, fl.now_ms - rng.integers(0, 200_000, size=nm), 0).astype(np.int64)
    return ts, lul


def _load(lib, fl, ts, lul, ni=None):
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, ni or fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    for m in range(fl.n_models):
        s.model_times(m, ts[fl.edge_off[m]:fl.edge_off[m + 1]], int(lul[m]))
    s.commit()
    return s


def _records(fl, rng, n, models):
    rec = np.zeros(n, dtype=L.SCALE_IN)
    rec["model"] = models
    # the entry belongs to a pod that holds a copy (at any position) when the model has copies, to any pod otherwise
    for r in range(n):
        m = int(models[r])
        k = int(fl.n_loaded[m])
        rec["instance"][r] = int(fl.edge_inst[fl.edge_off[m] + rng.integers(0, k)]) if k and rng.uniform() < 0.9 else int(rng.integers(0, fl.n_instances))
    rec["count"] = np.where(rng.uniform(size=n) < 0.5, rng.integers(0, 50, size=n), rng.integers(0, 20_000, size=n))
    rec["last_used"] = np.where(rng.uniform(size=n) < 0.05, 0, fl.now_ms - rng.integers(0, 40 * HOUR, size=n))
    rec["last_heavy"] = np.where(rng.uniform(size=n) < 0.4, 0, fl.now_ms - rng.integers(0, 30 * HOUR, size=n))
    rec["flags"] = (rng.uniform(size=n) < 0.15).astype(np.int32)  # MMP_SCALE_NO_LOCAL_STATS
    it = 5000
    rec["i1"] = it - rng.integers(0, 400, size=n)
    rec["i2"] = np.minimum(it, rec["i1"] + rng.integers(0, 300, size=n))
    return rec


def _params(now, thr, can_remove, lru_thr):
    p = np.zeros(1, dtype=L.SCALE_PARAMS)
    p["now"], p["last_check_time"], p["iteration"], p["scale_up_rpm_threshold"] = now, now - 10_000, 5000, thr
    p["second_copy_min_age_iters"], p["second_copy_max_age_iters"], p["second_copy_lru_threshold_ms"] = 42, 240, lru_thr
    p["rate_check_interval_ms"], p["assume_completed_ms"], p["second_copy_remove_max_age_ms"], p["can_remove"] = 10_000, 30_000, 36 * HOUR, can_remove
    return p


def _scale(lib, s, rec, p):
    out = np.zeros(len(rec), dtype=L.SCALE_OUT)
    s._ck(lib.mmp_scale_eval(s.h, vp(rec), len(rec), vp(p), vp(out)))
    return out


def _same_scale(x, y) -> bool:
    """Field by field: mmp_scale_out ends in 4 bytes of padding that the library does not write."""
    return all(np.array_equal(x[k], y[k]) for k in x.dtype.names)


def _oracle_scale(oracle_lib, o, fl, ts, lul, rec, p):
    """orc_rate_task_eval / orc_janitor_eval with each record's model as CSR edge lists: every registration, loaded first."""
    n = len(rec)
    m64 = rec["model"].astype(np.int64)
    deg = (fl.edge_off[m64 + 1] - fl.edge_off[m64]).astype(np.int64)
    eoff = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=eoff[1:])
    einst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64]).astype(np.int32)
    ets = np.concatenate([ts[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64]).astype(np.int64)
    nl = fl.n_loaded[m64].astype(np.int32)
    tidx = fl.model_type[m64].astype(np.int32)
    orec = np.zeros(n, dtype=ob.SCALE_IN)
    for k in ("instance", "model", "count", "last_used", "last_heavy", "i1", "i2", "flags"):
        orec[k] = rec[k]
    op = np.zeros(1, dtype=ob.SCALE_PARAMS)
    for k in op.dtype.names:
        if k != "pad":
            op[k] = p[k]
    up = np.zeros(n, dtype=ob.SCALE_OUT)
    down = np.zeros(n, dtype=ob.SCALE_OUT)
    names = (C.c_char_p * len(fl.type_names))(*[t.encode() for t in fl.type_names])
    assert oracle_lib.orc_rate_task_eval(o.h, n, vp(orec), vp(op), names, len(fl.type_names), vp(tidx), vp(eoff), vp(einst), vp(ets), vp(nl), vp(up)) == 0
    lulr = lul[m64].astype(np.int64)
    assert oracle_lib.orc_janitor_eval(o.h, n, vp(orec), vp(op), vp(eoff), vp(einst), vp(ets), vp(nl), vp(lulr), vp(down)) == 0
    return up, down


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 4000, 500, 3), ("C5", 3000, 400, 5), ("MIX", 1500, 160, 14), ("HEAVY", 3000, 500, 41)])
def test_scale_eval_over_every_registration(product_lib, oracle_lib, config, nm, ni, seed):
    rng = np.random.default_rng(seed)
    fl = _fleet(config, nm, ni, seed)
    ts, lul = _times(fl, rng)
    deg = np.diff(fl.edge_off)
    o = oracle_from_synth(fl)
    n = 6000
    saturated = np.nonzero(fl.n_loaded > 255)[0]
    plain = np.setdiff1d(np.arange(nm), saturated)
    # half of the records on models with more than four registrations, where there are any
    wide = np.setdiff1d(np.nonzero(deg > 4)[0], saturated)
    models = plain[rng.integers(0, len(plain), size=n)]
    if len(wide):
        models = np.where(rng.uniform(size=n) < 0.5, wide[rng.integers(0, len(wide), size=n)], models)
    rec = _records(fl, rng, n, models)
    pos = np.full(n, -1)
    for r in range(n):
        a, b = fl.edge_off[models[r]], fl.edge_off[models[r] + 1]
        hit = np.nonzero(fl.edge_inst[a:b] == rec["instance"][r])[0]
        pos[r] = hit[0] if len(hit) else -1
    if config == "HEAVY":
        assert (pos >= 4).sum() > 500  # entries owned by the pod whose copy sits past the inline edges
    s = _load(product_lib, fl, ts, lul)
    ovf = deg[models] > 4
    seen = np.zeros(3, dtype=np.int64)
    for thr, can_remove, lru_thr in PARAM_SETS:
        p = _params(fl.now_ms, thr, can_remove, lru_thr)
        out = _scale(product_lib, s, rec, p)
        up, down = _oracle_scale(oracle_lib, o, fl, ts, lul, rec, p)
        for k in ("action", "copies_to_load", "load_last_used", "rpm", "i1", "i2", "set_heavy"):
            bad = np.nonzero(out[k] != up[k])[0]
            assert len(bad) == 0, (thr, k, len(bad), bad[:5], out[bad[:5]], up[bad[:5]], rec[bad[:5]], deg[models[bad[:5]]])
        bad = np.nonzero(out["remove"] != down["remove"])[0]
        assert len(bad) == 0, (thr, "remove", len(bad), bad[:5], rec[bad[:5]], deg[models[bad[:5]]])
        assert not (out["action"] == -1).any(), thr
        seen += [np.count_nonzero(ovf & (out["action"] == 1)), np.count_nonzero(ovf & (out["action"] == 2)), np.count_nonzero(ovf & (out["remove"] == 1))]
        if len(saturated):  # copy_count 255 over 300 registrations: loaded and failed cannot be told apart
            srec = _records(fl, rng, 64, np.full(64, saturated[0]))
            sout = _scale(product_lib, s, srec, p)
            assert (sout["action"] == -1).all() and not sout["remove"].any()
    if config == "HEAVY":
        assert (seen > 0).all(), seen
    o.close()
    s.close()


def _oracle_prune(oracle_lib, o, fl, ts, self_idx, now, missing, first=None):
    """orc_prune_missing over every model (or its first `first` registrations): (model, instance) pairs and per-model masks."""
    pairs, masks = [], {}
    pruned = np.zeros(max(1, int(np.diff(fl.edge_off).max())), dtype=np.uint8)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if first is not None:
            b = min(b, a + first)
        if a == b:
            continue
        k = oracle_lib.orc_prune_missing(o.h, self_idx, vp(fl.edge_inst[a:b]), vp(ts[a:b]), b - a, now, GONE_MS, vp(missing), vp(pruned))
        if k:
            pairs += [(m, int(fl.edge_inst[a + j])) for j in range(b - a) if pruned[j]]
            masks[m] = sum(int(pruned[j]) << j for j in range(b - a))
    return pairs, masks


def test_registry_prune_over_every_registration(product_lib, oracle_lib):
    nm, ni = 8000, 600
    fl = _overflow_heavy(nm, ni, 9)
    rng = np.random.default_rng(9)
    ts, lul = _times(fl, rng)
    ts = np.where(rng.uniform(size=len(ts)) < 0.7, ts - 2 * HOUR, ts)  # most registrations older than the gone interval
    s = _load(product_lib, fl, ts, lul)
    o = oracle_from_synth(fl)
    # 40 pods leave: 30 of them among those holding the most registrations at positions past the fourth
    at_ovf = np.concatenate([fl.edge_inst[fl.edge_off[m] + 4:fl.edge_off[m + 1]] for m in range(nm)])
    ranked = np.argsort(-np.bincount(at_ovf, minlength=ni), kind="stable")
    gone = np.concatenate([ranked[:30], rng.choice(ranked[30:], size=10, replace=False)])
    self_idx = int(ranked[-1])
    for i in gone:
        s.instance_remove(int(i))
        o.instance_event(ob.DELETED, int(i), None, fl.inst_ids[int(i)], now_ms=fl.now_ms)
    s.commit()
    miss_p, miss_o = np.zeros(ni, dtype=np.int64), np.zeros(ni, dtype=np.int64)
    miss_pi, miss_oi = np.zeros(ni, dtype=np.int64), np.zeros(ni, dtype=np.int64)
    total = 0
    for rnd, now in enumerate((fl.now_ms, fl.now_ms + 360_000, fl.now_ms + 720_000)):
        before = miss_p.copy()
        n, pm, pi = s.registry_prune_ids(self_idx, now, GONE_MS, miss_p, 1 << 20)
        want, _ = _oracle_prune(oracle_lib, o, fl, ts, self_idx, now, miss_o)
        assert n == len(want) and list(zip(pm.tolist(), pi.tolist())) == want, (rnd, n, len(want))
        assert np.array_equal(miss_p, miss_o), rnd
        assert not np.array_equal(before, miss_p) or rnd > 0
        # the same `now` again: the stamping is idempotent, so the same pairs; and a cap below the count: the first ones
        again = miss_p.copy()
        n2, pm2, pi2 = s.registry_prune_ids(self_idx, now, GONE_MS, again, 1 << 20)
        assert n2 == n and np.array_equal(pm2, pm) and np.array_equal(pi2, pi) and np.array_equal(again, miss_p), rnd
        if n > 3:
            cap = n // 3
            n3, pm3, pi3 = s.registry_prune_ids(self_idx, now, GONE_MS, miss_p.copy(), cap)
            assert n3 == n and np.array_equal(pm3, pm[:cap]) and np.array_equal(pi3, pi[:cap]), rnd
        total += n
        # the four-registration view on the same fleet: masks and missing_since as the oracle on the first four
        outm = np.zeros(nm, dtype=np.int32)
        outk = np.zeros(nm, dtype=np.uint8)
        k = s._ck(product_lib.mmp_registry_prune(s.h, self_idx, now, GONE_MS, vp(miss_pi), vp(outm), vp(outk), nm))
        _, masks = _oracle_prune(oracle_lib, o, fl, ts, self_idx, now, miss_oi, first=4)
        assert {int(outm[i]): int(outk[i]) for i in range(k)} == masks, rnd
        assert np.array_equal(miss_pi, miss_oi), rnd
    deg = np.diff(fl.edge_off)
    assert total > 0 and any(deg[m] > 4 for m, _ in want)
    # some pruned registrations sit past the fourth position
    posn = [int(np.nonzero(fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]] == i)[0][0]) for m, i in want]
    assert max(posn) >= 4
    o.close()
    s.close()


def test_json_and_index_ingest_agree(product_lib):
    """Model records with more than four instanceIds / failedIn entries, ingested as JSON with their times, answer the scans
    as the same records upserted by index with mmp_model_times; also after pods leave, when a JSON record's ids resolve to
    fewer registrations and the times move with their ids (index side: the same record upserted without those pods)."""
    nm, ni = 2000, 400
    fl = _overflow_heavy(nm, ni, 17)
    rng = np.random.default_rng(17)
    ts, lul = _times(fl, rng)
    deg = np.diff(fl.edge_off)
    as_json = np.nonzero((deg > 4) | (rng.uniform(size=nm) < 0.2))[0]
    a = _load(product_lib, fl, ts, lul)
    # b: the same records by index, but no times for the ones about to be re-ingested as JSON: their times come from the JSON
    js = np.isin(np.arange(nm), as_json)
    b = _load(product_lib, fl, np.where(np.repeat(js, deg), 0, ts), np.where(js, 0, lul))
    for m in as_json:
        e0, k = int(fl.edge_off[m]), int(fl.n_loaded[m])
        ids = [fl.inst_ids[int(i)] for i in fl.edge_inst[e0:fl.edge_off[m + 1]]]
        t = [int(x) for x in ts[e0:fl.edge_off[m + 1]]]
        doc = {"type": fl.type_names[int(fl.model_type[m])], "instanceIds": dict(zip(ids[:k], t[:k])), "failedIn": dict(zip(ids[k:], t[k:])),
               "lu": int(fl.model_last_used[m]), "lul": int(lul[m])}
        b._ck(product_lib.mmp_model_upsert_json(b.h, int(m), json.dumps(doc).encode(), int(fl.model_size[m])))
    b.commit()
    assert (deg[as_json] > 4).sum() > 300
    models = as_json[rng.integers(0, len(as_json), size=4000)]
    models = models[fl.n_loaded[models] <= 255]
    rec = _records(fl, rng, len(models), models)

    def same_scale(what):
        for thr, can_remove, lru_thr in PARAM_SETS:
            p = _params(fl.now_ms, thr, can_remove, lru_thr)
            assert _same_scale(_scale(product_lib, a, rec, p), _scale(product_lib, b, rec, p)), (what, thr)

    same_scale("ingest")
    # 40 pods leave, most of them named past the fourth position of JSON records
    at_ovf = np.concatenate([fl.edge_inst[fl.edge_off[m] + 4:fl.edge_off[m + 1]] for m in as_json])
    gone = np.argsort(-np.bincount(at_ovf, minlength=ni), kind="stable")[:40]
    tid = {t: a.type_id(t) for t in fl.type_names}
    for m in as_json:
        e0, e1 = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        keep = ~np.isin(fl.edge_inst[e0:e1], gone)
        row = np.zeros(1, dtype=L.MODEL_ROW)
        row["last_used"], row["size_units"], row["rpm"] = fl.model_last_used[m], fl.model_size[m], fl.model_rpm[m]
        row["type_id"], row["copy_count"], row["fail_count"] = tid[fl.type_names[int(fl.model_type[m])]], min(255, fl.n_loaded[m]), min(255, fl.n_failed[m])
        a.model_upsert(int(m), row, fl.edge_inst[e0:e1][keep])
        a.model_times(int(m), ts[e0:e1][keep], int(lul[m]))
    for f in (a, b):
        for i in gone:
            f.instance_remove(int(i))
        f.commit()
    same_scale("pods gone")
    self_idx = int(np.setdiff1d(np.arange(ni), gone)[0])
    ma, mb = np.zeros(ni, dtype=np.int64), np.zeros(ni, dtype=np.int64)
    for now in (fl.now_ms, fl.now_ms + 720_000):
        ra, rb = a.registry_prune_ids(self_idx, now, GONE_MS, ma, 1 << 20), b.registry_prune_ids(self_idx, now, GONE_MS, mb, 1 << 20)
        assert ra[0] == rb[0] and np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2]) and np.array_equal(ma, mb), now
    assert ra[0] > 0
    a.close()
    b.close()


class _TimedReplay(Replay):
    """A replayed stream whose index upserts come with a time for every registration (mmp_model_times before the commit, so
    that the window's own commit carries them).  JSON records carry none: their times read 0."""

    def __init__(self, fl, lib, seed):
        super().__init__(fl, lib, seed)
        self.trng = np.random.default_rng(seed + 1000)
        self.times = {}
        self.touched = set(range(self.n_used))
        self._give()
        self.touched = set()
        self.f.commit()

    def _give(self):
        edges = self.current_edges()
        for m in self.touched:
            if m in self.json_ids:
                self.times[m] = (np.zeros(0, dtype=np.int64), 0)
                continue
            k = len(edges[m])
            ts = np.where(self.trng.uniform(size=k) < 0.3, self.now - self.trng.integers(0, 900_000, size=k),
                          self.now - self.trng.integers(0, 4 * HOUR, size=k)).astype(np.int64)
            self.times[m] = (ts, int(self.now - self.trng.integers(0, 200_000)) if self.trng.uniform() < 0.3 else 0)
            self.f.model_times(m, *self.times[m])

    def commit(self, kind, n_model_edits, events=()):
        self._give()
        return super().commit(kind, n_model_edits, events)

    def timed_scratch(self):
        g = self.scratch()
        for m, (ts, lul) in self.times.items():
            g.model_times(m, ts, lul)
        g.commit()
        return g


@pytest.mark.parametrize("config,nm,ni,seed,n_windows", [("C3", 3000, 600, 3, 8), ("MIX", 2000, 400, 14, 8)])
def test_replayed_commits_match_scratch(product_lib, config, nm, ni, seed, n_windows):
    rp = _TimedReplay(make_fleet(config, nm, ni, seed), product_lib, seed)
    crossed = 0
    for w in range(n_windows):
        before = [len(e) > 4 for e in rp.current_edges()]
        run_window(rp, w)
        after = [len(e) > 4 for e in rp.current_edges()]
        crossed += sum(x != y for x, y in zip(before, after))
        f, g = rp.f, rp.timed_scratch()
        rng = np.random.default_rng(seed * 100 + w)
        live = rp._live()
        missing = np.where(rng.uniform(size=rp.ni_max) < 0.5, rp.now - 660_000, 0).astype(np.int64)
        missing[~rp.present] = rp.now - 660_000
        ma, mb = missing.copy(), missing.copy()
        ra = f.registry_prune_ids(int(live[0]), rp.now, GONE_MS, ma, 1 << 20)
        rb = g.registry_prune_ids(int(live[0]), rp.now, GONE_MS, mb, 1 << 20)
        assert ra[0] == rb[0] and np.array_equal(ra[1], rb[1]) and np.array_equal(ra[2], rb[2]) and np.array_equal(ma, mb), ("prune", w)
        n = 3000
        rec = np.zeros(n, dtype=L.SCALE_IN)
        rec["model"] = rng.integers(0, rp.n_used, size=n)
        edges = rp.current_edges()
        rec["instance"] = [e[int(rng.integers(0, len(e)))] if e and rng.uniform() < 0.8 else int(rng.integers(0, rp.n_ever))
                           for e in (edges[int(m)] for m in rec["model"])]
        rec["count"] = rng.integers(0, 20_000, size=n)
        rec["last_used"] = rp.now - rng.integers(0, 40 * HOUR, size=n)
        rec["last_heavy"] = np.where(rng.uniform(size=n) < 0.4, 0, rp.now - rng.integers(0, 30 * HOUR, size=n))
        rec["i1"] = 5000 - rng.integers(0, 400, size=n)
        rec["i2"] = np.minimum(5000, rec["i1"] + rng.integers(0, 300, size=n))
        for thr, can_remove, lru_thr in PARAM_SETS:
            p = _params(rp.now, thr, can_remove, lru_thr)
            assert _same_scale(_scale(product_lib, f, rec, p), _scale(product_lib, g, rec, p)), ("scale", w, thr)
        g.close()
    assert crossed > 0
