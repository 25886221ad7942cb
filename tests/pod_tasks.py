"""Plumbing of the pod-task tests (the janitor, janitor-task, rate, shutdown, eviction and reaper calls, and their edges):
the parameter record of each task, the fleets and workloads they run on, a replayed stream with registration times, a
committed solver with those times, a report struct as a dict, and the composed-route checks (the same decisions through
mmp_scale_eval and mmp_place_batch)."""
import ctypes as C
import dataclasses

import numpy as np

import rate_run_oracle as rro
from common import EXPIRY, HOUR, LONG_MAX, vp
from helpers import solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import NOW_MS, make_fleet
from replay import Replay
from upgrade import upgrade

IT = 5000                  # the iteration of the rate and janitor parameters
HAND_TIMEOUT = 60_000      # load_timeout_ms of the hand-built eviction cases
FREQ_S, LOAD_TIMEOUT = 360, 30_000
WINDOW = FREQ_S * 2000 + LOAD_TIMEOUT     # 750 000 ms: the janitor task's recent-use window under its default parameters
MIN_STALE = 6 * HOUR + 123_456


# ------------------------------------------------------------------------------------------------------------ parameters

def janitor_params(now, adjusted_capacity, flags=0):
    p = np.zeros(1, dtype=L.JANITOR_PARAMS)
    s = p["scale"]
    s["now"], s["last_check_time"], s["iteration"], s["scale_up_rpm_threshold"] = now, now - 10_000, 5000, 2000
    s["rate_check_interval_ms"], s["assume_completed_ms"], s["second_copy_remove_max_age_ms"] = 10_000, 30_000, 1000
    p["scale"] = s
    p["load_failure_expiry_ms"], p["adjusted_capacity"], p["flags"] = EXPIRY, adjusted_capacity, flags
    return p


def janitor_task_params(now, adjusted_capacity=1 << 40, flags=0, min_stale=MIN_STALE, freq=FREQ_S, timeout=LOAD_TIMEOUT):
    p = np.zeros(1, dtype=L.JANITOR_TASK_PARAMS)
    p["janitor"] = janitor_params(now, adjusted_capacity, flags)[0]
    p["janitor"]["scale"]["second_copy_remove_max_age_ms"] = 36 * HOUR
    p["min_stale_age_ms"], p["janitor_freq_secs"], p["load_timeout_ms"] = min_stale, freq, timeout
    return p


def rate_params(now, thr, delta=10_000, expiry=EXPIRY):
    p = np.zeros(1, dtype=L.RATE_PARAMS)
    s = p["scale"]
    s["now"], s["last_check_time"], s["iteration"], s["scale_up_rpm_threshold"] = now, now - delta, IT, thr
    s["second_copy_min_age_iters"], s["second_copy_max_age_iters"], s["second_copy_lru_threshold_ms"] = 42, 240, -1
    s["rate_check_interval_ms"], s["assume_completed_ms"], s["second_copy_remove_max_age_ms"] = 10_000, 30_000, HOUR
    p["scale"] = s
    p["load_failure_expiry_ms"] = expiry
    return p


def shutdown_params(now=NOW_MS, cutoff_age=HOUR, expiry=EXPIRY):
    p = np.zeros(1, dtype=L.SHUTDOWN_PARAMS)
    p["now"], p["cutoff_age_ms"], p["load_failure_expiry_ms"] = now, cutoff_age, expiry
    return p


def evict_params(now=NOW_MS, timeout=HAND_TIMEOUT, expiry=EXPIRY):
    p = np.zeros(1, dtype=L.EVICT_PARAMS)
    p["now"], p["load_timeout_ms"], p["load_failure_expiry_ms"] = now, timeout, expiry
    return p


# ---------------------------------------------------------------------------------------------------- fleets and streams

def set_regs(fl, changes):
    """replace the registrations of the models in changes {m: (loaded, failed)} (instance lists)"""
    lists = []
    for m in range(fl.n_models):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        lists.append(changes.get(m, (list(fl.edge_inst[a:a + k]), list(fl.edge_inst[a + k:b]))))
    fl.edge_off = np.zeros(fl.n_models + 1, dtype=np.int64)
    np.cumsum([len(x) + len(y) for x, y in lists], out=fl.edge_off[1:])
    fl.edge_inst = np.array([i for x, y in lists for i in list(x) + list(y)], dtype=np.int32)
    fl.n_loaded = np.array([len(x) for x, _ in lists], dtype=np.int32)
    fl.n_failed = np.array([len(y) for _, y in lists], dtype=np.int32)


def held_models(fl, S):
    """the models pod S is registered on (loaded or failed), ascending"""
    return sorted(set(int(m) for m in np.searchsorted(fl.edge_off, np.nonzero(fl.edge_inst == S)[0], side="right") - 1))


def busiest_pod(fl, ranked=None):
    """the instance with the most registrations; only among the instances `ranked` (an index array) where given"""
    if ranked is None:
        return int(np.argmax(np.bincount(fl.edge_inst, minlength=fl.n_instances)))
    cnt = np.bincount(fl.edge_inst, minlength=max(fl.n_instances, int(ranked.max()) + 1))
    mask = np.zeros(len(cnt), dtype=bool)
    mask[ranked] = True
    return int(np.argmax(np.where(mask, cnt, -1)))


TASK_FLEETS = [("C2", 3000, 400, 2), ("C3", 4000, 600, 3), ("C5", 3000, 500, 5), ("MIX", 1500, 320, 14), ("C3/upgrade", 4000, 600, 21)]


def task_fleet(config, nm, ni, seed):
    """make_fleet(config) or, for "BASE/upgrade", make_fleet(BASE) with half the pods on a newer version and the old
    replicasets likely-replaced"""
    base, _, upg = config.partition("/")
    fl = make_fleet(base, nm, ni, seed)
    if upg:
        fl = upgrade(fl, "half", seed)
        fl = dataclasses.replace(fl, replaced_replicasets=sorted({i[:6] for i in fl.inst_ids if len(i) >= 7}))
        assert fl.replaced_replicasets and len(set(fl.inst_rows["vers"])) == 2
    return fl


def janitor_workload(config, nm, ni, seed, wide=False, saturated=False):
    """(fleet, times, lastUnloadTime, self) with self's failed registrations on 60 more models, and optionally self as the sixth
    of seven loaded copies on 20 models and a model with 280 copies + 20 failed loads that include self"""
    fl = make_fleet(config, nm, ni, seed)
    fl.inst_rows["used"] = fl.inst_rows["capacity"] - fl.inst_rows["capacity"] // 50
    rng = np.random.default_rng(seed)
    S = int(np.argmax(np.bincount(fl.edge_inst[np.repeat(np.arange(nm), np.diff(fl.edge_off)) >= 0], minlength=ni)))
    held = set(held_models(fl, S))
    free = [m for m in range(nm) if m not in held]
    changes = {}
    for m in rng.choice(free, 60, replace=False):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        changes[int(m)] = (list(fl.edge_inst[a:a + k]), list(fl.edge_inst[a + k:b]) + [S])
    others = [i for i in range(ni) if i != S]
    if wide:
        for m in rng.choice([m for m in free if m not in changes], 20, replace=False):
            ids = list(rng.choice(others, 6, replace=False))
            changes[int(m)] = (ids[:5] + [S] + ids[5:], [])
    if saturated:
        m = int(free[-1])
        ids = list(rng.choice(others, min(299, len(others)), replace=False))
        changes[m] = (ids[:279] + [S], ids[279:])
    set_regs(fl, changes)
    n = len(fl.edge_inst)
    ts = np.where(rng.uniform(size=n) < 0.3, fl.now_ms - rng.integers(0, EXPIRY + 2, size=n),
                  fl.now_ms - rng.integers(EXPIRY, 4 * HOUR, size=n)).astype(np.int64)
    lul = np.where(rng.uniform(size=nm) < 0.3, fl.now_ms - rng.integers(0, 200_000, size=nm), 0).astype(np.int64)
    return fl, ts, lul, S


def janitor_entries(fl, ts, S, rng, n_unreg=40):
    """the pod's cache: most of the models it holds (some failed, some with a wrong load_ts, some lastUsed shared or
    Long.MAX_VALUE), entries on some of its failure records (failed or not, used within 3 minutes or not), and entries of
    models that do not reference it"""
    now, out = fl.now_ms, []
    shared = now - 7 * HOUR
    for m in range(fl.n_models):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        regs = list(fl.edge_inst[a:b])
        if S not in regs:
            continue
        j = regs.index(S)
        u = rng.uniform()
        if j < k:
            if u < 0.1:
                continue
            e = np.zeros(1, dtype=L.JANITOR_ENTRY)[0]
            e["model"], e["weight"] = m, int(rng.integers(1, 400))
            r = rng.uniform()
            e["last_used"] = shared if r < 0.1 else (LONG_MAX if r < 0.13 else now - int(rng.integers(1, 40 * HOUR)))
            e["load_ts"] = ts[a + j] if rng.uniform() < 0.85 else ts[a + j] + 1
            e["last_heavy"] = 0 if rng.uniform() < 0.5 else now - int(rng.integers(0, 30 * HOUR))
            e["count"] = int(rng.integers(0, 50))
            e["flags"] = L.JANITOR_FAILED if rng.uniform() < 0.1 else 0
        else:
            if u < 0.5:
                continue
            e = np.zeros(1, dtype=L.JANITOR_ENTRY)[0]
            e["model"], e["weight"] = m, int(rng.integers(1, 400))
            e["last_used"] = -1 if rng.uniform() < 0.3 else now - int(rng.choice([int(rng.integers(1, 179_999)), 179_999, 180_000, int(rng.integers(180_000, HOUR))]))
            e["flags"] = L.JANITOR_FAILED if rng.uniform() < 0.7 else 0
        out.append(e)
    mine = set(int(e["model"]) for e in out)
    for m in rng.choice([m for m in range(fl.n_models) if m not in mine], n_unreg, replace=False):
        e = np.zeros(1, dtype=L.JANITOR_ENTRY)[0]
        e["model"], e["weight"], e["last_used"] = m, 10, now - 1000
        out.append(e)
    ents = np.array(out, dtype=L.JANITOR_ENTRY)
    return ents[rng.permutation(len(ents))]


class TimedReplay(Replay):
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

    def view_times(self, v):
        """(the time of every registration of the view v, lastUnloadTime per model): what the last commit holds"""
        ts = np.zeros(len(v.edge_inst), dtype=np.int64)
        lul = np.zeros(v.n_models, dtype=np.int64)
        for m, (t, u) in self.times.items():
            a, b = int(v.edge_off[m]), int(v.edge_off[m + 1])
            k = min(len(t), b - a)
            ts[a:a + k] = t[:k]
            lul[m] = u
        return ts, lul


def timed_solver(lib, fl, ts, lul=None, gone=(), skip_empty=False, max_models=None):
    """the solver of fl with ts, the time of every registration, and lul, lastUnloadTime per model (0 for every model when
    None), the instances `gone` removed, committed; skip_empty: no mmp_model_times for a model without registrations"""
    s = solver_from_synth(fl, lib, max_models=max_models)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if a < b or not skip_empty:
            s.model_times(m, ts[a:b], 0 if lul is None else int(lul[m]))
    for i in gone:
        s.instance_remove(int(i))
    s.commit()
    return s


# ------------------------------------------------------------------------------------------------------------ checks

def report_dict(r, skip=("reserved",)):
    """a report struct as a dict of its fields (a nested report as a dict too), without the fields in skip"""
    return {k: report_dict(getattr(r, k), skip) if isinstance(getattr(r, k), C.Structure) else getattr(r, k)
            for k, _ in r._fields_ if k not in skip}


def same_out(x, y):
    return all(np.array_equal(x[k], y[k]) for k in x.dtype.names)


def composed_shutdown(s, S, ents, out, p, seed, fresh):
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


def composed_evict(s, S, ents, out, p, seed, fresh):
    """the placed entries as mmp_place_batch records with the same ids: the answers must be out's, byte for byte"""
    rows = np.nonzero(out["what"] & L.EV_PLACED)[0]
    if not len(rows):
        return 0
    d = np.zeros(len(rows), dtype=L.DECISION_IN)
    d["model"], d["self"], d["last_used"] = ents["model"][rows], S, ents["last_used"][rows]
    d["flags"] = L.DF_FAVOUR_SELF | L.DF_OWN_ID | (rows.astype(np.uint32) << 8)
    d["fresh"], d["extra_off"], d["extra_n"] = -1 if fresh is None else 0, 0, 1
    kw = dict(fresh=None if fresh is None else np.asarray(fresh, dtype=L.INSTANCE_ROW).reshape(1))
    res = s.place_batch(d, int(p["now"][0]), seed, extra=np.array([S], dtype=np.int32), **kw)
    assert res.tobytes() == out[["target", "n_candidates"]][rows].astype(res.dtype).tobytes()
    return len(rows)


def ids(fl, ts, ents, out, p):
    """each entry's first decision id (the exclusive prefix sum of its decisions), -1 where it places none"""
    now, expiry = int(p["scale"]["now"][0]), int(p["load_failure_expiry_ms"][0])
    ids, off = np.full(len(ents), -1), 0
    for r, (e, x) in enumerate(zip(ents, out)):
        if int(x["action"]) in (1, 2) and not rro.refused(fl, ts, int(e["model"]), now, expiry):
            ids[r] = off
            off += 1 if int(x["action"]) == 1 else min(int(x["copies_to_load"]), L.RATE_CHAIN_MAX)
    return ids


def cross_check_rate(s, fl, ts, S, ents, p, seed, out, loads, heavy, fresh):
    """out is mmp_scale_eval's (can_remove = 0) field by field; round-0 scale-up loads are mmp_place_batch_excluding's under
    the heavy set with the same MMP_DF_OWN_ID ids; second copies are mmp_place_batch's with extra {self}"""
    sp = p["scale"].copy()
    sp["can_remove"] = 0
    se = np.zeros(len(ents), dtype=L.SCALE_OUT)
    s._ck(s.lib.mmp_scale_eval(s.h, vp(ents), len(ents), vp(sp), vp(se)))
    assert same_out(out, se)
    first = ids(fl, ts, ents, out, p)
    now = int(p["scale"]["now"][0])
    kw = dict(fresh=None if fresh is None else np.asarray(fresh, dtype=L.INSTANCE_ROW).reshape(1))
    for second in (True, False):
        sel = [ld for ld in loads if ld[2] == 0 and bool(ld[7] & L.RL_SECOND_COPY) == second]
        if not sel:
            continue
        d = np.zeros(len(sel), dtype=L.DECISION_IN)
        for q, ld in enumerate(sel):
            r, m = ld[0], ld[1]
            a, k = int(fl.edge_off[m]), int(fl.n_loaded[m])
            fav = second or S in set(int(i) for i in fl.edge_inst[a:a + k])
            d["model"][q], d["self"][q], d["last_used"][q] = m, S, ld[6]
            d["flags"][q] = (L.DF_FAVOUR_SELF if fav else 0) | L.DF_OWN_ID | (int(first[r]) << 8)
            d["fresh"][q] = -1 if fresh is None else 0
            d["extra_off"][q], d["extra_n"][q] = 0, 1 if second else 0
        if second:
            res = s.place_batch(d, now, seed, extra=np.array([S], dtype=np.int32), **kw)
        else:
            res = s.place_batch(d, now, seed, exclude=np.asarray(heavy, dtype=np.int32), **kw)
        assert [(int(x["target"]), int(x["n_candidates"])) for x in res] == [(ld[4], ld[5]) for ld in sel], second
