"""The closed loop on fleets whose models hold more than four registrations (loaded copies, then failed loads), against the
oracle's closed loop (oracle/mm_sim.inc), which keeps lists of any length.  Every window is compared as
test_churn_gpu.py compares it; after every window, each model that held more than four registrations at some point must hold,
on the device, the oracle's loaded copies followed by its failed loads (the loop never changes those).  After the trace, the
registry the loop left must place and scale exactly as a fleet committed from scratch with the oracle's registry."""
import dataclasses

import numpy as np
import pytest

from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet
from modelmesh_b200.synth import load_into_fleet, make_churn, make_churn_overflow
from test_churn_gpu import _build, _compare_window

pytestmark = pytest.mark.gpu


def _failed_lists(fl):
    return {int(m): [int(x) for x in fl.edge_inst[fl.edge_off[m] + fl.n_loaded[m]:fl.edge_off[m + 1]]]
            for m in np.nonzero(fl.n_failed > 0)[0]}


class _Registry:
    """the models to follow (more than four registrations at some point) and their failed loads"""

    def __init__(self, fl):
        self.fl = fl
        self.failed = _failed_lists(fl)
        self.watch = set(int(m) for m in np.nonzero(np.diff(fl.edge_off) > 4)[0])
        self.watch |= set(m for m, f in self.failed.items() if len(f) >= 4)  # one load away from a fifth registration

    def check(self, ep, sim, s):
        crossed = 0
        for m in sorted(self.watch):
            copies, lu = sim.model_copies(m)
            want = [int(x) for x in copies] + self.failed.get(m, [])
            row, ids = s.churn_model_ids(m)
            assert list(ids) == want and int(row["copy_count"]) == len(copies) and int(row["reserved"]) == len(want), \
                (ep, m, list(ids), want, int(row["copy_count"]))
            assert int(row["last_used"]) == lu, (ep, m)
            crossed += len(want) > 4
        return crossed


def _run(product_lib, w, windows, seed, slots=256, events=None):
    fl = w.fleet
    o, sim, s = _build(product_lib, w, slots=slots)
    reg = _Registry(fl)
    reg.check(-1, sim, s)
    for ep in range(windows):
        ev = events(ep) if events else w.events(ep, 2000, seed)
        now0 = fl.now_ms + ep * w.window_ms
        _compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, seed * 100 + ep)
        reg.check(ep, sim, s)
    return o, sim, s, reg


@pytest.mark.parametrize("with_types,fill,seed", [(False, 0.90, 4), (True, 0.90, 5), (False, 0.97, 6), (True, 0.97, 7)])
def test_overflow_closed_loop_matches_oracle_small(product_lib, oracle_lib, with_types, fill, seed):
    """12 windows of the 20k-model x 200-instance trace with 5 % of the models at 5-12 registrations"""
    w = make_churn_overflow(make_churn(20_000, 200, seed, fill=fill, with_types=with_types), 0.05, seed)
    fl = w.fleet
    assert (np.diff(fl.edge_off) > 4).sum() > 500 and (fl.n_loaded > 4).sum() > 100
    o, sim, s, reg = _run(product_lib, w, 12, seed)
    # some model went from four registrations to five (a first load of a model with four failed loads)
    pushed = [m for m in reg.watch if fl.n_loaded[m] == 0 and fl.n_failed[m] == 4 and len(sim.model_copies(m)[0]) > 0]
    assert pushed
    _check_registry_readers(product_lib, fl, o, sim, s, reg)


def _trimmed(w, keep_failed):
    """w with every model's failed loads cut to the first keep_failed (its copies and seeds unchanged)"""
    fl = w.fleet
    nf = np.minimum(fl.n_failed, keep_failed)
    cnt = (fl.n_loaded + nf).astype(np.int64)
    off = np.zeros(fl.n_models + 1, dtype=np.int64)
    np.cumsum(cnt, out=off[1:])
    inst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m] + cnt[m]] for m in range(fl.n_models)]).astype(np.int32)
    return dataclasses.replace(w, fleet=dataclasses.replace(fl, edge_off=off, edge_inst=inst, n_failed=nf.astype(np.int32)))


def test_overflow_edges_by_hand(product_lib, oracle_lib):
    """Crafted windows on a fleet where the overflow registrations are all loaded copies:
    window 0  a model with 6 copies hit with u = 0..5, then a REMOVE of every model with more than four registrations (the
              overflow table empties; a 6-copy REMOVE makes six LRU removals);
    window 1  requests of the models the REMOVEs left with failed loads only and of models with four failed loads (the table
              fills from empty: 4 failed + 1 load), beside an ordinary trace;
    then ordinary windows at 0.97 fill, where both copies of a two-copy model are evicted in one window."""
    base = make_churn(20_000, 200, 11, fill=0.97)
    w = _trimmed(make_churn_overflow(base, 0.01, 11, regs=(5, 8)), 4)
    fl = w.fleet
    regs = np.diff(fl.edge_off)
    # the copies of some two-copy models are the oldest entries of their caches: the first loads there evict both in one window
    aged = np.nonzero((fl.n_loaded == 2) & (regs == 2))[0][:20]
    sel = np.isin(w.seed_model, aged)
    lu = w.seed_last_used.copy()
    lu[sel] = fl.now_ms - 400_000_000 - w.seed_model[sel].astype(np.int64)
    rows = fl.inst_rows.copy()
    oldest = rows["lru_time"].astype(np.int64)
    np.minimum.at(oldest, w.seed_instance[sel], lu[sel])
    rows["lru_time"] = oldest
    mlu = fl.model_last_used.copy()
    mlu[w.seed_model[sel]] = lu[sel]
    w = dataclasses.replace(w, seed_last_used=lu, fleet=dataclasses.replace(fl, inst_rows=rows, model_last_used=mlu))
    fl = w.fleet
    six = [int(m) for m in np.nonzero(fl.n_loaded == 6)[0]] + [int(m) for m in np.nonzero(fl.n_loaded > 6)[0]]
    over = [int(m) for m in np.nonzero(regs > 4)[0]]
    four_failed = [int(m) for m in np.nonzero((fl.n_loaded == 0) & (fl.n_failed == 4))[0]]
    assert six and over and four_failed and all(fl.n_loaded[m] > 0 for m in over)
    left_failed = [m for m in over if fl.n_failed[m] > 0]
    evicted_two = 0

    def events(ep):
        now0 = fl.now_ms + ep * w.window_ms
        live = np.nonzero(fl.inst_rows["shutting_down"] == 0)[0]
        ev = []
        if ep == 0:
            ev += [(0, six[0], u, 10 + u) for u in range(int(fl.n_loaded[six[0]]))]
            ev += [(1, m, 0, 100 + k % 1500) for k, m in enumerate(over)]
        elif ep == 1:
            ev += [(0, m, 0, 10 + k % 1900) for k, m in enumerate(left_failed + four_failed[:100])]
        out = np.zeros(len(ev), dtype=L.CHURN_EVENT)
        for k, (ty, m, u, dt) in enumerate(ev):
            out[k] = (ty, m, int(live[(m * 7 + k) % len(live)]), u, now0 + dt)
        if ep == 0:
            return out
        if ep >= 2:
            return w.events(ep, 3000, 11)
        return np.sort(np.concatenate([out, w.events(ep, 600, 11)]), order="t", kind="stable")

    o, sim, s = _build(product_lib, w, slots=256)
    reg = _Registry(fl)
    for ep in range(8):
        ev = events(ep)
        now0 = fl.now_ms + ep * w.window_ms
        dec, evi, _ = _compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, 1100 + ep)
        crossed = reg.check(ep, sim, s)
        if ep == 0:
            assert crossed == 0, crossed  # nothing left past four: the overflow table is empty
            assert all(len(sim.model_copies(m)[0]) == 0 for m in over)
        if ep == 1:
            assert crossed > 0  # a fifth registration from an empty table
        pairs = {}
        for e in evi:
            pairs.setdefault(int(e["model"]), set()).add(int(e["instance"]))
        evicted_two += sum(1 for m, i in pairs.items() if len(i) > 1)
    assert evicted_two > 0
    _check_registry_readers(product_lib, fl, o, sim, s, reg)


def _fresh_fleet(product_lib, fl, sim, rows, rename=None):
    """a fleet committed once from the oracle's registry and the published rows"""
    nm = fl.n_models
    lists, n_loaded, lu = [], np.zeros(nm, dtype=np.int32), np.zeros(nm, dtype=np.int64)
    failed = _failed_lists(fl)
    for m in range(nm):
        c, lu[m] = sim.model_copies(m)
        n_loaded[m] = len(c)
        lists.append([int(x) for x in c] + failed.get(m, []))
    off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(x) for x in lists], out=off[1:])
    inst = np.asarray([i for x in lists for i in x], dtype=np.int32)
    ids = list(fl.inst_ids)
    if rename is not None:
        ids[rename] += "x"
    fl2 = dataclasses.replace(fl, inst_rows=rows, inst_ids=ids, model_last_used=lu, edge_off=off, edge_inst=inst, n_loaded=n_loaded,
                              n_failed=(np.diff(off) - n_loaded).astype(np.int32))
    f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, nm, lib=product_lib)
    load_into_fleet(fl2, f)
    return f


def _scale_entries(fl, s, models, rng):
    rec = np.zeros(len(models), dtype=L.SCALE_IN)
    rec["model"] = models
    for r, m in enumerate(models):
        _, ids = s.churn_model_ids(int(m))
        rec["instance"][r] = int(ids[rng.integers(0, len(ids))]) if len(ids) else int(rng.integers(0, fl.n_instances))
    rec["count"] = rng.integers(0, 20_000, size=len(models))
    rec["last_used"] = fl.now_ms - rng.integers(0, 40 * 3_600_000, size=len(models))
    rec["last_heavy"] = np.where(rng.uniform(size=len(models)) < 0.4, 0, fl.now_ms - rng.integers(0, 30 * 3_600_000, size=len(models)))
    rec["i1"] = 5000 - rng.integers(0, 400, size=len(models))
    rec["i2"] = np.minimum(5000, rec["i1"] + rng.integers(0, 300, size=len(models)))
    return rec


def _same_readers(fl, s, f, models, now, tag):
    nm = fl.n_models
    selfs = (np.arange(nm) * 13) % fl.n_instances
    a, b = s.place_sweep(0, nm, selfs, now, 77), f.place_sweep(0, nm, selfs, now, 77)
    assert a.tobytes() == b.tobytes(), (tag, np.nonzero(a != b)[0][:5])
    rec = _scale_entries(fl, s, models, np.random.default_rng(3))
    p = np.zeros(1, dtype=L.SCALE_PARAMS)
    p["now"], p["last_check_time"], p["iteration"], p["scale_up_rpm_threshold"] = now, now - 10_000, 5000, 400
    p["second_copy_min_age_iters"], p["second_copy_max_age_iters"], p["second_copy_lru_threshold_ms"] = 42, 240, 600_000
    p["rate_check_interval_ms"], p["assume_completed_ms"], p["second_copy_remove_max_age_ms"], p["can_remove"] = 10_000, 30_000, 36 * 3_600_000, 1
    outs = []
    for x in (s, f):
        out = np.zeros(len(rec), dtype=L.SCALE_OUT)
        x._ck(x.lib.mmp_scale_eval(x.h, rec.ctypes.data, len(rec), p.ctypes.data, out.ctypes.data))
        outs.append(out)
    assert all(np.array_equal(outs[0][k], outs[1][k]) for k in L.SCALE_OUT.names), tag
    assert np.count_nonzero(outs[0]["action"] > 0) + np.count_nonzero(outs[0]["remove"]) > 0, tag


def _check_registry_readers(product_lib, fl, o, sim, s, reg):
    """placement sweep over every model and the scale arithmetic on the followed models: the loop's fleet (right after a
    window: the device's overflow table; after a structural commit: the host tables synchronised from it) against a fleet
    committed from scratch"""
    t0 = fl.now_ms + 100 * 2000  # one empty window, for the published rows as both sides hold them
    _, _, rows_o, _, _ = sim.step(np.zeros(0, dtype=L.CHURN_EVENT), t0, t0 + 1, 1)
    _, _, rows, _ = s.churn_step(np.zeros(0, dtype=L.CHURN_EVENT), t0, t0 + 1, 1)
    for k in ("lru_time", "capacity", "used", "count", "l_in_prog", "rpm", "l_threads"):
        assert np.array_equal(rows[k], rows_o[k]), k
    models = np.asarray(sorted(reg.watch), dtype=np.int32)
    now = t0 + 5
    f = _fresh_fleet(product_lib, fl, sim, rows)
    _same_readers(fl, s, f, models, now, "after a window")
    s.instance_upsert(3, rows[3], fl.inst_ids[3] + "x", fl.inst_locs[3], fl.inst_zones[3], fl.inst_labels[3])  # structural
    s.commit()
    assert s.commit_info()[0] == 1
    reg.check("structural", sim, s)
    g = _fresh_fleet(product_lib, fl, sim, rows, rename=3)
    _same_readers(fl, s, g, models, now, "after a structural commit")


def test_overflow_closed_loop_c4_full_size(product_lib, oracle_lib):
    """The C4 shape (500k models x 2 500 instances, 97 % fill) with 0.2 % of the models at 6 registrations: 3 windows"""
    w = make_churn_overflow(make_churn(500_000, 2_500, 4), 0.002, 4, regs=(6, 6))
    fl = w.fleet
    assert (np.diff(fl.edge_off) > 4).sum() > 500
    o, sim, s = _build(product_lib, w, slots=512)
    reg = _Registry(fl)
    for ep in range(3):
        ev = w.events(ep, 20_000, 4)
        now0 = fl.now_ms + ep * w.window_ms
        _compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, 400 + ep)
        reg.check(ep, sim, s)
