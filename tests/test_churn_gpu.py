"""The closed loop on the device against the oracle's closed loop (oracle/mm_sim.inc), window by window:
every placement (target, candidates), every admission outcome, every eviction (in listener order, with its reload flag),
every republished instance record and the PLACEMENT_ORDER ranking after each window must be identical.
BASELINE.json configs[3] (C4): 500k models x 2 500 instances, 10k events/s, commit every 2 s; the small cases cover the
reload-elsewhere rule (a12) and type-set stats, the full-size case the headline shape."""
import os

import numpy as np
import pytest

from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet
from modelmesh_b200.synth import load_into_fleet, make_churn
from oracle import binding as ob

pytestmark = pytest.mark.gpu


def _build(product_lib, w, slots):
    fl = w.fleet
    o = oracle_from_synth(fl, bulk=False if fl.n_instances <= 300 else None)
    models = np.zeros(fl.n_models, dtype=ob.SIM_MODEL)
    models["last_used"], models["type_idx"], models["size_units"] = fl.model_last_used, fl.model_type, fl.model_size
    sim = ob.OracleSim(o, models, fl.type_names, fl.edge_off, fl.edge_inst, fl.n_loaded, w.capacity, w.load_timeout_ms,
                       fl.now_ms - 60_000)
    order = np.argsort(w.seed_instance, kind="stable")
    bounds = np.searchsorted(w.seed_instance[order], np.arange(fl.n_instances + 1))
    for i in range(fl.n_instances):
        sel = order[bounds[i]:bounds[i + 1]]
        if len(sel):
            sim.seed(i, w.seed_model[sel], w.seed_last_used[sel], w.seed_weight[sel], w.seed_load_ts[sel], fl.now_ms)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    load_into_fleet(fl, s)
    s.churn_init(w.load_timeout_ms, fl.now_ms - 60_000, slots)
    s.churn_seed(w.seed_instance, w.seed_model, w.seed_last_used, w.seed_weight, w.seed_load_ts, fl.now_ms)
    return o, sim, s


def _compare_window(ep, o, sim, s, ev, now0, now1, seed, path=2):
    """path: the commit path the window must end with (mmp_commit_info): 2, the device path; 1, the host path (a live set
    of more than one instance version, or commit_host_only)"""
    dec_o, evi_o, rows_o, npub_o, carry_o = sim.step(ev, now0, now1, seed)
    dec_p, evi_p, rows_p, rep = s.churn_step(ev, now0, now1, seed)
    assert len(dec_p) == len(dec_o), (ep, len(dec_p), len(dec_o))
    for k in ("event", "status", "model", "self", "target", "n_candidates"):
        a, b = dec_p[k], dec_o[k]
        if k in ("model", "target", "n_candidates"):  # a skipped reload carries no decision
            keep = dec_o["status"] != ob.SIM_SKIPPED
            a, b = a[keep], b[keep]
        assert np.array_equal(a, b), (ep, k, np.nonzero(a != b)[0][:5], a[a != b][:5], b[a != b][:5])
    key = lambda e: np.lexsort((e["model"], e["order"], e["instance"]))
    # the oracle appends evictions instance by instance in listener order; the device sorts by (instance, trace position, seq)
    assert len(evi_p) == len(evi_o), (ep, len(evi_p), len(evi_o))
    for k in ("instance", "model", "last_used", "weight", "order", "reload"):
        assert np.array_equal(evi_p[k], evi_o[k]), (ep, k)
    for k in ("lru_time", "capacity", "used", "count", "l_in_prog", "rpm", "l_threads"):
        assert np.array_equal(rows_p[k], rows_o[k]), (ep, k, np.nonzero(rows_p[k] != rows_o[k])[0][:5])
    assert rep.n_published == npub_o and rep.n_carry == carry_o, (ep, rep.n_published, npub_o, rep.n_carry, carry_o)
    assert np.array_equal(s.cluster_order(), o.cluster_order()), ep
    assert s.commit_info()[0] == path, (ep, s.commit_info()[0], path)
    return dec_o, evi_o, rep


@pytest.mark.parametrize("with_types,fill,seed", [(False, 0.90, 4), (True, 0.90, 5), (False, 0.97, 6), (True, 0.97, 7)])
def test_closed_loop_matches_oracle_small(product_lib, oracle_lib, with_types, fill, seed):
    run_small_closed_loop(product_lib, with_types, fill, seed, slots=256)


def run_small_closed_loop(product_lib, with_types, fill, seed, slots, w=None, path=2):
    """12 windows of a 20k-model x 200-instance churn trace (or of the workload w), compared window by window, then the
    registry and ingest after it; path: the commit path of every window"""
    w = w or make_churn(20_000, 200, seed, fill=fill, with_types=with_types)
    fl = w.fleet
    o, sim, s = _build(product_lib, w, slots=slots)
    totals = dict(dec=0, acc=0, evict=0, reload=0, rejected=0, pub=0)
    for ep in range(12):
        ev = w.events(ep, 2000, seed)
        now0 = fl.now_ms + ep * w.window_ms
        dec, evi, rep = _compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, seed * 100 + ep, path=path)
        totals["dec"] += len(dec); totals["acc"] += int(np.count_nonzero(dec["status"] == ob.SIM_ACCEPTED))
        totals["rejected"] += int(np.count_nonzero((dec["status"] >= 1) & (dec["status"] <= 5)))
        totals["evict"] += len(evi); totals["reload"] += int(evi["reload"].sum()); totals["pub"] += rep.n_published
    assert totals["acc"] > 500 and totals["evict"] > 300 and totals["pub"] > 50, totals
    if fill <= 0.9:
        assert totals["reload"] > 0, totals  # the reload-elsewhere rule fired (a12) and its queued placements were compared
    # registry: every model's copies as the oracle holds them
    for m in range(0, fl.n_models, 37):
        copies, lu = sim.model_copies(m)
        row, inst = s.churn_model(m)
        assert int(row["copy_count"]) == len(copies) and list(inst[:len(copies)]) == list(copies), (m, row, inst, copies)
        assert int(row["last_used"]) == lu, m
    # after the trace, ordinary ingest goes on from the device's state (host tables are synchronised on demand)
    r = fl.inst_rows[3].copy()
    s.instance_upsert(3, r, fl.inst_ids[3] + "x", fl.inst_locs[3], fl.inst_zones[3], fl.inst_labels[3])  # structural
    s.commit()
    assert s.commit_info()[0] == 1
    row2, inst2 = s.churn_model(0)
    copies, _ = sim.model_copies(0)
    assert int(row2["copy_count"]) == len(copies)


def test_closed_loop_c4_full_size(product_lib, oracle_lib):
    """BASELINE.json configs[3]: 500k models x 2 500 instances at 97 % fill, 20 000 events per 2 s window."""
    n_windows = int(os.environ.get("MMP_C4_WINDOWS", 6))
    w = make_churn(500_000, 2_500, 4)
    fl = w.fleet
    o, sim, s = _build(product_lib, w, slots=512)
    acc = ev_n = 0
    for ep in range(n_windows):
        ev = w.events(ep, 20_000, 4)
        now0 = fl.now_ms + ep * w.window_ms
        dec, evi, rep = _compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, 400 + ep)
        acc += int(np.count_nonzero(dec["status"] == ob.SIM_ACCEPTED)); ev_n += len(evi)
    assert acc > 1000 and ev_n > 1000


def test_checked_load_event_matches_oracle(product_lib, oracle_lib):
    """MMP_LRU_LOAD (a11) through mmp_lru_apply_status against the oracle's loadLocal restatement on one cache:
    churn guard, immediate fall-through, early reject, accepted, evicted while growing."""
    now = 1_760_000_000_000
    fl_min_space, churn_age = 2560, 600_000
    s = Fleet(fl_min_space, churn_age, 2560, 4, 64, lib=product_lib)
    row = np.zeros(1, dtype=L.INSTANCE_ROW)
    row["capacity"], row["l_threads"], row["active"], row["lru_time"] = 25_600, 8, 1, (1 << 63) - 1
    for i in range(4):
        s.instance_upsert(i, row[0], f"pod-{i}")
    s.commit()
    cap = 23_040
    s.lru_init(np.full(4, cap, dtype=np.int64), 64)
    lru = ob.OracleLru(cap)
    rng = np.random.default_rng(5)
    t = now
    seen = set()
    for step in range(400):
        t += int(rng.integers(1, 400_000))
        m = int(rng.integers(0, 40))
        size = int(rng.choice([256, 2560, 9000, 30_000]))
        lu = int(rng.choice([0, t - 5, t - 3_000_000, now - 10_000_000]))
        # oracle: the literal sequence of mm_sim.inc
        k0, t0, w0 = lru.dump()
        oldest = lru.oldest_time()
        want_ev = []
        if oracle_lib.orc_churn_reject(cap, lru.weighted_size(), oldest, fl_min_space, churn_age, t):
            want = 2
        else:
            exists = m in set(int(x) for x in k0)
            e = np.zeros(1, dtype=ob.LRU_EVENT); e["op"], e["key"], e["weight"], e["last_used"] = 0, m, 1, lu
            want_ev += list(lru.apply(e, t))
            if exists:
                want = 6
            elif m not in set(int(x) for x in lru.dump()[0]):
                want = 3
            elif oracle_lib.orc_early_reject(size, cap, lru.weighted_size(), lru.oldest_time(), lu):
                e["op"] = 3
                lru.apply(e, t)
                want = 4
            else:
                e["op"], e["weight"] = 2, size
                want_ev += list(lru.apply(e, t))
                want = 0 if m in set(int(x) for x in lru.dump()[0]) else 5
        ev = np.zeros(1, dtype=L.LRU_EVENT)
        ev["op"], ev["instance"], ev["model"], ev["weight"], ev["last_used"] = L.LRU_LOAD, 1, m, size, lu
        got_ev, status = s.lru_apply_status(ev, t)
        assert int(status[0]) == want, (step, status, want)
        assert [(int(x["model"]), int(x["last_used"])) for x in got_ev] == [(int(x["key"]), int(x["last_used"])) for x in want_ev], step
        oldest_p, weighted_p, count_p = s.lru_state()
        assert int(weighted_p[1]) == lru.weighted_size() and int(count_p[1]) == lru.size() and int(oldest_p[1]) == lru.oldest_time()
        seen.add(want)
    assert seen >= {0, 4, 6}, seen

    def both(m, size, lu, t):
        """one checked load through both sides (the literal sequence of oracle/mm_sim.inc); returns the common status"""
        if oracle_lib.orc_churn_reject(cap, lru.weighted_size(), lru.oldest_time(), fl_min_space, churn_age, t):
            want, want_ev = 2, []
        else:
            e = np.zeros(1, dtype=ob.LRU_EVENT); e["op"], e["key"], e["weight"], e["last_used"] = 0, m, 1, lu
            exists = m in set(int(x) for x in lru.dump()[0])
            want_ev = list(lru.apply(e, t))
            if exists:
                want = 6
            elif m not in set(int(x) for x in lru.dump()[0]):
                want = 3
            elif oracle_lib.orc_early_reject(size, cap, lru.weighted_size(), lru.oldest_time(), lu):
                e["op"] = 3; lru.apply(e, t); want = 4
            else:
                e["op"], e["weight"] = 2, size
                want_ev += list(lru.apply(e, t))
                want = 0 if m in set(int(x) for x in lru.dump()[0]) else 5
        ev = np.zeros(1, dtype=L.LRU_EVENT)
        ev["op"], ev["instance"], ev["model"], ev["weight"], ev["last_used"] = L.LRU_LOAD, 1, m, size, lu
        got_ev, status = s.lru_apply_status(ev, t)
        assert int(status[0]) == want, (status, want)
        assert [(int(x["model"]), int(x["last_used"])) for x in got_ev] == [(int(x["key"]), int(x["last_used"])) for x in want_ev]
        return want

    # fill the cache to the last unit with fresh entries, then: an older-than-everything load falls through (MM:5145-5148) ...
    free = cap - lru.weighted_size()
    k = 1000
    while free > 0:
        sz = min(free, 2000)
        t += 1
        assert both(k, sz, t, t) == 0
        free -= sz; k += 1
    assert lru.weighted_size() == cap
    t += 700_000  # past the churn window: the guard is quiet, the placeholder itself is the eviction victim
    assert both(2000, 256, 5, t) == 3
    # ... and while the oldest entry is younger than minChurnAgeMs a full cache rejects new loads (MM:3872-3884)
    t2 = int(lru.oldest_time()) + 1000
    assert both(2001, 256, t2, t2) == 2


def test_device_commit_equals_host_commit(product_lib, oracle_lib):
    """A non-structural commit (numeric instance updates + model-record deltas) takes the device path: re-ranking by
    counting under the literal comparator, table build, bitmap from device-resident edges.  The snapshot must be the one the
    host path builds from the same tables: ranking, type sets, decisions, stats."""
    from modelmesh_b200.synth import make_decisions, make_fleet
    for config, nm, ni, seed in (("C3", 6000, 1300, 3), ("C5", 4000, 700, 5), ("MIX", 1500, 300, 14)):
        fl = make_fleet(config, nm, ni, seed)
        a = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, ni, nm, lib=product_lib)
        os.environ["MMP_COMMIT"] = "host"
        try:
            b = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, ni, nm, lib=product_lib)
        finally:
            del os.environ["MMP_COMMIT"]
        load_into_fleet(fl, a); load_into_fleet(fl, b)
        rng = np.random.default_rng(seed)
        rows = fl.inst_rows.copy()
        mrow = np.zeros(1, dtype=L.MODEL_ROW)
        for rnd in range(4):
            live = np.nonzero(rows["shutting_down"] == 0)[0]
            for i in rng.choice(live, size=min(len(live), 40 + 200 * rnd), replace=False):
                rows[i]["used"] = int(rng.integers(0, rows[i]["capacity"] + 1))
                rows[i]["count"] = int(rng.integers(0, 400))
                rows[i]["lru_time"] = int(fl.now_ms - rng.integers(0, 10_000_000))
                rows[i]["rpm"] = int(rng.integers(0, 5000))
                rows[i]["l_in_prog"] = int(rng.integers(0, 4))
                a.instance_update(int(i), rows[i]); b.instance_update(int(i), rows[i])
            for m in rng.integers(0, nm, size=300):
                ids = [int(x) for x in rng.choice(ni, size=int(rng.integers(0, 4)), replace=False)]
                mrow["last_used"], mrow["size_units"], mrow["type_id"] = int(fl.now_ms - rng.integers(0, 1e7)), 1000, a.type_id(fl.type_names[fl.model_type[m]])
                mrow["copy_count"] = len(ids)
                a.model_upsert(int(m), mrow[0], ids); b.model_upsert(int(m), mrow[0], ids)
            a.commit(); b.commit()
            assert a.commit_info()[0] == 2 and b.commit_info()[0] == 1
            assert np.array_equal(a.cluster_order(), b.cluster_order())
            for t in range(len(fl.type_names)):
                ta, tb = a.type_sets(a.type_id(fl.type_names[t]), ni), b.type_sets(b.type_id(fl.type_names[t]), ni)
                for x, y in zip(ta, tb):
                    assert (x is None) == (y is None) and (x is None or np.array_equal(x, y))
            sd = make_decisions(fl, 3000, seed + rnd)
            kw = dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
            oa, ta_, ma = a.place_batch(sd.dec, fl.now_ms, 9, trace=True, masks=True, **kw)
            ob_, tb_, mb = b.place_batch(sd.dec, fl.now_ms, 9, trace=True, masks=True, **kw)
            assert np.array_equal(oa, ob_) and np.array_equal(ta_, tb_) and np.array_equal(ma, mb)
            assert np.array_equal(a.place_batch(sd.dec, fl.now_ms, 9, **kw), oa)
            sa, ia = a.stats(); sb, ib = b.stats()
            # the same partition stats (partition ids are opaque per fleet, and they break ties of PARTITION_STATS_COMP: compare as sets)
            assert np.array_equal(np.sort(sa, order=list(sa.dtype.names)), np.sort(sb, order=list(sb.dtype.names))), (sa, sb)
            for i in rng.choice(ni, size=50, replace=False):
                pa, pb = a.instance_partition(int(i)), b.instance_partition(int(i))
                assert (pa < 0) == (pb < 0)
                if pa >= 0:
                    assert np.array_equal(sa[ia == pa], sb[ib == pb])
