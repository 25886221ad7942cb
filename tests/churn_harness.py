"""The closed loop on the device against the oracle's closed loop (oracle/mm_sim.inc): build() makes a churn workload's
oracle, oracle loop and device loop, compare_window() steps both through one window and compares everything, and
run_small_closed_loop() runs 12 windows of it.  The reaper's workloads (with_failed, reaper_workload) and its selection on the
device (device_selection) go with them."""
import dataclasses

import numpy as np

from helpers import oracle_from_synth
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import load_into_fleet, make_churn
from oracle import binding as ob


def build_oracle(w, last_published_ms=None):
    """(the oracle fleet of w, its closed loop seeded with w's caches); every pod last published at last_published_ms
    (default: a minute before the fleet's clock)"""
    fl = w.fleet
    o = oracle_from_synth(fl, bulk=False if fl.n_instances <= 300 else None)
    models = np.zeros(fl.n_models, dtype=ob.SIM_MODEL)
    models["last_used"], models["type_idx"], models["size_units"] = fl.model_last_used, fl.model_type, fl.model_size
    sim = ob.OracleSim(o, models, fl.type_names, fl.edge_off, fl.edge_inst, fl.n_loaded, w.capacity, w.load_timeout_ms,
                       fl.now_ms - 60_000 if last_published_ms is None else last_published_ms)
    order = np.argsort(w.seed_instance, kind="stable")
    bounds = np.searchsorted(w.seed_instance[order], np.arange(fl.n_instances + 1))
    for i in range(fl.n_instances):
        sel = order[bounds[i]:bounds[i + 1]]
        if len(sel):
            sim.seed(i, w.seed_model[sel], w.seed_last_used[sel], w.seed_weight[sel], w.seed_load_ts[sel], fl.now_ms)
    return o, sim


def build(product_lib, w, slots, last_published_ms=None):
    fl = w.fleet
    o, sim = build_oracle(w, last_published_ms)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    load_into_fleet(fl, s)
    s.churn_init(w.load_timeout_ms, fl.now_ms - 60_000 if last_published_ms is None else last_published_ms, slots)
    s.churn_seed(w.seed_instance, w.seed_model, w.seed_last_used, w.seed_weight, w.seed_load_ts, fl.now_ms)
    return o, sim, s


def compare_window(ep, o, sim, s, ev, now0, now1, seed, path=2, out=None):
    """path: the commit path the window must end with (mmp_commit_info): 2, the device path; 1, the host path (a live set
    of more than one instance version, or commit_host_only); out: a dict that receives both sides' instance rows"""
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
    if out is not None:
        out.update(rows_o=rows_o, rows_p=rows_p)
    return dec_o, evi_o, rep


def run_small_closed_loop(product_lib, with_types, fill, seed, slots, w=None, path=2):
    """12 windows of a 20k-model x 200-instance churn trace (or of the workload w), compared window by window, then the
    registry and ingest after it; path: the commit path of every window"""
    w = w or make_churn(20_000, 200, seed, fill=fill, with_types=with_types)
    fl = w.fleet
    o, sim, s = build(product_lib, w, slots=slots)
    totals = dict(dec=0, acc=0, evict=0, reload=0, rejected=0, pub=0)
    for ep in range(12):
        ev = w.events(ep, 2000, seed)
        now0 = fl.now_ms + ep * w.window_ms
        dec, evi, rep = compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, seed * 100 + ep, path=path)
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


def device_selection(s, t: int):
    """mmp_reaper_select over the partitions in mmp_stats order with one `taken` array; a size estimate of 0 ends the run"""
    _, ids = s.stats()
    parts = [int(p) for p in ids[1:]] if len(ids) > 1 else [-1]
    taken = np.zeros(s.max_models, dtype=np.uint8)
    sel = []
    for p in parts:
        try:
            sel += [int(x) for x in s.reaper_select(p, t, taken)]
        except MmpError as e:
            assert e.code == -1 and "size estimate is zero" in str(e), e
            break
    return sel


def with_failed(w, fails: dict):
    """w with model m registering fails[m] failed loads (on instances 0, 1, ...) after its loaded copies"""
    fl = w.fleet
    nf = fl.n_failed.copy()
    for m, k in fails.items():
        nf[m] = k
    cnt = (fl.n_loaded + nf).astype(np.int64)
    off = np.zeros(fl.n_models + 1, dtype=np.int64)
    np.cumsum(cnt, out=off[1:])
    inst = np.zeros(int(off[-1]), dtype=np.int32)
    for m in range(fl.n_models):
        a, nl = int(fl.edge_off[m]), int(fl.n_loaded[m])
        inst[off[m]:off[m] + nl] = fl.edge_inst[a:a + nl]
        held = set(int(x) for x in fl.edge_inst[a:a + nl])
        inst[off[m] + nl:off[m + 1]] = [i for i in range(fl.n_instances) if i not in held][:int(nf[m])]
    return dataclasses.replace(w, fleet=dataclasses.replace(fl, edge_off=off, edge_inst=inst, n_failed=nf.astype(np.int32)))


def recent_unloaded(w, k):
    fl = w.fleet
    u = w.unloaded_models
    return u[np.argsort(-fl.model_last_used[u], kind="stable")[:k]]


def reaper_workload(case, seed):
    with_types = case.endswith("_tc")
    base = case.removesuffix("_tc")
    fill = {"free": 0.5, "cutoff": 0.9, "full": 0.97, "ties": 0.5, "none": 0.5, "zero": 0.5, "part0": 0.5}[base]
    w = make_churn(20_000, 200, seed, fill=fill, with_types=with_types)
    fl = w.fleet
    if base == "ties":  # equal-lastUsed runs among the most recent candidates, and 0 / 1 / 2 failed loads on them
        top = recent_unloaded(w, 60)
        for g in range(0, 60, 3):
            fl.model_last_used[top[g:g + 3]] = fl.model_last_used[top[g]]
        w = with_failed(w, {int(m): j % 3 for j, m in enumerate(top[:45])})
    elif base == "none":  # two failed loads on every unloaded model: no candidate at all
        w = with_failed(w, {int(m): 2 for m in w.unloaded_models})
    elif base == "zero":  # published records with copies but nothing used: the size estimate is 0 (MM:6626-6628)
        fl.inst_rows["used"] = 0
    elif base == "part0":  # one half of the fleet published full: its partition has no free space, counts 0
        fl.inst_rows["used"][1::2] = fl.inst_rows["capacity"][1::2]
    return w
