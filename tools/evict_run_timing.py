"""Timing of one pod's eviction listener over a burst of evictions: mmp_evict_run against the composed route a pod would
otherwise take, on C3 (1 000 000 models x 10 000 instances) with a load / failure time for every registration, for the pod
with the most registrations, at two burst sizes: 16 of its copies, and every model it is registered on.  Each entry's
load_ts / load_complete_ts is the time of the pod's registration, lastUsed spread over the last two hours.

The composed route: the classification on the host (the deregistration edit, attemptReload, the rebalance gate from the
type-set stats the pod holds, a live copy elsewhere among the epoch's ranked instances, checkLoadFailureCount without the
dropped failure record) over registry slices gathered once, and one mmp_place_batch of the reloads it places with the same
MMP_DF_OWN_ID ids and extra {self}.  The first call of each route is checked to return the same answers.

    python tools/evict_run_timing.py --out result.json [--reps 30]

Reports the host clock around each call (both end in a device synchronise), with preallocated output buffers: median, min
and max over `reps` calls of each, the routes alternated after three warm-up calls of each, and the composed route's
mmp_place_batch call on its own (its classification is a Python loop here, a Java one in a pod); the median of
mmp_last_timing("evict_run"); the report of the call; and the card's name, power limit and SM clock limit, read in the same
run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HOUR = 3_600_000
EXPIRY = 900_000
TIMEOUT = 120_000
vp = lambda a: a.ctypes.data_as(C.c_void_p)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def gate_by_type(fl):
    """the rebalance gate (MM:2918-2920) per type index, from typeSetStats as the pod holds them (read once, not timed)"""
    from oracle import binding as ob
    o = ob.OracleFleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units)
    o.types_set(fl.type_config)
    o.bulk_add(fl.inst_rows, fl.inst_ids, fl.inst_locs, fl.inst_zones, fl.inst_labels)
    o.set_replaced_replicasets(fl.replaced_replicasets)
    out = []
    for t in fl.type_names:
        s = o.type_stats(t)
        cap, free = int(s["total_capacity"]), int(s["total_free"])
        out.append(cap > 0 and int(s["instance_count"]) > 1 and 20 * free // cap >= 1)   # (free >= 0 here)
    o.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from modelmesh_b200 import _lib as L
    from modelmesh_b200.fleet import Fleet
    from modelmesh_b200.synth import load_into_fleet, make_fleet

    lib = L.load_product()
    res = {"card": card()}
    rng = np.random.default_rng(3)
    fl = make_fleet("C3", 1_000_000, 10_000, 3)
    now = fl.now_ms
    n = len(fl.edge_inst)
    ts = np.where(rng.uniform(size=n) < 0.2, now - rng.integers(0, EXPIRY, size=n), now - rng.integers(EXPIRY, 4 * HOUR, size=n)).astype(np.int64)
    lul = np.where(rng.uniform(size=fl.n_models) < 0.3, now - rng.integers(0, 200_000, size=fl.n_models), 0).astype(np.int64)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if a < b:
            s._ck(lib.mmp_model_times(s.h, m, vp(ts[a:b]), int(b - a), int(lul[m])))
    s.commit()
    gate = gate_by_type(fl)
    ranked = set(int(i) for i in s.cluster_order())

    S = int(np.argmax(np.bincount(fl.edge_inst, minlength=fl.n_instances)))
    mine = np.array(sorted(set(int(m) for m in np.searchsorted(fl.edge_off, np.nonzero(fl.edge_inst == S)[0], side="right") - 1)),
                    dtype=np.int32)
    rng.shuffle(mine)
    p = np.zeros(1, dtype=L.EVICT_PARAMS)
    p["now"], p["load_timeout_ms"], p["load_failure_expiry_ms"] = now, TIMEOUT, EXPIRY
    since = now - EXPIRY // 2
    extra = np.array([S], dtype=np.int32)
    res["pod_models"] = len(mine)

    for burst in (16, len(mine)):
        models = mine[:burst]
        ents = np.zeros(len(models), dtype=L.EVICT_ENTRY)
        ents["model"] = models
        ents["last_used"] = now - rng.integers(0, 2 * HOUR, size=len(models))
        # the per-entry registry slices the composed route reads, gathered once (the pod's own registry lookups):
        # (loaded instances, their times, failed instances, their times, lastUsed, lastUnloadTime, gate)
        sl = []
        for r, m in enumerate(models):
            a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
            li, lt, fi, ft = fl.edge_inst[a:a + k], ts[a:a + k], fl.edge_inst[a + k:b], ts[a + k:b]
            hit = np.nonzero(li == S)[0]
            ents["load_ts"][r] = lt[hit[0]] if len(hit) else 0
            hit = np.nonzero(fi == S)[0]
            ents["load_complete_ts"][r] = ft[hit[0]] if len(hit) else 0
            sl.append((li, lt, fi, ft, int(fl.model_last_used[m]), int(lul[m]), gate[int(fl.model_type[m])]))
        d_all = np.zeros(len(ents), dtype=L.DECISION_IN)
        r_all = np.zeros(len(ents), dtype=L.DECISION_OUT)
        out = np.zeros(len(ents), dtype=L.EVICT_ACTION)
        rep = L.EvictReport()
        placed_rows = []

        def one_call():
            s._ck(lib.mmp_evict_run(s.h, S, vp(ents), len(ents), vp(p), None, 7, vp(out), C.byref(rep)))

        def composed():
            """per entry (what, last_used, last_unload_time), and the placed entries' (entry, target, n_candidates)"""
            acts, rows = [], []
            for r, e in enumerate(ents):
                li, lt, fi, ft, lu_rec, lul_rec, open_ = sl[r]
                lpos, fpos = np.nonzero(li == S)[0], np.nonzero(fi == S)[0]
                unreg = len(lpos) > 0 and lt[lpos[0]] == e["load_ts"]
                drop = len(fpos) > 0 and ft[fpos[0]] == e["load_complete_ts"]
                what = (L.EV_UNREGISTER if unreg else 0) | (L.EV_DROP_FAILURE if drop else 0)
                if unreg or drop:
                    lu_rec = max(lu_rec, int(e["last_used"]) or now)
                    if unreg:
                        lul_rec = 0 if len(li) - 1 <= 2 else now
                t = lt[lpos[0]] if len(lpos) else (ft[fpos[0]] if len(fpos) else None)
                if t is not None and now - int(t) > 2 * TIMEOUT:
                    what |= L.EV_RELOAD
                    if not open_:
                        what |= L.EV_CLUSTER_FULL
                    elif any(int(i) != S and int(i) in ranked for i in li):
                        what |= L.EV_LOADED_ELSEWHERE
                    elif int(np.count_nonzero(ft > since)) - (1 if drop and ft[fpos[0]] > since else 0) >= 3:
                        what |= L.EV_REFUSED
                    else:
                        what |= L.EV_PLACED
                        rows.append(r)
                acts.append((what, lu_rec, lul_rec))
            d = d_all[:len(rows)]
            d["model"] = ents["model"][rows]
            d["self"], d["last_used"] = S, ents["last_used"][rows]
            d["flags"] = [L.DF_FAVOUR_SELF | L.DF_OWN_ID | (r << 8) for r in rows]
            d["fresh"], d["extra_off"], d["extra_n"] = -1, 0, 1
            got = s.place_batch(d, now, 7, extra=extra, out=r_all[:len(rows)])
            placed_rows[:] = rows
            return acts, [(r, int(x["target"]), int(x["n_candidates"])) for r, x in zip(rows, got)]

        def place_only():
            """the composed route's mmp_place_batch alone, on the records its classification built last"""
            k = len(placed_rows)
            s.place_batch(d_all[:k], now, 7, extra=extra, out=r_all[:k])

        one_call()
        acts, placed = composed()
        assert acts == [(int(a["what"]), int(a["last_used"]), int(a["last_unload_time"])) for a in out], "the two routes disagree"
        assert placed == [(int(r), int(out["target"][r]), int(out["n_candidates"][r]))
                          for r in np.nonzero(out["what"] & L.EV_PLACED)[0]], "the two routes disagree"
        row = {"entries": len(ents), "report": {k: getattr(rep, k) for k, _ in L.EvictReport._fields_}}

        def timed(k):
            t0 = time.perf_counter()
            (one_call, composed, place_only)[k]()
            return (time.perf_counter() - t0) * 1e3

        for _ in range(3):
            timed(0), timed(1), timed(2)
        host, dev = [[], [], []], []
        t = C.c_double()
        for _ in range(args.reps):
            for k in (0, 1, 2):
                host[k].append(timed(k))
                if k == 0:
                    s._ck(lib.mmp_last_timing(s.h, b"evict_run", C.byref(t)))
                    dev.append(t.value)
        for k, name in ((0, "evict_run"), (1, "composed"), (2, "composed_place_batch_only")):
            h = np.array(host[k])
            row[name] = {"host_ms_median": float(np.median(h)), "host_ms_min": float(h.min()), "host_ms_max": float(h.max())}
        d = np.array(dev)
        row["evict_run"].update(device_ms_median=float(np.median(d)), device_ms_min=float(d.min()), device_ms_max=float(d.max()))
        res[f"burst_{burst}"] = row
    res["reps"] = args.reps
    s.close()
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
