"""Timing of one pod's rate-tracking task: mmp_rate_run against the composed route a pod would otherwise take, on C3
(1 000 000 models x 10 000 instances) with a load / failure time for every registration, for the pod with the most
registrations: an entry for every model it holds or has failed on and 100 entries of models it does not hold, with interval
counts chosen so that second copies and scale-ups of up to 20 copies fire at a threshold of 300 rpm.

The composed route: mmp_scale_eval, the heavy set built on the host from the published rows the pod holds, checkLoadFailureCount
on the host, one mmp_place_batch for the second copies (extra {self}), then one mmp_place_batch_excluding per chain round.
Both routes place the same decisions with the same ids, and the first call of each is checked to return the same loads.

    python tools/rate_run_timing.py --out result.json [--reps 30]

Reports the host clock around each call (both end in a device synchronise): median, min and max over `reps` calls of each,
alternating the two routes after three warm-up calls of each; the median of mmp_last_timing("rate_run"), the CUDA-event time
from its stats kernel to its last placement round; the report of the call; and the card's name, power limit and SM clock
limit, read in the same run.
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
THR = 300
vp = lambda a: a.ctypes.data_as(C.c_void_p)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def composed(L, s, fl, ts, S, ents, p, seed, live, rpm_live):
    """the route through the per-step calls: loads as (entry, model, chain_pos, self, target, n_candidates) tuples"""
    sc = p["scale"][0]
    now = int(sc["now"])
    sp = p["scale"].copy()
    sp["can_remove"] = 0
    out = np.zeros(len(ents), dtype=L.SCALE_OUT)
    s._ck(s.lib.mmp_scale_eval(s.h, vp(ents), len(ents), vp(sp), vp(out)))
    rk = np.nonzero(live == S)[0]
    our = int(rpm_live[rk[0]]) if len(rk) else 0
    bound = max(4 * THR, our - 2 * THR)
    heavy = live[(rpm_live > bound) & (live != S)].astype(np.int32)
    since = now - EXPIRY // 2
    sec, chains, off = [], [], 0
    for r, (e, x) in enumerate(zip(ents, out)):
        act, m = int(x["action"]), int(e["model"])
        if act not in (1, 2):
            continue
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        if int(np.count_nonzero(ts[a + k:b] > since)) >= 3:
            continue
        if act == 1:
            sec.append((r, m, off, int(x["load_last_used"])))
            off += 1
        else:
            n = min(int(x["copies_to_load"]), L.RATE_CHAIN_MAX)
            fav = S in set(int(i) for i in fl.edge_inst[a:a + k])
            chains.append([r, m, off, int(x["load_last_used"]), n, fav, S, []])
            off += n
    loads = {}
    if sec:
        d = np.zeros(len(sec), dtype=L.DECISION_IN)
        d["model"], d["self"], d["last_used"] = [c[1] for c in sec], S, [c[3] for c in sec]
        d["flags"] = [L.DF_FAVOUR_SELF | L.DF_OWN_ID | (c[2] << 8) for c in sec]
        d["fresh"], d["extra_n"] = -1, 1
        res = s.place_batch(d, now, seed, extra=np.array([S], dtype=np.int32))
        for c, x in zip(sec, res):
            loads[(c[0], 0)] = (c[0], c[1], 0, S, int(x["target"]), int(x["n_candidates"]))
    active, j = chains, 0
    while active:
        d = np.zeros(len(active), dtype=L.DECISION_IN)
        d["model"], d["self"], d["last_used"] = [c[1] for c in active], [c[6] for c in active], [c[3] for c in active]
        d["flags"] = [(L.DF_FAVOUR_SELF if (j or c[5]) else 0) | L.DF_OWN_ID | ((c[2] + j) << 8) for c in active]
        d["fresh"], d["extra_n"] = -1, j
        d["extra_off"] = np.arange(len(active)) * j
        ext = np.array([t for c in active for t in c[7]], dtype=np.int32)
        res = s.place_batch(d, now, seed, extra=ext if len(ext) else None, exclude=heavy)
        nxt = []
        for c, x in zip(active, res):
            t = int(x["target"])
            loads[(c[0], j)] = (c[0], c[1], j, c[6], t, int(x["n_candidates"]))
            if t in (L.TARGET_NONE, L.TARGET_INVALID) or j + 1 >= c[4]:
                continue
            c[6] = S if t == L.TARGET_SELF else t
            c[7].append(c[6])
            nxt.append(c)
        active, j = nxt, j + 1
    return [loads[k] for k in sorted(loads)]


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
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if a < b:
            s._ck(lib.mmp_model_times(s.h, m, vp(ts[a:b]), int(b - a), 0))
    s.commit()

    S = int(np.argmax(np.bincount(fl.edge_inst, minlength=fl.n_instances)))
    mine = sorted(set(int(m) for m in np.searchsorted(fl.edge_off, np.nonzero(fl.edge_inst == S)[0], side="right") - 1))
    rest = np.setdiff1d(rng.choice(fl.n_models, 200, replace=False), mine)[:100]
    models = np.array(mine + [int(m) for m in rest], dtype=np.int32)
    ents = np.zeros(len(models), dtype=L.SCALE_IN)
    ents["instance"], ents["model"] = S, models
    u = rng.uniform(size=len(models))
    ents["count"] = np.where(u < 0.6, rng.integers(0, 30, size=len(models)), rng.integers(30, 1000, size=len(models)))
    ents["last_used"] = now - rng.integers(0, HOUR, size=len(models))
    ents["i1"] = 5000 - rng.integers(0, 400, size=len(models))
    ents["i2"] = np.minimum(5000, ents["i1"] + rng.integers(0, 300, size=len(models)))
    p = np.zeros(1, dtype=L.RATE_PARAMS)
    sc = p["scale"]
    sc["now"], sc["last_check_time"], sc["iteration"], sc["scale_up_rpm_threshold"] = now, now - 10_000, 5000, THR
    sc["second_copy_min_age_iters"], sc["second_copy_max_age_iters"], sc["second_copy_lru_threshold_ms"] = 42, 240, 3 * HOUR
    sc["rate_check_interval_ms"], sc["assume_completed_ms"], sc["second_copy_remove_max_age_ms"] = 10_000, 30_000, HOUR
    p["scale"] = sc
    p["load_failure_expiry_ms"] = EXPIRY
    live = np.asarray(s.cluster_order(), dtype=np.int32)
    rpm_live = fl.inst_rows["rpm"][live].astype(np.int64)

    seed = 7
    out, loads, rep = s.rate_run(S, ents, p, seed)
    got = [tuple(int(x) for x in ld)[:6] for ld in loads]
    assert got == composed(L, s, fl, ts, S, ents, p, seed, live, rpm_live), "the two routes disagree"
    res["report"] = {k: getattr(rep, k) for k, _ in L.RateReport._fields_ if k != "reserved"}
    res["entries"] = len(ents)

    def one(k):
        t0 = time.perf_counter()
        if k == 0:
            s.rate_run(S, ents, p, seed)
        else:
            composed(L, s, fl, ts, S, ents, p, seed, live, rpm_live)
        return (time.perf_counter() - t0) * 1e3

    for _ in range(3):
        one(0), one(1)
    host = [[], []]
    dev = []
    t = C.c_double()
    for _ in range(args.reps):
        for k in (0, 1):
            host[k].append(one(k))
            if k == 0:
                s._ck(lib.mmp_last_timing(s.h, b"rate_run", C.byref(t)))
                dev.append(t.value)
    for k, name in ((0, "rate_run"), (1, "composed")):
        h = np.array(host[k])
        res[name] = {"host_ms_median": float(np.median(h)), "host_ms_min": float(h.min()), "host_ms_max": float(h.max())}
    res["rate_run"]["device_ms_median"] = float(np.median(dev))
    res["reps"] = args.reps
    s.close()
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
