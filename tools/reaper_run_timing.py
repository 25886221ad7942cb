"""Timing of one run of the leader's reaper task: mmp_reaper_run against the composed route a leader has without it
(mmp_registry_prune_ids + mmp_reaper_select per partition in mmp_stats order + mmp_place_batch of the selections), alternated
call by call in one run, on two fleets:
  C3             1 000 000 models x 10 000 instances, a load / failure time for every registration, 40 pods gone and first
                 seen missing 11 minutes ago
  C4 at 80 %     500 000 models x 2 500 instances at 80 % fill (the free-space count: the reaper selects ~150 k models)

    python tools/reaper_run_timing.py --out result.json [--reps 30]

Each number is the host clock around the whole call (every call ends in a device synchronise): median, min and max over
`reps` calls after three warm-up calls; for mmp_reaper_run also mmp_last_timing("reaper_run"), the CUDA-event time from its
prune sweep to its last placement kernel.  Both routes see the same missing_since on every call and prune the same
registrations; where nothing is pruned they must also select the same models and place them on the same targets (with
registrations pruned, the composed route selects on the unpruned counts: the difference mmp_reaper_run exists for).  The
card's name, power limit and SM clock limit are read in the same run.
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

GONE_MS = 600_000
vp = lambda a: a.ctypes.data_as(C.c_void_p)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def _stats(ms):
    return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms)), "calls": len(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from modelmesh_b200 import _lib as L
    from modelmesh_b200.fleet import Fleet, MmpError
    from modelmesh_b200.synth import load_into_fleet, make_churn, make_fleet

    lib = L.load_product()
    res = {"card": card()}
    for name in ("C3", "C4 at 80 % fill"):
        rng = np.random.default_rng(5)
        fl = make_fleet("C3", 1_000_000, 10_000, 3) if name == "C3" else make_churn(500_000, 2_500, 4, fill=0.8).fleet
        s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
        load_into_fleet(fl, s)
        gone = np.zeros(0, dtype=np.int64)
        missing0 = np.zeros(fl.n_instances, dtype=np.int64)
        if name == "C3":
            ts = (fl.now_ms - rng.integers(0, 4 * 3_600_000, size=len(fl.edge_inst))).astype(np.int64)
            for m in range(fl.n_models):
                a, b = fl.edge_off[m], fl.edge_off[m + 1]
                if a != b:
                    s._ck(lib.mmp_model_times(s.h, m, vp(ts[a:b]), int(b - a), 0))
            gone = rng.choice(fl.n_instances, size=40, replace=False)
            for i in gone:
                s.instance_remove(int(i))
            missing0[gone] = fl.now_ms - 660_000
            s.commit()
        leader = int(np.setdiff1d(np.arange(fl.n_instances), gone)[0])
        now, seed = fl.now_ms + 500, 77
        _, ids = s.stats()
        parts = [int(p) for p in ids[1:]] if len(ids) > 1 else [-1]

        pm_buf = np.zeros(len(fl.edge_inst), dtype=np.int32)
        pi_buf = np.zeros(len(fl.edge_inst), dtype=np.int32)
        sel_buf = np.zeros(fl.n_models, dtype=np.int32)
        rep_buf = np.zeros(fl.n_models, dtype=np.int32)
        load_buf = np.zeros(fl.n_models, dtype=L.REAPER_LOAD)

        def run():  # (the buffers are allocated once, as for the composed route)
            miss = missing0.copy()
            r = L.ReaperReport()
            t0 = time.perf_counter()
            n = s._ck(lib.mmp_reaper_run(s.h, leader, now, GONE_MS, vp(miss), seed, vp(pm_buf), vp(pi_buf), len(pm_buf), vp(rep_buf),
                                         len(rep_buf), vp(load_buf), len(load_buf), C.byref(r)))
            t = (time.perf_counter() - t0) * 1e3
            ms = C.c_double()
            s._ck(lib.mmp_last_timing(s.h, b"reaper_run", C.byref(ms)))
            return t, float(ms.value), load_buf[:n].copy(), r

        def composed():
            miss = missing0.copy()
            t0 = time.perf_counter()
            n_pr = s._ck(lib.mmp_registry_prune_ids(s.h, leader, now, GONE_MS, vp(miss), vp(pm_buf), vp(pi_buf), len(pm_buf)))
            taken = np.zeros(fl.n_models, dtype=np.uint8)
            sel = []
            for p in parts:
                try:
                    n = s._ck(lib.mmp_reaper_select(s.h, p, now, vp(taken), vp(sel_buf), len(sel_buf)))
                except MmpError:
                    break
                sel.append(sel_buf[:n].copy())
            sel = np.concatenate(sel) if sel else np.zeros(0, dtype=np.int32)
            dec = np.zeros(len(sel), dtype=L.DECISION_IN)
            dec["model"], dec["self"], dec["fresh"] = sel, leader, -1
            dec["last_used"] = fl.model_last_used[sel]
            out = s.place_batch(dec, now, seed) if len(sel) else np.zeros(0, dtype=L.DECISION_OUT)
            return (time.perf_counter() - t0) * 1e3, n_pr, sel, out

        t_run, t_dev, t_cmp = [], [], []
        for k in range(args.reps + 3):  # the first three calls of each are warm-up
            a, d, loads, r = run()
            b, n_pr, sel, out = composed()
            assert r.n_pruned == n_pr, (r.n_pruned, n_pr)
            if k == 0 and n_pr == 0:  # (with registrations pruned the composed route selects on the unpruned counts)
                assert np.array_equal(loads["model"], sel), (len(loads), len(sel))
                assert np.array_equal(loads["target"], out["target"]) and np.array_equal(loads["n_candidates"], out["n_candidates"])
            if k >= 3:
                t_run.append(a); t_dev.append(d); t_cmp.append(b)
        res[name] = {"mmp_reaper_run": _stats(t_run), "t_reaper_run": _stats(t_dev), "composed_route": _stats(t_cmp),
                     "registrations_pruned": int(r.n_pruned), "repaired": int(r.n_repaired), "loads": int(r.n_loads),
                     "composed_route_loads": int(len(sel)),
                     "partitions": len(parts), "stopped_partition": int(r.stopped_partition)}
        print(name, json.dumps(res[name]), flush=True)
        s.close()
    print(json.dumps(res, indent=1))
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
