"""Timing of one pod's janitor registry loop: mmp_janitor_run on C3 (1 000 000 models x 10 000 instances), a load / failure
time for every registration, the cluster 2 % from full (so that scale-downs fire), for the pod with the most registrations: an
entry for most of the models it holds (some of them failed, some with a loadTimestamp that does not match), entries on half of
its failure records, and 100 entries of models it does not hold.

    python tools/janitor_run_timing.py --out result.json [--reps 30]

Reports the host clock around the whole call (it ends in a device synchronise): median, min and max over `reps` calls after
three warm-up calls, and the median of mmp_last_timing("janitor_run"), the CUDA-event time from its stats kernel to its
budget walk; the report of the call; and the card's name, power limit and SM clock limit, read in the same run.
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
vp = lambda a: a.ctypes.data_as(C.c_void_p)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


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
    fl.inst_rows["used"] = fl.inst_rows["capacity"] - fl.inst_rows["capacity"] // 50
    now = fl.now_ms
    n = len(fl.edge_inst)
    ts = (now - rng.integers(0, 4 * HOUR, size=n)).astype(np.int64)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if a < b:
            s._ck(lib.mmp_model_times(s.h, m, vp(ts[a:b]), int(b - a), 0))
    s.commit()

    S = int(np.argmax(np.bincount(fl.edge_inst, minlength=fl.n_instances)))
    hit = np.nonzero(fl.edge_inst == S)[0]
    models = np.searchsorted(fl.edge_off, hit, side="right") - 1
    loaded = (hit - fl.edge_off[models]) < fl.n_loaded[models]
    ents = []
    for q, m, ld in zip(hit, models, loaded):
        u = rng.uniform()
        if (ld and u < 0.1) or (not ld and u < 0.5):
            continue  # a stale registration / a failure record without an entry
        e = np.zeros(1, dtype=L.JANITOR_ENTRY)[0]
        e["model"], e["weight"] = int(m), int(rng.integers(1, 400))
        e["last_used"] = now - int(rng.integers(1, 40 * HOUR))
        e["load_ts"] = ts[q] if rng.uniform() < 0.9 else ts[q] + 1
        e["flags"] = L.JANITOR_FAILED if (not ld or rng.uniform() < 0.05) else 0
        ents.append(e)
    mine = set(int(m) for m in models)
    for m in rng.choice(fl.n_models, 200, replace=False):
        if int(m) not in mine and len(ents) < len(mine) + 100 + len(hit):
            e = np.zeros(1, dtype=L.JANITOR_ENTRY)[0]
            e["model"], e["weight"], e["last_used"] = int(m), 10, now - 1000
            ents.append(e)
    ents = np.array(ents, dtype=L.JANITOR_ENTRY)
    p = np.zeros(1, dtype=L.JANITOR_PARAMS)
    sp = p["scale"]
    sp["now"], sp["last_check_time"], sp["iteration"], sp["scale_up_rpm_threshold"] = now, now - 10_000, 5000, 2000
    sp["rate_check_interval_ms"], sp["assume_completed_ms"], sp["second_copy_remove_max_age_ms"] = 10_000, 30_000, 16 * HOUR
    p["scale"] = sp
    p["load_failure_expiry_ms"], p["adjusted_capacity"] = 900_000, int(fl.inst_rows["capacity"][S])

    host, dev = [], []
    t = C.c_double()
    for k in range(args.reps + 3):
        t0 = time.perf_counter()
        edits, r = s.janitor_run(S, ents, p)
        t1 = time.perf_counter()
        s._ck(lib.mmp_last_timing(s.h, b"janitor_run", C.byref(t)))
        if k >= 3:
            host.append((t1 - t0) * 1e3)
            dev.append(t.value)
    res["fleet"] = {"config": "C3", "models": fl.n_models, "instances": fl.n_instances, "self": S, "registrations_of_self": int(len(hit)),
                    "entries": int(len(ents))}
    res["report"] = {"n_referencing": r.n_referencing, "n_edits": r.n_edits, "n_candidates": r.n_candidates, "n_removed": r.n_removed,
                     "weight_removed": int(r.weight_removed)}
    res["janitor_run"] = {"median_ms": float(np.median(host)), "min_ms": float(np.min(host)), "max_ms": float(np.max(host)),
                          "calls": len(host), "device_median_ms": float(np.median(dev))}
    s.close()
    print(json.dumps(res))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
