"""Timing of one pod's whole janitor task: mmp_janitor_task next to mmp_janitor_run on the same entries, on C3 (1 000 000 models x
10 000 instances), a load / failure time for every registration, the cluster 2 % from full, for the pod with the most
registrations.  Two cache sizes, about 2 000 and 20 000 entries: an entry for most of the models the pod holds (some failed,
some with a loadTimestamp that does not match), the rest models it does not hold (undone, recent, not live or unloaded
recently, or to re-register), most recently used first with no Long.MAX_VALUE entry, so both passes run.

    python tools/janitor_task_timing.py --out result.json [--reps 30]

Per size, the two calls alternate, `reps` times each after three warm-up calls of each: the host clock around the call (it
ends in a device synchronise) and mmp_last_timing ("janitor_task": its plan kernel to its budget walk; "janitor_run": its
stats kernel to its budget walk), median, min and max; the reports; and the card's name, power limit and SM clock limit, read
in the same run.
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


def stats(xs):
    return {"median_ms": float(np.median(xs)), "min_ms": float(np.min(xs)), "max_ms": float(np.max(xs)), "calls": len(xs)}


def entries(L, fl, ts, S, n, rng):
    """about n JANITOR_TASK_ENTRY records of pod S, most recently used first"""
    now = fl.now_ms
    hit = np.nonzero(fl.edge_inst == S)[0]
    models = np.searchsorted(fl.edge_off, hit, side="right") - 1
    loaded = (hit - fl.edge_off[models]) < fl.n_loaded[models]
    out = []
    for q, m, ld in zip(hit, models, loaded):
        if rng.uniform() < (0.1 if ld else 0.5):
            continue
        t = np.zeros(1, dtype=L.JANITOR_TASK_ENTRY)[0]
        t["e"]["model"], t["e"]["weight"] = int(m), int(rng.integers(1, 400))
        t["e"]["last_used"] = now - int(rng.integers(1, 40 * HOUR))
        t["e"]["load_ts"] = ts[q] if rng.uniform() < 0.9 else ts[q] + 1
        t["e"]["flags"] = (L.JANITOR_FAILED | L.JANITOR_NOT_LIVE) if not ld else 0
        t["load_complete_ts"] = ts[q]
        out.append(t)
    mine = set(int(m) for m in models)
    others = [int(m) for m in rng.choice(fl.n_models, 2 * n, replace=False) if int(m) not in mine][:max(n - len(out), 0)]
    for m in others:
        t = np.zeros(1, dtype=L.JANITOR_TASK_ENTRY)[0]
        t["e"]["model"], t["e"]["weight"] = m, 10
        u = rng.uniform()
        t["e"]["last_used"] = now - int(rng.integers(1, 600_000)) if u < 0.2 else now - int(rng.integers(1, 40 * HOUR))
        t["e"]["load_ts"] = now - 50 * HOUR
        t["e"]["flags"] = L.JANITOR_NOT_DONE if u > 0.95 else (L.JANITOR_NOT_LIVE if u > 0.6 else 0)
        out.append(t)
    te = np.array(out, dtype=L.JANITOR_TASK_ENTRY)
    return np.ascontiguousarray(te[np.argsort(-te["e"]["last_used"], kind="stable")])


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
    ts = (now - rng.integers(0, 4 * HOUR, size=len(fl.edge_inst))).astype(np.int64)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if a < b:
            s._ck(lib.mmp_model_times(s.h, m, vp(ts[a:b]), int(b - a), 0))
    s.commit()
    S = int(np.argmax(np.bincount(fl.edge_inst, minlength=fl.n_instances)))

    p = np.zeros(1, dtype=L.JANITOR_TASK_PARAMS)
    jp = p["janitor"]
    sp = jp["scale"]
    sp["now"], sp["last_check_time"], sp["iteration"], sp["scale_up_rpm_threshold"] = now, now - 10_000, 5000, 2000
    sp["rate_check_interval_ms"], sp["assume_completed_ms"], sp["second_copy_remove_max_age_ms"] = 10_000, 30_000, 16 * HOUR
    jp["scale"] = sp
    jp["load_failure_expiry_ms"], jp["adjusted_capacity"] = 900_000, int(fl.inst_rows["capacity"][S])
    p["janitor"] = jp
    p["min_stale_age_ms"], p["janitor_freq_secs"], p["load_timeout_ms"] = 6 * HOUR + 1_800_000, 360, 30_000
    run_p = np.ascontiguousarray(p["janitor"])

    res["fleet"] = {"config": "C3", "models": fl.n_models, "instances": fl.n_instances, "self": S,
                    "registrations_of_self": int(np.count_nonzero(fl.edge_inst == S))}
    res["sizes"] = []
    t = C.c_double()
    for n in (2_000, 20_000):
        te = entries(L, fl, ts, S, n, rng)
        run_e = np.ascontiguousarray(te["e"])
        times = {"janitor_task": ([], []), "janitor_run": ([], [])}
        for k in range(args.reps + 3):
            for key in ("janitor_task", "janitor_run"):
                t0 = time.perf_counter()
                if key == "janitor_task":
                    out, edits, r = s.janitor_task(S, te, p)
                else:
                    edits_run, rr = s.janitor_run(S, run_e, run_p)
                t1 = time.perf_counter()
                s._ck(lib.mmp_last_timing(s.h, key.encode(), C.byref(t)))
                if k >= 3:
                    times[key][0].append((t1 - t0) * 1e3)
                    times[key][1].append(t.value)
        assert r.registry_ran == 1
        row = {"entries": int(len(te))}
        for key, (host, dev) in times.items():
            row[key] = {"host": stats(host), "device": stats(dev)}
        row["janitor_task_report"] = {f: getattr(r, f) for f, _ in r._fields_ if f != "registry"}
        row["janitor_task_report"]["registry"] = {f: int(getattr(r.registry, f)) for f, _ in r.registry._fields_}
        row["janitor_run_report"] = {f: int(getattr(rr, f)) for f, _ in rr._fields_}
        res["sizes"].append(row)
    s.close()
    print(json.dumps(res))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
