"""Cost of the reaper's proactive loads in the closed loop: mmp_churn_step on C4 (500k models x 2 500 instances, 20 000 events
per 2 s window) as bench.py runs it, then the same windows with one REAPER event each (caller = a live instance, t = the middle
of the window), on two fleets: C4 itself (97 % fill: the cluster's capacity minus its free space overflows the reference's
int cast, the size estimate is negative and the reaper selects nothing, so the pass runs to no effect) and C4 at 80 % fill
(the free-space count: ~150 k models per run, until the loads have filled the caches and the lastUsed cutoff decides).
Prints one JSON line per workload: medians over the timed windows of the host clock around the step, the step's CUDA-event
total and its reaper pass (ms_reaper, its one read-back included), the models the reaper decided in each timed window and
the median of all decisions per window, and the GPU's name and power limit with the clocks and throttle reasons sampled in
the timed region.  A second leg times mmp_reaper_select on each fleet's committed snapshot: one round calls it for every
partition in mmp_stats order (the cluster, -1, on a fleet without type constraints) with one taken array, as the leader's
reaper does; medians over the timed rounds of the host clock around each call (its read-backs included) and of its
CUDA-event time (mmp_last_timing "reaper"), and the models a round selects.  MMP_LIB selects another build of the library.

    python tools/churn_reaper_timing.py [--windows 10] [--warmup 3] [--calls 30]
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

from modelmesh_b200 import _lib  # noqa: E402
from modelmesh_b200.fleet import Fleet  # noqa: E402
from modelmesh_b200.synth import load_into_fleet, make_churn  # noqa: E402


def nvidia_smi(fields: str) -> str:
    try:
        return subprocess.check_output(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def time_windows(lib, w, windows: int, warmup: int, events: int, seed: int, reaper: bool) -> dict:
    fl = w.fleet
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    s.churn_init(w.load_timeout_ms, fl.now_ms - 60_000, 512)
    s.churn_seed(w.seed_instance, w.seed_model, w.seed_last_used, w.seed_weight, w.seed_load_ts, fl.now_ms)
    wall, total, ms_reaper, picked, decided, clocks = [], [], [], [], [], []
    for ep in range(warmup + windows):
        ev = w.events(ep, events, seed)
        now0 = fl.now_ms + ep * w.window_ms
        k = len(ev) // 2
        if reaper:
            r = np.zeros(1, dtype=_lib.CHURN_EVENT)
            r["type"], r["caller"], r["t"] = _lib.CHURN_REAPER, ev["caller"][k], ev["t"][k]
            ev = np.concatenate([ev[:k], r, ev[k:]])
        s._ck(lib.mmp_flush_l2(s.h))
        t0 = time.perf_counter()
        dec, _, _, rep = s.churn_step(ev, now0, now0 + w.window_ms, 400 + ep, want_rows=False)
        dt = time.perf_counter() - t0
        if ep >= warmup:
            wall.append(1e3 * dt); total.append(rep.ms_total); ms_reaper.append(rep.ms_reaper)
            picked.append(int(np.count_nonzero(dec["event"] == k)) if reaper else 0); decided.append(len(dec))
            if ep == warmup + windows // 2:
                clocks.append(nvidia_smi("clocks.sm,clocks.max.sm,clocks_event_reasons.active"))
    s.close()
    return {"windows": windows, "reaper": reaper, "ms_window_wall": float(np.median(wall)), "ms_window_total": float(np.median(total)),
            "ms_reaper": float(np.median(ms_reaper)), "ms_reaper_max": float(np.max(ms_reaper)),
            "reaper_decisions": picked, "decisions": int(np.median(decided)), "clocks_sm_max_throttle": clocks}


def time_select(lib, w, calls: int, warmup: int) -> dict:
    fl = w.fleet
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    _, ids = s.stats()
    parts = [int(p) for p in ids[1:]] or [-1]
    taken = np.zeros(s.max_models, dtype=np.uint8)
    out = np.zeros(s.max_models, dtype=np.int32)
    ms = C.c_double()
    wall, dev, picked = [], [], []
    for it in range(warmup + calls):
        taken[:] = 0
        n_round = 0
        for p in parts:
            s._ck(lib.mmp_flush_l2(s.h))
            t0 = time.perf_counter()
            n = s._ck(lib.mmp_reaper_select(s.h, p, fl.now_ms, taken.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), len(out)))
            dt = time.perf_counter() - t0
            s._ck(lib.mmp_last_timing(s.h, b"reaper", C.byref(ms)))
            n_round += n
            if it >= warmup:
                wall.append(1e3 * dt); dev.append(float(ms.value))
        if it >= warmup:
            picked.append(n_round)
    s.close()
    return {"leg": "mmp_reaper_select", "calls": calls, "partitions": len(parts), "ms_call_wall": float(np.median(wall)),
            "ms_call_wall_min_max": [float(np.min(wall)), float(np.max(wall))], "ms_reaper": float(np.median(dev)),
            "ms_reaper_min_max": [float(np.min(dev)), float(np.max(dev))], "selected_per_round": int(np.median(picked))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--events", type=int, default=20_000)
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--select-only", action="store_true", help="only the mmp_reaper_select leg")
    args = ap.parse_args()
    lib = _lib.load_product()
    gpu = nvidia_smi("name,power.limit")
    for name in ("C4", "C4 at 80 % fill"):
        w = make_churn(500_000, 2_500, 4, fill=0.8 if "80" in name else 0.97)
        legs = [] if args.select_only else [lambda r=r: time_windows(lib, w, args.windows, args.warmup, args.events, 4, r) for r in (False, True)]
        legs.append(lambda: time_select(lib, w, args.calls, args.warmup))
        for leg in legs:
            res = leg()
            res.update({"workload": name, "gpu": gpu, "lib": os.environ.get("MMP_LIB", "in-tree")})
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
