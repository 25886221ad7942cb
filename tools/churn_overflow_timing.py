"""Cost of overflow registrations in the closed loop: mmp_churn_step on the C4 fleet (500k models x 2 500 instances, 97 % fill,
20 000 events per 2 s window) as bench.py runs it, and on the same fleet with 0.2 % of its models at 6 registrations
(synth.make_churn_overflow).  Prints one JSON line per workload: the median window time (host clock around the step, and the
step's own CUDA-event total), the median and largest registry phase (ms_registry, which holds the overflow re-lay), and the
GPU's name and power limit.  MMP_LIB selects another build of the library.

    python tools/churn_overflow_timing.py [--windows 10] [--warmup 3] [--frac 0.002]
"""
from __future__ import annotations

import argparse
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
from modelmesh_b200.synth import load_into_fleet, make_churn, make_churn_overflow  # noqa: E402


def gpu_name_and_power() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def time_windows(lib, w, windows: int, warmup: int, events: int, seed: int) -> dict:
    fl = w.fleet
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    s.churn_init(w.load_timeout_ms, fl.now_ms - 60_000, 512)
    s.churn_seed(w.seed_instance, w.seed_model, w.seed_last_used, w.seed_weight, w.seed_load_ts, fl.now_ms)
    wall, total, registry = [], [], []
    for ep in range(warmup + windows):
        ev = w.events(ep, events, seed)
        now0 = fl.now_ms + ep * w.window_ms
        s._ck(lib.mmp_flush_l2(s.h))
        t0 = time.perf_counter()
        _, _, _, rep = s.churn_step(ev, now0, now0 + w.window_ms, 400 + ep, want_rows=False)
        dt = time.perf_counter() - t0
        if ep >= warmup:
            wall.append(1e3 * dt); total.append(rep.ms_total); registry.append(rep.ms_registry)
    s.close()
    return {"windows": windows, "ms_window_wall": float(np.median(wall)), "ms_window_total": float(np.median(total)),
            "ms_registry": float(np.median(registry)), "ms_registry_max": float(np.max(registry)),
            "events_per_s": events / (float(np.median(wall)) / 1e3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frac", type=float, default=0.002)
    ap.add_argument("--events", type=int, default=20_000)
    args = ap.parse_args()
    lib = _lib.load_product()
    gpu = gpu_name_and_power()
    base = make_churn(500_000, 2_500, 4)
    for name, w in (("C4", base), (f"C4 with {args.frac:.2%} of the models at 6 registrations",
                                   make_churn_overflow(base, args.frac, 4, regs=(6, 6)))):
        res = time_windows(lib, w, args.windows, args.warmup, args.events, 4)
        res.update({"workload": name, "models_over_four": int((np.diff(w.fleet.edge_off) > 4).sum()), "gpu": gpu,
                    "lib": os.environ.get("MMP_LIB", "in-tree")})
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
