"""Cost of reading every device LRU cache: mmp_lru_read over all 2 500 caches of the C4 closed loop (500k models x 2 500
instances, 97 % fill, 512 slots per cache) after a few windows of 20 000 events, as descendingLruMap() (used_since = 0) and
with a cutoff at the median lastUsed.  Prints one JSON line per cutoff: the median over `reps` calls of the kernel time
(mmp_last_timing("lru_read"): count + scan + emit, without the offsets copy between them) and of the call end to end (host
clock around mmp_lru_read into preallocated buffers, both copies included), the bytes the kernels move (every slot's model
column read twice, the time and sequence of every live slot, each returned entry read and written) over the kernel time
against the H100 SXM's 3.35 TB/s, and the GPU's name and power limit.

    python tools/lru_read_timing.py [--windows 3] [--reps 50]
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
from modelmesh_b200.fleet import Fleet, _ptr  # noqa: E402
from modelmesh_b200.synth import load_into_fleet, make_churn  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s
SLOTS = 512


def gpu_name_and_power() -> str:
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return "unknown"


def bytes_moved(n_caches: int, live: int, returned: int) -> int:
    """count: model of every slot, time of every live one; emit: model of every slot, time + seq of every live one, then
    model, weight, time and load time read and the 24 B entry written per returned entry; offsets written and read"""
    return n_caches * SLOTS * 4 * 2 + live * 8 + live * 16 + returned * (24 + 24) + n_caches * 8 * 3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    lib = _lib.load_product()
    gpu = gpu_name_and_power()
    w = make_churn(500_000, 2_500, 4)
    fl = w.fleet
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    s.churn_init(w.load_timeout_ms, fl.now_ms - 60_000, SLOTS)
    s.churn_seed(w.seed_instance, w.seed_model, w.seed_last_used, w.seed_weight, w.seed_load_ts, fl.now_ms)
    for ep in range(args.windows):
        now0 = fl.now_ms + ep * w.window_ms
        s.churn_step(w.events(ep, 20_000, 4), now0, now0 + w.window_ms, 400 + ep, want_rows=False)
    n = fl.n_instances
    _, everything = s.lru_read()
    live = len(everything)
    median_t = int(np.median(everything["last_used"]))
    for name, used_since in (("descendingLruMap", 0), ("descendingMapWithCutoff(median lastUsed)", median_t)):
        offsets = np.zeros(n + 1, dtype=np.int64)
        out = np.zeros(live, dtype=_lib.LRU_ENTRY)
        kernel, wall = [], []
        ms = C.c_double()
        for r in range(args.warmup + args.reps):
            t0 = time.perf_counter()
            s._ck(lib.mmp_lru_read(s.h, None, n, used_since, _ptr(offsets), _ptr(out), live))
            dt = time.perf_counter() - t0
            s._ck(lib.mmp_last_timing(s.h, b"lru_read", C.byref(ms)))
            if r >= args.warmup:
                kernel.append(ms.value); wall.append(1e3 * dt)
        returned = int(offsets[n])
        k_ms = float(np.median(kernel))
        moved = bytes_moved(n, live, returned)
        print(json.dumps({"read": name, "caches": n, "slots": SLOTS, "live_entries": live, "returned": returned, "reps": args.reps,
                          "ms_kernel": k_ms, "ms_kernel_min": float(np.min(kernel)), "ms_kernel_max": float(np.max(kernel)),
                          "ms_end_to_end": float(np.median(wall)), "bytes_moved": moved,
                          "gb_per_s": moved / (k_ms / 1e3) / 1e9, "share_of_hbm_peak": moved / (k_ms / 1e3) / HBM_PEAK,
                          "gpu": gpu}), flush=True)
    s.close()


if __name__ == "__main__":
    main()
