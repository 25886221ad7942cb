"""Latency of single decisions under a call-wide exclude set (mmp_place_batch_excluding) and throughput of a 1 M-decision
batch under one, on C3 (1 000 000 models x 10 000 instances).

    python tools/exclude_set_latency.py --out result.json [--calls 3000] [--batch-reps 5]

B = 1: p50 / p99 over `calls` calls (after a warm-up) of one decision with sets of 17, 200 and 2 000 instance ids, next to
mmp_place_one without a set (the resident server, one_mode 3, the default).  A call with a set derives its own slot tables
(k_exclude_slots + k_slot_lists) and is launched as k_place_small.  1 M decisions -- the C3 registry sweep, pinned host
buffers, host clock around each call -- with sets of 0, 16, 500 and 5 000 ids, alternated with mmp_place_batch (the same
route as the empty set) so that the spread of that call is measured in the same run.  The card's name, power limit and SM
clock limit are read in the same run and written beside the numbers.
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def _stats(ts):
    return {"p50_us": float(np.percentile(ts, 50)), "p99_us": float(np.percentile(ts, 99)), "calls": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--batch-reps", type=int, default=5)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from modelmesh_b200 import _lib as L
    from modelmesh_b200.fleet import Fleet
    from modelmesh_b200.synth import load_into_fleet, make_decisions, make_fleet

    lib = L.load_product()
    fl = make_fleet("C3", 1_000_000, 10_000, 3)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, s)
    res = {"card": card(), "config": "C3 1 000 000 models x 10 000 instances"}
    rng = np.random.default_rng(7)
    sets = {k: np.ascontiguousarray(rng.integers(0, fl.n_instances, size=k), dtype=np.int32) for k in (16, 17, 200, 500, 2000, 5000)}
    sets[0] = np.zeros(0, dtype=np.int32)
    P = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731

    # ---- single decisions ----
    base = make_decisions(fl, args.calls + args.warmup, 7, plain=True).dec
    out = np.zeros(1, dtype=L.DECISION_OUT)
    lat = {}
    for case in ("place_one_no_set", "set_17", "set_200", "set_2000"):
        xs = None if case == "place_one_no_set" else sets[int(case.split("_")[1])]
        ts = []
        for i in range(len(base)):
            d = np.ascontiguousarray(base[i:i + 1])
            t0 = time.perf_counter()
            if xs is None:
                rc = lib.mmp_place_one(s.h, P(d), None, None, P(out), fl.now_ms, 11)
            else:
                rc = lib.mmp_place_batch_excluding(s.h, P(d), 1, None, 0, None, 0, P(xs), len(xs), P(out), None, None, fl.now_ms, 11)
            t1 = time.perf_counter()
            s._ck(rc)
            if i >= args.warmup:
                ts.append(1e6 * (t1 - t0))
        lat[case] = _stats(ts)
        print(case, lat[case], flush=True)
    res["b1"] = lat

    # ---- the 1 M-decision batch ----
    sweep = np.ascontiguousarray(make_decisions(fl, fl.n_models, 3, sweep=True, plain=True).dec)
    n = len(sweep)
    h_in, h_out = C.c_void_p(), C.c_void_p()
    s._ck(lib.mmp_host_alloc(s.h, sweep.nbytes, C.byref(h_in)))
    s._ck(lib.mmp_host_alloc(s.h, n * L.DECISION_OUT.itemsize, C.byref(h_out)))
    C.memmove(h_in, P(sweep), sweep.nbytes)
    names = ["place_batch", "set_0", "set_16", "set_500", "set_5000"]
    ts = {k: [] for k in names}
    outs = {}
    for rep in range(args.batch_reps + 1):
        for k in names:
            xs = None if k == "place_batch" else sets[int(k.split("_")[1])]
            t0 = time.perf_counter()
            if xs is None:
                rc = lib.mmp_place_batch(s.h, h_in, n, None, 0, None, 0, h_out, fl.now_ms, 3)
            else:
                rc = lib.mmp_place_batch_excluding(s.h, h_in, n, None, 0, None, 0, P(xs), len(xs), h_out, None, None, fl.now_ms, 3)
            dt = time.perf_counter() - t0
            s._ck(rc)
            if rep:
                ts[k].append(dt)
            outs[k] = np.frombuffer((C.c_char * (n * 8)).from_address(h_out.value), dtype=L.DECISION_OUT).copy()
    batch = {}
    for k in names:
        batch[k] = {"ms_median": float(1e3 * np.median(ts[k])), "ms_min": float(1e3 * np.min(ts[k])), "ms_max": float(1e3 * np.max(ts[k])),
                    "decisions_per_s_median": float(n / np.median(ts[k])), "reps": len(ts[k])}
        print(k, batch[k], flush=True)
    batch["set_0_identical_to_place_batch"] = bool(np.array_equal(outs["set_0"], outs["place_batch"]))
    res["batch_1m_e2e"] = batch
    for p in (h_in, h_out):
        lib.mmp_host_free(s.h, p)
    s.close()
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
