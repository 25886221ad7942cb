"""Timing of the registry-side scans on C3 (1 000 000 models x 10 000 instances) with a load / failure time for every
registration, 40 pods gone and first seen missing 11 minutes ago.

    python tools/registry_scans_timing.py --out result.json [--reps 30] [--parent-lib path/to/libmmplace.so]

prune: the median (and min / max) over `reps` calls of the kernel time, mmp_last_timing("prune"), of mmp_registry_prune (the
four-registration view) and mmp_registry_prune_ids (every registration).  --parent-lib: another build of the library (the
parent commit's) loads the same fleet, and its mmp_registry_prune is called alternately with this build's, so that the
run-to-run spread of both is measured in the same run.  scale: host-clock time of mmp_scale_eval on 100 000 cache entries
(the call ends in a device synchronise).  The card's name, power limit and SM clock limit are read in the same run.
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
    ap.add_argument("--parent-lib", default=None)
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from modelmesh_b200 import _lib as L
    from modelmesh_b200.fleet import Fleet
    from modelmesh_b200.synth import load_into_fleet, make_fleet

    fl = make_fleet("C3", 1_000_000, 10_000, 3)
    rng = np.random.default_rng(5)
    ts = (fl.now_ms - rng.integers(0, 4 * 3_600_000, size=len(fl.edge_inst))).astype(np.int64)
    lul = np.where(rng.uniform(size=fl.n_models) < 0.3, fl.now_ms - rng.integers(0, 200_000, size=fl.n_models), 0).astype(np.int64)
    gone = rng.choice(fl.n_instances, size=40, replace=False)
    self_idx = int(np.setdiff1d(np.arange(fl.n_instances), gone)[0])
    missing0 = np.zeros(fl.n_instances, dtype=np.int64)
    missing0[gone] = fl.now_ms - 660_000

    def fleet(lib):
        s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
        load_into_fleet(fl, s)
        for m in range(fl.n_models):
            a, b = fl.edge_off[m], fl.edge_off[m + 1]
            if a != b:
                s._ck(lib.mmp_model_times(s.h, m, ts[a:b].ctypes.data_as(C.c_void_p), int(b - a), int(lul[m])))
        for i in gone:
            s.instance_remove(int(i))
        s.commit()
        return s

    def prune(lib, s, ids):
        miss = missing0.copy()
        outm = np.zeros(fl.n_models, dtype=np.int32)
        outx = np.zeros(fl.n_models, dtype=np.int32 if ids else np.uint8)
        fn = lib.mmp_registry_prune_ids if ids else lib.mmp_registry_prune
        n = s._ck(fn(s.h, self_idx, fl.now_ms, GONE_MS, miss.ctypes.data_as(C.c_void_p), outm.ctypes.data_as(C.c_void_p),
                     outx.ctypes.data_as(C.c_void_p), fl.n_models))
        ms = C.c_double()
        s._ck(lib.mmp_last_timing(s.h, b"prune", C.byref(ms)))
        return float(ms.value), n, outm[:n].tobytes() + outx[:n].tobytes()

    lib = L.load_product()
    s = fleet(lib)
    parent = None
    if args.parent_lib:
        plib = L.load(args.parent_lib, require_all=False)
        parent = (plib, fleet(plib))
    res = {"card": card(), "config": "C3 1 000 000 models x 10 000 instances, times for every registration, 40 pods gone",
           "overflow_models": int(np.count_nonzero(np.diff(fl.edge_off) > 4)), "registrations": int(len(fl.edge_inst))}
    t_inl, t_ids, t_par = [], [], []
    for k in range(args.reps + 3):  # the first three calls are warm-up
        a, n_inl, out_inl = prune(lib, s, False)
        b, n_ids, _ = prune(lib, s, True)
        if parent:
            c, n_par, out_par = prune(parent[0], parent[1], False)
            assert n_par == n_inl and out_par == out_inl, "the four-registration view differs from the parent build"
        if k >= 3:
            t_inl.append(a); t_ids.append(b)
            if parent:
                t_par.append(c)
    res["prune"] = {"mmp_registry_prune": _stats(t_inl), "mmp_registry_prune_ids": _stats(t_ids),
                    "models_pruned": n_inl, "registrations_pruned": n_ids}
    if parent:
        res["prune"]["parent_mmp_registry_prune"] = _stats(t_par)
    n = 100_000
    rec = np.zeros(n, dtype=L.SCALE_IN)
    rec["model"] = rng.integers(0, fl.n_models, size=n)
    k = fl.n_loaded[rec["model"]]
    pick = fl.edge_inst[np.minimum(fl.edge_off[rec["model"]] + (rng.uniform(size=n) * np.maximum(k, 1)).astype(np.int64), len(fl.edge_inst) - 1)]
    rec["instance"] = np.where(k > 0, pick, rng.integers(0, fl.n_instances, size=n))
    rec["count"] = rng.integers(0, 20_000, size=n)
    rec["last_used"] = fl.now_ms - rng.integers(0, 40 * 3_600_000, size=n)
    rec["i1"] = 5000 - rng.integers(0, 400, size=n)
    rec["i2"] = np.minimum(5000, rec["i1"] + rng.integers(0, 300, size=n))
    p = np.zeros(1, dtype=L.SCALE_PARAMS)
    p["now"], p["last_check_time"], p["iteration"], p["scale_up_rpm_threshold"] = fl.now_ms, fl.now_ms - 10_000, 5000, 2000
    p["second_copy_min_age_iters"], p["second_copy_max_age_iters"], p["second_copy_lru_threshold_ms"] = 42, 240, 6 * 3_600_000
    p["rate_check_interval_ms"], p["assume_completed_ms"], p["second_copy_remove_max_age_ms"], p["can_remove"] = 10_000, 30_000, 36_000_000, 1
    out = np.zeros(n, dtype=L.SCALE_OUT)
    t_scale = []
    for k in range(args.reps + 3):
        t0 = time.perf_counter()
        s._ck(lib.mmp_scale_eval(s.h, rec.ctypes.data_as(C.c_void_p), n, p.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
        if k >= 3:
            t_scale.append((time.perf_counter() - t0) * 1e3)
    res["scale_eval_100k"] = _stats(t_scale)
    res["scale_eval_100k"]["actions"] = {str(a): int(np.count_nonzero(out["action"] == a)) for a in (-1, 0, 1, 2)}
    print(json.dumps(res, indent=1))
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
