"""Latency of single request-model decisions (MMP_DF_REQUEST_MODEL) and throughput of a flagged batch, on C3.

    python tools/request_model_latency.py --out result.json [--calls 3000] [--unflagged-only]

For the resident server (one_mode 3) and the replayed graph (one_mode 2) it times mmp_place_one, p50 / p99 over `calls`
calls after a warm-up, for: a committed model without extras; a request-model decision with 0 and with 3 instance ids; an
unflagged decision with 3 extra excludes (the server takes it as one line-1 request with the extras inline).  Then one
batch of 1 M decisions -- the C3 registry sweep -- through mmp_place_batch with pinned host buffers, unflagged and with
every model's record carried by its decision (models with more than 16 ids stay unflagged), decisions/s on the host clock.
--unflagged-only skips the flagged cases (a library without the flag).  The card's name, power limit and SM clock limit are
read in the same run and written beside the numbers.  MMP_LIB selects another build of the library.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--batch-reps", type=int, default=5)
    ap.add_argument("--unflagged-only", action="store_true")
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from modelmesh_b200 import _lib as L
    from modelmesh_b200.fleet import Fleet
    from modelmesh_b200.synth import load_into_fleet, make_decisions, make_fleet

    lib = L.load_product()
    fl = make_fleet("C3", 1_000_000, 10_000, 3)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    tid = load_into_fleet(fl, s)
    tmap = np.asarray([tid[t] for t in fl.type_names], dtype=np.int32)
    res = {"card": card(), "library": os.environ.get("MMP_LIB", L.PRODUCT_SO), "config": "C3 1 000 000 models x 10 000 instances"}

    # ---- single decisions ----
    rng = np.random.default_rng(7)
    live = np.nonzero(fl.inst_rows["shutting_down"] == 0)[0]
    base = make_decisions(fl, args.calls + args.warmup, 7, plain=True).dec
    base["flags"] &= np.uint32(L.DF_FAVOUR_SELF)  # explicit last_used (a request-model decision has no model row)
    base["last_used"] = fl.now_ms - 60_000
    ids3 = live[rng.integers(0, len(live), size=(len(base), 3))].astype(np.int32)
    cases = {"committed_no_extras": (False, 0), "unflagged_3_extras": (False, 3)}
    if not args.unflagged_only:
        cases.update({"request_model_0_ids": (True, 0), "request_model_3_ids": (True, 3)})
    out = np.zeros(1, dtype=L.DECISION_OUT)
    lat = {}
    for mode_name, mode in (("server", 3), ("graph", 2)):
        s._ck(lib.mmp_tune(s.h, b"one_mode", mode))
        for case, (flag, nx) in cases.items():
            ts = []
            for i in range(len(base)):
                d = base[i:i + 1].copy()
                if flag:
                    d["model"] = tmap[fl.model_type[d["model"][0]]]
                    d["flags"] |= np.uint32(L.DF_REQUEST_MODEL)
                d["extra_off"], d["extra_n"] = 0, nx
                x = np.ascontiguousarray(ids3[i])
                t0 = time.perf_counter()
                rc = lib.mmp_place_one(s.h, d.ctypes.data_as(C.c_void_p), None, x.ctypes.data_as(C.c_void_p) if nx else None,
                                       out.ctypes.data_as(C.c_void_p), fl.now_ms, 11)
                t1 = time.perf_counter()
                s._ck(rc)
                assert out["target"][0] != L.TARGET_INVALID
                if i >= args.warmup:
                    ts.append(1e6 * (t1 - t0))
            lat[f"{mode_name}/{case}"] = {"p50_us": float(np.percentile(ts, 50)), "p99_us": float(np.percentile(ts, 99)),
                                          "calls": len(ts)}
            print(mode_name, case, lat[f"{mode_name}/{case}"], flush=True)
    res["place_one"] = lat
    s._ck(lib.mmp_tune(s.h, b"one_mode", 3))

    # ---- a 1 M-decision batch: the registry sweep, unflagged and carrying every model's record ----
    sweep = make_decisions(fl, fl.n_models, 3, sweep=True, plain=True).dec
    sweep["flags"] &= np.uint32(L.DF_FAVOUR_SELF)
    sweep["last_used"] = fl.model_last_used
    deg = np.diff(fl.edge_off)
    rq = sweep.copy()
    fit = deg <= L.MAX_EXTRA
    rq["model"] = np.where(fit, tmap[fl.model_type], rq["model"])
    rq["flags"] = np.where(fit, rq["flags"] | np.uint32(L.DF_REQUEST_MODEL), rq["flags"])
    rq["extra_off"] = np.where(fit, fl.edge_off[:-1], 0)
    rq["extra_n"] = np.where(fit, deg, 0)
    extra = np.ascontiguousarray(fl.edge_inst, dtype=np.int32)
    n = len(sweep)
    h_in, h_out, h_ex = C.c_void_p(), C.c_void_p(), C.c_void_p()
    s._ck(lib.mmp_host_alloc(s.h, sweep.nbytes, C.byref(h_in)))
    s._ck(lib.mmp_host_alloc(s.h, n * L.DECISION_OUT.itemsize, C.byref(h_out)))
    s._ck(lib.mmp_host_alloc(s.h, max(extra.nbytes, 4), C.byref(h_ex)))
    C.memmove(h_ex, extra.ctypes.data_as(C.c_void_p), extra.nbytes)
    batches = {"unflagged": (sweep, 0)}
    if not args.unflagged_only:
        batches["request_model"] = (rq, len(extra))
    outs, rates = {}, {}
    for name, (dec, ne) in batches.items():
        dec = np.ascontiguousarray(dec)
        C.memmove(h_in, dec.ctypes.data_as(C.c_void_p), dec.nbytes)
        ts = []
        for rep in range(args.batch_reps + 1):
            t0 = time.perf_counter()
            s._ck(lib.mmp_place_batch(s.h, h_in, n, None, 0, h_ex if ne else None, ne, h_out, fl.now_ms, 3))
            if rep:
                ts.append(time.perf_counter() - t0)
        outs[name] = np.frombuffer((C.c_char * (n * 8)).from_address(h_out.value), dtype=L.DECISION_OUT).copy()
        rates[name] = {"decisions_per_s_median": float(n / np.median(ts)), "ms_median": float(1e3 * np.median(ts)),
                       "ms_min": float(1e3 * np.min(ts)), "reps": len(ts)}
        print(name, rates[name], flush=True)
    if "request_model" in outs:
        rates["request_model"]["flagged_fraction"] = float(fit.mean())
        rates["identical_results"] = bool(np.array_equal(outs["unflagged"], outs["request_model"]))
    res["batch_1m_e2e"] = rates
    for p in (h_in, h_out, h_ex):
        lib.mmp_host_free(s.h, p)
    s.close()
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
