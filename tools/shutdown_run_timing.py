"""Timing of one pod's pre-shutdown migration: mmp_shutdown_run against the composed route a pod would otherwise take, on C3
(1 000 000 models x 10 000 instances) with a load / failure time for every registration, for the pod with the most
registrations: an entry for every model it is registered on and 100 entries of models it does not hold, lru_t values spread
over the last six hours.

The composed route: the classification on the host (the registry test over the fleet's registrations, the stale and
lruTime tests, checkLoadFailureCount) and one mmp_place_batch of the placed entries with the same MMP_DF_OWN_ID ids and
extra {self}.  The first call of each route is checked to return the same answers.

    python tools/shutdown_run_timing.py --out result.json [--reps 30]

Reports the host clock around each call (both end in a device synchronise), with preallocated output buffers: median, min
and max over `reps` calls of each, the routes alternated after three warm-up calls of each, and the composed route's
mmp_place_batch call on its own (its classification is a Python loop here, a Java one in a pod); the median of
mmp_last_timing("shutdown_run"); the report of the call; and the card's name, power limit and SM clock limit, read in the
same run.
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
    ents = np.zeros(len(models), dtype=L.SHUTDOWN_ENTRY)
    ents["model"] = models
    ents["lru_t"] = now - rng.integers(0, 6 * HOUR, size=len(models))
    ents["last_used"] = -1
    ents = ents[np.argsort(-ents["lru_t"], kind="stable")]
    p = np.zeros(1, dtype=L.SHUTDOWN_PARAMS)
    p["now"], p["cutoff_age_ms"], p["load_failure_expiry_ms"] = now, HOUR, EXPIRY
    since = now - EXPIRY // 2
    # the per-entry registry slices the composed route reads, gathered once (the pod's own registry lookups)
    sl = [(fl.edge_inst[fl.edge_off[m]:fl.edge_off[m] + fl.n_loaded[m]], ts[fl.edge_off[m] + fl.n_loaded[m]:fl.edge_off[m + 1]])
          for m in ents["model"]]
    d_all = np.zeros(len(ents), dtype=L.DECISION_IN)
    r_all = np.zeros(len(ents), dtype=L.DECISION_OUT)
    extra = np.array([S], dtype=np.int32)

    out = np.zeros(len(ents), dtype=L.SHUTDOWN_ACTION)
    rep = L.ShutdownReport()

    def one_call():
        s._ck(lib.mmp_shutdown_run(s.h, S, vp(ents), len(ents), vp(p), None, 7, vp(out), C.byref(rep)))

    def composed():
        """the placed entries' (entry, target, n_candidates)"""
        rows = []
        for r, e in enumerate(ents):
            loaded, fts = sl[r]
            if S not in loaded:
                continue
            lru = int(e["lru_t"]) if int(e["lru_t"]) != 0 else int(e["last_used"])
            if lru > 0 and int(np.count_nonzero(fts > since)) < 3:
                rows.append((r, lru))
        d = d_all[:len(rows)]
        d["model"] = [int(ents["model"][r]) for r, _ in rows]
        d["self"], d["last_used"] = S, [lru for _, lru in rows]
        d["flags"] = [L.DF_FAVOUR_SELF | L.DF_OWN_ID | (r << 8) for r, _ in rows]
        d["fresh"], d["extra_off"], d["extra_n"] = -1, 0, 1
        got = s.place_batch(d, now, 7, extra=extra, out=r_all[:len(rows)])
        return [(r, int(x["target"]), int(x["n_candidates"])) for (r, _), x in zip(rows, got)]

    def place_only():
        """the composed route's mmp_place_batch alone, on the records its classification built last"""
        k = int(rep.n_placed)
        s.place_batch(d_all[:k], now, 7, extra=extra, out=r_all[:k])

    one_call()
    placed = np.nonzero(out["what"] & L.SD_PLACED)[0]
    assert composed() == [(int(r), int(out["target"][r]), int(out["n_candidates"][r])) for r in placed], "the two routes disagree"
    res["report"] = {k: getattr(rep, k) for k, _ in L.ShutdownReport._fields_ if k != "reserved"}
    res["entries"] = len(ents)

    def timed(k):
        t0 = time.perf_counter()
        (one_call, composed, place_only)[k]()
        return (time.perf_counter() - t0) * 1e3

    for _ in range(3):
        timed(0), timed(1), timed(2)
    host, dev = [[], [], []], []
    t = C.c_double()
    for _ in range(args.reps):
        for k in (0, 1, 2):
            host[k].append(timed(k))
            if k == 0:
                s._ck(lib.mmp_last_timing(s.h, b"shutdown_run", C.byref(t)))
                dev.append(t.value)
    for k, name in ((0, "shutdown_run"), (1, "composed"), (2, "composed_place_batch_only")):
        h = np.array(host[k])
        res[name] = {"host_ms_median": float(np.median(h)), "host_ms_min": float(h.min()), "host_ms_max": float(h.max())}
    res["shutdown_run"]["device_ms_median"] = float(np.median(dev))
    res["reps"] = args.reps
    s.close()
    with open(args.out, "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
