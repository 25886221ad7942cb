"""Latency of mmp_place_one under concurrent request threads: the resident server's slots (one_mode 3) against the replayed
CUDA graph (one_mode 2, the path colliding callers took when the server answered one caller at a time), on C3.

    python tools/server_slots_latency.py --out result.json [--calls 3000] [--warmup 300] [--rounds 2] [--compare-lib PATH]

For each thread count in --threads (default 1 2 4 8 16) and each mode, alternated in the same process, the threads are
released together and each makes `warmup` + `calls` mmp_place_one calls (a committed model, no extras: kind 1) with a host
clock (CLOCK_MONOTONIC) around each call; p50 and p99 are taken per thread over the timed calls, and mmp_server_stats is
read before and after the run.  The threads are pthreads of a small C driver compiled into a temporary directory at start,
so that the timings hold the library call and nothing of Python's interpreter lock.  --rounds repeats the whole sweep: the
spread between rounds is the run-to-run spread.  --compare-lib times another build of the library (a library without
mmp_server_stats too) on its own fleet with the same data, alternated with this one in every round.  The card's name,
power limit and SM clock limit are read in the same run and written beside the numbers.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

DRIVER = r"""
#include <pthread.h>
#include <stdint.h>
#include <time.h>
typedef int32_t (*place_one_t)(void *, const void *, const void *, const void *, void *, int64_t, uint64_t);
typedef struct {
  place_one_t fn; void *h; const char *dec; int n_dec, dec_size, warmup, calls, tid; int64_t now; double *lat;
  pthread_barrier_t *bar; int rc;
} arg_t;
static double now_us(void) { struct timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e6 + t.tv_nsec * 1e-3; }
static void *worker(void *p) {
  arg_t *a = (arg_t *)p;
  char out[8];
  pthread_barrier_wait(a->bar);
  for (int j = 0; j < a->warmup + a->calls; j++) {
    const char *d = a->dec + (size_t)((a->tid * 7919 + j) % a->n_dec) * a->dec_size;
    double t0 = now_us();
    int rc = a->fn(a->h, d, 0, 0, out, a->now, 11);
    double t1 = now_us();
    if (rc < 0) { a->rc = rc; break; }
    if (j >= a->warmup) a->lat[j - a->warmup] = t1 - t0;
  }
  return 0;
}
/* n_threads threads released together; lat[t * calls + j]: call j of thread t in microseconds.  Returns 0 or the first
   negative return code of the library */
int run(void *fn, void *h, const char *dec, int n_dec, int dec_size, int n_threads, int warmup, int calls, int64_t now, double *lat) {
  pthread_t th[64];
  arg_t a[64];
  pthread_barrier_t bar;
  if (n_threads < 1 || n_threads > 64) return -1;
  pthread_barrier_init(&bar, 0, (unsigned)n_threads);
  for (int t = 0; t < n_threads; t++) {
    arg_t x = {(place_one_t)fn, h, dec, n_dec, dec_size, warmup, calls, t, now, lat + (size_t)t * calls, &bar, 0};
    a[t] = x;
    pthread_create(&th[t], 0, worker, &a[t]);
  }
  int rc = 0;
  for (int t = 0; t < n_threads; t++) { pthread_join(th[t], 0); if (a[t].rc < 0 && rc == 0) rc = a[t].rc; }
  pthread_barrier_destroy(&bar);
  return rc;
}
"""


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (x.strip() for x in q.stdout.splitlines()[0].split(","))
    return {"name": name, "power_limit": power, "sm_clock_max": clock}


def driver(tmp):
    src, so = os.path.join(tmp, "driver.c"), os.path.join(tmp, "driver.so")
    with open(src, "w") as f:
        f.write(DRIVER)
    subprocess.check_call(["cc", "-O2", "-shared", "-fPIC", "-pthread", "-o", so, src])
    d = C.CDLL(so)
    d.run.restype = C.c_int
    d.run.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_void_p]
    return d


def server_stats(lib, h):
    if not hasattr(lib, "mmp_server_stats"):
        return None
    v = np.zeros(4, dtype=np.int64)
    assert lib.mmp_server_stats(h, v.ctypes.data_as(C.c_void_p)) == 0
    return v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--calls", type=int, default=3000)
    ap.add_argument("--warmup", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--threads", type=int, nargs="+", default=[1, 2, 4, 8, 16])
    ap.add_argument("--compare-lib", default=None, help="another build of the library, timed alternately on its own fleet")
    args = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from modelmesh_b200 import _lib as L
    from modelmesh_b200.fleet import Fleet
    from modelmesh_b200.synth import load_into_fleet, make_decisions, make_fleet

    fl = make_fleet("C3", 1_000_000, 10_000, 3)
    libs = {"this": L.load_product()}
    if args.compare_lib:
        libs["compare"] = L.load(args.compare_lib, require_all=False)
    fleets = {}
    for name, lib in libs.items():
        s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
        load_into_fleet(fl, s)
        fleets[name] = s
    dec = np.ascontiguousarray(make_decisions(fl, 4096, 7, plain=True).dec)  # committed models, no extras, no fresh rows
    res = {"card": card(), "config": "C3 1 000 000 models x 10 000 instances", "call": "mmp_place_one, committed model, no extras",
           "calls_per_thread": args.calls, "warmup_per_thread": args.warmup,
           "libraries": {k: (args.compare_lib if k == "compare" else os.environ.get("MMP_LIB", L.PRODUCT_SO)) for k in libs},
           "runs": []}
    with tempfile.TemporaryDirectory() as tmp:
        drv = driver(tmp)
        for rnd in range(args.rounds):
            for nt in args.threads:
                for name, lib in libs.items():
                    s = fleets[name]
                    for mode_name, mode in (("server", 3), ("graph", 2)):
                        s._ck(lib.mmp_tune(s.h, b"one_mode", mode))
                        lat = np.zeros(nt * args.calls, dtype=np.float64)
                        before = server_stats(lib, s.h)
                        rc = drv.run(C.cast(lib.mmp_place_one, C.c_void_p), s.h, dec.ctypes.data_as(C.c_void_p), len(dec),
                                     dec.itemsize, nt, args.warmup, args.calls, fl.now_ms, lat.ctypes.data_as(C.c_void_p))
                        if rc < 0:
                            raise RuntimeError(lib.mmp_last_error(s.h))
                        after = server_stats(lib, s.h)
                        lat = lat.reshape(nt, args.calls)
                        p50 = np.percentile(lat, 50, axis=1)
                        p99 = np.percentile(lat, 99, axis=1)
                        run = {"round": rnd, "threads": nt, "library": name, "mode": mode_name,
                               "p50_us_median_thread": float(np.median(p50)), "p99_us_median_thread": float(np.median(p99)),
                               "p50_us_per_thread": [round(float(x), 2) for x in p50],
                               "p99_us_per_thread": [round(float(x), 2) for x in p99]}
                        if before is not None:
                            d = after - before
                            run["server_stats"] = {"answered": int(d[0]), "fallbacks": int(d[1]), "launches": int(d[2]),
                                                   "max_busy_since_create": int(after[3])}
                        res["runs"].append(run)
                        print(json.dumps({k: v for k, v in run.items() if not k.endswith("per_thread")}), flush=True)
                    s._ck(lib.mmp_tune(s.h, b"one_mode", 3))
    for s in fleets.values():
        s.close()
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
