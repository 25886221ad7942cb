"""Kernel times of the two-pass placement path against the one-pass one (mmp_tune "split" 1 / 0), for the bench
workloads C2 / C3 / C5: the bench's sweep batch placed through mmp_place_batch_device under torch.profiler, each kernel's
mean device time per call by name (k_slot_summary, k_place_split, k_place_tail, k_place_direct, the slot sort), and the
call's CUDA-event time; for k_place_split also the rate at which it streams a plain sweep's 56 B per decision (32 B record,
16 B SplitKey, 8 B result).  GPU only.

    python tools/split_timing.py [--configs C2,C3,C5] [--calls 20]
"""
import argparse
import ctypes as C
import os
import sys
from collections import defaultdict

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SIZES = {"C2": (100_000, 1_000, 2), "C3": (1_000_000, 10_000, 3), "C5": (1_000_000, 10_000, 5)}
SPLIT_BYTES = 32 + 16 + 8  # what k_place_split streams per plain decision: record, the model's SplitKey, result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C3,C5")
    ap.add_argument("--calls", type=int, default=20)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    from modelmesh_b200 import _lib
    from modelmesh_b200._lib import DECISION_OUT
    from modelmesh_b200.fleet import Fleet
    from modelmesh_b200.synth import load_into_fleet, make_decisions, make_fleet

    lib = _lib.load_product()
    torch.cuda.init()
    print(torch.cuda.get_device_name(0))
    try:
        import subprocess
        print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip())
    except OSError:
        pass
    for cfg in args.configs.split(","):
        nm, ni, seed = SIZES[cfg]
        fl = make_fleet(cfg, nm, ni, seed)
        dec = np.ascontiguousarray(make_decisions(fl, nm, seed, sweep=True, plain=True).dec)
        s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, nm, lib=lib)
        load_into_fleet(fl, s)
        d_in, d_out = C.c_void_p(), C.c_void_p()
        s._ck(lib.mmp_device_alloc(s.h, dec.nbytes, C.byref(d_in)))
        s._ck(lib.mmp_device_alloc(s.h, nm * DECISION_OUT.itemsize, C.byref(d_out)))
        s._ck(lib.mmp_device_upload(s.h, d_in, dec.ctypes.data_as(C.c_void_p), dec.nbytes))
        kms = C.c_float()
        for split in (0, 1):
            s._ck(lib.mmp_tune(s.h, b"split", split))
            for _ in range(5):
                s._ck(lib.mmp_place_batch_device(s.h, d_in, nm, d_out, fl.now_ms, seed, C.byref(kms)))
            ev = []
            for _ in range(args.calls):
                s._ck(lib.mmp_place_batch_device(s.h, d_in, nm, d_out, fl.now_ms, seed, C.byref(kms)))
                ev.append(kms.value)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(args.calls):
                    s._ck(lib.mmp_place_batch_device(s.h, d_in, nm, d_out, fl.now_ms, seed, C.byref(kms)))
                torch.cuda.synchronize()
            per = defaultdict(float)
            for e in prof.events():
                if e.device_type == torch.autograd.DeviceType.CUDA:
                    name = e.name.split("<")[0].split("(")[0]
                    per[name] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            print(f"{cfg} split={split}: call median {np.median(ev) * 1000:.1f} us (min {np.min(ev) * 1000:.1f})")
            for k, v in sorted(per.items(), key=lambda kv: -kv[1]):
                rate = f"  {SPLIT_BYTES * nm / (v / args.calls) / 1e6:6.2f} TB/s" if k == "k_place_split" else ""
                print(f"    {k[:60]:60s} {v / args.calls:9.1f} us/call{rate}")
        s._ck(lib.mmp_tune(s.h, b"split", 2))
        s.close()


if __name__ == "__main__":
    main()
