"""The two-pass placement path's CPU harness (tests/emul/split_place.cpp): `split_lib` (a module fixture) compiles it,
place_split() resolves a batch through it, and oracle_same() checks its answers against the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import oracle_inputs
from modelmesh_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def split_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("split_place") / "libmmplace_emul_split.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wl,-Bsymbolic", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "split_place.cpp")])
    lib = _lib.load(so, require_all=False)
    lib.mmp_emul_place_split.restype = C.c_int32
    lib.mmp_emul_place_split.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                         C.c_void_p, C.c_int64, C.c_uint64, C.c_void_p]
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def place_split(lib, s, sd, now_ms, seed):
    dec = np.ascontiguousarray(sd.dec, dtype=_lib.DECISION_IN)
    fresh = np.ascontiguousarray(sd.fresh, dtype=_lib.INSTANCE_ROW) if len(sd.fresh) else None
    extra = np.ascontiguousarray(sd.extra, dtype=np.int32) if len(sd.extra) else None
    out = np.zeros(len(dec), dtype=_lib.DECISION_OUT)
    counts = np.zeros(6, dtype=np.int64)
    s._ck(lib.mmp_emul_place_split(s.h, _ptr(dec), len(dec), _ptr(fresh), 0 if fresh is None else len(fresh), _ptr(extra),
                                   0 if extra is None else len(extra), _ptr(out), now_ms, seed, _ptr(counts)))
    return out, counts


def oracle_same(o, fl, sd, out, seed):
    od, off, idx = oracle_inputs(fl, sd)
    want = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)
    assert np.array_equal(out["target"], want["target"]) and np.array_equal(out["n_candidates"], want["n_candidates"])
