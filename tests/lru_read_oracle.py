"""The oracle with the read side of its LRU (tests/emul/lru_read_oracle.cpp): orderedMap / descendingLruMap, getLastUsedTime
and getWeight on ob.OracleLru caches, and the same walk with registration times on the caches of ob.OracleSim.

`read_oracle` (a module fixture) builds that library -- the whole oracle plus the four read functions -- and makes it the
library oracle/binding.py hands out while the module runs, so every OracleLru / OracleFleet / OracleSim the module creates
lives in it and the functions below can read them."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import binding as ob

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emul", "lru_read_oracle.cpp")


@pytest.fixture(scope="session")
def _read_oracle_so(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("lru_read_oracle") / "libmm_oracle_read.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-pthread", "-shared", "-o", so, SRC])
    return so


@pytest.fixture(scope="module")
def read_oracle(oracle_lib, _read_oracle_so):
    saved = ob.SO, ob._lib
    ob.SO, ob._lib = _read_oracle_so, None
    try:
        L = ob.lib()
        P, I32, I64 = C.c_void_p, C.c_int32, C.c_int64
        for name, res, args in (("orc_lru_read", I64, [P, I64, P, P, P, I64]), ("orc_lru_last_used", I64, [P, I32]),
                                ("orc_lru_weight", I64, [P, I32]), ("orc_sim_lru_read", I64, [P, I32, I64, P, P, P, P, I64])):
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        yield L
    finally:
        ob.SO, ob._lib = saved


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def lru_read(lru: ob.OracleLru, used_since: int = 0):
    """descendingMapWithCutoff(used_since): keys / lastUsed / weights, most recently used first"""
    n = lru.size()
    k = np.zeros(n, dtype=np.int32)
    t, w = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int64)
    got = lru.L.orc_lru_read(lru.h, used_since, _p(k), _p(t), _p(w), n)
    assert 0 <= got <= n
    return k[:got].copy(), t[:got].copy(), w[:got].copy()


def lru_last_used(lru: ob.OracleLru, key: int) -> int:
    return int(lru.L.orc_lru_last_used(lru.h, key))


def lru_weight(lru: ob.OracleLru, key: int) -> int:
    return int(lru.L.orc_lru_weight(lru.h, key))


def sim_lru_read(sim: ob.OracleSim, instance: int, used_since: int = 0):
    """descendingMapWithCutoff(used_since) of the instance's cache: keys / lastUsed / weights / loadTs (-1 if absent)"""
    n = sim.lru_state(instance)[2]
    k = np.zeros(n, dtype=np.int32)
    t, w, lt = (np.zeros(n, dtype=np.int64) for _ in range(3))
    got = sim.L.orc_sim_lru_read(sim.h, instance, used_since, _p(k), _p(t), _p(w), _p(lt), n)
    assert 0 <= got <= n
    return k[:got].copy(), t[:got].copy(), w[:got].copy(), lt[:got].copy()
