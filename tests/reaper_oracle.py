"""The oracle's closed loop with REAPER events (tests/emul/reaper_sim.cpp): orc_sim_step_reaper is oracle/mm_sim.inc's
orc_sim_step plus the reaper's proactive loads as a third event type.

`reaper_oracle` (a module fixture) builds that library -- the whole oracle plus the one step function -- and makes it the
library oracle/binding.py hands out while the module runs, so every OracleFleet / OracleSim the module creates lives in it.
`with_reaper(sim)` then makes sim.step run orc_sim_step_reaper; reaper_sim(w) builds a churn workload's oracle and loop that
way, and reaper_event() is one REAPER event of it."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import oracle_from_synth
from modelmesh_b200._lib import CHURN_REAPER
from oracle import binding as ob

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emul", "reaper_sim.cpp")
REAPER = 2


@pytest.fixture(scope="session")
def _reaper_oracle_so(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("reaper_oracle") / "libmm_oracle_reaper.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-pthread", "-shared", "-o", so, SRC])
    return so


@pytest.fixture(scope="module")
def reaper_oracle(oracle_lib, _reaper_oracle_so):
    saved = ob.SO, ob._lib
    ob.SO, ob._lib = _reaper_oracle_so, None
    try:
        L = ob.lib()
        P, I32, I64, U64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
        L.orc_sim_step_reaper.restype = I64
        L.orc_sim_step_reaper.argtypes = [P, P, I32, I64, I64, U64, P, I32, C.POINTER(I32), P, I32, C.POINTER(I32), P, C.POINTER(I32)]
        yield L
    finally:
        ob.SO, ob._lib = saved


def step(sim: ob.OracleSim, events: np.ndarray, now0: int, now1: int, seed: int):
    """OracleSim.step through orc_sim_step_reaper; the report buffers hold one decision per model for every REAPER event"""
    ev = np.ascontiguousarray(events, dtype=ob.SIM_EVENT)
    n_rp = int(np.count_nonzero(ev["type"] == REAPER)) * sim.reaper_models
    cap_d = len(ev) + 65536 + n_rp
    cap_e = 4 * (len(ev) + n_rp) + 65536
    dec = np.zeros(cap_d, dtype=ob.SIM_DECISION)
    evi = np.zeros(cap_e, dtype=ob.SIM_EVICTION)
    rows = np.zeros(sim.n_instances, dtype=ob.INST)
    nd, ne, npub = C.c_int32(), C.c_int32(), C.c_int32()
    carry = sim.L.orc_sim_step_reaper(sim.h, ob._ptr(ev), len(ev), now0, now1, seed, ob._ptr(dec), cap_d, C.byref(nd), ob._ptr(evi),
                                      cap_e, C.byref(ne), ob._ptr(rows), C.byref(npub))
    assert carry >= 0 and nd.value <= cap_d and ne.value <= cap_e
    return dec[:nd.value].copy(), evi[:ne.value].copy(), rows, int(npub.value), int(carry)


def with_reaper(sim: ob.OracleSim, n_models: int) -> ob.OracleSim:
    """sim, its step() now orc_sim_step_reaper (the sim must live in the reaper_oracle library)"""
    assert hasattr(sim.L, "orc_sim_step_reaper"), "create the sim while the reaper_oracle fixture is active"
    sim.reaper_models = n_models
    sim.step = lambda ev, now0, now1, seed: step(sim, ev, now0, now1, seed)
    return sim


def reaper_sim(w):
    """(the oracle fleet of w, its closed loop seeded with w's caches and stepping with REAPER events)"""
    fl = w.fleet
    o = oracle_from_synth(fl, bulk=False)
    models = np.zeros(fl.n_models, dtype=ob.SIM_MODEL)
    models["last_used"], models["type_idx"], models["size_units"] = fl.model_last_used, fl.model_type, fl.model_size
    sim = with_reaper(ob.OracleSim(o, models, fl.type_names, fl.edge_off, fl.edge_inst, fl.n_loaded, w.capacity, w.load_timeout_ms,
                                   fl.now_ms - 60_000), fl.n_models)
    order = np.argsort(w.seed_instance, kind="stable")
    bounds = np.searchsorted(w.seed_instance[order], np.arange(fl.n_instances + 1))
    for i in range(fl.n_instances):
        sel = order[bounds[i]:bounds[i + 1]]
        if len(sel):
            sim.seed(i, w.seed_model[sel], w.seed_last_used[sel], w.seed_weight[sel], w.seed_load_ts[sel], fl.now_ms)
    return o, sim


def reaper_event(caller: int, t: int) -> np.ndarray:
    e = np.zeros(1, dtype=ob.SIM_EVENT)
    e["type"], e["caller"], e["t"] = CHURN_REAPER, caller, t
    return e
