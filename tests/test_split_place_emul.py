"""CPU checks of the two-pass placement path: the per-slot summaries (slot_summary, both values of c_self) and the
answer they give a decision clear of its slot's reach (split_answer), compiled by g++ from place_core.cuh.

The tests/emul/split_place.cpp harness resolves a batch as k_place_direct does, then answers from the summaries every
decision k_place_split would answer, and counts the answers that differ from the walk."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from modelmesh_b200 import _lib
from modelmesh_b200._lib import DF_FAVOUR_SELF
from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import oracle_from_synth, oracle_inputs, solver_from_synth

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
    counts = np.zeros(4, dtype=np.int64)
    s._ck(lib.mmp_emul_place_split(s.h, _ptr(dec), len(dec), _ptr(fresh), 0 if fresh is None else len(fresh), _ptr(extra),
                                   0 if extra is None else len(extra), _ptr(out), now_ms, seed, _ptr(counts)))
    return out, counts


def _oracle_same(o, fl, sd, out, seed):
    od, off, idx = oracle_inputs(fl, sd)
    want = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)
    assert np.array_equal(out["target"], want["target"]) and np.array_equal(out["n_candidates"], want["n_candidates"])


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 3000, 1300, 33), ("C5", 1500, 500, 5), ("MIX", 800, 300, 14),
                                               ("MIX", 800, 700, 41), ("C2", 2000, 400, 2)])
def test_summary_answers_equal_the_walk(split_lib, oracle_lib, config, nm, ni, seed):
    """Plain sweeps (most decisions answered from the summaries), favour_self sweeps, and mixed batches (fresh records,
    extras, request-model decisions): every answer from a summary equals the decision's walk, and the walk the oracle."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, split_lib)
    sweep = make_decisions(fl, 3000, seed, sweep=True, plain=True)
    fav = make_decisions(fl, 2000, seed + 3, sweep=True, plain=True)
    fav.dec["flags"] |= DF_FAVOUR_SELF
    answered = 0
    for k, sd in enumerate((sweep, fav, make_decisions(fl, 2000, seed + 1))):
        out, counts = place_split(split_lib, s, sd, fl.now_ms, seed + k)
        assert counts[1] == 0, (config, k, counts)
        _oracle_same(o, fl, sd, out, seed + k)
        answered += counts[0]
    assert answered > 0
    s.close()


def test_reach_edges_on_a_front_loaded_fleet(split_lib, oracle_lib):
    """Every model's inline edges and every self among the first 64 ranks: exclusions and selves at, just before and just
    past best, the shortlist and its cut."""
    fl = make_fleet("C3", 3000, 1500, 21)
    order = oracle_from_synth(fl).cluster_order()
    rng = np.random.default_rng(21)
    nm = fl.n_models
    front = order[:64]
    edges = [list(rng.choice(front, size=rng.integers(0, 5), replace=False)) for _ in range(nm)]
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([int(x) for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, split_lib)
    sd = make_decisions(fl, 3000, 21, sweep=True, plain=True)
    sd.dec["self"] = rng.choice(front, size=len(sd.dec))
    for k in range(2):
        out, counts = place_split(split_lib, s, sd, fl.now_ms, 21 + k)
        assert counts[1] == 0, counts
        _oracle_same(o, fl, sd, out, 21 + k)
        sd.dec["flags"] |= DF_FAVOUR_SELF
    s.close()
