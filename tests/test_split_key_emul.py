"""CPU checks of the per-model entry k_place_split reads (SplitKey: the model row's last_used, the lowest live rank of its
inline edges, its type slot and overflow mark, built by make_split_key as the commit kernels build it): for every
decision, split_answer on the entry gives the same verdict and the same output as the rule it replaced, which read the
model row and the model's excluded ranks (restated in tests/emul/split_key.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from modelmesh_b200 import _lib
from modelmesh_b200._lib import DF_FAVOUR_SELF, DF_MODEL_LAST_USED, DF_REQUEST_MODEL
from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import oracle_from_synth, solver_from_synth
from upgrade import upgrade

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def split_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("split_key") / "libmmplace_emul_split_key.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wl,-Bsymbolic", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "split_key.cpp")])
    return _lib.load(so, require_all=False)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _rule_counts(lib, s, sd, now_ms, seed):
    fn = lib.mmp_emul_split_key_rule
    fn.restype = C.c_int32
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_uint64, C.c_void_p]
    dec = np.ascontiguousarray(sd.dec, dtype=_lib.DECISION_IN)
    fresh = np.ascontiguousarray(sd.fresh, dtype=_lib.INSTANCE_ROW) if len(sd.fresh) else None
    counts = np.zeros(5, dtype=np.int64)
    s._ck(fn(s.h, _ptr(dec), len(dec), _ptr(fresh), 0 if fresh is None else len(fresh), len(sd.extra), now_ms, seed, _ptr(counts)))
    return counts


def _batches(fl, seed):
    """A plain sweep with and without the model's last_used, a favour_self sweep, a mixed batch (fresh records, extras,
    request-model decisions) and the sweep with malformed records among it."""
    sweep = make_decisions(fl, 3000, seed, sweep=True, plain=True)
    own = make_decisions(fl, 3000, seed + 1, sweep=True, plain=True)
    own.dec["flags"] &= ~np.uint32(DF_MODEL_LAST_USED)
    own.dec["last_used"] = np.random.default_rng(seed).choice(
        np.asarray([-(1 << 63), (1 << 63) - 1, fl.now_ms - 5 * 86_400_000, fl.now_ms], dtype=np.int64), size=len(own.dec))
    fav = make_decisions(fl, 2000, seed + 3, sweep=True, plain=True)
    fav.dec["flags"] |= DF_FAVOUR_SELF
    mixed = make_decisions(fl, 2000, seed + 1)
    bad = make_decisions(fl, 2000, seed + 5, sweep=True, plain=True)
    bad.dec["model"][::7] = fl.n_models + 3
    bad.dec["self"][3::11] = -1
    bad.dec["flags"][5::13] |= np.uint32(DF_REQUEST_MODEL)
    bad.dec["model"][5::13] = np.asarray(fl.model_type)[bad.dec["model"][5::13] % fl.n_models]
    return sweep, own, fav, mixed, bad


CASES = [("C2", 2000, 400, 2, None), ("C3", 3000, 1300, 33, None), ("C5", 1500, 500, 5, None), ("MIX", 800, 300, 14, None),
         ("MIX", 800, 700, 41, None), ("C3", 3000, 1300, 33, "half"), ("MIX", 800, 300, 14, "saturated")]


@pytest.mark.parametrize("config,nm,ni,seed,pattern", CASES)
def test_keyed_rule_equals_row_rule(split_lib, config, nm, ni, seed, pattern):
    fl = make_fleet(config, nm, ni, seed)
    if pattern is not None:
        fl = upgrade(fl, pattern, seed)
    s = solver_from_synth(fl, split_lib)
    answered = 0
    for k, sd in enumerate(_batches(fl, seed)):
        c = _rule_counts(split_lib, s, sd, fl.now_ms, seed + k)
        assert c[0] == len(sd.dec)
        assert c[3] == 0 and c[4] == 0 and c[1] == c[2], (config, pattern, k, c)
        answered += c[2]
    assert answered > 0
    s.close()


def test_keyed_rule_on_overflow_models_and_front_edges(split_lib):
    """Models with 0-8 instances among the first 64 ranks: overflow marks, and lowest ranks at and around every reach."""
    fl = make_fleet("C3", 3000, 1500, 21)
    order = oracle_from_synth(fl).cluster_order()
    rng = np.random.default_rng(21)
    nm = fl.n_models
    edges = [list(rng.choice(order[:64], size=rng.integers(0, 9), replace=False)) for _ in range(nm)]
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([int(x) for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    s = solver_from_synth(fl, split_lib)
    sd = make_decisions(fl, 3000, 21, sweep=True, plain=True)
    sd.dec["self"] = rng.choice(order[:80], size=len(sd.dec))
    answered = 0
    for k in range(2):
        c = _rule_counts(split_lib, s, sd, fl.now_ms, 21 + k)
        assert c[3] == 0 and c[4] == 0 and c[1] == c[2], c
        answered += c[2]
        sd.dec["flags"] |= DF_FAVOUR_SELF
    assert answered > 0
    s.close()
