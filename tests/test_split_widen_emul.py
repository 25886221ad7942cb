"""CPU checks of the widened fast-path rule of k_place_split (DESIGN.md §5.2.1): keys built as the commit builds them --
the lowest rank among every live edge of a model, inline and overflow, that is a member of its slot's cand -- and a self
that is not a candidate of its slot left out of the test.  tests/emul/split_widen.cpp answers each decision by the old
rule and by the widened one, and walks it as k_place_direct does: every widened answer must equal the walk, and every
decision the old rule answered must still be answered."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from modelmesh_b200 import _lib
from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import oracle_from_synth, oracle_inputs, solver_from_synth
from split_widen import GROUPS, front_cases
from upgrade import upgrade

HERE = os.path.dirname(os.path.abspath(__file__))
SLOT_SUMMARY = np.dtype([("best_rem", "<i8"), ("best_lru", "<i8"), ("best_idx", "<i4"), ("best_rpm", "<i4"), ("best_full", "<i4"),
                         ("reach", "<i4", (2,)), ("n_in", "<i4", (2,)), ("pad_", "<i4")])


@pytest.fixture(scope="module")
def widen_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("split_widen") / "libmmplace_emul_split_widen.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wl,-Bsymbolic", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "split_widen.cpp")])
    lib = _lib.load(so, require_all=False)
    lib.mmp_emul_split_widen.restype = C.c_int32
    lib.mmp_emul_split_widen.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                         C.c_void_p, C.c_int64, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.mmp_emul_slot_summaries.restype = C.c_int32
    lib.mmp_emul_slot_summaries.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_int32]
    lib.mmp_emul_model_slot.restype = C.c_int32
    lib.mmp_emul_model_slot.argtypes = [C.c_void_p, C.c_int32]
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _widen(lib, s, sd, now_ms, seed):
    dec = np.ascontiguousarray(sd.dec, dtype=_lib.DECISION_IN)
    fresh = np.ascontiguousarray(sd.fresh, dtype=_lib.INSTANCE_ROW) if len(sd.fresh) else None
    extra = np.ascontiguousarray(sd.extra, dtype=np.int32) if len(sd.extra) else None
    out = np.zeros(len(dec), dtype=_lib.DECISION_OUT)
    verdict = np.zeros(len(dec), dtype=np.int8)
    counts = np.zeros(5, dtype=np.int64)
    s._ck(lib.mmp_emul_split_widen(s.h, _ptr(dec), len(dec), _ptr(fresh), 0 if fresh is None else len(fresh), _ptr(extra),
                                   0 if extra is None else len(extra), _ptr(out), now_ms, seed, _ptr(verdict), _ptr(counts)))
    return out, verdict, counts


def _oracle_same(o, fl, sd, out, seed):
    od, off, idx = oracle_inputs(fl, sd)
    want = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)
    assert np.array_equal(out["target"], want["target"]) and np.array_equal(out["n_candidates"], want["n_candidates"])


def _batches(fl, seed):
    sweep = make_decisions(fl, 3000, seed, sweep=True, plain=True)
    fav = make_decisions(fl, 2000, seed + 3, sweep=True, plain=True)
    fav.dec["flags"] |= _lib.DF_FAVOUR_SELF
    return sweep, fav, make_decisions(fl, 2000, seed + 1)


CASES = [("C2", 2000, 400, 2, None), ("C3", 3000, 1300, 33, None), ("C5", 1500, 500, 5, None), ("MIX", 800, 300, 14, None),
         ("MIX", 800, 700, 41, None), ("C3", 3000, 1300, 33, "half"), ("MIX", 800, 300, 14, "saturated")]


@pytest.mark.parametrize("config,nm,ni,seed,pattern", CASES)
def test_widened_answers_equal_the_walk(widen_lib, oracle_lib, config, nm, ni, seed, pattern):
    fl = make_fleet(config, nm, ni, seed)
    if pattern is not None:
        fl = upgrade(fl, pattern, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, widen_lib)
    old = new = 0
    for k, sd in enumerate(_batches(fl, seed)):
        out, verdict, c = _widen(widen_lib, s, sd, fl.now_ms, seed + k)
        assert c[0] == len(sd.dec) and c[3] == 0 and c[4] == 0, (config, pattern, k, c)
        _oracle_same(o, fl, sd, out, seed + k)
        old += c[1]
        new += c[2]
    assert new >= old > 0
    s.close()


def test_widened_rule_on_overflow_models_at_the_front(widen_lib, oracle_lib):
    """Models with 0-8 instances among the first 64 ranks, selves among the first 80: overflow ids with and without a
    candidate below the reach, candidate and non-candidate exclusions and selves around every reach."""
    fl = make_fleet("C3", 3000, 1500, 21)
    o = oracle_from_synth(fl)
    order = o.cluster_order()
    rng = np.random.default_rng(21)
    nm = fl.n_models
    edges = [list(rng.choice(order[:64], size=rng.integers(0, 9), replace=False)) for _ in range(nm)]
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([int(x) for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, widen_lib)
    sd = make_decisions(fl, 3000, 21, sweep=True, plain=True)
    sd.dec["self"] = rng.choice(order[:80], size=len(sd.dec))
    gained = 0
    for k in range(2):
        out, verdict, c = _widen(widen_lib, s, sd, fl.now_ms, 21 + k)
        assert c[3] == 0 and c[4] == 0, c
        _oracle_same(o, fl, sd, out, 21 + k)
        gained += c[2] - c[1]
        sd.dec["flags"] |= _lib.DF_FAVOUR_SELF
    assert gained > 0
    s.close()


def test_hand_built_cases(widen_lib, oracle_lib):
    """Each group of split_widen.front_cases, checked where its construction lies where it means to against the reach of
    the decision's slot (both values of c_self): A, C, D, F and G answered by the widened rule (A, C and D walked by the
    old one), B and E walked."""
    fl, sd, group, rank, allowed = front_cases()
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, widen_lib)
    sums = np.zeros(256, dtype=SLOT_SUMMARY)
    members = np.zeros(256 * 2 * 256, dtype=np.int32)
    s._ck(widen_lib.mmp_emul_slot_summaries(s.h, fl.now_ms, _ptr(sums), _ptr(members), 256))
    out, verdict, c = _widen(widen_lib, s, sd, fl.now_ms, 5)
    assert c[3] == 0 and c[4] == 0, c
    _oracle_same(o, fl, sd, out, 5)
    seen = {g: 0 for g in GROUPS}
    for i, d in enumerate(sd.dec):
        m = int(d["model"])
        reach = sums[widen_lib.mmp_emul_model_slot(s.h, m)]["reach"]
        if reach.min() < 0:
            continue
        lo, hi = int(reach.min()), int(reach.max())
        e = fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]]
        er, sr = rank[e], int(rank[d["self"]])
        cand = allowed[e]
        g = GROUPS[group[i]]
        assert sr >= 0
        if g == "A":
            ok, want_new, want_old = sr < lo and not allowed[d["self"]], True, False
        elif g == "B":
            ok, want_new, want_old = sr < lo, False, False
        elif g == "C":
            ok, want_new, want_old = er[0] < lo and not cand[0] and sr >= hi, True, False
        elif g == "D":
            ok, want_new, want_old = (er[~cand] < lo).all() and (er[cand] >= hi).all() and sr >= hi, True, False
        elif g == "E":
            ok, want_new, want_old = 0 <= er[4] < lo and cand[4], False, False
        else:  # F, G: the edge that is not live has no rank
            ok = (er[er >= 0] >= hi).all() and (er < 0).any() and sr >= hi
            want_new, want_old = True, g == "F"
        if not ok:
            continue
        seen[g] += 1
        assert bool(verdict[i] & 2) == want_new, (g, i, int(verdict[i]), lo, hi, sr, list(er))
        assert bool(verdict[i] & 1) == want_old, (g, i, int(verdict[i]), lo, hi, sr, list(er))
    assert all(v > 0 for v in seen.values()), seen
    s.close()
