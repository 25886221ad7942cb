"""CPU checks of call-wide exclude sets (mmp_place_batch_excluding): every decision of a call avoids the same instances,
however many.  tests/emul/exclude_set.cpp derives the call's slot tables on the host (the set's ranks cleared from
cand / candx / pref, the word lists rebuilt by HostState::slot_word_lists) and resolves the batch in the three shapes of
tests/emul/request_model.cpp; the oracle reads each decision's exclusion list extended by the set."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from modelmesh_b200 import _lib
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import SynthDecisions, load_into_fleet, make_decisions, make_fleet

from exclude_set import named_sets, oracle_excluding, rs_retry_type
from helpers import oracle_from_synth
from request_model import as_request_model

HERE = os.path.dirname(os.path.abspath(__file__))
FLEETS = [("C3", 2000, 1300, 33), ("C5", 1500, 500, 5), ("MIX", 500, 300, 14), ("MIX", 500, 700, 41)]
# (shape, lane window, lane budget): 0 tile routine, 1 lane routine on the row's window, 2 k_place_direct's ranks window
SHAPES = [(0, 12, 192), (1, 12, 192), (1, 5, 64), (1, 1, 2), (2, 12, 192), (2, 5, 64), (2, 1, 2)]


@pytest.fixture(scope="module")
def xs_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("exclude_set") / "libmmplace_emul_xs.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wl,-Bsymbolic", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "exclude_set.cpp")])
    lib = _lib.load(so, require_all=False)
    lib.mmp_emul_place_excluding.restype = C.c_int32
    lib.mmp_emul_place_excluding.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                             C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_int64, C.c_uint64]
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def place(lib, s, sd, xs, now_ms, seed, shape, window=12, budget=192, trace=False, masks=False, n_xs=None):
    dec = np.ascontiguousarray(sd.dec, dtype=_lib.DECISION_IN)
    fresh = np.ascontiguousarray(sd.fresh, dtype=_lib.INSTANCE_ROW) if len(sd.fresh) else None
    extra = np.ascontiguousarray(sd.extra, dtype=np.int32) if len(sd.extra) else None
    xs = None if xs is None else np.ascontiguousarray(xs, dtype=np.int32)
    out = np.zeros(len(dec), dtype=_lib.DECISION_OUT)
    tr = np.zeros(len(dec), dtype=_lib.DECISION_TRACE) if trace else None
    cm = np.zeros((len(dec), 2, s.row_words()), dtype=np.uint32) if masks else None
    s._ck(lib.mmp_emul_place_excluding(s.h, _ptr(dec), len(dec), _ptr(fresh), 0 if fresh is None else len(fresh), _ptr(extra),
                                       0 if extra is None else len(extra), _ptr(xs), len(xs) if n_xs is None else n_xs, shape,
                                       window, budget, _ptr(out), _ptr(tr), _ptr(cm), now_ms, seed))
    return out, tr, cm


def _fleet(lib, fl, **kw):
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib, **kw)
    return s, load_into_fleet(fl, s)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def _all_shapes(lib, s, sd, xs, want, fl, seed, what):
    for shape, window, budget in SHAPES:
        got, _, _ = place(lib, s, sd, xs, fl.now_ms, seed, shape, window, budget)
        _same(got, want, what + (shape, window, budget))
    got, tr, _ = place(lib, s, sd, xs, fl.now_ms, seed, 0, trace=True, masks=True)
    _same(got, want, what + ("traced",))
    has = want["n_candidates"] > 0
    assert np.array_equal(tr["best"], want["best"]), what
    assert np.array_equal(tr["n_remaining"][has], want["n_remaining"][has]), what
    assert np.array_equal(tr["pick_index"][has], want["pick_index"][has]), what
    assert np.array_equal(tr["flags"] & 15, want["flags"] & 15), what
    return tr


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_sets_of_every_size_equal_the_oracle(xs_lib, oracle_lib, config, nm, ni, seed):
    """Sets of 1 / 17 / 200 / 2 000 ids, every candidate of one type, every instance, and the batch's selves with their
    unconstrained answers: every shape equals the oracle with each decision's exclusions extended by the set."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s, _ = _fleet(xs_lib, fl)
    sd = make_decisions(fl, 600, seed)
    first, _, _ = place(xs_lib, s, sd, None, fl.now_ms, seed, 0, n_xs=0)
    for name, xs in named_sets(s, fl, sd, first, seed):
        _all_shapes(xs_lib, s, sd, xs, oracle_excluding(o, fl, sd, xs, seed), fl, seed, (config, name))
    # an empty set is the plain call
    plain = s.place_batch(sd.dec, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
    assert np.array_equal(first, plain)
    s.close()


def test_set_of_unflagged_candidates_forces_the_replicaset_retry(xs_lib, oracle_lib):
    """A set holding every candidate of a type outside the likely-replaced replicaset: the filter drops to nothing and is
    retried without the replicaset rule (MM:4798-4802, MMP_TF_RS_RETRY), and the answers lie inside that replicaset."""
    fl = make_fleet("C3", 2000, 1300, 33)
    assert fl.replaced_replicasets
    o = oracle_from_synth(fl)
    s, _ = _fleet(xs_lib, fl)
    t, free, flagged = rs_retry_type(s, fl)
    sd = make_decisions(fl, 6000, 34)
    keep = fl.model_type[sd.dec["model"]] == fl.type_names.index(t)
    sd = SynthDecisions(sd.dec[keep], sd.fresh, sd.extra)
    assert len(sd.dec) >= 50
    want = oracle_excluding(o, fl, sd, free, 5)
    tr = _all_shapes(xs_lib, s, sd, free, want, fl, 5, ("rs", t))
    tgt = want["target"]
    assert np.isin(tgt[tgt >= 0], flagged).all() and (tgt >= 0).any()
    assert ((tr["flags"] & _lib.TF_RS_RETRY) != 0).mean() > 0.5
    s.close()


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_request_model_decisions_under_a_set(xs_lib, oracle_lib, config, nm, ni, seed):
    """MMP_DF_REQUEST_MODEL decisions (the model's record in the decision's extras) keep their meaning under a set."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s, tid = _fleet(xs_lib, fl)
    sd = make_decisions(fl, 600, seed + 1)
    rq, flagged = as_request_model(fl, sd, tid)
    rq = SynthDecisions(rq.dec[flagged], rq.fresh, rq.extra)
    type_idx = fl.model_type[sd.dec["model"][flagged]]
    first, _, _ = place(xs_lib, s, rq, None, fl.now_ms, seed, 0, n_xs=0)
    for name, xs in named_sets(s, fl, sd, first, seed)[1::2]:  # 17, 2 000, every instance
        want = oracle_excluding(o, fl, rq, xs, seed, names=fl.type_names, type_idx=type_idx)
        for shape, window, budget in SHAPES:
            got, _, _ = place(xs_lib, s, rq, xs, fl.now_ms, seed, shape, window, budget)
            _same(got, want, (config, name, shape, window, budget))
    s.close()


def test_malformed_sets_fail_the_call_and_write_nothing(xs_lib):
    fl = make_fleet("C3", 300, 200, 3)
    s, _ = _fleet(xs_lib, fl)
    sd = make_decisions(fl, 40, 3)
    for xs, n_xs in ((np.asarray([3, 200], dtype=np.int32), None), (np.asarray([-1], dtype=np.int32), None), (None, 2)):
        with pytest.raises(MmpError) as e:
            place(xs_lib, s, sd, xs, fl.now_ms, 1, 0, n_xs=n_xs)
        assert e.value.code == _lib.E_ARG
    # duplicates and not-live ids are fine: same answers as the de-duplicated live part
    live = np.asarray(s.cluster_order()[:10], dtype=np.int32)
    a, _, _ = place(xs_lib, s, sd, np.concatenate([live, live, live[:3]]), fl.now_ms, 1, 0)
    b, _, _ = place(xs_lib, s, sd, live, fl.now_ms, 1, 0)
    assert np.array_equal(a, b)
    s.close()
    sh, _ = _fleet(xs_lib, make_fleet("C3", 300, 400, 3), shard_rank=0, shard_count=2)
    with pytest.raises(MmpError) as e:
        place(xs_lib, sh, sd, np.asarray([1], dtype=np.int32), fl.now_ms, 1, 0)
    assert e.value.code == _lib.E_STATE
    sh.close()
