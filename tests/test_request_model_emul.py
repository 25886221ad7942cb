"""CPU checks of request-model decisions (MMP_DF_REQUEST_MODEL): the model's type id in `model`, its loaded ∪ failed
instances among the decision's extras, no registry state of the snapshot read.

tests/emul/request_model.cpp resolves a batch the way each kernel family reads a decision's exclusion row (tile routine
with traces and candidate masks; the lane routine over a window copied from the row; k_place_direct's window rebuilt from
the model's excluded ranks), all through the helpers the kernels use (excl_row_id / excl_row and prepare_ctx_a).
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from modelmesh_b200 import _lib
from modelmesh_b200.fleet import Fleet
from modelmesh_b200.sharding import combine_shard_keys, decode_shard_keys
from modelmesh_b200.synth import SynthDecisions, load_into_fleet, make_decisions, make_fleet

from helpers import oracle_from_synth, oracle_inputs
from request_model import as_request_model, hold_front, oracle_request, random_records

HERE = os.path.dirname(os.path.abspath(__file__))
FLEETS = [("C3", 2000, 1300, 33), ("C5", 1500, 500, 5), ("MIX", 500, 300, 14), ("MIX", 500, 700, 41)]
# (shape, lane window, lane budget): 0 tile routine, 1 lane routine on the row's window, 2 k_place_direct's ranks window
SHAPES = [(0, 12, 192), (1, 12, 192), (1, 5, 64), (1, 1, 2), (2, 12, 192), (2, 5, 64), (2, 1, 2)]


@pytest.fixture(scope="module")
def rm_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("request_model") / "libmmplace_emul_rm.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wl,-Bsymbolic", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "request_model.cpp")])
    lib = _lib.load(so, require_all=False)
    lib.mmp_emul_place_request.restype = C.c_int32
    lib.mmp_emul_place_request.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                           C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_uint64]
    lib.mmp_emul_set_keys.argtypes = [C.c_void_p, C.c_void_p]
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def place(lib, s, sd, now_ms, seed, shape, window=12, budget=192, trace=False, masks=False):
    dec = np.ascontiguousarray(sd.dec, dtype=_lib.DECISION_IN)
    fresh = np.ascontiguousarray(sd.fresh, dtype=_lib.INSTANCE_ROW) if len(sd.fresh) else None
    extra = np.ascontiguousarray(sd.extra, dtype=np.int32) if len(sd.extra) else None
    out = np.zeros(len(dec), dtype=_lib.DECISION_OUT)
    tr = np.zeros(len(dec), dtype=_lib.DECISION_TRACE) if trace else None
    cm = np.zeros((len(dec), 2, s.row_words()), dtype=np.uint32) if masks else None
    s._ck(lib.mmp_emul_place_request(s.h, _ptr(dec), len(dec), _ptr(fresh), 0 if fresh is None else len(fresh), _ptr(extra),
                                     0 if extra is None else len(extra), shape, window, budget, _ptr(out), _ptr(tr), _ptr(cm),
                                     now_ms, seed))
    return out, tr, cm


def _fleet(lib, fl, **kw):
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib, **kw)
    return s, load_into_fleet(fl, s)


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_committed_record_in_the_decision_equals_the_registry_row(rm_lib, oracle_lib, config, nm, ni, seed):
    """For every committed model, the decision that carries its record (type, ids ∪ the decision's extras) equals the one
    that reads it from the registry: results on every shape, trace and both candidate-mask planes on the tile routine."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    fl = hold_front(fl, o.cluster_order())
    s, tid = _fleet(rm_lib, fl)
    sd = make_decisions(fl, fl.n_models, seed, sweep=True)  # one decision per model, with fresh rows and extra excludes
    rq, flagged = as_request_model(fl, sd, tid)
    assert flagged.mean() > 0.95
    if config == "MIX":
        assert (np.diff(fl.edge_off) > 4).any()  # overflow models are among them
    od, off, idx = oracle_inputs(fl, sd)
    want = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh)
    for shape, window, budget in SHAPES:
        a, _, _ = place(rm_lib, s, sd, fl.now_ms, seed, shape, window, budget)
        b, _, _ = place(rm_lib, s, rq, fl.now_ms, seed, shape, window, budget)
        assert np.array_equal(a["target"], want["target"]) and np.array_equal(a["n_candidates"], want["n_candidates"])
        assert np.array_equal(a, b), (shape, window, budget, np.nonzero(a != b)[0][:5])
    a, ta, ma = place(rm_lib, s, sd, fl.now_ms, seed, 0, trace=True, masks=True)
    b, tb, mb = place(rm_lib, s, rq, fl.now_ms, seed, 0, trace=True, masks=True)
    assert np.array_equal(a, b) and np.array_equal(ta, tb) and np.array_equal(ma, mb)
    # without masks the unflagged decisions may take the one-window fast path (trace flag 256, internal): same fields
    a, ta, _ = place(rm_lib, s, sd, fl.now_ms, seed, 0, trace=True)
    b, tb, _ = place(rm_lib, s, rq, fl.now_ms, seed, 0, trace=True)
    assert np.array_equal(a, b)
    for k in ("best", "n_remaining", "pick_index", "cut_rank", "best_rank"):
        assert np.array_equal(ta[k], tb[k]), k
    assert np.array_equal(ta["flags"] & 255, tb["flags"] & 255)


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_request_records_equal_the_oracle(rm_lib, oracle_lib, config, nm, ni, seed):
    """Records the snapshot has never seen: types interned after the commit, other instance sets (non-live instances and
    self among them), 0 / 4 / 5 / 16 ids, favourSelf -- every shape equals the oracle on the same record."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    fl = hold_front(fl, o.cluster_order())
    s, tid = _fleet(rm_lib, fl)
    new = [f"late-type-{k}" for k in range(2)]
    names = list(fl.type_names) + new
    ids = [tid[t] for t in fl.type_names] + [s.type_id(t) for t in new]  # interned now: past the snapshot's type table
    assert min(ids[-2:]) > max(tid.values())
    sd = make_decisions(fl, 2000, seed + 7)
    rq, k = random_records(fl, sd, ids, seed)
    assert set(np.unique(rq.dec["extra_n"])) == {0, 4, 5, 16}
    assert ((rq.dec["flags"] & _lib.DF_FAVOUR_SELF) != 0).any() and (k >= len(fl.type_names)).any()
    want = oracle_request(o, names, k, rq, fl.now_ms, seed)
    for shape, window, budget in SHAPES:
        got, _, _ = place(rm_lib, s, rq, fl.now_ms, seed, shape, window, budget)
        assert np.array_equal(got["target"], want["target"]), (shape, window, budget)
        assert np.array_equal(got["n_candidates"], want["n_candidates"]), (shape, window, budget)
    got, tr, _ = place(rm_lib, s, rq, fl.now_ms, seed, 0, trace=True, masks=True)
    has = want["n_candidates"] > 0
    assert np.array_equal(tr["best"], want["best"])
    assert np.array_equal(tr["pick_index"][has], want["pick_index"][has])


def test_malformed_request_model_decisions(rm_lib):
    fl = make_fleet("C3", 300, 200, 3)
    s, tid = _fleet(rm_lib, fl)
    base = make_decisions(fl, 1, 3, plain=True).dec[0].copy()
    base["flags"] = _lib.DF_REQUEST_MODEL
    base["model"] = tid[fl.type_names[0]]
    extra = np.arange(17, dtype=np.int32)
    cases = []
    for model, flags, n_x, off_x in [(-1, 0, 0, 0), (65535, 0, 0, 0), (1 << 20, 0, 0, 0),  # type id outside [0, 65535)
                                     (None, _lib.DF_MODEL_LAST_USED, 0, 0),                   # no model row to take it from
                                     (None, 0, 17, 0), (None, 0, 4, 14)]:                     # more than 16 / slice past the table
        d = base.copy()
        if model is not None:
            d["model"] = model
        d["flags"] |= flags
        d["extra_n"], d["extra_off"] = n_x, off_x
        cases.append(d)
    good = base.copy()
    good["model"], good["extra_n"] = 65534, 16  # an unknown type id and a full extra[]: well formed
    dec = np.asarray(cases + [good], dtype=_lib.DECISION_IN)
    for shape in (0, 1, 2):
        out, _, _ = place(rm_lib, s, SynthDecisions(dec, np.zeros(0, dtype=_lib.INSTANCE_ROW), extra), fl.now_ms, 1, shape)
        assert (out["target"][:-1] == _lib.TARGET_INVALID).all(), shape
        assert out["target"][-1] != _lib.TARGET_INVALID


@pytest.mark.parametrize("config,nm,ni,seed,world", [("C3", 1500, 4000, 3, 2), ("MIX", 500, 700, 8, 3)])
def test_instance_sharded_fleets_refuse_request_model_decisions(rm_lib, config, nm, ni, seed, world):
    """Every shard answers a request-model decision MMP_TARGET_INVALID (no zero row: rows are column blocks there); the
    unflagged decisions of the same batch are combined as usual."""
    fl = make_fleet(config, nm, ni, seed)
    ref, tid = _fleet(rm_lib, fl)
    sd = make_decisions(fl, 600, seed)
    rq, flagged = as_request_model(fl, sd, tid)
    mixed = rq.dec.copy()
    mixed[::2] = sd.dec[::2]  # even positions unflagged (their extra slices index the same table as before: re-point them)
    extra = np.concatenate([rq.extra, sd.extra]).astype(np.int32)
    mixed["extra_off"][::2] = sd.dec["extra_off"][::2] + len(rq.extra)
    batch = SynthDecisions(mixed, sd.fresh, extra)
    is_req = (mixed["flags"] & _lib.DF_REQUEST_MODEL) != 0
    assert is_req.sum() > 200
    keys = []
    for r in range(world):
        f, _ = _fleet(rm_lib, fl, shard_rank=r, shard_count=world)
        k = np.zeros(len(mixed), dtype=np.uint64)
        rm_lib.mmp_emul_set_keys(f.h, k.ctypes.data_as(C.c_void_p))
        out, _, _ = place(rm_lib, f, batch, fl.now_ms, 77, 0)
        rm_lib.mmp_emul_set_keys(f.h, None)
        assert (out["target"][is_req] == _lib.TARGET_INVALID).all()
        assert (out["target"][~is_req] != _lib.TARGET_INVALID).all()
        keys.append(k)
        f.close()
    target, ncand, is_open = decode_shard_keys(combine_shard_keys(np.stack(keys)))
    assert (target[is_req] == _lib.TARGET_INVALID).all() and not is_open[is_req].any()
    want, _, _ = place(rm_lib, ref, SynthDecisions(sd.dec, sd.fresh, sd.extra), fl.now_ms, 77, 0)
    closed = ~is_req & ~is_open
    assert np.array_equal(target[closed], want["target"][closed])
