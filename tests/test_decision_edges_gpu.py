"""Every placement route of the H100 library at the decision arithmetic's edges (tests/decision_edges.py), exactly against
the oracle: the traced tile kernel with masks (full ordered shortlists and survivors) and without (the window fast path),
the mapped tiny-batch path, and on batches large enough for launch_place: k_place_direct with and without the slot
sort, the two-pass path forced on and off, k_place_lanes, and the two-pass path at its default threshold through
mmp_place_batch_device; the four one-decision launch paths (k_place_server with an inline fresh record included), the
micro-batcher, request-model copies of the decisions, and a call-wide exclude set that removes each fleet's first entry."""
import ctypes as C

import numpy as np
import pytest

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthDecisions

from decision_edges import all_cases, check_built
from exclude_set import oracle_excluding
from helpers import compare_decisions, oracle_from_synth, oracle_inputs_fast, solver_from_synth
from request_model import as_request_model

pytestmark = pytest.mark.gpu

CASES = all_cases()
SEED = 5


def _kw(sd):
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


def _oracle(c, o, sd, seed, ids=None):
    od, off, idx = oracle_inputs_fast(c.fl, sd)
    if ids is not None:
        od["decision_id"] = ids
    return o.get_next_batch(od, c.fl.type_names, off, idx, c.fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def _tiled(sd, n):
    return SynthDecisions(np.resize(sd.dec, n), sd.fresh, sd.extra)


@pytest.fixture(scope="module")
def built(product_lib, oracle_lib):
    out = {}
    for c in CASES:
        o = oracle_from_synth(c.fl)
        s = solver_from_synth(c.fl, product_lib)
        out[c.id] = (o, s)
    yield out
    for _, s in out.values():
        s.close()


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_batch_routes(built, product_lib, case):
    """traced with and without masks and untraced (helpers.compare_decisions; a batch this small is placed untraced from
    the mapped buffer by k_place_server or k_place_small), and request-model copies of the same decisions"""
    o, s = built[case.id]
    assert np.array_equal(s.cluster_order(), case.order)
    ores, out, tr = compare_decisions(case.fl, case.sd, o, s, seed=SEED)
    check_built(case, o, ores)
    if case.family in ("full-best", "pref-b"):
        assert (tr["flags"] & L.TF_BEST_FULL).any()
    if case.family == "pref-b":
        assert (tr["flags"] & L.TF_PREF_B).any()
    tid = {t: s.type_id(t) for t in case.fl.type_names}
    rq, flagged = as_request_model(case.fl, case.sd, tid)
    assert flagged.all()
    _same(s.place_batch(rq.dec, case.fl.now_ms, SEED, **_kw(rq)), out, "request model")


def _launched(s, place):
    """place() and the number of kernel launches it took"""
    k0 = s.kernel_launches()
    got = place()
    return got, s.kernel_launches() - k0


def _device_place(s, lib, dec, now_ms, seed):
    """mmp_place_batch_device: the records in device memory, placed as one batch (no chunks, no mapped buffer)"""
    d_in, d_out = C.c_void_p(), C.c_void_p()
    s._ck(lib.mmp_device_alloc(s.h, dec.nbytes, C.byref(d_in)))
    s._ck(lib.mmp_device_alloc(s.h, len(dec) * L.DECISION_OUT.itemsize, C.byref(d_out)))
    try:
        s._ck(lib.mmp_device_upload(s.h, d_in, dec.ctypes.data_as(C.c_void_p), dec.nbytes))
        ms = C.c_float()
        s._ck(lib.mmp_place_batch_device(s.h, d_in, len(dec), d_out, now_ms, seed, C.byref(ms)))
        got = np.zeros(len(dec), dtype=L.DECISION_OUT)
        s._ck(lib.mmp_device_download(s.h, got.ctypes.data_as(C.c_void_p), d_out, got.nbytes))
    finally:
        s._ck(lib.mmp_device_free(s.h, d_in))
        s._ck(lib.mmp_device_free(s.h, d_out))
    return got


MAPPED_BYTES = 16384  # the mapped buffer of tiny untraced batches (PlaceCtx::MAPPED_BYTES)
CHUNK = 1 << 17       # host batches above this are placed in chunks of it


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_large_batches_each_kernel(built, product_lib, case):
    """the edge decisions repeated to 8 269 decisions, a batch that leaves the mapped buffer and is placed by launch_place
    in one piece: k_place_direct with sort_slots 0 and 1, the two-pass path forced on and off (byte for byte), and
    k_place_lanes (mmp_tune direct = 0); then the plain decisions from device memory"""
    o, s = built[case.id]
    lib = product_lib
    sd = _tiled(case.sd, 8192 + 77)
    n = len(sd.dec)
    assert n * (L.DECISION_IN.itemsize + L.DECISION_OUT.itemsize) + 64 > MAPPED_BYTES and n <= CHUNK
    want = _oracle(case, o, sd, SEED)
    got, launches = {}, {}
    try:
        for sort in (0, 1):
            s._ck(lib.mmp_tune(s.h, b"sort_slots", sort))
            for split in (1, 0):
                s._ck(lib.mmp_tune(s.h, b"split", split))
                got[f"k_place_direct sort_slots={sort} split={split}"], launches[sort, split] = \
                    _launched(s, lambda: s.place_batch(sd.dec, case.fl.now_ms, SEED, **_kw(sd)))
        s._ck(lib.mmp_tune(s.h, b"sort_slots", 2))
        s._ck(lib.mmp_tune(s.h, b"split", 0))
        s._ck(lib.mmp_tune(s.h, b"direct", 0))
        got["k_place_lanes"] = s.place_batch(sd.dec, case.fl.now_ms, SEED, **_kw(sd))
    finally:
        s._ck(lib.mmp_tune(s.h, b"direct", 1))
        s._ck(lib.mmp_tune(s.h, b"sort_slots", 2))
        s._ck(lib.mmp_tune(s.h, b"split", 2))
    wrong = {k: int(np.count_nonzero((g["target"] != want["target"]) | (g["n_candidates"] != want["n_candidates"]))) for k, g in got.items()}
    assert not any(wrong.values()), "; ".join(f"{k}: {v} wrong" for k, v in wrong.items())  # every route, by name
    assert launches[0, 1] > launches[0, 0] >= 1, launches  # k_place_direct; the two-pass path launches more kernels
    plain = np.ascontiguousarray(case.sd.dec[case.sd.dec["fresh"] < 0])
    if len(plain):
        _same(_device_place(s, lib, plain, case.fl.now_ms, SEED),
              _oracle(case, o, SynthDecisions(plain, case.sd.fresh, case.sd.extra), SEED), "device batch")


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_single_decisions_and_exclude_set(built, product_lib, case):
    """each decision alone through one_mode 0 .. 3 (decision id 0; k_place_server reads the caller's fresh record inline),
    the micro-batcher, and the whole batch under an exclude set that holds the fleet's first entry"""
    o, s = built[case.id]
    lib = product_lib
    sd = case.sd
    n = min(len(sd.dec), 200)
    idx = np.linspace(0, len(sd.dec) - 1, n).astype(np.int64)
    want = _oracle(case, o, SynthDecisions(sd.dec[idx], sd.fresh, sd.extra), SEED, ids=np.zeros(n, dtype=np.uint64))
    out = np.zeros(1, dtype=L.DECISION_OUT)
    try:
        for mode in (0, 1, 2, 3):
            s._ck(lib.mmp_tune(s.h, b"one_mode", mode))
            got, one = np.zeros(n, dtype=L.DECISION_OUT), np.zeros(n, dtype=L.DECISION_OUT)
            for j, i in enumerate(idx):
                d = sd.dec[i:i + 1].copy()  # (a copy: its fresh index is rewritten below)
                f1 = None
                if d["fresh"][0] >= 0:  # its own fresh record, at index 0
                    f1 = np.ascontiguousarray(sd.fresh[d["fresh"][0]:d["fresh"][0] + 1])
                    d["fresh"] = 0
                got[j] = s.place_batch(d, case.fl.now_ms, SEED, fresh=f1)[0]
                if mode:
                    s._ck(lib.mmp_place_one(s.h, d.ctypes.data_as(C.c_void_p), None if f1 is None else f1.ctypes.data_as(C.c_void_p),
                                            None, out.ctypes.data_as(C.c_void_p), case.fl.now_ms, SEED))
                    one[j] = out[0]
            _same(got, want, ("one_mode", mode))
            if mode:
                _same(one, want, ("mmp_place_one", mode))
    finally:
        s._ck(lib.mmp_tune(s.h, b"one_mode", 3))
    bt = C.c_void_p()
    s._ck(lib.mmp_batcher_create(s.h, 64, 50, 99, C.byref(bt)))
    try:
        fresh = np.ascontiguousarray(sd.fresh if len(sd.fresh) else np.zeros(1, dtype=L.INSTANCE_ROW), dtype=L.INSTANCE_ROW)
        extra = np.zeros(1, dtype=np.int32)
        did = C.c_uint32()
        got = np.zeros(n, dtype=L.DECISION_OUT)
        dids = np.zeros(n, dtype=np.uint64)
        for j, i in enumerate(idx):
            d = np.ascontiguousarray(sd.dec[i:i + 1])
            s._ck(lib.mmp_place_submit(bt, d.ctypes.data_as(C.c_void_p), fresh.ctypes.data_as(C.c_void_p),
                                       extra.ctypes.data_as(C.c_void_p), case.fl.now_ms, out.ctypes.data_as(C.c_void_p), C.byref(did)))
            got[j], dids[j] = out[0], did.value
    finally:
        lib.mmp_batcher_destroy(bt)
    _same(got, _oracle(case, o, SynthDecisions(sd.dec[idx], sd.fresh, sd.extra), 99, ids=dids), "batcher")
    first = np.asarray(case.order[:1], dtype=np.int32)
    _same(s.place_batch(sd.dec, case.fl.now_ms, SEED, exclude=first, **_kw(sd)), oracle_excluding(o, case.fl, sd, first, SEED),
          "exclude the first entry")


# fleets with at least 24 candidates in a decision's window: on sparser snapshots the default keeps k_place_direct
@pytest.mark.parametrize("cid", ["count-cut:violator-rank-33", "count-cut:violator-rank-1025", "full-best:long-max", "full-best:a10-450000"])
def test_default_threshold_batch(built, product_lib, cid):
    """2^18 + 33 plain decisions of an edge fleet from device memory (one batch: mmp_place_batch_device does not chunk),
    the size at which the two-pass path is the default: the default takes it (as many launches as forcing it on) and
    equals the path forced on and off, byte for byte, and the oracle"""
    lib = product_lib
    case = next(c for c in CASES if c.id == cid)
    o, s = built[cid]
    plain = case.sd.dec[case.sd.dec["fresh"] < 0]
    assert len(plain)
    dec = np.ascontiguousarray(np.resize(plain, (1 << 18) + 33))
    got, launches = {}, {}
    try:
        for split in (2, 1, 0):
            s._ck(lib.mmp_tune(s.h, b"split", split))
            got[split], launches[split] = _launched(s, lambda: _device_place(s, lib, dec, case.fl.now_ms, SEED))
    finally:
        s._ck(lib.mmp_tune(s.h, b"split", 2))
    assert launches[2] == launches[1] > launches[0], launches
    assert got[2].tobytes() == got[1].tobytes() == got[0].tobytes()
    _same(got[2], _oracle(case, o, SynthDecisions(dec, case.sd.fresh, case.sd.extra), SEED), cid)
