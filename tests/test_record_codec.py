"""KV-record codecs (mmp_instance_upsert_json / mmp_model_upsert_json): a fleet ingested from the registry's jackson JSON
(InstanceRecord IR:37-69, ModelRecord MR:61-114) is the fleet ingested through the struct API -- same PLACEMENT_ORDER,
same type sets, same decisions.  Host logic only: runs on the CPU harness (it compiles the product's host_state.hpp)."""
import json

import numpy as np
import pytest

from modelmesh_b200 import _lib as L
from modelmesh_b200._lib import MODEL_ROW
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import LONG_MAX, load_into_fleet, make_decisions, make_fleet


def instance_json(fl, i, extra=None):
    r = fl.inst_rows[i]
    d = {"lruTime": int(r["lru_time"]), "count": int(r["count"]), "cap": int(r["capacity"]), "used": int(r["used"]),
         "lThreads": int(r["l_threads"]), "lInProg": int(r["l_in_prog"]), "rpm": int(r["rpm"]), "shutdown": bool(r["shutting_down"]),
         "startTime": int(r["start_time"]), "vers": int(r["vers"]), "loc": fl.inst_locs[i], "zone": fl.inst_zones[i],
         "labels": list(fl.inst_labels[i])}
    if extra:
        d.update(extra)
    return json.dumps(d)


def model_json(fl, m, tname):
    a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
    ids = [fl.inst_ids[int(x)] for x in fl.edge_inst[a:b]]
    nl = int(fl.n_loaded[m])
    loaded = {iid: 1700000000000 + k for k, iid in enumerate(ids[:nl])}
    failed = {iid: 1700000001000 + k for k, iid in enumerate(ids[nl:])}
    return json.dumps({"type": tname, "encKey": None, "mPath": "s3://bucket/m%d" % m, "instanceIds": loaded, "failedIn": failed,
                       "fails": {}, "refs": 0, "autoDel": False, "lu": int(fl.model_last_used[m]), "lul": 0})


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 600, 300, 3), ("MIX", 400, 97, 21), ("C5", 500, 200, 5)])
def test_fleet_from_json_records_equals_struct_ingest(emul_lib, config, nm, ni, seed):
    lib = emul_lib
    fl = make_fleet(config, nm, ni, seed)
    a = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    load_into_fleet(fl, a)
    b = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
    b.types_set_json(fl.type_json())
    b.replicasets_set(fl.replaced_replicasets)
    for i in range(fl.n_instances):
        extra = {"futureField": {"x": [1, 2, {"y": "z"}]}, "kvVersion": 7} if i % 3 == 0 else None  # unknown properties are ignored
        b._ck(lib.mmp_instance_upsert_json(b.h, i, fl.inst_ids[i].encode(), instance_json(fl, i, extra).encode(), int(fl.inst_rows[i]["active"])))
    for m in range(fl.n_models):
        b._ck(lib.mmp_model_upsert_json(b.h, m, model_json(fl, m, fl.type_names[int(fl.model_type[m])]).encode(), int(fl.model_size[m])))
    b.commit()
    assert np.array_equal(a.cluster_order(), b.cluster_order())
    for t in fl.type_names:  # type ids are interned in encounter order (opaque); the sets behind them must agree
        sa, sb = a.type_sets(a.type_id(t), fl.n_instances), b.type_sets(b.type_id(t), fl.n_instances)
        for x, y in zip(sa, sb):
            assert (x is None) == (y is None) and (x is None or np.array_equal(x, y))
    sd = make_decisions(fl, 1500, seed)
    kw = dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
    ra = a.place_batch(sd.dec, fl.now_ms, 5, **kw)
    rb = b.place_batch(sd.dec, fl.now_ms, 5, **kw)
    assert np.array_equal(ra, rb)


def test_record_defaults_and_errors(emul_lib):
    lib = emul_lib
    f = Fleet(2560, 600000, 2560, 8, 8, lib=lib)
    # jackson-constructor defaults (IR:76-78): everything absent -> zeros, null loc/zone, no labels
    f._ck(lib.mmp_instance_upsert_json(f.h, 0, b"pod-a", b"{}", 1))
    f._ck(lib.mmp_instance_upsert_json(f.h, 1, b"pod-b", json.dumps({"lruTime": LONG_MAX, "cap": 25600, "used": 100, "lThreads": 8,
                                                                     "labels": None, "loc": None, "zone": "zé中"}).encode(), 1))
    f._ck(lib.mmp_instance_upsert_json(f.h, 2, b"pod-c", b' { "cap" : 25600 , "used":25600, "shutdown" : true } ', 1))
    f._ck(lib.mmp_model_upsert_json(f.h, 0, json.dumps({"type": "t1", "instanceIds": {"pod-b": 5, "pod-zzz": 6}, "lu": 123}).encode(), 256))
    f._ck(lib.mmp_model_upsert_json(f.h, 1, b'{"type":null}', 256))
    f.commit()
    # pod-c is shutting down: treated as deleted (MM:1462-1464); pod-a has no capacity at all: full, ranks after pod-b
    assert list(f.cluster_order()) == [1, 0]
    for bad in (b"", b"[]", b'{"cap": 1.5}', b'{"cap": }', b'{"labels": [1]}', b'{"lruTime": 99999999999999999999}', b'{"cap":1} x'):
        with pytest.raises(MmpError):
            f._ck(lib.mmp_instance_upsert_json(f.h, 3, b"pod-d", bad, 1))
    for bad in (b'{"instanceIds": []}', b'{"lu": "x"}', b"{"):
        with pytest.raises(MmpError):
            f._ck(lib.mmp_model_upsert_json(f.h, 2, bad, 1))
    # values outside the supported domain are refused like the struct API refuses them
    with pytest.raises(MmpError):
        f._ck(lib.mmp_instance_upsert_json(f.h, 3, b"pod-d", b'{"rpm": 600000000}', 1))


def test_json_readers_survive_garbage(emul_lib):
    """The three JSON readers of the host code (type constraints, instance record, model record) take bytes that come from
    a KV store: any input must end in MMP_OK or MMP_E_ARG, never in a crash or a hang (mutations of valid documents,
    truncations, random bytes; NUL-free because the ABI takes C strings)."""
    import random
    lib = emul_lib
    f = Fleet(2560, 600000, 2560, 8, 8, lib=lib)
    f._ck(lib.mmp_instance_upsert_json(f.h, 0, b"pod-a", b'{"cap": 25600}', 1))
    valid = [
        b'{"lruTime":9223372036854775807,"count":3,"cap":131072,"used":5,"lThreads":8,"lInProg":0,"rpm":12,"shutdown":false,'
        b'"startTime":1700000000000,"vers":7,"loc":null,"zone":"z\\u00e9\\ud83d\\ude00","labels":["b","a"]}',
        b'{"type":"t1","encKey":null,"mPath":"p","instanceIds":{"pod-a":5,"x":6},"failedIn":{"pod-a":9},"fails":{"pod-a":{"msg":"m"}},"refs":0,"autoDel":false,"lu":12,"lul":0}',
        b'{"t1":{"required":["l1","l2"],"preferred":["l3"]},"_default":{"preferred":[]},"t2":{}}',
    ]
    rng = random.Random(7)
    def mutate(b):
        b = bytearray(b)
        for _ in range(rng.randint(1, 4)):
            k = rng.randint(0, 3)
            if k == 0 and b:
                del b[rng.randrange(len(b))]
            elif k == 1:
                b.insert(rng.randrange(len(b) + 1), rng.choice(b'{}[]",:\\u0123456789-.eEtfn '))
            elif k == 2 and b:
                b[rng.randrange(len(b))] = rng.randrange(1, 256)
            else:
                b = b[:rng.randrange(len(b) + 1)]
        return bytes(x for x in b if x != 0)
    calls = 0
    for it in range(4000):
        src = valid[it % 3] if it % 5 else bytes(rng.randrange(1, 256) for _ in range(rng.randint(0, 40)))
        doc = mutate(src)
        for rc in (lib.mmp_instance_upsert_json(f.h, 1, b"pod-b", doc, 1), lib.mmp_model_upsert_json(f.h, 1, doc, 10),
                   lib.mmp_types_set_json(f.h, doc)):
            assert rc in (0, -1), (rc, doc)
            calls += 1
    assert calls == 12000
    f._ck(lib.mmp_types_set_json(f.h, valid[2]))
    f.commit()  # the host state is still consistent


def _two_pod_fleet(lib):
    f = Fleet(2560, 600000, 2560, 8, 8, lib=lib)
    rec = json.dumps({"lruTime": LONG_MAX, "cap": 25600, "used": 100, "lThreads": 8}).encode()
    return f, rec


def _place(f, model, self_idx=0):
    d = np.zeros(1, dtype=L.DECISION_IN)
    d["model"], d["self"], d["fresh"], d["last_used"] = model, self_idx, -1, 1
    return f.place_batch(d, 1_760_000_000_000, 1)[0]


def test_model_record_may_arrive_before_its_instances(emul_lib):
    """ADVICE r1: the two KV listeners deliver in any order (INTEGRATION.md §6).  A model record that names an instance
    not yet in the table keeps the id and the exclusion edge appears at the first commit after the instance registers;
    an instance that re-registers under another index keeps its edges (membership is by id, MM:4735-4743)."""
    lib = emul_lib
    f = Fleet(2560, 600000, 2560, 8, 8, lib=lib)
    rec = lambda used, cap=25600: json.dumps({"lruTime": LONG_MAX, "cap": cap, "used": used, "lThreads": 8}).encode()
    # the caller (pod-c, index 2) is full and not in the service-instance list: never a candidate, and its fresh record
    # makes every non-self candidate fail the walk test (N2), so the answer is always the first filtered entry
    f._ck(lib.mmp_instance_upsert_json(f.h, 2, b"pod-c", rec(25600), 0))
    f._ck(lib.mmp_model_upsert_json(f.h, 0, json.dumps({"type": "t", "instanceIds": {"pod-b": 5}, "lu": 9}).encode(), 256))
    f._ck(lib.mmp_model_upsert_json(f.h, 1, json.dumps({"type": "t", "lu": 9}).encode(), 256))
    f._ck(lib.mmp_instance_upsert_json(f.h, 0, b"pod-a", rec(20000), 1))
    f.commit()
    assert _place(f, 0, 2)["target"] == 0  # only pod-a can take it
    f._ck(lib.mmp_instance_upsert_json(f.h, 1, b"pod-b", rec(0, 51200), 1))
    f.commit()
    assert list(f.cluster_order())[:2] == [1, 0]
    assert _place(f, 1, 2)["target"] == 1  # pod-b wins on free space ...
    assert _place(f, 0, 2)["target"] == 0  # ... unless the model is already loaded there: the edge named by id is now resolved
    # pod-b re-registers under index 5
    f.instance_remove(1)
    f._ck(lib.mmp_instance_upsert_json(f.h, 5, b"pod-b", rec(0, 51200), 1))
    f.commit()
    assert _place(f, 1, 2)["target"] == 5
    assert _place(f, 0, 2)["target"] == 0
    # an index-based upsert replaces the record held by id
    row = np.zeros(1, dtype=L.MODEL_ROW)
    f.model_upsert(0, row[0], [])
    f.commit()
    assert _place(f, 0, 2)["target"] == 5


def test_absent_type_is_nlclassifier(emul_lib):
    """ADVICE r1: a ModelRecord without "type" is DEFAULT_TYPE "NLCLASSIFIER" (MR:117-130), not an unconstrained type."""
    lib = emul_lib
    f = Fleet(2560, 600000, 2560, 8, 8, lib=lib)
    f.types_set_json(json.dumps({"NLCLASSIFIER": {"required": ["gpu"]}}))
    base = {"lruTime": LONG_MAX, "cap": 25600, "used": 0, "lThreads": 8}
    f._ck(lib.mmp_instance_upsert_json(f.h, 0, b"pod-a", json.dumps(base).encode(), 1))
    f._ck(lib.mmp_instance_upsert_json(f.h, 1, b"pod-b", json.dumps(dict(base, labels=["gpu"], used=20000)).encode(), 1))
    f._ck(lib.mmp_model_upsert_json(f.h, 0, b'{"lu": 5}', 256))
    f._ck(lib.mmp_model_upsert_json(f.h, 1, b'{"type": "other", "lu": 5}', 256))
    f.commit()
    assert _place(f, 0)["target"] == 1             # legacy record: only the labelled pod is allowed
    assert _place(f, 1)["target"] == L.TARGET_SELF  # unconstrained type: the empty caller pod-a (pod-b is too full to be shortlisted)


def test_extra_slice_out_of_bounds_is_invalid(emul_lib):
    """ADVICE r1: a decision whose extra[] slice does not lie inside the table passed with the call is answered
    MMP_TARGET_INVALID; the table is never read out of bounds."""
    lib = emul_lib
    f, rec = _two_pod_fleet(lib)
    for i, name in enumerate((b"pod-a", b"pod-b", b"pod-c")):
        f._ck(lib.mmp_instance_upsert_json(f.h, i, name, rec, 1))
    f._ck(lib.mmp_model_upsert_json(f.h, 0, b'{"lu": 5}', 256))
    f.commit()
    d = np.zeros(6, dtype=L.DECISION_IN)
    d["model"], d["self"], d["fresh"], d["last_used"] = 0, 0, -1, 1
    d["extra_off"] = [0, 1, 2, -1, 0, 1 << 30]
    d["extra_n"] = [2, 1, 1, 1, 17, 1]
    extra = np.asarray([1, 2], dtype=np.int32)
    out = f.place_batch(d, 1_760_000_000_000, 1, extra=extra)
    assert list(out["target"] == L.TARGET_INVALID) == [False, False, True, True, True, True]
    assert out["target"][0] == L.TARGET_SELF  # both other pods excluded
    d["extra_n"][:] = 1
    d["extra_off"][:] = 0
    assert np.all(f.place_batch(d, 1_760_000_000_000, 1)["target"] == L.TARGET_INVALID)  # no table at all
