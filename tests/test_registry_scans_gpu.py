"""Registry-side batch scans against the oracle (SURVEY.md §8a row a14, §8f-2):
  mmp_scale_eval      = rateTrackingTask's loop body (MM:5684-5806, exclude set MM:5835-5856, loadedSince MM:5858-5870) and the
                        janitor's removeModelCopies (MM:6197-6335) for a batch of cache entries
  mmp_registry_prune  = pruneMissingInstances (MM:6752-6784) over the whole registry in one sweep
Parity unpinned by reference tests (testSecondCopyTrigger pins the second-copy arithmetic through the oracle's own golden
test); bit-exact against the literal restatements orc_rate_task_eval / orc_janitor_eval / orc_prune_missing."""
import ctypes as C

import numpy as np
import pytest

from common import vp
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet
from modelmesh_b200.synth import load_into_fleet, make_fleet
from oracle import binding as ob

pytestmark = pytest.mark.gpu


def _fleet_with_times(lib, config, nm, ni, seed, rng):
    fl = make_fleet(config, nm, ni, seed)
    # keep at most 4 registered instances per model (the inline list) and give every edge a load / failure time
    keep = np.minimum(fl.edge_off[1:] - fl.edge_off[:-1], 4)
    off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(keep, out=off[1:])
    inst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m] + keep[m]] for m in range(nm)]) if nm else np.zeros(0, np.int32)
    fl.n_loaded = np.minimum(fl.n_loaded, keep).astype(np.int32)
    fl.n_failed = (keep - fl.n_loaded).astype(np.int32)
    fl.edge_off, fl.edge_inst = off, inst.astype(np.int32)
    ts = (fl.now_ms - rng.integers(0, 4 * 3_600_000, size=len(inst))).astype(np.int64)
    ts = np.where(rng.uniform(size=len(inst)) < 0.3, fl.now_ms - rng.integers(0, 120_000, size=len(inst)), ts).astype(np.int64)
    lul = np.where(rng.uniform(size=nm) < 0.3, fl.now_ms - rng.integers(0, 200_000, size=nm), 0).astype(np.int64)
    s = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, ni, nm, lib=lib)
    load_into_fleet(fl, s)
    for m in range(nm):
        e = ts[off[m]:off[m + 1]]
        s._ck(lib.mmp_model_times(s.h, m, np.ascontiguousarray(e).ctypes.data_as(C.c_void_p), len(e), int(lul[m])))
    s.commit()
    return fl, s, ts, lul


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 4000, 300, 2), ("C3", 4000, 500, 3), ("C5", 3000, 400, 5), ("MIX", 1500, 160, 14)])
def test_scale_eval_matches_oracle(product_lib, oracle_lib, config, nm, ni, seed):
    lib = product_lib
    rng = np.random.default_rng(seed)
    fl, s, ts, lul = _fleet_with_times(lib, config, nm, ni, seed, rng)
    o = oracle_from_synth(fl)
    n = 6000
    rec = np.zeros(n, dtype=L.SCALE_IN)
    models = rng.integers(0, nm, size=n)
    rec["model"] = models
    # the entry belongs to a pod that holds the model when it has copies, to any pod otherwise
    for r in range(n):
        m = int(models[r])
        k = int(fl.n_loaded[m])
        rec["instance"][r] = int(fl.edge_inst[fl.edge_off[m] + rng.integers(0, k)]) if k and rng.uniform() < 0.9 else int(rng.integers(0, ni))
    rec["count"] = np.where(rng.uniform(size=n) < 0.5, rng.integers(0, 50, size=n), rng.integers(0, 20_000, size=n))
    rec["last_used"] = np.where(rng.uniform(size=n) < 0.05, 0, fl.now_ms - rng.integers(0, 40 * 3_600_000, size=n))
    rec["last_heavy"] = np.where(rng.uniform(size=n) < 0.4, 0, fl.now_ms - rng.integers(0, 30 * 3_600_000, size=n))
    rec["flags"] = (rng.uniform(size=n) < 0.15).astype(np.int32)  # MMP_SCALE_NO_LOCAL_STATS (quirk N13)
    it = 5000
    rec["i1"] = it - rng.integers(0, 400, size=n)
    rec["i2"] = np.minimum(it, rec["i1"] + rng.integers(0, 300, size=n))
    for thr, can_remove, lru_thr in ((2000, 1, 6 * 3_600_000), (300, 1, 1000), (5, 0, 6 * 3_600_000)):
        p = np.zeros(1, dtype=L.SCALE_PARAMS)
        p["now"], p["last_check_time"], p["iteration"], p["scale_up_rpm_threshold"] = fl.now_ms, fl.now_ms - 10_000, it, thr
        p["second_copy_min_age_iters"], p["second_copy_max_age_iters"], p["second_copy_lru_threshold_ms"] = 42, 240, lru_thr
        p["rate_check_interval_ms"], p["assume_completed_ms"], p["second_copy_remove_max_age_ms"], p["can_remove"] = 10_000, 30_000, 36_000_000, can_remove
        out = np.zeros(n, dtype=L.SCALE_OUT)
        s._ck(lib.mmp_scale_eval(s.h, rec.ctypes.data_as(C.c_void_p), n, p.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)))
        # oracle: per record the model's edges (loaded first) with their times
        m64 = models.astype(np.int64)
        deg = (fl.edge_off[m64 + 1] - fl.edge_off[m64]).astype(np.int64)
        eoff = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(deg, out=eoff[1:])
        einst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64]).astype(np.int32)
        ets = np.concatenate([ts[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64]).astype(np.int64)
        nl = fl.n_loaded[m64].astype(np.int32)
        tidx = fl.model_type[m64].astype(np.int32)
        orec = np.zeros(n, dtype=ob.SCALE_IN)
        for k in ("instance", "model", "count", "last_used", "last_heavy", "i1", "i2", "flags"):
            orec[k] = rec[k]
        op = np.zeros(1, dtype=ob.SCALE_PARAMS)
        for k in op.dtype.names:
            if k != "pad":
                op[k] = p[k]
        up = np.zeros(n, dtype=ob.SCALE_OUT)
        down = np.zeros(n, dtype=ob.SCALE_OUT)
        names = (C.c_char_p * len(fl.type_names))(*[t.encode() for t in fl.type_names])
        assert oracle_lib.orc_rate_task_eval(o.h, n, vp(orec), vp(op), names, len(fl.type_names), vp(tidx), vp(eoff), vp(einst), vp(ets), vp(nl), vp(up)) == 0
        lulr = lul[m64].astype(np.int64)
        assert oracle_lib.orc_janitor_eval(o.h, n, vp(orec), vp(op), vp(eoff), vp(einst), vp(ets), vp(nl), vp(lulr), vp(down)) == 0
        for k in ("action", "copies_to_load", "load_last_used", "rpm", "i1", "i2", "set_heavy"):
            bad = np.nonzero(out[k] != up[k])[0]
            assert len(bad) == 0, (thr, k, len(bad), bad[:5], out[bad[:5]], up[bad[:5]], rec[bad[:5]])
        bad = np.nonzero(out["remove"] != down["remove"])[0]
        assert len(bad) == 0, (thr, "remove", len(bad), bad[:5], rec[bad[:5]])
        if thr == 2000:
            seen = (int(np.count_nonzero(out["action"] == 1)), int(np.count_nonzero(out["action"] == 2)), int(out["remove"].sum()))
    assert seen[0] + seen[1] > 0, seen


def test_registry_prune_matches_oracle(product_lib, oracle_lib):
    lib = product_lib
    rng = np.random.default_rng(9)
    fl, s, ts, lul = _fleet_with_times(lib, "C3", 20_000, 600, 3, rng)
    o = oracle_from_synth(fl)
    # 40 instances leave the table; the prune pass runs three times, 6 minutes apart (ASSUME_INSTANCE_GONE_AFTER_MS = 10 min)
    gone = rng.choice(600, size=40, replace=False)
    for i in gone:
        s.instance_remove(int(i))
        o.instance_event(ob.DELETED, int(i), None, fl.inst_ids[int(i)], now_ms=fl.now_ms)
    s.commit()
    missing_p = np.zeros(600, dtype=np.int64)
    missing_o = np.zeros(600, dtype=np.int64)
    self_idx = int(np.setdiff1d(np.arange(600), gone)[0])
    total = 0
    for rnd, now in enumerate((fl.now_ms, fl.now_ms + 360_000, fl.now_ms + 720_000)):
        outm = np.zeros(20_000, dtype=np.int32)
        outk = np.zeros(20_000, dtype=np.uint8)
        n = s._ck(lib.mmp_registry_prune(s.h, self_idx, now, 600_000, missing_p.ctypes.data_as(C.c_void_p), outm.ctypes.data_as(C.c_void_p),
                                         outk.ctypes.data_as(C.c_void_p), len(outm)))
        want = {}
        pruned = np.zeros(8, dtype=np.uint8)
        for m in range(fl.n_models):
            a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
            if a == b:
                continue
            k = oracle_lib.orc_prune_missing(o.h, self_idx, fl.edge_inst[a:b].ctypes.data_as(C.c_void_p), ts[a:b].ctypes.data_as(C.c_void_p), b - a,
                                             now, 600_000, missing_o.ctypes.data_as(C.c_void_p), pruned.ctypes.data_as(C.c_void_p))
            if k:
                want[m] = sum(int(pruned[j]) << j for j in range(b - a))
        got = {int(outm[i]): int(outk[i]) for i in range(n)}
        assert got == want, (rnd, len(got), len(want))
        # first sightings are stamped with this pass's clock on both sides (the sweep is order-free: any pass stamps `now`)
        assert np.array_equal(missing_p != 0, missing_o != 0) and np.array_equal(missing_p, missing_o), rnd
        total += n
    assert total > 0
