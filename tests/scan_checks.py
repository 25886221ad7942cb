"""Checks of the batch scans shared by the scan tests: the partition-id map between the oracle and the product, the oracle
with every subset's LRU converged, mmp_scale_eval with its parameter record, and orc_rate_task_eval / orc_janitor_eval /
orc_prune_missing over every registration of a model."""
import ctypes as C

import numpy as np

from common import GONE_MS, HOUR, vp
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from oracle import binding as ob


def partition_maps(fl, o, s):
    """partition id correspondence through instance membership (numbering differs between the two)."""
    m = {}
    for i in range(fl.n_instances):
        po, ps = o.instance_partition(i), s.instance_partition(i)
        if fl.inst_rows["shutting_down"][i]:
            continue
        assert (po < 0) == (ps < 0)
        if po >= 0:
            assert m.setdefault(ps, po) == po
    return m


def converged_oracle(fl):
    """The oracle with every subset's LRU recomputed over the final fleet (N10): bulk_add above 3 000 instances, else the
    ADDED events and then one UPDATED event per instance (as test_stats_match_oracle)."""
    o = oracle_from_synth(fl)
    if fl.n_instances <= 3000:
        for i in range(fl.n_instances):
            if not fl.inst_rows["shutting_down"][i]:
                r = fl.inst_rows[i].copy()
                r["l_in_prog"] += 1
                o.instance_event(ob.UPDATED, i, r, fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i], fl.now_ms)
                o.instance_event(ob.UPDATED, i, fl.inst_rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i],
                                 fl.inst_labels[i], fl.now_ms)
    return o


def scale_params(now, thr, can_remove, lru_thr):
    p = np.zeros(1, dtype=L.SCALE_PARAMS)
    p["now"], p["last_check_time"], p["iteration"], p["scale_up_rpm_threshold"] = now, now - 10_000, 5000, thr
    p["second_copy_min_age_iters"], p["second_copy_max_age_iters"], p["second_copy_lru_threshold_ms"] = 42, 240, lru_thr
    p["rate_check_interval_ms"], p["assume_completed_ms"], p["second_copy_remove_max_age_ms"], p["can_remove"] = 10_000, 30_000, 36 * HOUR, can_remove
    return p


def scale_eval(lib, s, rec, p):
    out = np.zeros(len(rec), dtype=L.SCALE_OUT)
    s._ck(lib.mmp_scale_eval(s.h, vp(rec), len(rec), vp(p), vp(out)))
    return out


def oracle_scale(oracle_lib, o, fl, ts, lul, rec, p):
    """orc_rate_task_eval / orc_janitor_eval with each record's model as CSR edge lists: every registration, loaded first."""
    n = len(rec)
    m64 = rec["model"].astype(np.int64)
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
    return up, down


def oracle_prune(oracle_lib, o, fl, ts, self_idx, now, missing, first=None):
    """orc_prune_missing over every model (or its first `first` registrations): (model, instance) pairs and per-model masks."""
    pairs, masks = [], {}
    pruned = np.zeros(max(1, int(np.diff(fl.edge_off).max())), dtype=np.uint8)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        if first is not None:
            b = min(b, a + first)
        if a == b:
            continue
        k = oracle_lib.orc_prune_missing(o.h, self_idx, vp(fl.edge_inst[a:b]), vp(ts[a:b]), b - a, now, GONE_MS, vp(missing), vp(pruned))
        if k:
            pairs += [(m, int(fl.edge_inst[a + j])) for j in range(b - a) if pruned[j]]
            masks[m] = sum(int(pruned[j]) << j for j in range(b - a))
    return pairs, masks
