"""One pod's rate-tracking task (rateTrackingTask MM:5619-5858) composed from the oracle's entry points, the reference
mmp_rate_run is checked against (tests/test_rate_run_gpu.py; its own check without a GPU: tests/test_rate_run_oracle.py):
  gates     timeDelta * 5 < RATE_CHECK_INTERVAL_MS * 3 (too soon), clusterStats.instanceCount < 2, no entries (MM:5646-5670)
  evaluate  orc_rate_task_eval per entry: rpm, set_heavy, i1 / i2, action, copies_to_load and the loads' lastUsed
  refuse    checkLoadFailureCount (MM:4607-4627): a model with 3 or more failure records younger than half of
            LOAD_FAILURE_EXPIRY_MS gets no load
  heavy     orc_scaleup_exclude_set: getExcludeSet (MM:5835-5856) for ourRpm = the pod's published rpm (0 outside the table)
  place     OracleFleet.get_next_batch round by round.  A second copy is getNext(model, pod, lastCheckTime) excluding the
            model's registrations and the pod, favourSelf set.  Decision j of a scale-up chain excludes the registrations, the
            heavy set and the chain's targets 0..j-1, with self = the pod (j = 0, or a target that was the pod) or target j-1,
            favourSelf set for j > 0 and for j = 0 when the pod is a loaded registration.  The pod's fresh row goes with every
            decision whose self is the pod.  Decision j of the chain of entry r draws with id off[r] + j, off the exclusive
            prefix sum of each entry's decisions (1 per second copy, min(copies, 17) per chain)."""
import ctypes as C

import numpy as np

from modelmesh_b200 import _lib as L
from oracle import binding as ob

vp = lambda a: a.ctypes.data_as(C.c_void_p)
FAILURE_LIMIT = 3   # checkLoadFailureCount's MAX_LOAD_FAILURES


def jlong(x: int) -> int:
    return ((int(x) + (1 << 63)) % (1 << 64)) - (1 << 63)


def jdiv(a: int, b: int) -> int:
    """Java long a / b (truncates toward zero)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def saturated(fl, m: int) -> bool:
    """the committed record's copy count (min(255, loaded)) is saturated over more than 255 registrations: where its loaded
    copies end is unknown, and the library decides nothing for the model (mmp_scale_eval's -1, MMP_*_UNDECIDED)"""
    return min(int(fl.n_loaded[m]), 255) == 255 and int(fl.edge_off[m + 1] - fl.edge_off[m]) > 255


def too_soon(scale) -> bool:
    delta = jlong(int(scale["now"]) - int(scale["last_check_time"]))
    return jlong(delta * 5) < jlong(int(scale["rate_check_interval_ms"]) * 3)


def evaluate(o: ob.OracleFleet, fl, ts, entries, scale):
    """orc_rate_task_eval per entry (can_remove has no part in it) as L.SCALE_OUT records; a saturated record's entry is
    action -1 with i1 / i2 kept and nothing else, as mmp_scale_eval answers it"""
    n = len(entries)
    m64 = entries["model"].astype(np.int64)
    deg = (fl.edge_off[m64 + 1] - fl.edge_off[m64]).astype(np.int64)
    eoff = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=eoff[1:])
    einst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64] + [np.zeros(0)]).astype(np.int32)
    ets = np.concatenate([ts[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64] + [np.zeros(0)]).astype(np.int64)
    nl = fl.n_loaded[m64].astype(np.int32)
    tidx = fl.model_type[m64].astype(np.int32)
    orec = np.zeros(n, dtype=ob.SCALE_IN)
    for k in ("instance", "model", "count", "last_used", "last_heavy", "i1", "i2", "flags"):
        orec[k] = entries[k]
    op = np.zeros(1, dtype=ob.SCALE_PARAMS)
    for k in op.dtype.names:
        if k != "pad":
            op[k] = scale[k]
    op["can_remove"] = 0
    up = np.zeros(n, dtype=ob.SCALE_OUT)
    names = (C.c_char_p * max(1, len(fl.type_names)))(*[t.encode() for t in fl.type_names])
    assert ob.lib().orc_rate_task_eval(o.h, n, vp(orec), vp(op), names, len(fl.type_names), vp(tidx), vp(eoff), vp(einst), vp(ets),
                                       vp(nl), vp(up)) == 0
    out = np.zeros(n, dtype=L.SCALE_OUT)
    for k in L.SCALE_OUT.names:
        out[k] = up[k]
    for r in range(n):
        if saturated(fl, int(m64[r])):
            out[r] = (-1, 0, 0, 0, entries["i1"][r], entries["i2"][r], 0, 0)
    return out


def refused(fl, ts, m: int, now: int, expiry: int) -> bool:
    """checkLoadFailureCount: FAILURE_LIMIT or more failure records with a time after now - expiry / 2"""
    a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
    since = jlong(now - jdiv(expiry, 2))
    return sum(1 for t in ts[a + k:b] if int(t) > since) >= FAILURE_LIMIT


def heavy_set(o: ob.OracleFleet, fl, pod: int, thr: int):
    """getExcludeSet: the instance indices, ascending"""
    live = set(int(i) for i in o.cluster_order())
    our = int(fl.inst_rows["rpm"][pod]) if pod in live else 0
    marks = np.zeros(fl.n_instances, dtype=np.uint8)
    n = ob.lib().orc_scaleup_exclude_set(o.h, pod, thr, our, vp(marks), fl.n_instances)
    xs = np.nonzero(marks)[0].astype(np.int32)
    assert n == len(xs)
    return xs


def empty_out(entries):
    out = np.zeros(len(entries), dtype=L.SCALE_OUT)
    out["i1"], out["i2"] = entries["i1"], entries["i2"]
    return out


def rate_run(o: ob.OracleFleet, fl, ts, pod: int, entries, params, seed: int, fresh_self=None):
    """(out (L.SCALE_OUT per entry), loads [(entry, model, chain_pos, self, target, n_candidates, last_used, flags,
    remaining)] in (entry, chain_pos) order, report dict).  ts: the time of every registration of fl.edge_inst; entries:
    L.SCALE_IN records of the pod; params: one L.RATE_PARAMS record; fresh_self: the pod's INSTANCE_ROW or None."""
    p = params[0] if params.shape else params
    scale = p["scale"]
    now, thr, expiry = int(scale["now"]), int(scale["scale_up_rpm_threshold"]), int(p["load_failure_expiry_ms"])
    rep = dict(gate=L.RATE_RAN, n_second=0, n_scale_up=0, n_loads=0, n_heavy=0, n_chains_cut=0, n_refused_failures=0)
    if too_soon(scale):
        rep["gate"] = L.RATE_TOO_SOON
    elif int(o.cluster_stats()["instance_count"]) < 2:
        rep["gate"] = L.RATE_FEW_INSTANCES
    elif len(entries) == 0:
        rep["gate"] = L.RATE_NO_ENTRIES
    if rep["gate"] != L.RATE_RAN:
        return empty_out(entries), [], rep
    # (a pod outside the table places through its fresh row: without one its decisions are malformed, which the oracle does
    # not model)
    assert fresh_self is not None or pod in set(int(i) for i in o.cluster_order())
    out = evaluate(o, fl, ts, entries, scale)
    heavy = heavy_set(o, fl, pod, thr)
    rep["n_heavy"] = len(heavy)
    fresh = None if fresh_self is None else np.asarray(fresh_self, dtype=ob.INST).reshape(1)
    # one plan per entry that loads: its chain (a second copy is a chain of one) and the loads it placed
    plans, off = [], 0
    for r, (e, x) in enumerate(zip(entries, out)):
        act, m = int(x["action"]), int(e["model"])
        if act not in (1, 2):
            continue
        rep["n_second" if act == 1 else "n_scale_up"] += 1
        if refused(fl, ts, m, now, expiry):
            rep["n_refused_failures"] += 1
            continue
        a, k = int(fl.edge_off[m]), int(fl.n_loaded[m])
        copies = 1 if act == 1 else int(x["copies_to_load"])
        favour0 = act == 1 or pod in [int(i) for i in fl.edge_inst[a:a + k]]
        plans.append(dict(entry=r, model=m, copies=copies, id0=off, favour=favour0, second=act == 1, self=pod, targets=[],
                          last_used=int(x["load_last_used"]), loads=[]))
        off += min(copies, L.RATE_CHAIN_MAX)
    active = list(plans)
    j = 0
    while active:
        od = np.zeros(len(active), dtype=ob.DECISION)
        lists = []
        for q, c in enumerate(active):
            m = c["model"]
            od["type_idx"][q], od["self"][q], od["last_used"][q] = fl.model_type[m], c["self"], c["last_used"]
            od["fresh_idx"][q] = 0 if (c["self"] == pod and fresh is not None) else -1
            od["favour_self"][q] = 1 if (j > 0 or c["favour"]) else 0
            od["decision_id"][q] = c["id0"] + j
            own = fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]]
            more = [pod] if c["second"] else list(heavy) + c["targets"]
            lists.append(np.concatenate([own, np.asarray(more, dtype=np.int32)]))
        eoff = np.zeros(len(active) + 1, dtype=np.int64)
        np.cumsum([len(x) for x in lists], out=eoff[1:])
        res = o.get_next_batch(od, fl.type_names, eoff, np.concatenate(lists).astype(np.int32), now, seed, fresh=fresh)
        nxt = []
        for c, d, x in zip(active, od, res):
            t = int(x["target"])
            c["loads"].append([c["entry"], c["model"], j, int(d["self"]), t, int(x["n_candidates"]), c["last_used"],
                               L.RL_SECOND_COPY if c["second"] else 0, 0])
            if c["second"] or t in (L.TARGET_NONE, L.TARGET_INVALID) or j + 1 >= c["copies"]:
                continue
            if j + 1 >= L.RATE_CHAIN_MAX:   # decision j + 1 would need more than MAX_EXTRA extras: the chain is cut
                c["loads"][-1][7] |= L.RL_CHAIN_CUT
                c["loads"][-1][8] = c["copies"] - L.RATE_CHAIN_MAX
                rep["n_chains_cut"] += 1
                continue
            nt = pod if t == L.TARGET_SELF else t
            c["targets"].append(nt)
            c["self"] = nt
            nxt.append(c)
        active = nxt
        j += 1
    loads = [tuple(ld) for c in plans for ld in c["loads"]]
    rep["n_loads"] = len(loads)
    return out, loads, rep
