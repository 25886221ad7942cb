"""One pod's eviction listener (onEviction MM:2867-2933) over a burst of evictions, restated from the Java text, with every
getNext answered by OracleFleet.get_next_batch: the reference mmp_evict_run is checked against (tests/test_evict_run_gpu.py;
its own check without a GPU: tests/test_evict_run_oracle.py).

For each eviction, in listener order (the task each one puts on taskPool, MM:2882-2932):
    a saturated record (rate_run_oracle.saturated): MMP_EV_UNDECIDED alone, the record's own values; the pod decides it
    attemptReload (MM:2886-2896), on the record before the write: !ce.isFailed() and the record holds the pod;
        loadedTime = instanceIds.get(pod), else loadFailedInstanceIds.get(pod); now - loadedTime > 2 * loadTimeoutMs
    deregisterModel(key, lastUsed, ce.loadTimestamp, ce.loadCompleteTimestamp) (MM:2936-2962):
        wasThere = instanceIds.remove(pod, loadTimestamp); failedWasThere = removeLoadFailure(pod, loadCompleteTimestamp)
        (MR:173-179); neither -> no write; else updateLastUsed(lastUsed) (MR:239-246: 0 means now) and, where wasThere,
        updateLastUnloadTime (MR:260-262: instanceIds.size() <= 2 ? 0 : now)
    the rebalance gate (MM:2918-2920) for a reload: typeSetStats(type) (OracleFleet.type_stats), totalCapacity > 0 &&
        instanceCount > 1 && 20 * totalFree / totalCapacity >= 1
    ensureLoadedElsewhere(key, lastUsed) (MM:6905-6907) on the record after the write, {pod} excluded:
        a loaded copy on another instance of clusterState -> forwarded to it, LOADED, no load (MM:3540-3760)
        checkLoadFailureCount (rate_run_oracle.refused over the failure records the write left) -> refused
        getNext(model, pod, lastUsed) excluding the model's registrations and the pod, favourSelf (the pod is in toExclude,
        MM:6940-6943)
The decision of entry r draws with id r.  A pod outside clusterState without its fresh row makes a malformed decision, which
the library answers MMP_TARGET_INVALID; the restatement gives that answer without asking the oracle."""
from types import SimpleNamespace

import numpy as np

from modelmesh_b200 import _lib as L
from oracle import binding as ob
from rate_run_oracle import jdiv, jlong, refused, saturated

REPORT_KEYS = ("n_unregister", "n_drop_failure", "n_reload", "n_cluster_full", "n_loaded_elsewhere", "n_refused", "n_placed")
BITS = (L.EV_UNREGISTER, L.EV_DROP_FAILURE, L.EV_RELOAD, L.EV_CLUSTER_FULL, L.EV_LOADED_ELSEWHERE, L.EV_REFUSED, L.EV_PLACED)


def gate_open(o: ob.OracleFleet, type_name: str) -> bool:
    """the cluster is less than 95 % full and has more than one instance (MM:2918-2920)"""
    s = o.type_stats(type_name)
    cap, free = int(s["total_capacity"]), int(s["total_free"])
    return cap > 0 and int(s["instance_count"]) > 1 and jdiv(jlong(20 * free), cap) >= 1


def evict_run(o: ob.OracleFleet, fl, ts, lul, pod: int, entries, params, seed: int, fresh_self=None):
    """(out (L.EVICT_ACTION per entry), report dict).  ts: the time of every registration of fl.edge_inst; lul: lastUnloadTime
    per model; entries: L.EVICT_ENTRY records; params: one L.EVICT_PARAMS record; fresh_self: the pod's INSTANCE_ROW or None."""
    p = params[0] if params.shape else params
    now, timeout, expiry = int(p["now"]), int(p["load_timeout_ms"]), int(p["load_failure_expiry_ms"])
    out = np.zeros(len(entries), dtype=L.EVICT_ACTION)
    out["model"] = entries["model"]
    out["target"] = L.TARGET_INVALID
    cluster = set(int(i) for i in o.cluster_order())
    tasks = []   # (r, model, lastUsed) of each getNext
    for r, ent in enumerate(entries):
        m = int(ent["model"])
        if saturated(fl, m):   # the pod decides it itself: no edit, the record's own values
            out["what"][r] = L.EV_UNDECIDED
            out["last_used"][r], out["last_unload_time"][r] = int(fl.model_last_used[m]), int(lul[m])
            continue
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        regs = [int(i) for i in fl.edge_inst[a:b]]
        loaded_at = next((j for j in range(k) if regs[j] == pod), None)
        failed_at = next((j for j in range(k, b - a) if regs[j] == pod), None)
        # attemptReload, on the record as the task read it
        reload = False
        if not int(ent["flags"]) & L.EV_ENTRY_FAILED:
            at = loaded_at if loaded_at is not None else failed_at
            reload = at is not None and jlong(now - int(ts[a + at])) > jlong(2 * timeout)
        # deregisterModel
        was_there = loaded_at is not None and int(ts[a + loaded_at]) == int(ent["load_ts"])
        failed_was_there = failed_at is not None and int(ts[a + failed_at]) == int(ent["load_complete_ts"])
        lu_rec, lul_rec = int(fl.model_last_used[m]), int(lul[m])
        what = (L.EV_UNREGISTER if was_there else 0) | (L.EV_DROP_FAILURE if failed_was_there else 0)
        if was_there or failed_was_there:
            lu = int(ent["last_used"]) or now
            lu_rec = max(lu_rec, lu)
            if was_there:
                lul_rec = 0 if k - 1 <= 2 else now
        out["last_used"][r], out["last_unload_time"][r] = lu_rec, lul_rec
        if reload:
            what |= L.EV_RELOAD
            gone = {j for j, hit in ((loaded_at, was_there), (failed_at, failed_was_there)) if hit}
            after = [j for j in range(b - a) if j not in gone]   # the record after the write
            k_after = sum(1 for j in after if j < k)
            if not gate_open(o, fl.type_names[int(fl.model_type[m])]):
                what |= L.EV_CLUSTER_FULL
            elif any(regs[j] != pod and regs[j] in cluster for j in after[:k_after]):
                what |= L.EV_LOADED_ELSEWHERE
            elif refused(SimpleNamespace(edge_off=np.array([0, len(after)]), n_loaded=np.array([k_after])),
                         np.array([ts[a + j] for j in after], dtype=np.int64), 0, now, expiry):
                what |= L.EV_REFUSED
            else:
                what |= L.EV_PLACED
                tasks.append((r, m, int(ent["last_used"])))
        out["what"][r] = what
    rep = {key: int(np.count_nonzero(out["what"] & bit)) for key, bit in zip(REPORT_KEYS, BITS)}
    rep["n_none"] = 0
    if not tasks:
        return out, rep
    if fresh_self is None and pod not in cluster:
        return out, rep
    fresh = None if fresh_self is None else np.asarray(fresh_self, dtype=ob.INST).reshape(1)
    od = np.zeros(len(tasks), dtype=ob.DECISION)
    lists = []
    for q, (r, m, lu) in enumerate(tasks):
        od["type_idx"][q], od["self"][q], od["last_used"][q] = fl.model_type[m], pod, lu
        od["fresh_idx"][q] = -1 if fresh is None else 0
        od["favour_self"][q], od["decision_id"][q] = 1, r
        lists.append(np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]], np.array([pod], dtype=np.int32)]))
    eoff = np.zeros(len(tasks) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in lists], out=eoff[1:])
    res = o.get_next_batch(od, fl.type_names, eoff, np.concatenate(lists).astype(np.int32), now, seed, fresh=fresh)
    for (r, m, lu), x in zip(tasks, res):
        out["target"][r], out["n_candidates"][r] = int(x["target"]), int(x["n_candidates"])
        rep["n_none"] += int(x["target"]) == L.TARGET_NONE
    return out, rep
