"""One pod's pre-shutdown migration (preShutdown MM:6959-7147, its distribution loop MM:6990-7047) restated from the Java text,
with every getNext answered by OracleFleet.get_next_batch: the reference mmp_shutdown_run is checked against
(tests/test_shutdown_run_gpu.py; its own check without a GPU: tests/test_shutdown_run_oracle.py).

    foundOther   clusterState holds an instance other than the pod (MM:6968-6976); without one no entry is evaluated
    for each entry of descendingLruMap(), most recently used first (MM:7005):
      a saturated record (rate_run_oracle.saturated)             ->  MMP_SD_UNDECIDED alone: the pod decides it itself
      mr == null || !mr.getInstanceIds().containsKey(instanceId)  ->  skipped (MM:7007-7010)
      lruT < cutoff                                               ->  willBeSkipped++ (MM:7011-7014)
      the task (MM:7016-7045):
        ce == null || ce.isFailed()                               ->  nothing more
        lruTime = lruT != 0 ? lruT : getLastUsedTime(model)
        lruTime >= 0                                              ->  ce.remove()
        ce.isAborted()                                            ->  deregisterModelAsync now
        lruTime > 0                                               ->  triggerNewModelCopyElsewhere(model, mr, lruTime): one
            getNext excluding the record's registrations and the pod (favourSelf: the pod is in toExclude, MM:6940-6943),
            refused by checkLoadFailureCount (rate_run_oracle.refused: 3 or more failures younger than expiry / 2);
            Status.LOADING && lruTime >= cutoff                  ->  return ent (the pod waits for it)
The decision of entry r draws with id r."""
import numpy as np

from modelmesh_b200 import _lib as L
from oracle import binding as ob
from rate_run_oracle import jlong, refused, saturated


def shutdown_run(o: ob.OracleFleet, fl, ts, pod: int, entries, params, seed: int, fresh_self=None):
    """(out (L.SHUTDOWN_ACTION per entry), report dict).  ts: the time of every registration of fl.edge_inst; entries:
    L.SHUTDOWN_ENTRY records; params: one L.SHUTDOWN_PARAMS record; fresh_self: the pod's INSTANCE_ROW or None."""
    p = params[0] if params.shape else params
    now, expiry = int(p["now"]), int(p["load_failure_expiry_ms"])
    out = np.zeros(len(entries), dtype=L.SHUTDOWN_ACTION)
    out["model"] = entries["model"]
    out["target"] = L.TARGET_INVALID
    rep = dict(found_other=0, n_registered=0, will_be_skipped=0, n_placed=0, n_none=0, n_refused=0, n_wait=0)
    cluster = [int(i) for i in o.cluster_order()]
    found_other = any(i != pod for i in cluster)
    rep["found_other"] = int(found_other)
    if not found_other:
        return out, rep
    # (a pod outside clusterState places through its fresh row: without one its decisions are malformed, which the oracle
    # does not model)
    assert fresh_self is not None or pod in cluster
    cutoff = jlong(now - int(p["cutoff_age_ms"]))
    tasks = []   # (r, model, lruTime) of each triggerNewModelCopyElsewhere
    for r, ent in enumerate(entries):
        m = int(ent["model"])
        if saturated(fl, m):
            out["what"][r] = L.SD_UNDECIDED
            continue
        a, k = int(fl.edge_off[m]), int(fl.n_loaded[m])
        if pod not in set(int(i) for i in fl.edge_inst[a:a + k]):
            out["what"][r] = L.SD_NOT_REGISTERED
            continue
        rep["n_registered"] += 1
        what = 0
        lru_t = int(ent["lru_t"])
        if lru_t < cutoff:
            what |= L.SD_STALE
            rep["will_be_skipped"] += 1
        flags = int(ent["flags"])
        if not flags & (L.SD_ENTRY_GONE | L.SD_ENTRY_FAILED):
            lru_time = lru_t if lru_t != 0 else int(ent["last_used"])
            out["last_used"][r] = lru_time
            if lru_time >= 0:
                what |= L.SD_REMOVE_LOCAL
            if flags & L.SD_ENTRY_ABORTED:
                what |= L.SD_DEREGISTER_NOW
            if lru_time > 0:
                if refused(fl, ts, m, now, expiry):
                    what |= L.SD_REFUSED
                    rep["n_refused"] += 1
                else:
                    what |= L.SD_PLACED
                    tasks.append((r, m, lru_time))
        out["what"][r] = what
    if not tasks:
        return out, rep
    fresh = None if fresh_self is None else np.asarray(fresh_self, dtype=ob.INST).reshape(1)
    od = np.zeros(len(tasks), dtype=ob.DECISION)
    lists = []
    for q, (r, m, lru_time) in enumerate(tasks):
        od["type_idx"][q], od["self"][q], od["last_used"][q] = fl.model_type[m], pod, lru_time
        od["fresh_idx"][q] = -1 if fresh is None else 0
        od["favour_self"][q], od["decision_id"][q] = 1, r
        lists.append(np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]], np.array([pod], dtype=np.int32)]))
    eoff = np.zeros(len(tasks) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in lists], out=eoff[1:])
    res = o.get_next_batch(od, fl.type_names, eoff, np.concatenate(lists).astype(np.int32), now, seed, fresh=fresh)
    for (r, m, lru_time), x in zip(tasks, res):
        t = int(x["target"])
        out["target"][r], out["n_candidates"][r] = t, int(x["n_candidates"])
        rep["n_placed"] += 1
        if t == L.TARGET_NONE:
            rep["n_none"] += 1
        elif t >= 0 and lru_time >= cutoff:
            out["what"][r] |= L.SD_WAIT
            rep["n_wait"] += 1
    return out, rep
