"""The leader's reaper task (MM:6436-6494) composed from the oracle's entry points, the reference mmp_reaper_run is checked
against (tests/test_reaper_run_gpu.py; its own check without a GPU: tests/test_reaper_run_oracle.py):
  prune     orc_prune_missing per model over its loaded, then its failed registrations, one `missings` map (MM:6752-6784)
  repair    a lastUsed of Long.MAX_VALUE becomes now - 3 x LASTUSED_AGE_ON_ADD_MS (repairLastUsedTimeIfNeeded, MM:6837-6850)
  select    orc_reaper_select per partition in getPartitionStats order with one taken array, over the pruned and repaired
            records; a size estimate of 0 (the oracle's -4, the reference's ArithmeticException) ends the run
  place     OracleFleet.get_next_batch of the selected models: self = leader, lastUsed = the (repaired) value, exclusions =
            the surviving loaded and failed registrations, decision id = emission position
  cleanup   the `missings` map after the loop (MM:6601-6607)."""
import ctypes as C
from dataclasses import dataclass

import numpy as np

from oracle import binding as ob

HOUR = 3_600_000
REPAIR_AGE_MS = 3 * HOUR   # LASTUSED_AGE_ON_ADD_MS x 3
LONG_MAX = np.iinfo(np.int64).max
vp = lambda a: a.ctypes.data_as(C.c_void_p)


@dataclass
class Pruned:
    pairs: list            # (model, instance) in (model, registration position) order
    keep: np.ndarray       # bool per registration of fl.edge_inst: survives the prune
    n_loaded: np.ndarray   # per model after the prune
    n_failed: np.ndarray


def prune(o: ob.OracleFleet, fl, ts: np.ndarray, leader: int, now: int, gone_ms: int, missing: np.ndarray) -> Pruned:
    """orc_prune_missing over each model's loaded, then failed registrations; missing (int64[n]) is stamped in place"""
    L = ob.lib()
    keep = np.ones(len(fl.edge_inst), dtype=bool)
    nl, nf = fl.n_loaded.astype(np.int64).copy(), fl.n_failed.astype(np.int64).copy()
    pairs = []
    buf = np.zeros(max(1, int(np.diff(fl.edge_off).max(initial=0))), dtype=np.uint8)
    inst = np.ascontiguousarray(fl.edge_inst, dtype=np.int32)
    ts = np.ascontiguousarray(ts, dtype=np.int64)
    for m in range(fl.n_models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        k = int(fl.n_loaded[m])
        for count, lo, hi in ((nl, a, a + k), (nf, a + k, b)):
            if lo == hi:
                continue
            if L.orc_prune_missing(o.h, leader, vp(inst[lo:hi]), vp(ts[lo:hi]), hi - lo, now, gone_ms, vp(missing), vp(buf)) == 0:
                continue
            for j in np.nonzero(buf[:hi - lo])[0]:
                keep[lo + j] = False
                pairs.append((m, int(inst[lo + j])))
                count[m] -= 1
    return Pruned(pairs, keep, nl, nf)


def repair(last_used: np.ndarray, now: int):
    """(the lastUsed values after repairLastUsedTimeIfNeeded, the repaired model ids)"""
    bad = np.nonzero(last_used == LONG_MAX)[0]
    lu = last_used.astype(np.int64).copy()
    lu[bad] = now - REPAIR_AGE_MS
    return lu, [int(m) for m in bad]


def select(o: ob.OracleFleet, fl, pr: Pruned, last_used: np.ndarray, now: int):
    """(selected models in emission order, mmp_stats index of the partition a size estimate of 0 stopped at or -1)"""
    L = ob.lib()
    om = np.zeros(fl.n_models, dtype=ob.MODEL)
    om["last_used"], om["type_idx"], om["n_loaded"], om["n_failed"] = last_used, fl.model_type, pr.n_loaded, pr.n_failed
    parts = [-1] if fl.type_config is None else [int(p) for p in o.partition_stats()[1]]
    names = (C.c_char_p * max(1, len(fl.type_names)))(*[t.encode() for t in fl.type_names])
    taken = np.zeros(fl.n_models, dtype=np.uint8)
    out = np.zeros(fl.n_models, dtype=np.int32)
    sel = []
    for k, p in enumerate(parts):
        n = L.orc_reaper_select(o.h, fl.n_models, vp(om), names, len(fl.type_names), p, now, vp(taken), vp(out), len(out))
        if n == -4:  # the size estimate is 0
            return sel, (0 if p < 0 else 1 + k)
        assert n >= 0, n
        sel += [int(x) for x in out[:n]]
    return sel, -1


def place(o: ob.OracleFleet, fl, pr: Pruned, last_used: np.ndarray, sel, leader: int, now: int, seed: int):
    n = len(sel)
    if n == 0:
        return np.zeros(0, dtype=ob.RESULT)
    m = np.asarray(sel, dtype=np.int64)
    od = np.zeros(n, dtype=ob.DECISION)
    od["type_idx"], od["self"], od["fresh_idx"], od["last_used"] = fl.model_type[m], leader, -1, last_used[m]
    od["decision_id"] = np.arange(n, dtype=np.uint64)
    lists = [fl.edge_inst[fl.edge_off[x]:fl.edge_off[x + 1]][pr.keep[fl.edge_off[x]:fl.edge_off[x + 1]]] for x in m]
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(e) for e in lists], out=off[1:])
    idx = np.concatenate(lists).astype(np.int32) if off[-1] else np.zeros(0, dtype=np.int32)
    return o.get_next_batch(od, fl.type_names, off, idx, now, seed)


def cleanup(missing: np.ndarray, in_table: np.ndarray, now: int, gone_ms: int):
    """missings.entrySet().removeIf(now - v > ASSUME_INSTANCE_GONE_AFTER_MS || instanceInfo.contains(k)), in place"""
    drop = (missing != 0) & (((now - missing) > gone_ms) | in_table[:len(missing)])
    missing[drop] = 0


def reaper_run(o: ob.OracleFleet, fl, ts, leader: int, now: int, gone_ms: int, missing: np.ndarray, in_table: np.ndarray, seed: int):
    """The whole task: {pairs, repaired, loads (model, target, n_candidates, last_used), stopped, pruned}; missing updated in
    place"""
    pr = prune(o, fl, ts, leader, now, gone_ms, missing)
    lu, repaired = repair(fl.model_last_used, now)
    sel, stopped = select(o, fl, pr, lu, now)
    # (a leader outside the table has no getNext on the oracle; mmp_reaper_run answers its decisions MMP_TARGET_INVALID)
    res = place(o, fl, pr, lu, sel, leader, now, seed) if in_table[leader] else np.full(len(sel), -3, dtype=ob.RESULT)
    cleanup(missing, in_table, now, gone_ms)
    loads = [(m, int(r["target"]), int(r["n_candidates"]), int(lu[m])) for m, r in zip(sel, res)]
    return {"pairs": pr.pairs, "repaired": repaired, "loads": loads, "stopped": stopped, "pruned": pr}
