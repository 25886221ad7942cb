"""The registry loop of one pod's janitor task (MM:6013-6145), restated in plain Python over a synth fleet's edge lists and
registration times -- the reference mmp_janitor_run is checked against (tests/test_janitor_run_gpu.py; its own check without
a GPU: tests/test_janitor_run_oracle.py).  removeModelCopies (MM:6197-6335) is orc_janitor_eval, one candidate at a time with
canRemove from the budget; the registration-time check of removeLocalModelCopyAsync (MM:6347-6349), which orc_janitor_eval
leaves out, is added here.

Quirk N15 (the janitor's TreeSet): scaleCopiesCandidates is a TreeSet ordered by VALUE_COMP (MM:6875-6880), which compares the
lastUsed value only, so of candidates with equal lastUsed the set keeps the first one added and drops the others.  The
reference adds them in registry iteration order; model index order stands in for it, as it does for the reaper's bounded set
(N12)."""
import numpy as np

from common import jsub, vp
from modelmesh_b200 import _lib as L
from oracle import binding as ob
from rate_run_oracle import saturated

SHORT_EXPIRY_RECENT_USE_TIME_MS = 180_000


def remove_model_copies(o: ob.OracleFleet, fl, ts, lul, self_idx: int, m: int, ce, params, can_remove: int) -> int:
    """orc_janitor_eval for self's copy of model m under the entry ce (a JANITOR_ENTRY record)"""
    a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
    rec = np.zeros(1, dtype=ob.SCALE_IN)
    rec["instance"], rec["model"], rec["count"], rec["last_used"], rec["last_heavy"] = self_idx, m, ce["count"], ce["last_used"], ce["last_heavy"]
    rec["flags"] = int(params["flags"]) & 1
    op = np.zeros(1, dtype=ob.SCALE_PARAMS)
    for k in op.dtype.names:
        if k != "pad":
            op[k] = params["scale"][k]
    op["can_remove"] = can_remove
    eoff = np.array([0, b - a], dtype=np.int64)
    einst = np.ascontiguousarray(fl.edge_inst[a:b], dtype=np.int32)
    ets = np.ascontiguousarray(ts[a:b], dtype=np.int64)
    nl = np.array([fl.n_loaded[m]], dtype=np.int32)
    lulr = np.array([lul[m]], dtype=np.int64)
    down = np.zeros(1, dtype=ob.SCALE_OUT)
    assert ob.lib().orc_janitor_eval(o.h, 1, vp(rec), vp(op), vp(eoff), vp(einst), vp(ets), vp(nl), vp(lulr), vp(down)) == 0
    return int(down["remove"][0])


def janitor_run(o: ob.OracleFleet, fl, ts, lul, self_idx: int, entries, params):
    """(edits [(model, what, last_used, last_unload_time)] in model order, report dict).  ts: the time of every registration
    of fl.edge_inst; lul: lastUnloadTime per model; entries: JANITOR_ENTRY records; params: one JANITOR_PARAMS record."""
    p = params[0] if params.shape else params
    now, expiry = int(p["scale"]["now"]), int(p["load_failure_expiry_ms"])
    by_model = {int(e["model"]): e for e in entries}
    hits = np.nonzero(fl.edge_inst == self_idx)[0]
    models = np.unique(np.searchsorted(fl.edge_off, hits, side="right") - 1)
    edits, cands = {}, []
    for m in (int(x) for x in models):
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        nl = int(fl.n_loaded[m])
        rec_lu, rec_lul = int(fl.model_last_used[m]), int(lul[m])
        if saturated(fl, m):
            edits[m] = [L.JE_UNDECIDED, rec_lu, rec_lul]
            continue
        pos = [q - a for q in range(a, b) if fl.edge_inst[q] == self_idx]
        loaded_at = next((q for q in pos if q < nl), None)
        failed_at = next((q for q in pos if q >= nl), None)
        loaded = loaded_at is not None
        ce = by_model.get(m)
        ce_failed = ce is not None and bool(int(ce["flags"]) & L.JANITOR_FAILED)
        rem_loaded = loaded and (ce is None or ce_failed)
        rem_failed = False
        if failed_at is not None:
            if ce is not None and not ce_failed:
                rem_failed = True
            else:
                lu = int(ce["last_used"]) if ce is not None else -1
                age = expiry // 2 if lu > 0 and jsub(now, lu) < SHORT_EXPIRY_RECENT_USE_TIME_MS else expiry
                rem_failed = jsub(now, int(ts[a + failed_at])) > age
        what, lu_rec, lul_rec = 0, rec_lu, rec_lul
        if rem_loaded or rem_failed:
            if rem_loaded:  # instanceIds.remove(self); updateLastUnloadTime()
                what |= L.JE_UNREGISTER
                lul_rec = 0 if nl - 1 <= 2 else now
            if rem_failed:
                what |= L.JE_DROP_FAILURE
            if ce is not None and int(ce["last_used"]) > 0:
                lu_rec = max(lu_rec, int(ce["last_used"]))
        if rem_failed and ce_failed:
            what |= L.JE_REMOVE_LOCAL
        if what:
            edits[m] = [what, lu_rec, lul_rec]
        if loaded and not rem_loaded and int(ce["last_used"]) > 0:
            cands.append((int(ce["last_used"]), m, int(ts[a + loaded_at])))
    # TreeSet(VALUE_COMP): ascending lastUsed, the first of equal values (N15)
    tree = []
    for c in sorted(cands):
        if not tree or tree[-1][0] != c[0]:
            tree.append(c)
    budget, removed, weight_removed = int(p["adjusted_capacity"]) // 20, 0, 0
    for lu, m, reg_ts in tree:
        ce = by_model[m]
        w = int(ce["weight"])
        can = 1 if removed == 0 or w <= budget else 0
        if not (remove_model_copies(o, fl, ts, lul, self_idx, m, ce, p, can) and reg_ts == int(ce["load_ts"])):
            continue
        removed += 1
        budget -= w
        weight_removed += w
        e = edits.setdefault(m, [0, int(fl.model_last_used[m]), int(lul[m])])
        e[0] |= L.JE_SCALE_DOWN
        e[1] = max(e[1], lu)
        e[2] = 0 if int(fl.n_loaded[m]) - 1 <= 2 else now
    out = [(m, *edits[m]) for m in sorted(edits)]
    return out, dict(n_referencing=len(models), n_edits=len(out), n_candidates=len(tree), n_removed=removed,
                     weight_removed=weight_removed)
