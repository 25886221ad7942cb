"""One run of one pod's whole janitor task (MM:5876-6145), restated in plain Python -- the reference mmp_janitor_task is checked
against (tests/test_janitor_task_gpu.py; its own check without a GPU: tests/test_janitor_task_oracle.py).  The cache loop
(MM:5892-6008) runs over the entries in order and writes the records it changes into a copy of the fleet's registry; the
registry loop is tests/janitor_run_oracle.py on that copy, with the entries the loop removed reading lastUsed -1.

Quirk N16 (the early stop): the first entry that passes the skips with lastUsed == Long.MAX_VALUE force-sets it to
now - 3 x LASTUSED_AGE_ON_ADD_MS, repairs a record at Long.MAX_VALUE to the same value, and `return`s from the task's run()
(MM:5929): the rest of the cache loop and the whole registry loop do not run.

A model without a record is one at or past the fleet's model count (never upserted)."""
import copy

import numpy as np

import janitor_run_oracle as jro
from janitor_run_oracle import jsub
from modelmesh_b200 import _lib as L
from rate_run_oracle import saturated

LONG_MAX = (1 << 63) - 1
LASTUSED_AGE_ON_ADD_MS = 3_600_000


def jlong(x: int) -> int:
    return ((int(x) + (1 << 63)) % (1 << 64)) - (1 << 63)


def _self_regs(fl, ts, S, m):
    """(loaded time or None, failed time or None): the pod's first loaded and first failed registration of model m"""
    a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
    loaded = next((int(ts[q]) for q in range(a, a + k) if fl.edge_inst[q] == S), None)
    failed = next((int(ts[q]) for q in range(a + k, b) if fl.edge_inst[q] == S), None)
    return loaded, failed


def cache_pass(fl, ts, S, entries, params):
    """(actions [(model, what, last_used, replaced_ts)] in entry order, counts dict, stopped_at, records {m: (lastUsed,
    reregistered load_ts or None)}, removed models)"""
    p = params[0] if params.shape else params
    now = int(p["janitor"]["scale"]["now"])
    window = jlong(int(p["janitor_freq_secs"]) * 2000 + int(p["load_timeout_ms"]))
    min_stale = int(p["min_stale_age_ms"])
    out, recs, removed = [], {}, set()
    last_last, stopped = LONG_MAX, -1

    def stale(m, lu, rec_lu):
        """updateLastUsedTimeInRegistryIfStale (MM:6165-6183): (what, the record's lastUsed)"""
        if jsub(lu, rec_lu) < min_stale:
            return 0, rec_lu
        recs[m] = (max(rec_lu, lu), None)
        return L.JC_STALE_UPDATE, max(rec_lu, lu)

    for r, te in enumerate(entries):
        e = te["e"]
        m, lu, flags = int(e["model"]), int(e["last_used"]), int(e["flags"])
        has_rec = m < fl.n_models
        rec_lu = int(fl.model_last_used[m]) if has_rec else 0
        if stopped >= 0:
            out.append((m, L.JC_NOT_REACHED, rec_lu, -1))
            continue
        what, shown, replaced = 0, None, -1
        if flags & L.JANITOR_NOT_DONE:
            what = L.JC_NOT_DONE
        elif lu <= 0:
            what = L.JC_NOT_CACHED
        else:
            if lu > last_last:
                what |= L.JC_OUT_OF_ORDER
            last_last = lu
            if lu == LONG_MAX:
                what |= L.JC_STOP
                shown = jsub(now, 3 * LASTUSED_AGE_ON_ADD_MS)
                if has_rec and rec_lu == LONG_MAX:
                    what |= L.JC_REPAIR
                    rec_lu = shown
                stopped = r
            elif jsub(now, lu) < window:
                if has_rec:
                    w, rec_lu = stale(m, lu, rec_lu)
                    what |= w
            elif has_rec and saturated(fl, m):
                what |= L.JC_UNDECIDED
            else:
                failed = bool(flags & L.JANITOR_FAILED)
                loaded_ts, failed_ts = _self_regs(fl, ts, S, m) if has_rec else (None, None)
                reg, local = (failed_ts, int(te["load_complete_ts"])) if failed else (loaded_ts, int(e["load_ts"]))
                if has_rec and reg is not None and reg == local:
                    w, rec_lu = stale(m, lu, rec_lu)
                    what |= w
                elif not has_rec or flags & (L.JANITOR_NOT_LIVE | L.JANITOR_UNLOAD_RECENT):
                    what |= L.JC_REMOVE
                    removed.add(m)
                else:
                    what |= L.JC_REREGISTER
                    if not failed and loaded_ts is not None:
                        replaced = loaded_ts
                    rec_lu = max(rec_lu, lu)
                    recs[m] = (rec_lu, int(e["load_ts"]))
        out.append((m, what, shown if what & L.JC_STOP else rec_lu, replaced))
    names = ["n_not_done", "n_not_cached", "n_out_of_order", "n_stop", "n_repair", "n_not_reached", "n_stale_update", "n_remove",
             "n_reregister", "n_undecided"]
    counts = {k: sum(1 for _, w, _, _ in out if w & (1 << b)) for b, k in enumerate(names)}
    return out, counts, stopped, recs, removed


def records_after(fl, ts, S, recs):
    """(fleet, times) with the cache pass's writes: a re-registered model holds the pod among its loaded copies at load_ts
    (appended where it was not loaded) and no failure record of it; lastUsed as written"""
    if not recs:
        return fl, ts
    f2 = copy.copy(fl)
    f2.model_last_used = fl.model_last_used.copy()
    inst, times, nl, nf = [], [], [], []
    for m in range(fl.n_models):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        li, lt = list(fl.edge_inst[a:a + k]), list(ts[a:a + k])
        fi, ft = list(fl.edge_inst[a + k:b]), list(ts[a + k:b])
        if m in recs:
            lu, load_ts = recs[m]
            f2.model_last_used[m] = lu
            if load_ts is not None:
                if S in li:
                    lt[li.index(S)] = load_ts
                else:
                    li.append(S)
                    lt.append(load_ts)
                keep = [q for q, i in enumerate(fi) if i != S]
                fi, ft = [fi[q] for q in keep], [ft[q] for q in keep]
        inst += li + fi
        times += lt + ft
        nl.append(len(li))
        nf.append(len(fi))
    f2.edge_inst = np.array(inst, dtype=np.int32)
    f2.n_loaded = np.array(nl, dtype=np.int32)
    f2.n_failed = np.array(nf, dtype=np.int32)
    f2.edge_off = np.zeros(fl.n_models + 1, dtype=np.int64)
    np.cumsum(np.array(nl) + np.array(nf), out=f2.edge_off[1:])
    return f2, np.array(times, dtype=np.int64)


def janitor_task(o, fl, ts, lul, S, entries, params):
    """(actions, edits [(model, what, last_used, last_unload_time)] in model order, report dict).  entries: JANITOR_TASK_ENTRY
    records, most recently used first; params: one JANITOR_TASK_PARAMS record; o: the oracle fleet of fl's instances."""
    p = params[0] if params.shape else params
    out, counts, stopped, recs, removed = cache_pass(fl, ts, S, entries, p)
    rep = dict(counts, stopped_at=stopped, registry_ran=int(stopped < 0), cache_changed=int(counts["n_remove"] > 0))
    if stopped >= 0:
        return out, [], dict(rep, registry=dict(n_referencing=0, n_edits=0, n_candidates=0, n_removed=0, weight_removed=0))
    f2, ts2 = records_after(fl, ts, S, recs)
    ents = np.array([te["e"] for te in entries], dtype=L.JANITOR_ENTRY)
    for r, te in enumerate(entries):
        if int(te["e"]["model"]) in removed:
            ents[r]["last_used"] = -1
    jp = np.array([p["janitor"]], dtype=L.JANITOR_PARAMS)
    edits, jr = jro.janitor_run(o, f2, ts2, lul, S, ents, jp)
    return out, edits, dict(rep, registry=jr)
