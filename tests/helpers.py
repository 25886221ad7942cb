"""Shared test plumbing: feed one SynthFleet to the oracle and to a solver, then compare decision by decision."""
from __future__ import annotations

import socket

import numpy as np

from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, candidates_from_masks
from modelmesh_b200.synth import SynthDecisions, SynthFleet, load_into_fleet, make_fleet
from oracle import binding as ob


def oracle_from_synth(fl: SynthFleet, bulk=None, gone=()) -> ob.OracleFleet:
    """Config first (as a pod does at start-up, MM:777), instances as ADDED events, then one converged refresh.  gone: the
    instances left out (they left the table and a commit dropped them; one event at a time only)."""
    o = ob.OracleFleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units)
    o.types_set(fl.type_config)
    if bulk is None:
        bulk = fl.n_instances > 3000
    gone = set(int(i) for i in gone)
    assert not (bulk and gone), "bulk_add adds every instance"
    if bulk:  # same final state (checked in test_host_logic.py) without the per-event O(N) work
        o.bulk_add(fl.inst_rows, fl.inst_ids, fl.inst_locs, fl.inst_zones, fl.inst_labels)
    else:
        for i in range(fl.n_instances):
            if i in gone:
                continue
            o.instance_event(ob.ADDED, i, fl.inst_rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i],
                             fl.inst_labels[i], fl.now_ms)
        if fl.type_config is not None:
            o.tc_converge()
    o.set_replaced_replicasets(fl.replaced_replicasets)
    return o


def solver_from_synth(fl: SynthFleet, lib, max_models=None) -> Fleet:
    f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances,
              max_models or fl.n_models, lib=lib)
    load_into_fleet(fl, f)
    return f


def oracle_inputs(fl: SynthFleet, sd: SynthDecisions):
    """Translate mmp_decision_in rows into oracle decisions + exclusion CSR (loaded ∪ failed ∪ extra)."""
    dec = sd.dec
    n = len(dec)
    od = np.zeros(n, dtype=ob.DECISION)
    od["type_idx"] = fl.model_type[dec["model"]]
    od["self"] = dec["self"]
    od["fresh_idx"] = dec["fresh"]
    od["favour_self"] = (dec["flags"] & L.DF_FAVOUR_SELF) != 0
    use_model = (dec["flags"] & L.DF_MODEL_LAST_USED) != 0
    od["last_used"] = np.where(use_model, fl.model_last_used[dec["model"]], dec["last_used"])
    od["decision_id"] = np.arange(n, dtype=np.uint64)
    m = dec["model"].astype(np.int64)
    deg = (fl.edge_off[m + 1] - fl.edge_off[m]) + dec["extra_n"]
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=off[1:])
    idx = np.zeros(int(off[-1]), dtype=np.int32)
    for i in range(n):  # small n in tests
        a, b = fl.edge_off[m[i]], fl.edge_off[m[i] + 1]
        k = b - a
        idx[off[i]:off[i] + k] = fl.edge_inst[a:b]
        e0 = dec["extra_off"][i]
        idx[off[i] + k:off[i + 1]] = sd.extra[e0:e0 + dec["extra_n"][i]]
    return od, off, idx


def oracle_inputs_fast(fl: SynthFleet, sd: SynthDecisions):
    """Vectorised oracle_inputs for large batches."""
    dec = sd.dec
    n = len(dec)
    od = np.zeros(n, dtype=ob.DECISION)
    od["type_idx"] = fl.model_type[dec["model"]]
    od["self"] = dec["self"]
    od["fresh_idx"] = dec["fresh"]
    od["favour_self"] = (dec["flags"] & L.DF_FAVOUR_SELF) != 0
    use_model = (dec["flags"] & L.DF_MODEL_LAST_USED) != 0
    od["last_used"] = np.where(use_model, fl.model_last_used[dec["model"]], dec["last_used"])
    od["decision_id"] = np.arange(n, dtype=np.uint64)
    m = dec["model"].astype(np.int64)
    dm = (fl.edge_off[m + 1] - fl.edge_off[m]).astype(np.int64)
    dx = dec["extra_n"].astype(np.int64)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(dm + dx, out=off[1:])
    idx = np.zeros(int(off[-1]), dtype=np.int32)
    for deg, src_base, src, shift in ((dm, fl.edge_off[m], fl.edge_inst, np.zeros(n, dtype=np.int64)),
                                      (dx, dec["extra_off"].astype(np.int64), sd.extra, dm)):
        tot = int(deg.sum())
        if tot == 0:
            continue
        owner = np.repeat(np.arange(n, dtype=np.int64), deg)
        start = np.zeros(n, dtype=np.int64)
        np.cumsum(deg[:-1], out=start[1:])
        within = np.arange(tot, dtype=np.int64) - start[owner]
        idx[off[owner] + shift[owner] + within] = src[src_base[owner] + within]
    return od, off, idx


def compare_decisions(fl: SynthFleet, sd: SynthDecisions, oracle: ob.OracleFleet, solver: Fleet, seed: int,
                      full_lists: bool = True):
    """Bit-exact comparison of (target, n_candidates, best, n_remaining, pick, ordered shortlist, survivors)."""
    od, off, idx = oracle_inputs(fl, sd)
    fresh = sd.fresh if len(sd.fresh) else None
    extra = sd.extra if len(sd.extra) else None
    ores, coff, cidx, cload, ckeep = oracle.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=fresh,
                                                            want_candidates=True)
    out, tr, cm = solver.place_batch(sd.dec, fl.now_ms, seed, fresh=fresh, extra=extra, trace=True, masks=True)
    order = solver.cluster_order()
    n = len(sd.dec)
    # the untraced entry point runs the production kernel (k_place_ring on the GPU): same answers
    out_fast = solver.place_batch(sd.dec, fl.now_ms, seed, fresh=fresh, extra=extra)
    assert np.array_equal(out_fast, out), _first_diff(out_fast["target"], out["target"], sd, ores, out_fast, tr)
    # traced but without masks: the one-window fast path answers whatever it can resolve; same trace fields
    out2, tr2, _ = solver.place_batch(sd.dec, fl.now_ms, seed, fresh=fresh, extra=extra, trace=True, masks=False)
    assert np.array_equal(out2, out), _first_diff(out2["target"], out["target"], sd, ores, out2, tr2)
    for k in ("best", "n_remaining", "pick_index", "cut_rank", "best_rank"):
        assert np.array_equal(tr2[k], tr[k]), (k, _first_diff(tr2[k], tr[k], sd, ores, out2, tr2))
    assert np.array_equal(tr2["flags"] & 255, tr["flags"] & 255), _first_diff(tr2["flags"] & 255, tr["flags"] & 255, sd, ores, out2, tr2)
    compare_decisions.fast_fraction = float(np.mean((tr2["flags"] & 256) != 0))
    assert np.array_equal(out["target"], ores["target"]), _first_diff(out["target"], ores["target"], sd, ores, out, tr)
    assert np.array_equal(out["n_candidates"], ores["n_candidates"]), _first_diff(out["n_candidates"], ores["n_candidates"], sd, ores, out, tr)
    has = ores["n_candidates"] > 0
    assert np.array_equal(tr["n_remaining"][has], ores["n_remaining"][has])
    assert np.array_equal(tr["pick_index"][has], ores["pick_index"][has])
    assert np.array_equal(tr["best"], ores["best"]), _first_diff(tr["best"], ores["best"], sd, ores, out, tr)
    assert np.array_equal(tr["flags"] & 15, ores["flags"] & 15), _first_diff(tr["flags"] & 15, ores["flags"] & 15, sd, ores, out, tr)
    if full_lists:
        for i in np.nonzero(has)[0]:
            pref_b = bool(tr["flags"][i] & L.TF_PREF_B)
            want = [int(x) for x in cidx[coff[i]:coff[i + 1]]]
            got = candidates_from_masks(order, tr["best"][i], cm[i, 0], include_best=not pref_b)
            assert got == want, (i, got[:8], want[:8])
            keep = ckeep[coff[i]:coff[i + 1]].astype(bool)
            want_surv = [c for c, k in zip(want, keep) if k]
            got_surv = candidates_from_masks(order, tr["best"][i], cm[i, 1],
                                             include_best=(not pref_b) and bool(tr["flags"][i] & L.TF_KEEP_BEST))
            assert got_surv == want_surv, (i, got_surv[:8], want_surv[:8])
    return ores, out, tr


def _first_diff(a, b, sd, ores, out, tr):
    d = np.nonzero(a != b)[0]
    i = int(d[0])
    return f"{len(d)} mismatches; first at {i}: got {a[i]} want {b[i]} dec={sd.dec[i]} oracle={ores[i]} out={out[i]} trace={tr[i]}"


def place_kw(sd: SynthDecisions) -> dict:
    """place_batch's fresh and extra arguments for sd"""
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


def same_answers(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def word_edge_fleet(ni: int, nm: int, seed: int):
    """C3 with about a quarter of the models holding 5-12 instances; the first (inline) edges of every model are the
    instances at ranks 0, 31, 32 (word edge), 383, 384, 385 (edge of the 12-word window) and n_ranks-1."""
    fl = make_fleet("C3", nm, ni, seed)
    # the placement order depends on the instance rows only: take it from the oracle
    order = oracle_from_synth(fl).cluster_order()
    nr = len(order)
    special = order[[0, 31, 32, 383, 384, 385, nr - 1]]
    rng = np.random.default_rng(seed)
    deg = np.where(rng.uniform(size=nm) < 0.25, rng.integers(5, 13, size=nm), rng.integers(0, 5, size=nm))
    edges = []
    for m in range(nm):
        inl = list(rng.choice(special, size=min(4, deg[m]), replace=False))
        rest = [int(x) for x in rng.choice(ni, size=deg[m] + 8, replace=False) if x not in inl][:max(0, deg[m] - 4)]
        edges.append([int(x) for x in inl] + rest)
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([x for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    return fl, order, edges


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p
