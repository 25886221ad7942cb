"""Request-model decisions (MMP_DF_REQUEST_MODEL) for the tests: the model record travels with the decision -- its type id
in `model`, its loaded ∪ failed instances in the decision's extra[] slice together with the request's own excludes -- and
the oracle inputs for them (type index + per-decision exclusion CSR, as tests/helpers.py builds them for model indices)."""
from __future__ import annotations

import numpy as np

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthDecisions, SplitMix
from oracle import binding as ob


def _csr(slices):
    off = np.zeros(len(slices) + 1, dtype=np.int64)
    np.cumsum([len(s) for s in slices], out=off[1:])
    idx = np.concatenate([np.asarray(s, dtype=np.int32) for s in slices]) if len(slices) else np.zeros(0, dtype=np.int32)
    return off, idx.astype(np.int32)


def hold_front(fl, order, n_models: int = 64):
    """Models 0 .. n_models-1 hold the first 4 instances of PLACEMENT_ORDER (the usual answers).  Type ids are small model
    indices too, so a request-model decision that read the registry row of the model whose INDEX equals its type id instead
    of the zero row would exclude the instances it most likely picks: the checks below then fail."""
    keep = [fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]] if m >= n_models else np.asarray(order[:4], dtype=np.int32)
            for m in range(fl.n_models)]
    deg = np.asarray([len(e) for e in keep], dtype=np.int64)
    fl.edge_off = np.zeros(fl.n_models + 1, dtype=np.int64)
    np.cumsum(deg, out=fl.edge_off[1:])
    fl.edge_inst = np.concatenate(keep).astype(np.int32)
    fl.n_loaded = deg.astype(np.int32)
    fl.n_failed = np.zeros(fl.n_models, dtype=np.int32)
    return fl


def _explicit_last_used(fl, dec):
    """last_used as the model row gives it (a request-model decision has no model row to take it from)"""
    use_model = (dec["flags"] & L.DF_MODEL_LAST_USED) != 0
    return np.where(use_model, fl.model_last_used[np.maximum(dec["model"], 0)], dec["last_used"])


def as_request_model(fl, sd: SynthDecisions, tid: dict):
    """The same getNext calls with each model's COMMITTED record carried by the decision.  Returns the flagged decisions and
    a mask of those that were flagged: a decision whose model ids ∪ own extras exceed MMP_MAX_EXTRA stays as it was."""
    tmap = np.asarray([tid[t] for t in fl.type_names], dtype=np.int32)
    dec = sd.dec.copy()
    slices, flagged = [], np.zeros(len(dec), dtype=bool)
    for i, d in enumerate(sd.dec):
        m = int(d["model"])
        own = sd.extra[d["extra_off"]:d["extra_off"] + d["extra_n"]]
        ids = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]], own])
        flagged[i] = len(ids) <= L.MAX_EXTRA
        slices.append(ids if flagged[i] else own)
    off, extra = _csr(slices)
    dec["extra_off"] = off[:-1]
    dec["extra_n"] = np.diff(off)
    dec["last_used"] = np.where(flagged, _explicit_last_used(fl, sd.dec), dec["last_used"])
    dec["model"] = np.where(flagged, tmap[fl.model_type[sd.dec["model"]]], dec["model"])
    dec["flags"] = np.where(flagged, (dec["flags"] & ~np.uint32(L.DF_MODEL_LAST_USED)) | np.uint32(L.DF_REQUEST_MODEL), dec["flags"])
    return SynthDecisions(dec, sd.fresh, extra), flagged


def random_records(fl, sd: SynthDecisions, type_ids, seed: int, sizes=(0, 4, 5, 16)):
    """Request-model decisions on records the snapshot has never seen: decision i names type type_ids[k] (k drawn per
    decision: the caller lists committed types and types interned after the commit) and sizes[i % len(sizes)] instance
    ids drawn over the whole index space (instances that are not live included), self among them for a quarter.
    Returns the decisions and k per decision (the oracle's type index into the caller's name list)."""
    rng = SplitMix(seed ^ 0x5EC0)
    n = len(sd.dec)
    dec = sd.dec.copy()
    k = rng.randint(n, 0, len(type_ids)).astype(np.int32)
    sz = np.asarray([sizes[i % len(sizes)] for i in range(n)], dtype=np.int64)
    ids = rng.randint(int(sz.sum()), 0, fl.n_instances).astype(np.int32)
    has_self = rng.uniform(n) < 0.25
    slices, o = [], 0
    for i in range(n):
        s = ids[o:o + sz[i]].copy()
        o += sz[i]
        if has_self[i] and len(s):
            s[len(s) // 2] = dec["self"][i]
        slices.append(s)
    off, extra = _csr(slices)
    dec["extra_off"] = off[:-1]
    dec["extra_n"] = np.diff(off)
    dec["last_used"] = _explicit_last_used(fl, sd.dec)
    dec["model"] = np.asarray(type_ids, dtype=np.int32)[k]
    dec["flags"] = (dec["flags"] & ~np.uint32(L.DF_MODEL_LAST_USED)) | np.uint32(L.DF_REQUEST_MODEL)
    return SynthDecisions(dec, sd.fresh, extra), k


def oracle_inputs_request(type_idx, sd: SynthDecisions):
    """Oracle decisions + exclusion CSR for request-model decisions: the exclusions are exactly the extra[] slices."""
    dec = sd.dec
    n = len(dec)
    od = np.zeros(n, dtype=ob.DECISION)
    od["type_idx"] = type_idx
    od["self"] = dec["self"]
    od["fresh_idx"] = dec["fresh"]
    od["favour_self"] = (dec["flags"] & L.DF_FAVOUR_SELF) != 0
    od["last_used"] = dec["last_used"]
    od["decision_id"] = np.arange(n, dtype=np.uint64)
    off, idx = _csr([sd.extra[a:a + b] for a, b in zip(dec["extra_off"], dec["extra_n"])])
    return od, off, idx


def oracle_request(o, names, type_idx, sd: SynthDecisions, now_ms: int, seed: int):
    od, off, idx = oracle_inputs_request(type_idx, sd)
    return o.get_next_batch(od, names, off, idx, now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)
