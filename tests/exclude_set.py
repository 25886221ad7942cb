"""Call-wide exclude sets (mmp_place_batch_excluding) for the tests: the oracle inputs with the set appended to every
decision's exclusion list, and the sets the CPU and GPU tests place under."""
from __future__ import annotations

import numpy as np

from modelmesh_b200.synth import SplitMix, SynthDecisions

from helpers import oracle_inputs_fast
from request_model import oracle_inputs_request


def extend_csr(off, idx, xs):
    """Exclusion CSR with xs appended to every decision's list (the oracle's reading of a call-wide set)."""
    n = len(off) - 1
    xs = np.asarray(xs, dtype=np.int32)
    own = np.diff(off).astype(np.int64)
    noff = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(own + len(xs), out=noff[1:])
    nidx = np.empty(int(noff[-1]), dtype=np.int32)
    owner = np.repeat(np.arange(n, dtype=np.int64), own)
    nidx[noff[owner] + np.arange(len(idx), dtype=np.int64) - off[owner]] = idx
    if len(xs):
        nidx[(noff[:-1] + own)[:, None] + np.arange(len(xs), dtype=np.int64)[None, :]] = xs[None, :]
    return noff, nidx


def oracle_excluding(o, fl, sd, xs, seed, names=None, type_idx=None, candidates=False, positions=None):
    """The oracle on sd with xs added to every decision's CacheMissExcludeSet.  Request-model decisions: pass the type
    names and each decision's type index (tests/request_model.py).  positions: the decisions' places in the batch the
    solver placed (the hash-indexed pick numbers them), when sd is a sample of it."""
    od, off, idx = oracle_inputs_fast(fl, sd) if type_idx is None else oracle_inputs_request(type_idx, sd)
    if positions is not None:
        od["decision_id"] = np.asarray(positions, dtype=np.uint64)
    off, idx = extend_csr(off, idx, xs)
    return o.get_next_batch(od, fl.type_names if names is None else names, off, idx, fl.now_ms, seed,
                            fresh=sd.fresh if len(sd.fresh) else None, want_candidates=candidates)


def random_set(n_instances, size, seed):
    """size ids over the whole index space (not-live instances and duplicates among them)"""
    return SplitMix(seed ^ 0xE5E7).randint(size, 0, n_instances).astype(np.int32)


def type_candidates(s, fl, type_name):
    """instance indices the type allows (every live one when unconstrained), from the solver's committed type sets"""
    allowed, _ = s.type_sets(s.type_id(type_name), fl.n_instances)
    if allowed is None:
        return np.asarray(s.cluster_order(), dtype=np.int32)
    return np.nonzero(allowed)[0].astype(np.int32)


def self_and_best(sd, first):
    """the selves of the batch's first decisions and the targets they get without a set"""
    k = min(64, len(sd.dec))
    t = first["target"][:k]
    return np.unique(np.concatenate([sd.dec["self"][:k], t[t >= 0]])).astype(np.int32)


def unflagged_candidates(s, fl, type_name):
    """the type's candidates outside the likely-replaced replicasets (MM:4769-4770): a set of these leaves the flagged ones"""
    c = type_candidates(s, fl, type_name)
    flagged = np.asarray([len(fl.inst_ids[i]) >= 7 and fl.inst_ids[i][:6] in fl.replaced_replicasets for i in c], dtype=bool)
    return c[~flagged], c[flagged]


def named_sets(s, fl, sd, first, seed):
    """(name, set) pairs every test places under: sizes 1 / 17 / 200 / 2 000, every candidate of one type, every instance,
    the batch's selves and their unconstrained answers"""
    t0 = fl.type_names[int(fl.model_type[sd.dec["model"][0]])] if len(sd.dec) else fl.type_names[0]
    return [(f"random-{k}", random_set(fl.n_instances, k, seed + k)) for k in (1, 17, 200, 2000)] + [
        ("type-" + t0, type_candidates(s, fl, t0)),
        ("every-instance", np.arange(fl.n_instances, dtype=np.int32)),
        ("self-and-best", self_and_best(sd, first)),
    ]


def rs_retry_type(s, fl):
    """a type with candidates inside and outside the flagged replicasets"""
    for t in fl.type_names:
        free, flagged = unflagged_candidates(s, fl, t)
        if len(free) and len(flagged):
            return t, free, flagged
    raise AssertionError("no type with flagged and unflagged candidates")


def compact(sd, n):
    """the first n decisions with only the fresh rows and extras they use (a small call's own side tables)"""
    dec = sd.dec[:n].copy()
    fr = dec["fresh"] >= 0
    fresh = sd.fresh[dec["fresh"][fr]] if len(sd.fresh) else sd.fresh[:0]
    dec["fresh"][fr] = np.arange(int(fr.sum()))
    slices = [sd.extra[a:a + b] for a, b in zip(dec["extra_off"], dec["extra_n"])]
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(x) for x in slices], out=off[1:])
    dec["extra_off"] = off[:-1]
    extra = np.concatenate(slices).astype(np.int32) if n else np.zeros(0, dtype=np.int32)
    return SynthDecisions(dec, fresh, extra)
