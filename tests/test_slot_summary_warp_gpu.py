"""k_slot_summary on the device (one warp per type slot and c_self, the cooperative slot_summary) against the CPU harness's
summaries (the same routine one row word per step): every SlotSummary field and every listed shortlist member, read back
with mmp_slot_summaries.  The fleets: C2, C3 and C5 at the bench's instance counts, MIX 14 / 41, rolling upgrades (a
saturated front, where bests are full, and a replicaset roll, where the filter is retried), and a fleet of more than 64
type slots; `now` on both sides of the lruTime thresholds a full best's summary depends on.  On each fleet the batch placed
with the two passes forced on equals the one-pass placement and the oracle, byte for byte, with and without a call-wide
exclude set."""
import ctypes as C
import itertools

import numpy as np
import pytest

from exclude_set import oracle_excluding, random_set
from helpers import oracle_from_synth, oracle_inputs_fast, solver_from_synth
from modelmesh_b200.synth import make_decisions, make_fleet
from split_place import split_lib  # noqa: F401  (split_lib: module fixture)
from upgrade import upgrade

CAP = 256  # SPLIT_CAP: members listed per (slot, c_self)
SLOT_SUMMARY = np.dtype([("best_rem", "<i8"), ("best_lru", "<i8"), ("best_idx", "<i4"), ("best_rpm", "<i4"), ("best_full", "<i4"),
                         ("reach", "<i4", (2,)), ("n_in", "<i4", (2,)), ("pad", "<i4")])
FIELDS = [f for f in SLOT_SUMMARY.names if f != "pad"]


def _many_slot_fleet():
    """C3's instances (8 labels, 1-3 per instance) under 96 types that ask for label pairs, required and preferred: 74
    distinct type slots, pairs of required labels sparse enough that some shortlists run past the first 384 ranks."""
    nm, seed = 20_000, 61
    fl = make_fleet("C3", nm, 3000, seed)
    labs = [f"lbl-{k:02d}" for k in range(8)]
    pairs = list(itertools.combinations(labs, 2))
    cfg = {}
    for k in range(96):
        a, b = pairs[k % len(pairs)]
        if k % 3 == 0:
            ent = {"required": [a, b]}
        elif k % 3 == 1:
            ent = {"required": [labs[k % 8]], "preferred": [a, b] if (k // 8) % 2 else [b]}
        elif k < 56:
            ent = {"required": [a], "preferred": [b]}
        elif k < 84:
            ent = {"preferred": [a, b]}
        else:
            ent = {"required": [b, a], "preferred": [labs[k % 8]]}
        cfg[f"type-{k:02d}"] = ent
    fl.type_config = cfg
    fl.type_names = list(cfg) + ["untyped"]
    fl.model_type = np.random.default_rng(seed).integers(0, len(fl.type_names), nm).astype(np.int32)
    return fl


FLEETS = {
    "C2": lambda: make_fleet("C2", 20_000, 1_000, 2),
    "C3": lambda: make_fleet("C3", 20_000, 10_000, 3),
    "C5": lambda: make_fleet("C5", 20_000, 10_000, 5),
    "MIX14": lambda: make_fleet("MIX", 800, 300, 14),
    "MIX41": lambda: make_fleet("MIX", 800, 700, 41),
    "C3-saturated": lambda: upgrade(make_fleet("C3", 3000, 1300, 33), "saturated", 33),
    "C5-saturated": lambda: upgrade(make_fleet("C5", 1500, 500, 5), "saturated", 5),
    "C3-rsroll": lambda: upgrade(make_fleet("C3", 3000, 1300, 33), "rsroll", 33),
    "many-slots": _many_slot_fleet,
}


def _summaries(lib, fn, s, now):
    sums = np.zeros(CAP, dtype=SLOT_SUMMARY)
    members = np.full((CAP, 2, CAP), -1, dtype=np.int32)
    fn.restype = C.c_int32
    n = s._ck(fn(s.h, C.c_int64(now), sums.ctypes.data_as(C.c_void_p), members.ctypes.data_as(C.c_void_p), CAP))
    assert 0 < n <= CAP
    return sums[:n], members[:n]


def _same_summaries(dev, cpu, what):
    (ds, dm), (cs, cm) = dev, cpu
    assert len(ds) == len(cs), what
    for f in FIELDS:
        bad = np.nonzero((ds[f] != cs[f]).reshape(len(ds), -1).any(axis=1))[0]
        assert len(bad) == 0, (what, f, bad[:5], ds[f][bad[:5]], cs[f][bad[:5]])
    for sl in range(len(cs)):
        for c in range(2):
            if cs["reach"][sl, c] >= 0:
                k = int(cs["n_in"][sl, c])
                assert np.array_equal(dm[sl, c, :k], cm[sl, c, :k]), (what, sl, c)
    return int((cs["reach"] >= 0).sum())


def _threshold_nows(sums, now):
    """`now` just below and at the ages where a full best's summary changes: c_self's a10 = age / 10 passes 45 000 at age
    450 010, non-simple (b)'s a4 = age / 4 passes 120 000 at age 480 004"""
    full = np.nonzero(sums["best_full"] == 1)[0]
    if len(full) == 0:
        return [now]
    lru = int(sums["best_lru"][full[0]])
    return [now] + [lru + a for a in (450_009, 450_010, 480_003, 480_004)]


def _placements_agree(lib, s, o, fl, now, seed, exclude=None):
    """a plain sweep and a mixed batch, placed with split = 1 and 0: byte-identical, and equal to the oracle"""
    for sd in (make_decisions(fl, 20_000, seed, sweep=True, plain=True), make_decisions(fl, 5_000, seed + 1)):
        kw = dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None, exclude=exclude)
        got = {}
        for split in (1, 0):
            s._ck(lib.mmp_tune(s.h, b"split", split))
            try:
                got[split] = s.place_batch(sd.dec, now, seed, **kw)
            finally:
                s._ck(lib.mmp_tune(s.h, b"split", 2))
        assert got[1].tobytes() == got[0].tobytes(), (now, int(np.sum(got[1] != got[0])))
        if exclude is None:
            od, off, idx = oracle_inputs_fast(fl, sd)
            want = o.get_next_batch(od, fl.type_names, off, idx, now, seed, fresh=kw["fresh"])
        else:
            want = oracle_excluding(o, fl, sd, exclude, seed)
        bad = np.nonzero((got[1]["target"] != want["target"]) | (got[1]["n_candidates"] != want["n_candidates"]))[0]
        assert len(bad) == 0, (now, len(bad), bad[:5])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FLEETS))
def test_device_summaries_equal_the_harness(product_lib, oracle_lib, split_lib, name):  # noqa: F811
    fl = FLEETS[name]()
    o = oracle_from_synth(fl)
    dev = solver_from_synth(fl, product_lib)
    cpu = solver_from_synth(fl, split_lib)
    try:
        base = _summaries(split_lib, split_lib.mmp_emul_slot_summaries, cpu, fl.now_ms)
        listed = 0
        for now in _threshold_nows(base[0], fl.now_ms):
            want = base if now == fl.now_ms else _summaries(split_lib, split_lib.mmp_emul_slot_summaries, cpu, now)
            listed += _same_summaries(_summaries(product_lib, product_lib.mmp_slot_summaries, dev, now), want, (name, now))
        assert listed > 0, name
        _placements_agree(product_lib, dev, o, fl, fl.now_ms, 7)
        if name.endswith("saturated"):  # a full best at the thresholds: the two passes still place what one pass does
            assert base[0]["best_full"].any(), name
            for now in _threshold_nows(base[0], fl.now_ms)[1:]:
                _placements_agree(product_lib, dev, o, fl, now, 11)
        if name in ("C3", "C5", "MIX41"):
            xs = np.concatenate([dev.cluster_order()[:3], random_set(fl.n_instances, 40, 5)]).astype(np.int32)
            _placements_agree(product_lib, dev, o, fl, fl.now_ms, 13, exclude=xs)
    finally:
        dev.close()
        cpu.close()
