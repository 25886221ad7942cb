"""Deterministic synthetic fleets for the placement path (SURVEY.md §8d / BASELINE.json configs).

Everything is derived from a counter-mode SplitMix64 stream so a (config, sizes, seed) triple always yields the same
fleet, independent of numpy's own generators.  Used by tests/ (small sizes, against the oracle) and bench.py (full sizes).
"""
from __future__ import annotations

import json
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np

from ._lib import DECISION_IN, DF_FAVOUR_SELF, DF_MODEL_LAST_USED, INSTANCE_ROW, MODEL_ROW

NOW_MS = 1_760_000_000_000
LONG_MAX = (1 << 63) - 1
_G = np.uint64(0x9E3779B97F4A7C15)


class SplitMix:
    """Counter-mode SplitMix64: stream(k) is a pure function of (seed, k, index)."""

    def __init__(self, seed: int):
        self.seed = np.uint64(seed)
        self.k = 0

    def u64(self, n: int) -> np.ndarray:
        self.k += 1
        with np.errstate(over="ignore"):
            base = self.seed * np.uint64(0x2545F4914F6CDD1D) + np.uint64(self.k) * np.uint64(0xD1342543DE82EF95)
            z = base + _G * (np.arange(n, dtype=np.uint64) + np.uint64(1))
            z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
            z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
            return z ^ (z >> np.uint64(31))

    def uniform(self, n: int) -> np.ndarray:
        return (self.u64(n) >> np.uint64(11)).astype(np.float64) * (1.0 / (1 << 53))

    def randint(self, n: int, lo: int, hi: int) -> np.ndarray:  # [lo, hi)
        return (lo + (self.u64(n) % np.uint64(max(1, hi - lo))).astype(np.int64)).astype(np.int64)

    def exponential(self, n: int, mean: float) -> np.ndarray:
        return -np.log1p(-self.uniform(n)) * mean


@dataclass
class SynthFleet:
    name: str
    now_ms: int
    min_space_units: int
    min_churn_age_ms: int
    default_model_size_units: int
    inst_rows: np.ndarray                 # INSTANCE_ROW[n_i]
    inst_ids: List[str]
    inst_locs: List[Optional[str]]
    inst_zones: List[Optional[str]]
    inst_labels: List[List[str]]
    type_config: Optional[Dict[str, dict]]   # MM_TYPE_CONSTRAINTS document or None
    type_names: List[str]                 # model type names in use (index = model_type[m])
    model_type: np.ndarray                # int32[n_m] index into type_names
    model_last_used: np.ndarray           # int64[n_m]
    model_size: np.ndarray                # int32[n_m]
    model_rpm: np.ndarray                 # int32[n_m]
    edge_off: np.ndarray                  # int64[n_m+1] loaded ∪ failed
    edge_inst: np.ndarray                 # int32[]
    n_loaded: np.ndarray                  # int32[n_m]
    n_failed: np.ndarray                  # int32[n_m]
    replaced_replicasets: List[str] = field(default_factory=list)

    @property
    def n_instances(self) -> int:
        return len(self.inst_rows)

    @property
    def n_models(self) -> int:
        return len(self.model_type)

    def type_json(self) -> Optional[str]:
        return None if self.type_config is None else json.dumps(self.type_config)


def _zipf_weights(n: int, s: float) -> np.ndarray:
    w = 1.0 / np.power(np.arange(1, n + 1, dtype=np.float64), s)
    return w / w.sum()


def make_fleet(config: str, n_models: int, n_instances: int, seed: int) -> SynthFleet:
    """config in {"C1", "C2", "C3", "C5"}; sizes are free so the tests can shrink them."""
    rng = SplitMix(seed)
    now = NOW_MS
    ni, nm = n_instances, n_models
    rows = np.zeros(ni, dtype=INSTANCE_ROW)
    ids, locs, zones, labels = [], [], [], []
    type_config: Optional[Dict[str, dict]] = None
    replaced: List[str] = []

    if config == "C1":
        # DummyModelMesh-like: 10 x 20 MiB capacity, 20 MiB models, nothing loaded yet
        cap, size, min_space, default_size = 25600, 2560, 2560, 2560
        rows["capacity"] = cap - 2560  # unload reserve published out of cap (MM:5373-5378)
        rows["used"] = 0
        rows["lru_time"] = LONG_MAX
        rows["count"] = 0
        rows["l_threads"] = 8
        rows["rpm"] = 0
        rows["active"] = 1
        rows["start_time"] = now - 3_600_000
        ids = [f"mmdemo-{i:05d}" for i in range(ni)]
        locs = [None] * ni
        zones = [None] * ni
        labels = [[] for _ in range(ni)]
        type_names = ["ExampleType"]
        model_type = np.zeros(nm, dtype=np.int32)
        model_size = np.full(nm, size, dtype=np.int32)
        model_last = (now - np.arange(nm, dtype=np.int64) * 1000).astype(np.int64)
        model_rpm = np.zeros(nm, dtype=np.int32)
        edge_off = np.zeros(nm + 1, dtype=np.int64)
        edge_inst = np.zeros(0, dtype=np.int32)
        return SynthFleet(config, now, min_space, 600_000, default_size, rows, ids, locs, zones, labels, None, type_names,
                          model_type, model_last, model_size, model_rpm, edge_off, edge_inst,
                          np.zeros(nm, dtype=np.int32), np.zeros(nm, dtype=np.int32))

    if config == "MIX":
        return _make_mix(nm, ni, seed)
    cap = 4_000_000  # 32 GiB of 8 KiB units
    default_size = 6400
    adversarial = config == "C5"
    min_space = 51200  # max(6400*1, min(6400*8, cap/20)) for 8 loading threads with an unload manager (MM:767-769)
    rows["capacity"] = cap
    u = rng.uniform(ni)
    if adversarial:
        # every instance ~95 % full, remaining uniformly in [0.5, 1.5] * minSpaceUnits (about half "full")
        rem = (min_space * (0.5 + rng.uniform(ni))).astype(np.int64)
        rows["used"] = cap - rem
        rows["lru_time"] = now - 6 * 3_600_000 + rng.randint(ni, -60_000, 60_001)
    else:
        full = u < 0.30
        rem_full = (rng.uniform(ni) * min_space * 0.999).astype(np.int64)
        rem_free = (min_space + rng.uniform(ni) * (0.8 * cap - min_space)).astype(np.int64)
        rem = np.where(full, rem_full, rem_free)
        rows["used"] = cap - rem
        rows["lru_time"] = now - rng.exponential(ni, 6 * 3_600_000.0).astype(np.int64) - 1
    mean_size = 9000.0 if not adversarial else 16000.0
    rows["count"] = np.maximum(0, (rows["used"] / mean_size * (0.8 + 0.4 * rng.uniform(ni)))).astype(np.int32)
    rows["l_threads"] = 8
    rows["l_in_prog"] = np.where(rng.uniform(ni) < 0.2, rng.randint(ni, 1, 4), 0).astype(np.int32)
    zipf_i = _zipf_weights(ni, 1.1)
    perm = np.argsort(rng.u64(ni), kind="stable")
    rows["rpm"] = np.minimum(2_000_000, (zipf_i[perm] * 40_000.0 * ni / 8.0)).astype(np.int32)
    rows["start_time"] = now - rng.randint(ni, 3_600_000, 30 * 86_400_000)
    rows["vers"] = 7
    rows["active"] = 1
    rows["shutting_down"] = 0

    n_rs = max(2, ni // 200)
    rs_names = [f"mm{(0x1000 + k * 0x137) & 0xFFFF:04x}" for k in range(n_rs)]
    rs_of = rng.randint(ni, 0, n_rs)
    ids = [f"{rs_names[int(rs_of[i])]}-{i:05x}" for i in range(ni)]
    zone_pick = rng.randint(ni, 0, 4)
    zones = [None if int(z) == 3 else f"zone-{int(z)}" for z in zone_pick]
    loc_pick = rng.randint(ni, 0, max(2, ni // 8))
    locs = [f"node-{int(l):04d}" for l in loc_pick]

    if config == "C2":
        n_types = 4
        type_names = [f"type-{t}" for t in range(n_types)]
        labels = [[] for _ in range(ni)]
        type_config = None
    else:
        n_types = 32 if config == "C3" else 64
        n_labels = 8 if config == "C3" else 12
        type_names = [f"type-{t:02d}" for t in range(n_types)] + ["untyped"]
        lab_names = [f"lbl-{k:02d}" for k in range(n_labels)]
        # each instance carries 1..3 labels (a "label group" and extras); ~6 % carry none
        l1 = rng.randint(ni, 0, n_labels)
        l2 = rng.randint(ni, 0, n_labels)
        l3 = rng.randint(ni, 0, n_labels)
        nl = rng.randint(ni, 0, 16)
        labels = []
        for i in range(ni):
            k = int(nl[i])
            if k == 0:
                labels.append([])
            elif k < 8:
                labels.append(sorted({lab_names[int(l1[i])]}))
            elif k < 13:
                labels.append(sorted({lab_names[int(l1[i])], lab_names[int(l2[i])]}))
            else:
                labels.append(sorted({lab_names[int(l1[i])], lab_names[int(l2[i])], lab_names[int(l3[i])]}))
        type_config = {}
        pick = rng.randint(n_types, 0, 1 << 30)
        for t in range(n_types):
            p = int(pick[t])
            if config == "C3":
                kind = t % 4  # 25 % required, 25 % preferred, rest unconstrained
                if kind == 0:
                    type_config[type_names[t]] = {"required": [lab_names[p % n_labels]]}
                elif kind == 1:
                    type_config[type_names[t]] = {"preferred": [lab_names[p % n_labels], lab_names[(p >> 8) % n_labels]]}
            else:
                req = sorted({lab_names[p % n_labels], lab_names[(p >> 8) % n_labels]} |
                             ({lab_names[(p >> 16) % n_labels]} if (p >> 24) & 1 else set()))
                ent = {"required": req[:2] if len(req) > 2 and (p >> 25) & 1 else req}
                if t % 2 == 0:
                    ent["preferred"] = [lab_names[(p >> 4) % n_labels]]
                type_config[type_names[t]] = ent
        if config == "C3":
            # 0.5 % of instances shutting down, one replicaset (about 2 % of instances) flagged likely-replaced
            rows["shutting_down"] = (rng.uniform(ni) < 0.005).astype(np.int32)
            replaced = [rs_names[0]]
            rows["active"] = (rng.uniform(ni) >= 0.002).astype(np.int32)

    # ---- models ----
    nt_use = len(type_names)
    model_type = rng.randint(nm, 0, nt_use).astype(np.int32)
    if adversarial:
        model_size = np.where(rng.uniform(nm) < 0.5, 256, 32768).astype(np.int32)
    else:
        model_size = np.exp(np.log(256.0) + rng.uniform(nm) * (np.log(65536.0) - np.log(256.0))).astype(np.int32)
    model_last = (now - rng.exponential(nm, 6 * 3_600_000.0).astype(np.int64) - 1).astype(np.int64)
    # a few never-used (0) and very old (> 5 days) models
    r = rng.uniform(nm)
    model_last = np.where(r < 0.01, 0, np.where(r < 0.05, now - 6 * 86_400_000, model_last)).astype(np.int64)
    zipf_m = _zipf_weights(nm, 1.1)
    model_rpm = np.minimum(1_000_000, zipf_m[np.argsort(rng.u64(nm), kind="stable")] * 5.0e6).astype(np.int32)
    r = rng.uniform(nm)
    n_loaded = np.where(r < 0.40, 0, np.where(r < 0.97, 1, 2)).astype(np.int32)
    r = rng.uniform(nm)
    n_failed = np.where(r < 0.97, 0, np.where(r < 0.995, 1, 2)).astype(np.int32)
    r = rng.uniform(nm)
    n_loaded = np.where(r < 0.002, 6, n_loaded).astype(np.int32)  # a few widely replicated models (> 4 inline edges)
    deg = (n_loaded + n_failed).astype(np.int64)
    edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(deg, out=edge_off[1:])
    ne = int(edge_off[-1])
    edge_inst = rng.randint(ne, 0, ni).astype(np.int32)
    # make edges of one model distinct by shifting duplicates (cheap, deterministic)
    for _ in range(3):
        if ne == 0:
            break
        owner = np.repeat(np.arange(nm, dtype=np.int64), deg)
        key = owner * ni + edge_inst
        order = np.argsort(key, kind="stable")
        dup = np.zeros(ne, dtype=bool)
        dup[order[1:]] = key[order[1:]] == key[order[:-1]]
        if not dup.any():
            break
        edge_inst = np.where(dup, (edge_inst + 1 + np.arange(ne) % 7) % ni, edge_inst).astype(np.int32)

    return SynthFleet(config, now, min_space, 600_000, default_size, rows, ids, locs, zones, labels, type_config,
                      type_names, model_type, model_last, model_size, model_rpm, edge_off, edge_inst, n_loaded, n_failed,
                      replaced)


def _make_mix(nm: int, ni: int, seed: int) -> SynthFleet:
    """Regime-randomised small fleets that reach the rarely taken branches of getNext: all-full fleets with close LRU
    times (long full-case shortlists, non-simple case (b)), low counts (long non-full shortlists), large preferred
    sets, a replaced replicaset that covers every allowed instance of some types (filter retry), equal sort keys."""
    rng = SplitMix(seed * 7919 + 13)
    now = NOW_MS
    pick = [int(x) for x in rng.randint(12, 0, 1 << 30)]
    frac_full = [0.0, 0.35, 1.0, 0.9][pick[0] % 4]
    cmax = [6, 14, 200, 11][pick[1] % 4]
    lru_spread = [20_000, 200_000, 4 * 3_600_000][pick[2] % 3]
    cap, default_size, min_space = 1_000_000, 2000, 16_000
    rows = np.zeros(ni, dtype=INSTANCE_ROW)
    rows["capacity"] = cap
    full = rng.uniform(ni) < frac_full
    rem = np.where(full, rng.randint(ni, 0, min_space), rng.randint(ni, min_space, cap // 2))
    if pick[3] % 3 == 0:  # coarse remaining values -> many ties further down the comparator
        rem = (rem // 50_000) * 50_000 + np.where(full, 0, min_space)
    rows["used"] = cap - rem
    base = now - [60_000, 3_600_000, 86_400_000][pick[4] % 3]
    rows["lru_time"] = base + rng.randint(ni, -lru_spread, lru_spread + 1)
    rows["lru_time"] = np.where(rng.uniform(ni) < 0.03, LONG_MAX, rows["lru_time"])
    rows["count"] = rng.randint(ni, 0, cmax + 1).astype(np.int32)
    rows["l_threads"] = np.where(rng.uniform(ni) < 0.5, 8, 4).astype(np.int32)
    rows["l_in_prog"] = rng.randint(ni, 0, 3).astype(np.int32)
    rows["rpm"] = np.where(rng.uniform(ni) < 0.4, rng.randint(ni, 0, 90), rng.randint(ni, 90, 3000)).astype(np.int32)
    rows["start_time"] = now - rng.randint(ni, 60_000, 86_400_000)
    rows["vers"] = 3
    rows["active"] = (rng.uniform(ni) >= 0.03).astype(np.int32)
    rows["shutting_down"] = (rng.uniform(ni) < 0.02).astype(np.int32)
    rs_names = ["rsaaaa", "rsbbbb", "rscccc"]
    rs_of = rng.randint(ni, 0, 3)
    ids = [(f"{rs_names[int(rs_of[i])]}-{i:04x}" if i % 17 else f"s{i:x}") for i in range(ni)]  # some ids shorter than 7
    zones = [None if int(z) == 2 else f"z{int(z)}" for z in rng.randint(ni, 0, 3)]
    locs = [None if int(z) == 4 else f"n{int(z)}" for z in rng.randint(ni, 0, 5)]
    n_labels, n_types = 5, 10
    lab_names = [f"L{k}" for k in range(n_labels)]
    lb = rng.randint(ni * 3, 0, n_labels).reshape(ni, 3)
    nl = rng.randint(ni, 0, 8)
    labels = []
    for i in range(ni):
        k = int(nl[i])
        labels.append([] if k == 0 else sorted({lab_names[int(x)] for x in lb[i, : (1 if k < 4 else 2 if k < 7 else 3)]}))
    type_names = [f"t{t}" for t in range(n_types)] + ["other"]
    type_config: Optional[Dict[str, dict]] = {}
    tp = rng.randint(n_types, 0, 1 << 30)
    for t in range(n_types):
        p = int(tp[t])
        kind = p % 5
        a, b, c = lab_names[(p >> 3) % n_labels], lab_names[(p >> 7) % n_labels], lab_names[(p >> 11) % n_labels]
        if kind == 0:
            type_config[type_names[t]] = {"required": [a]}
        elif kind == 1:
            type_config[type_names[t]] = {"preferred": [a, b]}
        elif kind == 2:
            type_config[type_names[t]] = {"required": [a], "preferred": [b, c]}
        elif kind == 3:
            type_config[type_names[t]] = {"required": [a, b]}
        # kind 4: unconstrained
    if pick[5] % 4 == 0:
        type_config["_default"] = {"preferred": [lab_names[pick[6] % n_labels]]}
    if pick[7] % 5 == 0:
        type_config = None
        labels = [[] for _ in range(ni)]
    replaced = [["rsaaaa"], ["rsaaaa", "rsbbbb"], [], ["rsaaaa", "rsbbbb", "rscccc"]][pick[8] % 4]

    model_type = rng.randint(nm, 0, len(type_names)).astype(np.int32)
    model_size = rng.randint(nm, 100, 40_000).astype(np.int32)
    r = rng.uniform(nm)
    model_last = np.where(r < 0.05, 0, np.where(r < 0.15, now - 6 * 86_400_000,
                          now - rng.randint(nm, 0, 2 * 86_400_000))).astype(np.int64)
    model_rpm = rng.randint(nm, 0, 1000).astype(np.int32)
    n_loaded = np.where(rng.uniform(nm) < 0.5, 0, rng.randint(nm, 1, 4)).astype(np.int32)
    n_loaded = np.where(rng.uniform(nm) < 0.03, min(ni, 9), n_loaded).astype(np.int32)
    n_failed = np.where(rng.uniform(nm) < 0.9, 0, rng.randint(nm, 1, 3)).astype(np.int32)
    deg = np.minimum(ni, n_loaded + n_failed).astype(np.int64)
    edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(deg, out=edge_off[1:])
    ne = int(edge_off[-1])
    start = rng.randint(nm, 0, ni)
    owner = np.repeat(np.arange(nm, dtype=np.int64), deg)
    within = np.arange(ne, dtype=np.int64) - edge_off[owner]
    stride = 1 + (pick[9] % 3)
    edge_inst = ((start[owner] + within * stride) % ni).astype(np.int32)
    if stride > 1:  # keep edges of a model distinct
        edge_inst = ((start[owner] + within) % ni).astype(np.int32) if ni % stride == 0 else edge_inst
    return SynthFleet("MIX", now, min_space, 600_000, default_size, rows, ids, locs, zones, labels, type_config,
                      type_names, model_type, model_last, model_size, model_rpm, edge_off, edge_inst, n_loaded, n_failed,
                      replaced)


@dataclass
class SynthDecisions:
    dec: np.ndarray          # DECISION_IN[n]
    fresh: np.ndarray        # INSTANCE_ROW[n_fresh]
    extra: np.ndarray        # int32[]


def make_decisions(fl: SynthFleet, n: int, seed: int, sweep: bool = False, plain: bool = False) -> SynthDecisions:
    """n getNext calls.  sweep=True: decision i is for model i % n_models (a reaper-style pass over the registry).
    plain=True: no fresh overrides, no extra excludes, last_used from the model row (the bench workload)."""
    rng = SplitMix(seed ^ 0xDEC1510)
    ni, nm = fl.n_instances, fl.n_models
    dec = np.zeros(n, dtype=DECISION_IN)
    dec["model"] = (np.arange(n) % nm) if sweep else rng.randint(n, 0, nm)
    live = np.nonzero(fl.inst_rows["shutting_down"] == 0)[0]
    dec["self"] = live[rng.randint(n, 0, len(live))]
    fav = rng.uniform(n) < 0.3
    if plain:
        dec["flags"] = np.where(fav, DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(DF_MODEL_LAST_USED)
        dec["fresh"] = -1
        return SynthDecisions(dec, np.zeros(0, dtype=INSTANCE_ROW), np.zeros(0, dtype=np.int32))
    r = rng.uniform(n)
    use_model = r < 0.6
    lu = np.where(r < 0.7, fl.now_ms + 20_000,                       # load-triggered scale-up (MM:5675)
         np.where(r < 0.8, 0,                                         # "now"
         np.where(r < 0.9, fl.now_ms - rng.randint(n, 0, 3_000_000),  # recently used
                  fl.now_ms - 7 * 86_400_000)))                       # older than five days
    dec["last_used"] = lu
    dec["flags"] = (np.where(fav, DF_FAVOUR_SELF, 0) | np.where(use_model, DF_MODEL_LAST_USED, 0)).astype(np.uint32)
    # fresh rows for a subset of the instances: published row drifted a little, rpm 0 as the reference leaves it,
    # except a few with a non-zero rpm to exercise the filter arithmetic
    n_fresh = max(1, min(ni, 64))
    fresh_inst = live[rng.randint(n_fresh, 0, len(live))]
    fresh = fl.inst_rows[fresh_inst].copy()
    drift = rng.randint(n_fresh, -200_000, 200_001)
    fresh["used"] = np.clip(fresh["used"] + drift, 0, fresh["capacity"])
    fresh["count"] = np.maximum(0, fresh["count"] + rng.randint(n_fresh, -3, 4)).astype(np.int32)
    bump = rng.randint(n_fresh, 0, 120_000)
    lru0 = fresh["lru_time"].copy()
    fresh["lru_time"] = np.where((rng.uniform(n_fresh) < 0.1) | (lru0 > LONG_MAX - 200_000), LONG_MAX,
                                 np.minimum(lru0, LONG_MAX - 200_000) + bump)
    fresh["rpm"] = np.where(rng.uniform(n_fresh) < 0.25, rng.randint(n_fresh, 0, 5000), 0).astype(np.int32)
    if fl.name == "MIX":  # decouple the caller's fresh state from its published row
        wide = rng.uniform(n_fresh) < 0.5
        fresh["used"] = np.where(wide, rng.randint(n_fresh, 0, int(fresh["capacity"].max()) + 1), fresh["used"])
        fresh["used"] = np.minimum(fresh["used"], fresh["capacity"])
        fresh["count"] = np.where(wide, rng.randint(n_fresh, 0, 20), fresh["count"]).astype(np.int32)
    # decisions whose self has a fresh row use it half of the time
    slot_of = np.full(ni, -1, dtype=np.int64)
    slot_of[fresh_inst] = np.arange(n_fresh)
    s = slot_of[dec["self"]]
    dec["fresh"] = np.where((s >= 0) & (rng.uniform(n) < 0.7), s, -1).astype(np.int32)
    # extra excludes (tried-this-request ∪ explicit): 12 % of decisions carry 1..3, sometimes self
    k = np.where(rng.uniform(n) < 0.12, rng.randint(n, 1, 4), 0).astype(np.int32)
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(k, out=off[1:])
    extra = rng.randint(int(off[-1]), 0, ni).astype(np.int32)
    selfx = rng.uniform(int(off[-1])) < 0.15
    owner = np.repeat(np.arange(n), k)
    extra = np.where(selfx, dec["self"][owner], extra).astype(np.int32)
    dec["extra_off"] = off[:-1].astype(np.int32)
    dec["extra_n"] = k
    return SynthDecisions(dec, fresh, extra)


# ---------------------------------------------------------------------------------------------------------------
# feeding a solver (libmmplace or the CPU harness) — product-side helper, no oracle involved
# ---------------------------------------------------------------------------------------------------------------
def load_into_fleet(fl: SynthFleet, fleet, bulk_chunk: int = 1 << 18) -> Dict[str, int]:
    """Ingest a SynthFleet through the C ABI and commit.  Returns {type name: type id}."""
    fleet.types_set_json(fl.type_json())
    tid = {t: fleet.type_id(t) for t in fl.type_names}
    fleet.replicasets_set(fl.replaced_replicasets)
    for i in range(fl.n_instances):
        fleet.instance_upsert(i, fl.inst_rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i])
    rows = np.zeros(fl.n_models, dtype=MODEL_ROW)
    rows["last_used"] = fl.model_last_used
    rows["size_units"] = fl.model_size
    rows["rpm"] = fl.model_rpm
    tmap = np.asarray([tid[t] for t in fl.type_names], dtype=np.uint16)
    rows["type_id"] = tmap[fl.model_type]
    rows["copy_count"] = np.minimum(255, fl.n_loaded)
    rows["fail_count"] = np.minimum(255, fl.n_failed)
    for lo in range(0, fl.n_models, bulk_chunk):
        hi = min(fl.n_models, lo + bulk_chunk)
        off = fl.edge_off[lo:hi + 1] - fl.edge_off[lo]
        fleet.models_bulk(lo, rows[lo:hi], off, fl.edge_inst[fl.edge_off[lo]:fl.edge_off[hi]])
    fleet.commit()
    return tid


# ---------------------------------------------------------------------------------------------------------------
# C4: the churn workload (BASELINE.json configs[3], SURVEY.md §8d): a fleet at steady state (caches filled to `fill`), then a
# Poisson trace of requests -- cache hits on loaded models (Zipf), cache misses on unloaded ones (-> placement + load +
# evictions), removals -- in republish windows of 2 s.
# ---------------------------------------------------------------------------------------------------------------
@dataclass
class ChurnWorkload:
    fleet: SynthFleet
    capacity: np.ndarray          # int64[n_i] cache capacity per instance (= published capacity)
    seed_instance: np.ndarray     # resident copies at the start: instance, model, lastUsed, weight, registration time
    seed_model: np.ndarray
    seed_last_used: np.ndarray
    seed_weight: np.ndarray
    seed_load_ts: np.ndarray
    loaded_models: np.ndarray     # model ids with a copy at the start (hot set of the trace), hottest first
    unloaded_models: np.ndarray
    load_timeout_ms: int
    window_ms: int = 2000

    def events(self, epoch: int, n: int, seed: int, hit=0.70, miss=0.25):
        """Window `epoch` of the trace: n events sorted by time.  hit / miss / (rest = remove) fractions as SURVEY.md §8d."""
        from ._lib import CHURN_EVENT
        rng = SplitMix((seed * 1_000_003 + epoch) ^ 0xC4C4)
        fl = self.fleet
        now0 = fl.now_ms + epoch * self.window_ms
        ev = np.zeros(n, dtype=CHURN_EVENT)
        r = rng.uniform(n)
        kind = np.where(r < hit, 0, np.where(r < hit + miss, 1, 2))
        nl, nu = len(self.loaded_models), len(self.unloaded_models)
        # Zipf(1.1) over the loaded models by inverse-CDF on a precomputed table
        if not hasattr(self, "_zipf_cdf"):
            w = 1.0 / np.power(np.arange(1, nl + 1, dtype=np.float64), 1.1)
            self._zipf_cdf = np.cumsum(w / w.sum())
        hot = np.minimum(nl - 1, np.searchsorted(self._zipf_cdf, rng.uniform(n)))
        cold = rng.randint(n, 0, max(1, nu))
        anym = rng.randint(n, 0, fl.n_models)
        ev["model"] = np.where(kind == 0, self.loaded_models[hot], np.where(kind == 1, self.unloaded_models[cold % max(1, nu)], anym))
        ev["type"] = np.where(kind == 2, 1, 0)
        live = np.nonzero(fl.inst_rows["shutting_down"] == 0)[0]
        ev["caller"] = live[rng.randint(n, 0, len(live))]
        ev["u"] = (rng.u64(n) >> np.uint64(33)).astype(np.uint32)
        ev["t"] = now0 + np.sort(rng.randint(n, 0, self.window_ms))
        return ev


def make_churn(n_models: int, n_instances: int, seed: int, fill: float = 0.97, with_types: bool = False) -> ChurnWorkload:
    rng = SplitMix(seed ^ 0xC4)
    now = NOW_MS
    ni, nm = n_instances, n_models
    default_size = 6400
    model_size = np.exp(np.log(256.0) + rng.uniform(nm) * (np.log(65536.0) - np.log(256.0))).astype(np.int32)
    mean = float(model_size.mean())
    # ~70 % of the models resident once: capacity so that `fill` of it holds an even share of them
    cap = int(0.70 * nm * mean / ni / fill)
    cap = max(cap, 4 * 65536)
    min_space = max(default_size, min(default_size * 8, cap // 20))  # MM:767-769, 8 loading threads, unload manager
    perm = np.argsort(rng.u64(nm), kind="stable").astype(np.int64)
    # fill instance after instance with the shuffled models until `fill` of the capacity is used
    sizes = model_size[perm].astype(np.int64)
    csum = np.cumsum(sizes)
    target = int(fill * cap)
    inst_of = np.full(nm, -1, dtype=np.int64)
    start, pos = 0, 0
    for i in range(ni):
        if pos >= nm:
            break
        base = csum[pos - 1] if pos > 0 else 0
        end = int(np.searchsorted(csum, base + target, side="right"))
        end = max(end, pos)
        inst_of[pos:end] = i
        pos = end
    n_res = pos
    res_models = perm[:n_res]
    res_inst = inst_of[:n_res]
    last_used = (now - rng.exponential(n_res, 6 * 3_600_000.0).astype(np.int64) - 1 - np.arange(n_res) % 997).astype(np.int64)
    # 5 % of the resident models get a second copy on another instance (evicting nothing: only where it still fits)
    used = np.bincount(res_inst, weights=model_size[res_models].astype(np.float64), minlength=ni).astype(np.int64)
    second = np.nonzero(rng.uniform(n_res) < 0.05)[0]
    s_inst, s_model, s_lu = [], [], []
    other = rng.randint(len(second), 0, ni)
    for k, j in enumerate(second):
        m = int(res_models[j])
        i2 = int(other[k])
        if i2 == int(res_inst[j]) or used[i2] + model_size[m] > cap:
            continue
        used[i2] += model_size[m]
        s_inst.append(i2); s_model.append(m); s_lu.append(int(last_used[j]) + 7)
    seed_instance = np.concatenate([res_inst, np.asarray(s_inst, dtype=np.int64)]).astype(np.int32)
    seed_model = np.concatenate([res_models, np.asarray(s_model, dtype=np.int64)]).astype(np.int32)
    seed_lu = np.concatenate([last_used, np.asarray(s_lu, dtype=np.int64)]).astype(np.int64)
    seed_w = model_size[seed_model].astype(np.int32)
    load_timeout = 30_000
    seed_lt = np.full(len(seed_model), now - 3 * 3_600_000, dtype=np.int64)
    # registry: edges = loaded copies in seeding order per model
    order = np.argsort(seed_model, kind="stable")
    n_loaded = np.bincount(seed_model, minlength=nm).astype(np.int32)
    edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(n_loaded, out=edge_off[1:])
    edge_inst = seed_instance[order].astype(np.int32)
    # instance records as each pod would publish them (getFreshInstanceRecord MM:5369-5386)
    rows = np.zeros(ni, dtype=INSTANCE_ROW)
    rows["capacity"] = cap
    rows["used"] = used
    cnt = np.bincount(seed_instance, minlength=ni)
    rows["count"] = cnt
    oldest = np.full(ni, LONG_MAX, dtype=np.int64)
    np.minimum.at(oldest, seed_instance, seed_lu)
    rows["lru_time"] = oldest
    rows["l_threads"] = 8
    rows["rpm"] = rng.randint(ni, 0, 3000)
    rows["start_time"] = now - rng.randint(ni, 3_600_000, 30 * 86_400_000)
    rows["vers"] = 7
    rows["active"] = 1
    ids = [f"mmc4{(i * 7919) % 9973:04d}-{i:05x}" for i in range(ni)]
    zones = [None if i % 4 == 3 else f"zone-{i % 4}" for i in range(ni)]
    locs = [f"node-{i // 8:04d}" for i in range(ni)]
    type_config: Optional[Dict[str, dict]] = None
    type_names = [f"type-{t}" for t in range(4)]
    labels: List[List[str]] = [[] for _ in range(ni)]
    if with_types:  # a quarter of the types is pinned to half of the fleet: two partitions, subset stats in the rebalance rule
        labels = [(["gpu"] if i % 2 == 0 else []) for i in range(ni)]
        type_config = {"type-0": {"required": ["gpu"]}, "type-1": {"preferred": ["gpu"]}}
    model_type = rng.randint(nm, 0, 4).astype(np.int32)
    model_last = np.zeros(nm, dtype=np.int64)
    model_last[seed_model] = seed_lu
    model_last = np.where(model_last == 0, now - rng.exponential(nm, 12 * 3_600_000.0).astype(np.int64) - 1, model_last).astype(np.int64)
    fl = SynthFleet("C4", now, min_space, 600_000, default_size, rows, ids, locs, zones, labels, type_config, type_names, model_type,
                    model_last, model_size, np.zeros(nm, dtype=np.int32), edge_off, edge_inst, n_loaded, np.zeros(nm, dtype=np.int32), [])
    loaded = np.nonzero(n_loaded > 0)[0]
    hot_order = loaded[np.argsort(rng.u64(len(loaded)), kind="stable")]
    unloaded = np.nonzero(n_loaded == 0)[0]
    return ChurnWorkload(fl, rows["capacity"].astype(np.int64).copy(), seed_instance, seed_model, seed_lu, seed_w, seed_lt, hot_order,
                         unloaded, load_timeout)


def make_churn_overflow(w: ChurnWorkload, frac: float, seed: int, regs=(5, 12)) -> ChurnWorkload:
    """`w` with about `frac` of its models holding more registrations than the four inline ones.  A chosen model with a copy
    gets further copies on other instances where they fit the caches (seeded resident, registered after its first copies) and
    failed loads for the rest, regs[0]..regs[1] registrations in all; a chosen model without a copy gets failed loads only:
    every other one exactly four, so that its first load makes a fifth registration, the rest regs[0]..regs[1].  Its own
    random stream: `w`'s fleet, seeds and event trace stay as they are for the models not chosen."""
    rng = SplitMix(seed ^ 0x0F5C4)
    fl = w.fleet
    nm, ni = fl.n_models, fl.n_instances
    chosen = np.nonzero(rng.uniform(nm) < frac)[0]
    target = rng.randint(len(chosen), regs[0], regs[1] + 1)
    start = rng.randint(len(chosen), 0, ni)
    rows = fl.inst_rows.copy()
    used = rows["used"].astype(np.int64)
    lu_of = fl.model_last_used
    new_lists, s_inst, s_model, s_lu = {}, [], [], []
    for k, m in enumerate(chosen):
        m = int(m)
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        loaded = [int(x) for x in fl.edge_inst[a:a + int(fl.n_loaded[m])]]
        failed = [int(x) for x in fl.edge_inst[a + int(fl.n_loaded[m]):b]]
        want = int(target[k]) if loaded or k % 2 else 4
        size = int(fl.model_size[m])
        taken = set(loaded) | set(failed)
        for j in range(ni):
            if len(loaded) + len(failed) >= want:
                break
            i = (int(start[k]) + j) % ni
            if i in taken:
                continue
            taken.add(i)
            if loaded and used[i] + size <= w.capacity[i]:  # another resident copy
                used[i] += size
                loaded.append(i)
                s_inst.append(i); s_model.append(m); s_lu.append(int(lu_of[m]) - 11 * len(loaded))
            else:
                failed.append(i)
        new_lists[m] = (loaded, failed)
    n_loaded = fl.n_loaded.copy()
    n_failed = fl.n_failed.copy()
    for m, (ld, fd) in new_lists.items():
        n_loaded[m], n_failed[m] = len(ld), len(fd)
    cnt = (n_loaded + n_failed).astype(np.int64)
    edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(cnt, out=edge_off[1:])
    edge_inst = np.full(int(edge_off[-1]), -1, dtype=np.int32)
    old_cnt = np.diff(fl.edge_off)
    keep = np.ones(nm, dtype=bool)
    keep[chosen] = False
    owner = np.repeat(np.arange(nm), old_cnt)
    sel = keep[owner]
    pos = np.arange(len(fl.edge_inst)) - fl.edge_off[owner]
    edge_inst[(edge_off[owner] + pos)[sel]] = fl.edge_inst[sel]
    for m, (ld, fd) in new_lists.items():
        edge_inst[edge_off[m]:edge_off[m + 1]] = ld + fd
    s_inst_a, s_model_a = np.asarray(s_inst, dtype=np.int32), np.asarray(s_model, dtype=np.int32)
    s_lu_a = np.asarray(s_lu, dtype=np.int64)
    rows["used"] = used
    rows["count"] += np.bincount(s_inst_a, minlength=ni).astype(rows["count"].dtype)
    oldest = rows["lru_time"].astype(np.int64)
    np.minimum.at(oldest, s_inst_a, s_lu_a)
    rows["lru_time"] = oldest
    fl2 = SynthFleet(fl.name, fl.now_ms, fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, rows, fl.inst_ids,
                     fl.inst_locs, fl.inst_zones, fl.inst_labels, fl.type_config, fl.type_names, fl.model_type, fl.model_last_used,
                     fl.model_size, fl.model_rpm, edge_off, edge_inst, n_loaded, n_failed, fl.replaced_replicasets)
    return ChurnWorkload(fl2, w.capacity, np.concatenate([w.seed_instance, s_inst_a]), np.concatenate([w.seed_model, s_model_a]),
                         np.concatenate([w.seed_last_used, s_lu_a]), np.concatenate([w.seed_weight, fl.model_size[s_model_a].astype(np.int32)]),
                         np.concatenate([w.seed_load_ts, np.full(len(s_inst_a), fl.now_ms - 3 * 3_600_000, dtype=np.int64)]),
                         w.loaded_models, w.unloaded_models, w.load_timeout_ms, w.window_ms)
