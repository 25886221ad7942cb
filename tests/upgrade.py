"""Fleets in a rolling upgrade, some pods on a newer instance version (tests/test_rolling_upgrade_gpu.py says what that
changes): upgrade() and fleet_for() build them, bump() moves a replayed stream's pods to a new version, and the checks read
the comparator's total order and the decisions whose best is full."""
import dataclasses

import numpy as np

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthFleet, make_fleet
from oracle import binding as ob
from replay import Replay

PATTERNS = ("canary", "half", "rsroll", "saturated", "three")
NEW_RS = "mmupgr"  # the replicaset prefix of the pods an rsroll upgrade brings up


def upgrade(fl: SynthFleet, pattern: str, seed: int) -> SynthFleet:
    """fl with some of its pods moved to newer versions:
      canary     one to three live pods on vers + 1
      half       about half of the pods, drawn at random
      rsroll     up to a tenth of the pods, drawn among those without labels, on vers + 1 under the new replicaset
                 prefix NEW_RS; every old prefix is listed as likely-replaced (UpgradeTracker, MM:4769-4770): a type that
                 requires a label has every candidate flagged, and the candx filter is retried across the boundary
      saturated  about a third of the pods on vers + 1, every one of them full with an lruTime hours old: the best is
                 full and non-full older pods follow it
      three      three versions (about 50 / 30 / 20 %)
    Every full instance keeps an lruTime above 2 * minChurnAgeMs, so the comparator stays a strict total order."""
    rng = np.random.default_rng(seed ^ 0x5EED)
    rows = fl.inst_rows.copy()
    ni = len(rows)
    v0 = int(rows["vers"][0])
    assert (rows["vers"] == v0).all()
    ids, replaced = list(fl.inst_ids), list(fl.replaced_replicasets)
    live = np.nonzero(rows["shutting_down"] == 0)[0]
    if pattern == "canary":
        rows["vers"][rng.choice(live, size=int(rng.integers(1, 4)), replace=False)] = v0 + 1
    elif pattern == "half":
        rows["vers"][rng.uniform(size=ni) < 0.5] = v0 + 1
    elif pattern == "rsroll":
        pool = [int(i) for i in live if not fl.inst_labels[i]] or list(live)
        new = rng.choice(pool, size=max(1, min(len(pool), ni // 10)), replace=False)
        rows["vers"][new] = v0 + 1
        for i in new:
            ids[i] = f"{NEW_RS}-{i:05x}"
        replaced = sorted({ids[i][:6] for i in range(ni) if len(ids[i]) >= 7 and not ids[i].startswith(NEW_RS)})
    elif pattern == "saturated":
        new = np.nonzero(rng.uniform(size=ni) < 0.33)[0]
        rows["vers"][new] = v0 + 1
        rows["used"][new] = rows["capacity"][new] - rng.integers(0, fl.min_space_units, size=len(new))
        rows["lru_time"][new] = fl.now_ms - rng.integers(3_600_000, 12 * 3_600_000, size=len(new))
    elif pattern == "three":
        u = rng.uniform(size=ni)
        rows["vers"] = v0 + (u < 0.5) + (u < 0.2)
    else:
        raise ValueError(pattern)
    return dataclasses.replace(fl, inst_rows=rows, inst_ids=ids, replaced_replicasets=replaced)


def fleet_for(config: str, nm: int, ni: int, seed: int) -> SynthFleet:
    """make_fleet(config) or, for "BASE/pattern", make_fleet(BASE) in that rolling upgrade"""
    base, _, pattern = config.partition("/")
    fl = make_fleet(base, nm, ni, seed)
    return upgrade(fl, pattern, seed) if pattern else fl


def check_total_order(fl: SynthFleet, o: ob.OracleFleet, seed: int, n: int = 3000):
    """No full live instance at or below 2 * minChurnAgeMs (N1's non-transitive corner), and the oracle's comparator
    is antisymmetric and transitive on sampled triples of live instances."""
    r = fl.inst_rows
    live = np.nonzero(r["shutting_down"] == 0)[0]
    full = (np.maximum(0, r["capacity"] - r["used"]) < fl.min_space_units)[live]
    assert not (full & (r["lru_time"][live] <= 2 * fl.min_churn_age_ms)).any()
    rng = np.random.default_rng(seed)
    for a, b, c in live[rng.integers(0, len(live), size=(n, 3))]:
        a, b, c = int(a), int(b), int(c)
        if len({a, b, c}) < 3:
            continue
        ab, bc, ac = o.compare(a, b), o.compare(b, c), o.compare(a, c)
        assert np.sign(ab) == -np.sign(o.compare(b, a)) != 0, (a, b)
        if ab < 0 and bc < 0:
            assert ac < 0, (a, b, c)
        if ab > 0 and bc > 0:
            assert ac > 0, (a, b, c)


def versions(fl: SynthFleet) -> np.ndarray:
    return np.unique(fl.inst_rows["vers"][fl.inst_rows["shutting_down"] == 0])


def full_best_then_room(fl: SynthFleet, tr: np.ndarray, out: np.ndarray) -> int:
    """decisions whose best is full and whose answer is an instance with room: non-full candidates after a full best"""
    r = fl.inst_rows
    t = out["target"]
    ok = (t >= 0) & ((tr["flags"] & L.TF_BEST_FULL) != 0)
    room = np.zeros(len(t), dtype=bool)
    room[ok] = (r["capacity"][t[ok]] - r["used"][t[ok]]) >= fl.min_space_units
    return int(np.count_nonzero(room))


def bump(rp: Replay, idx, vers: int):
    """mmp_instance_update with a new version and nothing else changed (the same pod, restarted on a new image)"""
    for i in np.atleast_1d(idx):
        r = rp.rows[int(i)].copy()
        r["vers"] = vers
        rp.f.instance_update(int(i), r)
        rp.rows[int(i)] = r
