"""Edge fleets for the placement decision: small hand-ranked fleets and hand-made decisions whose values sit on both sides
of every threshold where getNext's answer changes (MM:4811-4986) -- the caller-record cut (N2), the count cut, the full
best's lruTime distance, non-simple case (b)'s distance and its own-rpm filter, and the rpm filter's bands.

Every fleet starts from make_fleet("C2") (no type constraints unless a case asks for a preferred label) and has its
instance rows overwritten so that PLACEMENT_ORDER puts pod r at rank r: pods with room by count ascending, remaining
descending, lruTime ascending; full pods after them by lruTime.  Instance indices are a shuffle of the ranks, and one extra
instance is shutting down (a "ghost" that is not in the order): a decision whose self is the ghost carries its own fresh
record and has no self rank, so the two-pass path can answer it from a slot summary.

A Case lists, besides the fleet and its decisions, the answers the fleet was built to give (`expect`: decision ->
n_candidates) and pairs of decisions on the two sides of one threshold, which must get different answers (`pairs`).
Both are checked against the oracle, so a builder mistake that moves a case off its threshold fails instead of testing
nothing."""
from __future__ import annotations

import dataclasses
from typing import Dict, List, Optional, Tuple

import numpy as np

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import LONG_MAX, NOW_MS, SynthDecisions, SynthFleet, make_fleet

CAP = 4_000_000
MS = 51_200  # C2's minSpaceUnits
NOW = NOW_MS
LONG_MIN = -(1 << 63)
# lastUsed ages at the rpm filter's band edges (MM:4966-4974) and the five-day cut (MM:4960)
AGO_EDGES = (-1001, -1000, -999, 4_999, 5_000, 5_001, 719_999, 720_000, 86_399_999, 86_400_000, 431_999_999, 432_000_000)


@dataclasses.dataclass
class Pod:
    count: int
    rem: int
    lru: int
    rpm: int = 0
    pref: bool = False


@dataclasses.dataclass
class Case:
    family: str
    name: str
    fl: SynthFleet
    sd: SynthDecisions
    order: np.ndarray                          # instance index by intended rank
    ghost: int                                 # the shutting-down instance
    expect: Dict[int, int] = dataclasses.field(default_factory=dict)            # decision -> n_candidates
    pairs: List[Tuple[int, int, str]] = dataclasses.field(default_factory=list)  # decisions either side of a threshold
    summarised: bool = False                   # built so that the two-pass path answers some decisions from summaries

    @property
    def id(self):
        return f"{self.family}:{self.name}"


def edge_fleet(pods: List[Pod], n_models: int, seed: int, preferred: bool = False, model_last_used=None,
               edges: Optional[Dict[int, List[int]]] = None):
    """The C2 fleet whose live pods are `pods` in rank order (instance index order[r] for rank r) plus one shutting-down
    ghost at the last index.  preferred: every model is of type-1, whose preferred instances are the pods with pref.  A
    type without required labels has the inferred default preference (quirk N11, TCM:706-707): the instances that no
    type's configured preferred set holds.  So type-1 is configured to prefer a label that only the pods WITHOUT pref
    carry, which makes them the configured set and the others the preferred ones.
    edges: model -> ranks of its registered instances (four inline, the rest in the overflow list)."""
    n = len(pods)
    fl = make_fleet("C2", n_models, n + 1, seed)
    order = np.random.default_rng(seed).permutation(n).astype(np.int32)
    ghost = n
    rows = fl.inst_rows
    rows["capacity"] = CAP
    rows["l_threads"] = 8
    rows["l_in_prog"] = 0
    rows["vers"] = 7
    rows["active"] = 1
    rows["shutting_down"] = 0
    labels = [[] for _ in range(n + 1)]
    for r, p in enumerate(pods):
        i = int(order[r])
        if preferred and not p.pref:
            labels[i] = ["not-preferred"]
        rows["used"][i] = CAP - p.rem
        rows["lru_time"][i] = p.lru
        rows["count"][i] = p.count
        rows["rpm"][i] = p.rpm
    rows["used"][ghost] = 0
    rows["lru_time"][ghost] = LONG_MAX
    rows["count"][ghost] = 0
    rows["rpm"][ghost] = 0
    rows["shutting_down"][ghost] = 1
    fl.inst_labels = labels
    if preferred:
        fl.type_config = {"type-1": {"preferred": ["not-preferred"]}}
    fl.model_type = np.full(n_models, 1 if preferred else 0, dtype=np.int32)
    fl.model_last_used = np.asarray(model_last_used if model_last_used is not None else [NOW - 1000] * n_models, dtype=np.int64)
    fl.model_rpm = np.zeros(n_models, dtype=np.int32)
    e = [[int(order[r]) for r in (edges or {}).get(m, [])] for m in range(n_models)]
    fl.edge_off = np.zeros(n_models + 1, dtype=np.int64)
    np.cumsum([len(x) for x in e], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([x for xs in e for x in xs], dtype=np.int32)
    fl.n_loaded = np.asarray([len(x) for x in e], dtype=np.int32)
    fl.n_failed = np.zeros(n_models, dtype=np.int32)
    return fl, order, ghost


class Decisions:
    """hand-made decisions and the fresh records they carry"""

    def __init__(self):
        self.rows, self.fresh = [], []

    def fresh_row(self, rem: int = CAP, lru: int = NOW - 1000, count: int = 0, rpm: int = 0) -> int:
        """a caller's record; rem < 0 publishes used > capacity, which reads as no free space"""
        f = np.zeros(1, dtype=L.INSTANCE_ROW)
        f["capacity"] = CAP
        f["used"] = CAP - rem
        f["lru_time"] = lru
        f["count"] = count
        f["rpm"] = rpm
        f["l_threads"] = 8
        f["vers"] = 7
        f["active"] = 1
        self.fresh.append(f[0])
        return len(self.fresh) - 1

    def add(self, model: int, self_: int, last_used: int = 0, favour: bool = False, fresh: int = -1, model_lu: bool = False) -> int:
        d = np.zeros(1, dtype=L.DECISION_IN)
        d["model"] = model
        d["self"] = self_
        d["last_used"] = 0 if model_lu else last_used
        d["flags"] = (L.DF_FAVOUR_SELF if favour else 0) | (L.DF_MODEL_LAST_USED if model_lu else 0)
        d["fresh"] = fresh
        self.rows.append(d[0])
        return len(self.rows) - 1

    def build(self) -> SynthDecisions:
        fresh = np.asarray(self.fresh, dtype=L.INSTANCE_ROW) if self.fresh else np.zeros(0, dtype=L.INSTANCE_ROW)
        return SynthDecisions(np.asarray(self.rows, dtype=L.DECISION_IN), fresh, np.zeros(0, dtype=np.int32))


def _case(family, name, pods, ds_fn, n_models=1, seed=1, summarised=False, **kw):
    fl, order, ghost = edge_fleet(pods, n_models, seed, **kw)
    c = Case(family, name, fl, None, order, ghost, summarised=summarised)
    ds = Decisions()
    ds_fn(c, ds)
    c.sd = ds.build()
    return c


def _members(n, count, rem0, lru=NOW - 5000, step=1000, rpm=0, pref=False):
    return [Pod(count, rem0 - k * step, lru, rpm, pref) for k in range(n)]


def _tail(count=1000, n=3):
    """pods with room past every cut: the first one is a count violator for every best count below 800"""
    return [Pod(count + k, 3_900_000, NOW - 5000) for k in range(n)]


# ---------------------------------------------------------------------------------------------------------------
# 1. the caller-record cut (N2) with a best that has room: c_self = fr.rem < minSpace || fr.rem < best_rem >> 2
# ---------------------------------------------------------------------------------------------------------------
def family_caller_cut() -> List[Case]:
    b0, b1 = 400_003, 150_001          # odd: >> 2 rounds down.  q = 100 000 > minSpace, and 37 500 < minSpace
    pods = [Pod(8, b0, NOW - 5000), Pod(8, b1, NOW - 5000)] + _members(6, 8, 140_000) + _tail()

    def decs(c, ds):
        g = c.ghost
        for model, q in ((0, b0 >> 2), (1, b1 >> 2)):  # model 1 excludes rank 0: its best is rank 1
            at = {}
            for rem in (MS - 1, MS, q - 1, q, q + 1, 3_000_000, -5):
                for lu in (0, NOW - 10_000_000):
                    at[(rem, lu)] = ds.add(model, g, lu, fresh=ds.fresh_row(rem=rem))
            n_all = 8 if model == 0 else 7
            for lu in (0, NOW - 10_000_000):
                c.expect[at[(3_000_000, lu)]] = n_all
                c.expect[at[(-5, lu)]] = 1
                if model == 0:
                    c.pairs.append((at[(q - 1, lu)], at[(q, lu)], "fr.rem < best_rem >> 2"))
                    c.expect[at[(q, lu)]] = n_all
                else:
                    c.pairs.append((at[(MS - 1, lu)], at[(MS, lu)], "fr.rem < minSpace"))
                    c.expect[at[(MS, lu)]] = n_all
            # self inside S reads its own fresh record for c_self; the first member (rank 1 or 2) and a later one
            for r in ((1, 3) if model == 0 else (2, 4)):
                s = int(c.order[r])
                lo = ds.add(model, s, 0, fresh=ds.fresh_row(rem=(q - 1) if model == 0 else MS - 1))
                hi = ds.add(model, s, 0, fresh=ds.fresh_row(rem=q if model == 0 else MS))
                c.pairs.append((lo, hi, "self in S: c_self"))
                for favour in (False, True):
                    for rem in (q - 1, q, MS - 1, MS):
                        ds.add(model, s, 0, favour=favour, fresh=ds.fresh_row(rem=rem))
            # self = best: best_rem comes from the fresh record (q from it, us)
            s = int(c.order[0 if model == 0 else 1])
            for rem in (MS - 1, MS, 4 * MS - 1, 4 * MS, 600_003, 3_000_001):
                ds.add(model, s, 0, fresh=ds.fresh_row(rem=rem))

    return [_case("caller-cut", "room", pods, decs, n_models=2, seed=11, summarised=True, edges={1: [0]})]


# ---------------------------------------------------------------------------------------------------------------
# 2. the count cut: a member fails when count >= 10 && count > thr, thr = best + (best >> 2)
# ---------------------------------------------------------------------------------------------------------------
def _cvmin(c):
    thr = c + (c >> 2)
    return max(10, thr + 1)


def family_count_cut() -> List[Case]:
    out = []
    for bc in (0, 7, 8, 9, 10, 11, 10 ** 9):
        thr = bc + (bc >> 2)
        counts = sorted({x for x in (bc, thr - 1, thr, thr + 1, 9, 10) if bc <= x <= 10 ** 9})
        pods = [Pod(bc, 3_000_001, NOW - 5000)]
        for k, cnt in enumerate(counts):
            pods += _members(2, cnt, 2_000_000 - k * 10_000)
        if bc < 10 ** 9:
            pods += _tail(max(_cvmin(bc) + 50, 1000))
        else:
            pods += _members(3, bc, 1_000_000)
        n_pass = 1 + sum(1 for p in pods[1:] if p.count < _cvmin(bc))

        def decs(c, ds, n_pass=n_pass, bc=bc):
            g = c.ghost
            for lu in (0, NOW - 10_000_000):
                c.expect[ds.add(0, g, lu, fresh=ds.fresh_row())] = n_pass
                ds.add(0, g, lu, favour=True, fresh=ds.fresh_row())
            # self = best: its fresh count is the best count
            b = int(c.order[0])
            if bc < 10 ** 9:
                for fc in (0, 7, 8, 9, 10, 11):
                    ds.add(0, b, 0, fresh=ds.fresh_row(count=fc))
            # self among the members, at each count
            for r in range(1, min(len(c.order), 14)):
                ds.add(0, int(c.order[r]), 0)
                ds.add(0, int(c.order[r]), 0, favour=True)

        out.append(_case("count-cut", f"best-count-{bc}", pods, decs, seed=20 + bc % 97, summarised=True))
    # us best: the fresh count 7 / 8 / 9 moves thr across the count-10 and count-11 members
    pods = [Pod(8, 3_000_001, NOW - 5000)] + _members(3, 8, 2_000_000) + _members(2, 10, 1_900_000) + _members(2, 11, 1_800_000) + \
        _members(2, 12, 1_700_000) + _tail()

    def us_decs(c, ds):
        b = int(c.order[0])
        at = {fc: ds.add(0, b, 0, fresh=ds.fresh_row(count=fc)) for fc in (0, 7, 8, 9, 10)}
        c.expect.update({at[0]: 4, at[7]: 4, at[8]: 6, at[9]: 8})
        c.pairs += [(at[7], at[8], "us: fresh count 7 / 8"), (at[8], at[9], "us: fresh count 8 / 9")]

    out.append(_case("count-cut", "us-best", pods, us_decs, seed=31))
    # the first violator at word, half-window and window edges; the word before it mixes thr and thr + 1 (a "mixed" word
    # whose csum.lo == thr), the word after it holds thr + 1 only
    for vr in (31, 32, 33, 511, 512, 1023, 1024, 1025, 1400):
        pods = [Pod(8, 3_000_001, NOW - 5000)] + _members(vr - 3, 8, 2_900_000, step=1) + _members(2, 10, 2_000_000) + \
            _members(70, 11, 1_900_000, step=1) + _tail()

        def v_decs(c, ds, vr=vr):
            g = c.ghost
            c.expect[ds.add(0, g, 0, fresh=ds.fresh_row())] = vr
            c.expect[ds.add(0, g, NOW - 10_000_000, fresh=ds.fresh_row())] = vr
            ds.add(0, g, 0, fresh=ds.fresh_row(rem=MS - 1))
            for r in (1, vr // 2, vr - 2, vr - 1, vr, vr + 1, vr + 40):
                ds.add(0, int(c.order[r]), 0)
                ds.add(0, int(c.order[r]), 0, favour=True)

        out.append(_case("count-cut", f"violator-rank-{vr}", pods, v_decs, seed=40 + vr % 89, summarised=vr <= 256))
    return out


# ---------------------------------------------------------------------------------------------------------------
# 3. a full best: c_self = df > 45 000 && df > age(best)/10, df = fresh lruTime - best lruTime (wrapping)
# ---------------------------------------------------------------------------------------------------------------
def _age(t):
    return 0 if t == 0 else NOW - t


def _jdiv(a, b):  # Java's truncating division
    q = abs(a) // b
    return q if a >= 0 else -q


def family_full_best() -> List[Case]:
    out = []
    for name, l0 in (("lru-0", 0), ("a10-44999", NOW - 449_999), ("a10-45000", NOW - 450_001), ("a10-450000", NOW - 4_500_007),
                     ("future", NOW + 100_007), ("long-max", LONG_MAX)):
        a10 = _jdiv(_age(l0), 10)
        if l0 == LONG_MAX:
            pods = [Pod(1 + k, MS - 1 - k, LONG_MAX) for k in range(30)]
        else:
            pods = [Pod(3, MS - 1, l0)] + [Pod(2, MS - 2 - k, l0 + 10 + 10 * k) for k in range(30)] + \
                [Pod(2, MS - 20, l0 + 10_000_000 + k) for k in range(3)]

        def decs(c, ds, l0=l0, a10=a10):
            g = c.ghost
            n_all = len(c.order)
            vals = [LONG_MAX, 0, NOW] if l0 == LONG_MAX else \
                sorted({l0 + 45_000, l0 + 45_001, l0 + a10, l0 + a10 + 1, l0, LONG_MAX} - {x for x in [l0 + a10, l0 + a10 + 1] if x < 0})
            at = {}
            for v in vals:
                for lu in (0, NOW - 10_000_000):
                    at[(v, lu)] = ds.add(0, g, lu, fresh=ds.fresh_row(rem=MS - 1, lru=v))
            for lu in (0, NOW - 10_000_000):
                if l0 != LONG_MAX:
                    lo, hi = (l0 + 45_000, l0 + 45_001) if a10 < 45_000 else (l0 + a10, l0 + a10 + 1)
                    c.pairs.append((at[(lo, lu)], at[(hi, lu)], "df > max(45 000, age/10)"))
                    c.expect[at[(lo, lu)]] = n_all
                    c.expect[at[(hi, lu)]] = 1
                    c.expect[at[(LONG_MAX, lu)]] = 1
                else:
                    c.expect[at[(LONG_MAX, lu)]] = n_all
            for r in (1, 3):
                s = int(c.order[r])
                for v in vals[:4]:
                    ds.add(0, s, 0, fresh=ds.fresh_row(rem=MS - 1, lru=v))
                    ds.add(0, s, 0, favour=True, fresh=ds.fresh_row(rem=MS - 1, lru=v))
                ds.add(0, s, 0)

        out.append(_case("full-best", name, pods, decs, seed=50 + len(out), summarised=True))
    return out


# ---------------------------------------------------------------------------------------------------------------
# 4. non-simple case (b): a full best that is not preferred.  An entry is far when its own lruTime is more than 120 000
# and more than age(best)/4 past the best's; preferred entries before the first far one are the candidates, each
# filtered on its own rpm.  And non-simple (a)'s self test, which reads the first entry's record.
# ---------------------------------------------------------------------------------------------------------------
NEAR_RPMS = (100, 110, 111, 150, 151, 300, 301, 401)


def family_pref_b() -> List[Case]:
    out = []
    for name, l0 in (("a4-50000", NOW - 200_000), ("a4-250001", NOW - 1_000_004), ("future", NOW + 400_000), ("lru-0", 0)):
        t = max(120_000, _jdiv(_age(l0), 4))
        a10 = max(0, _jdiv(_age(l0), 10))
        near = [Pod(1, MS - 3 - k, l0 + t - len(NEAR_RPMS) + 1 + k, rpm, True) for k, rpm in enumerate(NEAR_RPMS)]
        pods = [Pod(1, MS - 1, l0), Pod(1, MS - 2, l0 + 10)] + near + \
            [Pod(1, MS - 20, l0 + t + 1, 0, True), Pod(1, MS - 21, l0 + t + 2), Pod(1, MS - 22, l0 + t + 3, 0, True),
             Pod(1, MS - 23, l0 + t + 5_000_000)]
        # model 0: the near preferred pods are the candidates; model 1 excludes the last four of them; model 2 excludes the
        # first four: a pod at exactly t is near, one at t + 1 far.  Model 3 excludes all eight: no preferred pod before the
        # first far one, so the walk rewinds to the simple case over the entries before it
        edges = {1: [6, 7, 8, 9], 2: [2, 3, 4, 5], 3: list(range(2, 10))}

        def decs(c, ds, l0=l0, a10=a10):
            g = c.ghost
            for m in (0, 1, 2):
                at = {}
                for ago in AGO_EDGES + (None,):
                    lu = 0 if ago is None else NOW - ago
                    at[ago] = ds.add(m, g, lu, fresh=ds.fresh_row(rem=MS - 1, lru=NOW))
                if m == 0:
                    c.expect[at[None]] = len(NEAR_RPMS)
                    for a, b in ((-1001, -1000), (4_999, 5_000), (719_999, 720_000), (86_399_999, 86_400_000)):
                        c.pairs.append((at[a], at[b], f"own-rpm filter at ago {b}"))
                for lu in (LONG_MAX, LONG_MIN, 0):
                    ds.add(m, g, lu, fresh=ds.fresh_row(rem=MS - 1, lru=NOW))
                # N8: favourSelf with self among the candidates returns null; self outside them, and without favour
                for r in (3, 6, 9, 10, 11):
                    ds.add(m, int(c.order[r]), 0, favour=True)
                    ds.add(m, int(c.order[r]), 0)
            # the caller's record against the rewound simple case's distance test
            for m in range(4):
                for d in (45_000, 45_001, 45_000 + a10, 45_001 + a10):
                    ds.add(m, g, 0, fresh=ds.fresh_row(rem=MS - 1, lru=l0 + d))
            lo = ds.add(3, g, 0, fresh=ds.fresh_row(rem=MS - 1, lru=l0 + max(45_000, a10)))
            hi = ds.add(3, g, 0, fresh=ds.fresh_row(rem=MS - 1, lru=l0 + max(45_000, a10) + 1))
            c.expect.update({lo: 2, hi: 1})
            c.pairs.append((lo, hi, "rewound: df > max(45 000, age/10)"))

        out.append(_case("pref-b", name, pods, decs, n_models=4, seed=60 + len(out), preferred=True, edges=edges))
    # with only one / two near preferred pods: ccount 1 skips the filter
    for k in (1, 2):
        l0 = NOW - 200_000
        pods = [Pod(1, MS - 1, l0), Pod(1, MS - 2, l0 + 10)] + \
            [Pod(1, MS - 3 - j, l0 + 100_000 + j, (100, 401)[j], True) for j in range(k)] + \
            [Pod(1, MS - 20, l0 + 120_001, 0, True), Pod(1, MS - 21, l0 + 300_000)]

        def decs_k(c, ds, k=k):
            for ago in (0, -1001, 4_999, 5_000, 719_999, 720_000):
                c.expect[ds.add(0, c.ghost, NOW - ago, fresh=ds.fresh_row(rem=MS - 1, lru=NOW))] = k

        out.append(_case("pref-b", f"near-{k}", pods, decs_k, seed=70 + k, preferred=True))
    # non-simple (a): the first entry has room but no preference, the first preferred entry after it becomes best; self's
    # test reads the FIRST entry's published remaining against the new best's quarter (q = 100 000)
    q = 400_003 >> 2
    pods = [Pod(7, rem, NOW - 5000) for rem in (q + 1, q, q - 1, MS)] + [Pod(8, 400_003, NOW - 5000, 0, True)] + \
        _members(4, 8, 300_000, pref=True) + [Pod(8, 200_000, NOW - 5000)] + [Pod(11, 3_900_000, NOW - 5000, 0, True)] + _tail()

    def a_decs(c, ds):
        s = int(c.order[6])  # the second preferred member
        at = {m: ds.add(m, s, 0) for m in range(4)}
        c.expect.update({at[0]: 5, at[1]: 5, at[2]: 2, at[3]: 2})
        c.pairs.append((at[1], at[2], "self_viol: first entry's remaining < q"))
        for m in range(4):
            ds.add(m, s, 0, favour=True)
            for rem in (MS - 1, MS, q - 1, q):
                ds.add(m, c.ghost, 0, fresh=ds.fresh_row(rem=rem))
            lo, hi = ds.add(m, c.ghost, 0, fresh=ds.fresh_row(rem=q - 1)), ds.add(m, c.ghost, 0, fresh=ds.fresh_row(rem=q))
            c.pairs.append((lo, hi, "(a): c_self against the new best's quarter"))
            ds.add(m, int(c.order[m]), 0, fresh=ds.fresh_row(rem=q))  # self = the first entry

    out.append(_case("pref-a", "first-entry-record", pods, a_decs, n_models=4, seed=80, preferred=True,
                     edges={1: [0], 2: [0, 1], 3: [0, 1, 2]}))
    return out


# ---------------------------------------------------------------------------------------------------------------
# 5. the rpm filter of the simple case: best's rpm, the caller's fresh rpm for every member (N2), lastUsed's age bands
# ---------------------------------------------------------------------------------------------------------------
def _jd2i(x):
    return min(int(x), 2 ** 31 - 1)


def family_rpm() -> List[Case]:
    out = []
    lu_vals = [NOW - a for a in AGO_EDGES] + [0, LONG_MAX, LONG_MIN]
    for best_rpm in (99, 100, 101, 111, 500_000_000):
        m = max(100, best_rpm)
        m11, m15 = _jd2i(1.1 * m), _jd2i(1.5 * m)
        rpms = sorted({x for x in (99, 100, m11, m11 + 1, m15, m15 + 1, 3 * m, 3 * m + 1, 4 * m, 4 * m + 1, m) if m <= x <= 500_000_000 or x in (99, 100)})
        pods = [Pod(8, 3_000_001, NOW - 5000, best_rpm)] + _members(3, 8, 2_000_000, rpm=7) + _tail()

        def decs(c, ds, rpms=rpms, m11=m11, m15=m15, m=m):
            g = c.ghost
            at = {}
            for j, lu in enumerate(lu_vals):
                for f in rpms:
                    at[(lu, f)] = ds.add(0, g, lu, fresh=ds.fresh_row(rpm=f))
                    ds.add(1 + j, g, model_lu=True, fresh=ds.fresh_row(rpm=f))  # the same lastUsed from the model row
            for ago, lo, why in ((-1001, m11, "1.1 x minLoad"), (-999, m15, "1.5 x minLoad"), (4_999, m15, "1.5 x minLoad"),
                                 (5_000, 3 * m, "3 x minLoad"), (719_999, 3 * m, "3 x minLoad"), (720_000, 4 * m, "4 x minLoad"),
                                 (86_399_999, 4 * m, "4 x minLoad")):
                if lo + 1 <= 500_000_000:
                    c.pairs.append((at[(NOW - ago, lo)], at[(NOW - ago, lo + 1)], why))
            for ago_lo, ago_hi in ((-1001, -1000), (4_999, 5_000), (719_999, 720_000), (86_399_999, 86_400_000)):
                f = {(-1001): m11 + 1, 4_999: m15 + 1, 719_999: 3 * m + 1, 86_399_999: 4 * m + 1}[ago_lo]
                if f <= 500_000_000:
                    c.pairs.append((at[(NOW - ago_lo, f)], at[(NOW - ago_hi, f)], f"ago {ago_hi}"))
            for f in rpms:
                c.expect[at[(0, f)]] = 4
            s = int(c.order[1])  # self in the shortlist: its filter reads the first entry's rpm
            for f in (99, min(m15 + 1, 500_000_000)):
                ds.add(0, s, 0, fresh=ds.fresh_row(rpm=f))
                ds.add(0, s, NOW - 5000, fresh=ds.fresh_row(rpm=f))

        out.append(_case("rpm", f"best-rpm-{best_rpm}", pods, decs, n_models=1 + len(lu_vals), seed=90 + len(out),
                         summarised=True, model_last_used=[NOW - 1000] + lu_vals))
    # shortlists of one and of two
    for n_mem in (0, 1):
        pods = [Pod(8, 3_000_001, NOW - 5000, 100)] + _members(n_mem, 8, 2_000_000) + _tail()

        def decs_n(c, ds, n_mem=n_mem):
            for lu in (0, NOW + 1001, NOW - 5000):
                for f in (99, 100, 151, 401, 500_000_000):
                    c.expect[ds.add(0, c.ghost, lu, fresh=ds.fresh_row(rpm=f))] = 1 + n_mem

        out.append(_case("rpm", f"shortlist-{1 + n_mem}", pods, decs_n, seed=99 + n_mem, summarised=n_mem == 1))
    return out


def all_cases() -> List[Case]:
    return family_caller_cut() + family_count_cut() + family_full_best() + family_pref_b() + family_rpm()


def check_built(case: Case, oracle, ores):
    """the fleet is ranked as intended, and the oracle answers as the case was built to: the designed shortlist lengths
    and different answers on the two sides of every threshold"""
    assert np.array_equal(oracle.cluster_order(), case.order), case.id
    for i, n in case.expect.items():
        assert ores["n_candidates"][i] == n, (case.id, i, case.sd.dec[i], ores[i], n)
    key = lambda i: (int(ores["target"][i]), int(ores["n_candidates"][i]), int(ores["n_remaining"][i]))  # noqa: E731
    for a, b, why in case.pairs:
        assert key(a) != key(b), (case.id, why, a, b, key(a))
