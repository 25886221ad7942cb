"""The closed loop's republish (publishInstanceRecord MM:5390-5470) at its thresholds, as data: pods built to sit on either
side of one line each, and the fleets that hold them.  tests/test_publish_rule_oracle.py runs them through the oracle's
loop, tests/test_publish_edges_gpu.py through the device's; tests/publish_rule.py gives the answer.

A Pod is one pod's cache (capacity and entries) and its published record; a Pair is two pods (or one pod on two fleets)
either side of one threshold, with the runs where their answers must differ and the side that publishes there.  A run is a
fleet whose pods all last published `last_done` ms before the window's end, NOW1, with or without every pod forced: a
forced pod holds one more entry (the newest, weight 1) which a REMOVE in the window takes out again, so its cache at the
end of the window is the one the pod was built with.  A pod may also carry its own event, one of the sources of a forced
publish (an eviction, an accepted load, a REMOVE of a cached model) or a REMOVE of a model its cache does not hold."""
import dataclasses
from typing import Dict, List, Optional, Tuple

import numpy as np

import publish_rule
from common import HOUR, LONG_MAX
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import NOW_MS, ChurnWorkload, make_churn

NOW1 = NOW_MS                # the end of every window built here
NOW0 = NOW1 - 2_000
MIN_SPACE = 6_400            # minSpaceUnits of every fleet here
CAP = 100_000                # the default cache capacity
LOAD_TIMEOUT_MS = 30_000
LAST_DONE = (1_999, 2_000, 38_999, 39_000, 160_000, 160_001)
RUNS = tuple((d, f) for d in LAST_DONE for f in (False, True))
# the runs that reach the threshold test (the gates open, not "old") and the ones that reach the any-change test
OPEN = ((2_000, True), (38_999, True), (39_000, False), (39_000, True), (160_000, False), (160_000, True))
OLD = ((160_001, False), (160_001, True))
EVENTS = ("evict", "load", "remove", "absent")
EVICT_SIZE, LOAD_SIZE = 5_000, 2_000


@dataclasses.dataclass
class Pod:
    cap: int                                     # the cache's capacity
    entries: List[Tuple[int, int]]               # (lastUsed, weight), distinct times
    row: Dict[str, int]                          # the published record (INSTANCE_ROW fields)
    event: Optional[str] = None                  # one of EVENTS


@dataclasses.dataclass
class Pair:
    name: str
    a: Pod
    b: Pod
    where: Tuple[Tuple[Tuple[int, bool], Tuple[int, bool]], ...]   # (run of a, run of b) where the answers differ
    pub: int                                     # the side (0: a, 1: b) that publishes there


def pod(entries=(), cap=CAP, event=None, **row):
    """a pod whose published record matches its cache (capacity, used, count, oldest entry) except for `row`"""
    entries = [(int(t), int(w)) for t, w in entries]
    r = dict(capacity=cap, used=sum(w for _, w in entries), count=len(entries),
             lru_time=min((t for t, _ in entries), default=LONG_MAX), l_in_prog=0)
    r.update(row)
    return Pod(cap, entries, r, event)


def ents(n, w=1_000, t0=NOW1 - 10 * HOUR, step=1_000):
    """n entries, oldest first at t0, one every `step` ms, each of weight w"""
    return [(t0 + k * step, w) for k in range(n)]


def summing(total, n, t0=NOW1 - 10 * HOUR):
    """n entries whose weights add up to total"""
    w = [total // n] * n
    w[-1] += total - sum(w)
    return [(t0 + k * 1_000, x) for k, x in enumerate(w)]


def _both(name, a, b, pub, where=OPEN):
    return Pair(name, a, b, tuple((r, r) for r in where), pub)


def gate_pairs():
    p = pod(ents(3), l_in_prog=1)  # a record that any open gate republishes
    out = [Pair("lastDone 1999 vs 2000, forced", p, p, (((1_999, True), (2_000, True)),), 1),
           Pair("lastDone 38999 vs 39000, not forced", p, p, (((38_999, False), (39_000, False)),), 1)]
    where = tuple(((d, False), (d, False)) for d in (2_000, 38_999))
    absent = pod(ents(3), l_in_prog=1, event="absent")
    for ev in ("evict", "load", "remove"):
        if ev == "evict":  # full of old entries: the load evicts the oldest
            forced = pod(ents(10, w=9_900, t0=NOW1 - 2 * HOUR), l_in_prog=1, used=50_000, event=ev)
        else:
            forced = pod(ents(3), l_in_prog=1, event=ev)
        out.append(Pair(f"force by {ev} vs a REMOVE of an absent key", forced, absent, where, 0))
    # lastDone 160000 is not old (MM:5402: >, not >=): a change the thresholds tolerate publishes only past it
    q = pod(ents(40), count=41)
    out.append(Pair("old: lastDone 160000 vs 160001", q, q, (((160_000, False), (160_001, False)), ((160_000, True), (160_001, True))), 1))
    return out


def old_pairs():
    e = ents(5)
    base = pod(e)
    lru = e[0][0]
    return [_both(f"old: {k} equal vs off by one", base, pod(e, **{k: v}), 1, OLD)
            for k, v in (("capacity", CAP + 1), ("count", 6), ("lru_time", lru + 1), ("used", 5_001), ("l_in_prog", 1))] + \
        [_both("old: lru_time one older", base, pod(e, lru_time=lru - 1), 1, OLD),
         _both("old: used one less", base, pod(e, used=4_999), 1, OLD)]


def capacity_pairs():
    e = ents(4)
    out = []
    for sign in (1, -1):
        out.append(_both(f"capacity: |d| = cap/50 - 1 vs cap/50 ({'+' if sign > 0 else '-'})",
                         pod(e, capacity=CAP + sign * (CAP // 50 - 1)), pod(e, capacity=CAP + sign * (CAP // 50)), 1))
    # cap / 50 == 0: no capacity is within it, even an equal one
    out.append(_both("capacity: cap 49 vs 50, equal", pod(cap=49), pod(cap=50), 0))
    return out


def lru_pairs():
    t = NOW1 - 10 * HOUR
    out = []
    for sign in (1, -1):
        out.append(_both(f"lruTime: |d| 19999 vs 20000 ({'+' if sign > 0 else '-'})",
                         pod(ents(3, t0=t), lru_time=t - sign * 19_999), pod(ents(3, t0=t), lru_time=t - sign * 20_000), 1))
    # (now - lruTime) / 16 = 160015 / 16 = 10000 (truncated)
    c = NOW1 - 160_015
    out.append(_both("lruTime: d one under vs at (now - lruTime)/16", pod(ents(3, t0=c + 9_999), lru_time=c),
                     pod(ents(3, t0=c + 10_000), lru_time=c), 1))
    # a published lruTime in the future: (now - lruTime) / 16 < 0, so even a difference of 1 publishes
    out.append(_both("lruTime: published in the future vs in the past", pod(ents(2, t0=NOW1 + 100), lru_time=NOW1 + 101),
                     pod(ents(2, t0=NOW1 - 100_000), lru_time=NOW1 - 99_999), 0))
    # published Long.MAX_VALUE: the (now - lruTime) / 16 test is skipped, 20000 still applies
    out.append(_both("lruTime: published MAX, oldest MAX - 19999 vs MAX - 20000", pod(ents(1, t0=LONG_MAX - 19_999), lru_time=LONG_MAX),
                     pod(ents(1, t0=LONG_MAX - 20_000), lru_time=LONG_MAX), 1))
    out.append(_both("lruTime: empty cache published empty vs with a time", pod(), pod(lru_time=NOW1 - HOUR), 1))
    return out


def count_pairs():
    return [_both("count: d 9 vs 10", pod(ents(61), count=70), pod(ents(60), count=70), 1),
            _both("count: d 9 at count 60 vs 61", pod(ents(51), count=60), pod(ents(52), count=61), 0),
            _both("count: d 9 at count 60 vs 61 (cache above)", pod(ents(69), count=60), pod(ents(70), count=61), 0),
            _both("count: published 0, cache empty vs one entry", pod(), pod(ents(1), count=0), 1)]


def used_pairs():
    out = [_both("used: +20% vs +19.9%", pod(summing(12_000, 4), used=10_000), pod(summing(11_999, 4), used=10_000), 0),
           _both("used: -20% vs -19.9%", pod(summing(8_000, 4), used=10_000), pod(summing(8_001, 4), used=10_000), 0),
           _both("used: published 0, used 0 vs 1", pod(), pod(ents(1, w=1), used=0), 1)]
    # |d| * 100 past Long.MAX_VALUE wraps negative: "within" in Java (both records full, everything else equal)
    full = summing(CAP - 10, 10)
    out.append(_both("used: |d|*100 wraps vs just below the wrap", pod(full, used=93 * 10 ** 15), pod(full, used=92 * 10 ** 15), 1))
    return out


def full_pairs():
    nf = CAP - MIN_SPACE  # remaining exactly minSpace: not full
    return [_both("full: published not full, remaining minSpace - 1 vs minSpace", pod(summing(nf + 1, 5), used=nf - 100),
                  pod(summing(nf, 5), used=nf - 100), 0),
            _both("full: published full, remaining minSpace - 1 vs minSpace", pod(summing(nf + 1, 5), used=nf + 50),
                  pod(summing(nf, 5), used=nf + 50), 1)]


def loading_pairs():
    return [_both("loading: l_in_prog 0 vs 1", pod(ents(4)), pod(ents(4), l_in_prog=1), 1)]


def all_pairs():
    return gate_pairs() + old_pairs() + capacity_pairs() + lru_pairs() + count_pairs() + used_pairs() + full_pairs() + loading_pairs()


def event_free(pairs):
    """the pairs whose pods carry no event of their own"""
    return [p for p in pairs if p.a.event is None and p.b.event is None]


def pods_of(pairs):
    """every pair's two pods in order: pod 2k is pair k's side a, 2k + 1 its side b"""
    return [x for p in pairs for x in (p.a, p.b)]


# ---------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass
class Run:
    w: ChurnWorkload            # the fleet as ingested: every row's capacity is its cache's (mmp_churn_init sizes the caches)
    rows: np.ndarray            # the published records, capacity included: `updates` get them after churn_init
    updates: List[int]          # pods whose published capacity is not their cache's
    last_published: int
    events: np.ndarray          # the window's events (CHURN_EVENT)
    forced: set                 # the pods the window forces
    pods: List[Pod]
    spare: np.ndarray           # models without a registration (for decisions after the window)
    entry_models: List[List[int]]  # the model of each of pod i's entries, in the order of pods[i].entries


def build_run(pods: List[Pod], last_done: int, force, seed: int = 7, n_spare: int = 16, removed=()) -> Run:
    """One fleet holding `pods` (pod i = instance i), its caches, registry and the window's events.  force: True (every pod)
    or the pods that hold one more entry a REMOVE in the window takes out.  removed: pods that will leave the table (no
    event of theirs)."""
    ni = len(pods)
    seeds = []          # (instance, model, lastUsed, weight)
    regs = []           # per model: (loaded instances, failed instances, size)
    events = []         # (type, model, caller, t)
    forced = set()
    entry_models = []
    for i, p in enumerate(pods):
        first = len(regs)
        entry_models.append(list(range(first, first + len(p.entries))))
        for t, w in p.entries:
            seeds.append((i, len(regs), t, w))
            regs.append(([i], [], max(w, 1)))
        live = i not in removed
        if (force is True or (force and i in force)) and live:
            t = max([t for t, _ in p.entries], default=NOW1 - HOUR) + 1
            seeds.append((i, len(regs), t, 1))
            events.append((1, len(regs), i, NOW0 + 100 + i))
            regs.append(([i], [], 1))
            forced.add(i)
        if p.event and live:
            others = [j for j in range(ni) if j != i]
            if p.event in ("evict", "load"):  # a cache miss that only this pod can take: every other pod failed the model
                events.append((0, len(regs), i, NOW0 + 500 + i))
                regs.append(([], others, EVICT_SIZE if p.event == "evict" else LOAD_SIZE))
                forced.add(i)
            elif p.event == "remove":  # of the pod's newest entry
                k = max(range(len(p.entries)), key=lambda j: p.entries[j][0])
                events.append((1, first + k, i, NOW0 + 300 + i))
                forced.add(i)
            else:  # "absent": registered here, never in the cache
                events.append((1, len(regs), i, NOW0 + 300 + i))
                regs.append(([i], [], 1_000))
    nm = len(regs) + n_spare
    regs += [([], [], 1_000)] * n_spare
    w = make_churn(max(nm, 8), ni, seed)
    fl = dataclasses.replace(w.fleet, now_ms=NOW0, min_space_units=MIN_SPACE, type_config=None)
    fl.type_names = fl.type_names[:1]
    fl.model_type = np.zeros(nm, dtype=np.int32)
    fl.model_size = np.asarray([r[2] for r in regs], dtype=np.int32)
    fl.model_last_used = np.full(nm, NOW1 - 5 * HOUR, dtype=np.int64)
    fl.model_rpm = np.zeros(nm, dtype=np.int32)
    fl.n_loaded = np.asarray([len(r[0]) for r in regs], dtype=np.int32)
    fl.n_failed = np.asarray([len(r[1]) for r in regs], dtype=np.int32)
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(fl.n_loaded + fl.n_failed, out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([x for r in regs for x in r[0] + r[1]], dtype=np.int32)
    rows = fl.inst_rows.copy()
    rows["l_threads"], rows["vers"], rows["active"], rows["shutting_down"] = 8, 7, 1, 0
    for i, p in enumerate(pods):
        for k, v in p.row.items():
            rows[i][k] = v
    fl.inst_rows = rows.copy()
    fl.inst_rows["capacity"] = [p.cap for p in pods]
    s = np.asarray(seeds, dtype=np.int64).reshape(-1, 4)
    ev = np.zeros(len(events), dtype=L.CHURN_EVENT)
    if events:
        e = np.asarray(events, dtype=np.int64)
        ev["type"], ev["model"], ev["caller"], ev["t"] = e[:, 0], e[:, 1], e[:, 2], e[:, 3]
        ev["u"] = np.arange(len(events), dtype=np.uint32)
        ev = ev[np.argsort(ev["t"], kind="stable")]
    w2 = ChurnWorkload(fl, np.asarray([p.cap for p in pods], dtype=np.int64), s[:, 0].astype(np.int32), s[:, 1].astype(np.int32),
                       s[:, 2].astype(np.int64), s[:, 3].astype(np.int32), np.full(len(s), NOW0 - 1_000, dtype=np.int64),
                       np.nonzero(fl.n_loaded > 0)[0], np.nonzero(fl.n_loaded == 0)[0], LOAD_TIMEOUT_MS)
    updates = [i for i, p in enumerate(pods) if int(rows[i]["capacity"]) != p.cap]
    return Run(w2, rows, updates, NOW1 - last_done, ev, forced, pods, np.arange(nm - n_spare, nm, dtype=np.int32), entry_models)


def designed_cache(p: Pod):
    """(capacity, weightedSize, size, oldest or None) of the pod's cache as built"""
    return (p.cap, sum(w for _, w in p.entries), len(p.entries), min((t for t, _ in p.entries), default=None))


def cache_of(sim, i: int, cap: int):
    """(capacity, weightedSize, size, oldest or None) of the oracle loop's cache of pod i"""
    oldest, weighted, count = sim.lru_state(i)
    return (cap, weighted, count, None if oldest == -1 else oldest)


ROW_FIELDS = ("lru_time", "capacity", "used", "start_time", "vers", "count", "l_threads", "l_in_prog", "rpm", "shutting_down")


def expected(rows, last_published, forced, caches, present=None, now=NOW1):
    """publish_rule.publish for every pod at `now`: (bool[n] publish, the rows afterwards as dicts).  rows: the published
    records at the start of the window; caches[i]: pod i's cache at its end; present: pods still in the table."""
    pub, after = [], []
    for i, r in enumerate(rows):
        cur = {k: int(r[k]) for k in ROW_FIELDS}
        if present is not None and not present[i]:
            pub.append(False)
            after.append(cur)
            continue
        p, new = publish_rule.publish(cur, last_published[i], now, i in forced, caches[i], MIN_SPACE)
        pub.append(p)
        after.append(new)
    return np.asarray(pub, dtype=bool), after


def same_rows(got, want, what):
    """got: INSTANCE_ROW / INST rows; want: dicts from expected()"""
    for i, w in enumerate(want):
        g = {k: int(got[i][k]) for k in publish_rule.FIELDS + ("l_threads", "rpm")}
        assert all(g[k] == w[k] for k in g), (what, i, g, {k: w[k] for k in g})


def check_pairs(pairs, pub_by_run):
    """every pair answers differently where it says, on the side it names; pub_by_run[run]: bool[n] of a run of pods_of(pairs)"""
    for k, p in enumerate(pairs):
        for ra, rb in p.where:
            if ra not in pub_by_run or rb not in pub_by_run:  # (a fleet of some runs only)
                continue
            a, b = bool(pub_by_run[ra][2 * k]), bool(pub_by_run[rb][2 * k + 1])
            assert a != b and (b if p.pub else a), (p.name, ra, rb, a, b)


def random_pods(n: int, seed: int):
    """pods near every threshold at once: a random cache, and a record off it by amounts around each line"""
    rng = np.random.default_rng(seed)
    pods = []
    for _ in range(n):
        cap = int(rng.choice([49, 50, 2_000, CAP, 3 * CAP]))
        k = int(rng.integers(0, 9))
        t0 = int(NOW1 - rng.choice([HOUR, 160_015, 330_000, 10 * HOUR]))
        wts = [int(x) for x in rng.integers(0 if cap < 100 else 1, max(2, cap // 12), size=k)] if cap >= 100 else [1] * min(k, 40)
        e = [(t0 + 997 * j, w) for j, w in enumerate(wts)]
        if rng.random() < 0.05:
            e = [(LONG_MAX - 19_990 - 10 * j, w) for j, (_, w) in enumerate(e)][::-1]
        p = pod(e, cap=cap)
        r = p.row
        if rng.random() < 0.4:
            r["capacity"] += int(rng.choice([-1, 1])) * int(rng.choice([0, 1, cap // 50 - 1, cap // 50, cap // 50 + 1]))
        if rng.random() < 0.4:
            r["count"] = max(0, r["count"] + int(rng.integers(-11, 12)))
        if rng.random() < 0.4:
            base = r["lru_time"] if r["lru_time"] != LONG_MAX else NOW1 - HOUR
            d = int(rng.choice([-1, 1])) * int(rng.choice([1, 9_999, 10_000, 19_999, 20_000, 20_001]))
            r["lru_time"] = LONG_MAX if rng.random() < 0.2 else min(LONG_MAX, base + d)
        if rng.random() < 0.4:
            u = r["used"]
            r["used"] = max(0, int(rng.choice([0, u + 1, u - 1, u * 5 // 4, u * 4 // 5, u * 6 // 5, 93 * 10 ** 15, 92 * 10 ** 15])))
        if rng.random() < 0.2:
            r["used"] = max(0, r["capacity"] - MIN_SPACE + int(rng.integers(-2, 3)))
        if rng.random() < 0.15:
            r["l_in_prog"] = int(rng.integers(1, 4))
        pods.append(p)
    return pods
