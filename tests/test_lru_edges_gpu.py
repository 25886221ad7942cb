"""Plug point 3 at its edges: k_lru_events and k_lru_state, through mmp_lru_apply(_status) and mmp_lru_state, against the
oracle's LRU (ob.OracleLru, itself pinned by a plain Python list in test_oracle_properties.py), with MMP_LRU_LOAD against
loadLocal's literal sequence (oracle/mm_sim.inc).

An instance with 12 or more events in one call runs on a shared-memory copy of its slots when its block has room for
them (4 warps x 32 B per slot: up to 1 600 slots), so the shapes straddle both limits.  The state is compared after every
call (oldestTime() as CLHM caches it, weightedSize(), size()), and every scenario ends by setting every capacity to 0:
the evictions are then each cache's whole deque, in order, with keys, lastUsed values and weights."""
import numpy as np
import pytest

from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError, _ptr
from oracle import binding as ob

pytestmark = pytest.mark.gpu

INSERT, TOUCH, RESIZE, REMOVE, SETCAP, LOAD = range(6)
ACCEPTED, CHURN, FALLTHRU, EARLY, GROW_EVICTED, EXISTS = 0, 2, 3, 4, 5, 6
MIN_SPACE, CHURN_AGE = 2560, 600_000
NOW0 = 1_760_000_000_000
W_MAX = 2**31 - 1
FIELDS = ("op", "instance", "model", "weight", "last_used")


def events(rows):
    """(op, instance, model, weight, last_used) tuples -> mmp_lru_event array (SET_CAPACITY: last_used = the capacity)"""
    ev = np.zeros(len(rows), dtype=L.LRU_EVENT)
    for j, k in enumerate(FIELDS):
        ev[k] = [r[j] for r in rows]
    return ev


class Ref:
    """Every instance's cache on the oracle; an MMP_LRU_LOAD event as loadLocal's literal sequence (oracle/mm_sim.inc:
    churn guard on oldestTime(), placeholder putIfAbsent, fall-through, early reject, growth)."""

    def __init__(self, oracle_lib, caps, min_space=MIN_SPACE, churn_age=CHURN_AGE):
        self.L = oracle_lib
        self.lru = [ob.OracleLru(int(c)) for c in caps]
        self.cap = [int(c) for c in caps]
        self.min_space, self.churn_age = min_space, churn_age

    def _run(self, i, idx, ev, now, out):
        """a run of plain events of instance i, in one oracle call"""
        if not idx:
            return
        idx = np.array(idx)
        e = ev[idx]
        setcap = e["op"] == SETCAP
        oe = np.zeros(len(idx), dtype=ob.LRU_EVENT)
        oe["op"], oe["key"] = e["op"], e["model"]
        oe["weight"] = np.where(setcap, e["last_used"], e["weight"])
        oe["last_used"] = np.where(setcap, 0, e["last_used"])
        for x in self.lru[i].apply(oe, now):
            out.append((i, int(x["key"]), int(x["last_used"]), int(x["weight"]), int(idx[x["event"]])))
        if setcap.any():
            self.cap[i] = int(e["last_used"][setcap][-1])

    def _load(self, i, k, e, now, out):
        lru, m, size, lu = self.lru[i], int(e["model"]), int(e["weight"]), int(e["last_used"])
        if self.L.orc_churn_reject(self.cap[i], lru.weighted_size(), lru.oldest_time(), self.min_space, self.churn_age, now):
            return CHURN

        def put(op, w):
            for x in lru.apply(np.array([(op, m, w, lu)], dtype=ob.LRU_EVENT), now):
                out.append((i, int(x["key"]), int(x["last_used"]), int(x["weight"]), k))

        exists = m in lru.dump()[0]
        put(INSERT, 1)  # the placeholder (INSERTION_WEIGHT MM:5011)
        if exists:
            return EXISTS
        if m not in lru.dump()[0]:
            return FALLTHRU
        if self.L.orc_early_reject(abs(size), self.cap[i], lru.weighted_size(), lru.oldest_time(), lu):
            put(REMOVE, 0)
            return EARLY
        put(RESIZE, size)
        return ACCEPTED if m in lru.dump()[0] else GROW_EVICTED

    def apply(self, ev, now):
        """evictions as (instance, model, last_used, weight, event), grouped by instance in order; per-event status"""
        out, status = [], np.full(len(ev), -1, dtype=np.int32)
        order = np.argsort(ev["instance"], kind="stable")
        cuts = np.flatnonzero(np.diff(ev["instance"][order])) + 1
        for sel in np.split(order, cuts) if len(ev) else []:
            i, run = int(ev["instance"][sel[0]]), []
            for k in sel:
                if ev["op"][k] == LOAD:
                    self._run(i, run, ev, now, out)
                    run = []
                    status[k] = self._load(i, int(k), ev[k], now, out)
                else:
                    run.append(int(k))
            self._run(i, run, ev, now, out)
        return out, status

    def sizes(self):
        return sum(o.size() for o in self.lru)


def check_state(s, ref, tag=""):
    oldest, weighted, count = s.lru_state()
    for name, got, want in (("weightedSize", weighted, [o.weighted_size() for o in ref.lru]),
                            ("size", count, [o.size() for o in ref.lru]),
                            ("oldestTime", oldest, [o.oldest_time() for o in ref.lru])):
        bad = np.flatnonzero(np.asarray(got, dtype=np.int64) != np.asarray(want, dtype=np.int64))
        assert not len(bad), (tag, name, [(int(i), int(got[i]), int(want[i])) for i in bad[:5]])


def check(s, ref, ev, now, tag=""):
    """one call through both sides: evictions, statuses, then the state of every cache"""
    cap = 4 * len(ev) + ref.sizes() + 16  # no call evicts more than was resident plus what it inserts
    got, status = s.lru_apply_status(ev, now, cap=cap)
    want, want_status = ref.apply(ev, now)
    got_l = [tuple(int(x[k]) for k in ("instance", "model", "last_used", "weight", "event")) for x in got]
    if got_l != want:
        j = next((j for j, (a, b) in enumerate(zip(got_l, want)) if a != b), min(len(got_l), len(want)))
        raise AssertionError((tag, "evictions", len(got_l), len(want), j, got_l[j:j + 3], want[j:j + 3]))
    bad = np.flatnonzero(status != want_status)
    assert not len(bad), (tag, "status", [(int(k), tuple(int(ev[k][f]) for f in FIELDS), int(status[k]), int(want_status[k]))
                                          for k in bad[:5]])
    check_state(s, ref, tag)
    return want_status


def drain(s, ref, now, tag="drain"):
    """capacity 0 everywhere: the evictions are every deque, whole and in order"""
    check(s, ref, events([(SETCAP, i, 0, 0, 0) for i in range(len(ref.lru))]), now, tag)
    assert ref.sizes() == 0


def fleet(product_lib, churn_age=CHURN_AGE):
    return Fleet(MIN_SPACE, churn_age, 2560, 4, 64, lib=product_lib)


# ---------------------------------------------------------------------------------------------------------------------
# shapes: slot counts around a warp's width and the staging limit, partial blocks, 0 / 1 / 11 / 12 / 13 events per
# instance per call (staged and unstaged instances share blocks; each instance crosses the threshold from call to call)
# and one hot instance
# ---------------------------------------------------------------------------------------------------------------------
COUNTS = (0, 1, 11, 12, 13)


class Gen:
    """random events per cache: every op, keys that are never inserted, coarse times (equal lastUsed values are common),
    times in the future (a touch at `now` moves them back), weights and capacities up to int32 / 2^62 on `big` caches"""

    def __init__(self, rng, caps, keys, big):
        self.rng, self.caps, self.keys, self.big = rng, caps, keys, big

    def rows(self, i, n, now, p_load):
        r, cap, keys = self.rng, int(self.caps[i]), self.keys
        p = np.array([0.36, 0.24, 0.12, 0.10, 0.04, p_load])
        op = r.choice(6, size=n, p=p / p.sum())
        model = r.integers(0, keys, size=n)
        absent = np.isin(op, (TOUCH, RESIZE, REMOVE)) & (r.random(n) < 0.1)
        model = np.where(absent, keys + 1000 + r.integers(0, 10, size=n), model)
        pick = lambda *c: np.choose(r.integers(0, len(c), size=n), [np.broadcast_to(np.int64(x), n) for x in c])
        if self.big[i]:
            weight = pick(1, W_MAX, r.integers(1, W_MAX, size=n))
            capv = pick(0, 2**62, r.integers(2**31, 2**35, size=n))
        else:
            weight = r.integers(1, max(2, 3 * cap // keys) + 1, size=n)
            capv = np.where(r.random(n) < 0.1, 0, r.integers(cap // 2, 2 * cap, size=n))
        lu = np.where(r.random(n) < 0.2, 0, now + r.integers(-40, 41, size=n) * 1000)
        load_size = pick(1, 256, 2560, weight, min(cap + 1, W_MAX))
        load_lu = pick(0, now - 5, now - 3_000_000, lu)
        weight = np.where(op == LOAD, load_size, weight)
        lu = np.where(op == SETCAP, capv, np.where(op == LOAD, load_lu, lu))
        return op, model, weight, lu

    def batch(self, counts, now, p_load=0.14, hot=-1, n_hot=0):
        """counts[i] events on cache i (n_hot on `hot`, with fewer loads), the caches interleaved at random"""
        parts = [(i, self.rows(i, n_hot if i == hot else n, now, 0.02 if i == hot else p_load))
                 for i, n in enumerate(counts) if (n_hot if i == hot else n)]
        ev = np.zeros(sum(len(c[0]) for _, c in parts), dtype=L.LRU_EVENT)
        if not parts:
            return ev
        ev["instance"] = np.concatenate([np.full(len(c[0]), i) for i, c in parts])
        for j, k in enumerate(("op", "model", "weight", "last_used")):
            ev[k] = np.concatenate([c[j] for _, c in parts])
        out = np.empty_like(ev)
        out[np.argsort(self.rng.permutation(ev["instance"]), kind="stable")] = ev  # each cache's events keep their order
        return out


@pytest.mark.parametrize("slots,n_inst,hot", [(7, 1, False), (7, 5, True), (31, 3, False), (32, 37, False), (33, 5, True),
                                              (96, 37, True), (96, 4000, False), (33, 4003, True), (1600, 5, True),
                                              (1600, 37, False), (1601, 5, True), (1601, 37, False)])
def test_lru_shapes_match_oracle(product_lib, oracle_lib, slots, n_inst, hot):
    rng = np.random.default_rng(slots * 10_007 + n_inst)
    big = rng.random(n_inst) < 0.15
    caps = np.where(big, 2**33, rng.integers(20_000, 60_000, size=n_inst)).astype(np.int64)
    s = fleet(product_lib)
    s.lru_init(caps, slots)
    ref = Ref(oracle_lib, caps)
    gen = Gen(rng, caps, slots, big)
    now = NOW0
    hot_i = 1 % n_inst if hot else -1
    for call in range(6):
        counts = [COUNTS[(i + call) % len(COUNTS)] for i in range(n_inst)]
        ev = gen.batch(counts, now, hot=hot_i, n_hot=20_000 if call == 2 else counts[hot_i])
        check(s, ref, ev, now, (slots, n_inst, call))
        now += int(rng.integers(1, 400_000))
    drain(s, ref, now)


# ---------------------------------------------------------------------------------------------------------------------
# semantics edges, each on its own cache; one call (instances with 12+ events staged when slots <= 1600) or one call per
# event (never staged)
# ---------------------------------------------------------------------------------------------------------------------
def _semantics_scenario(slots, now):
    t0 = now - 100_000
    rows, caps = [], []
    # 0: ties -- equal lastUsed inserts, touches to the successor's time (seq chains), repeated equal touches
    caps.append(1_000_000)
    rows += [(INSERT, 0, j, 10, t0 + 1000 * j) for j in range(10)]
    rows += [(TOUCH, 0, j, 0, t0 + 1000 * (j + 1)) for j in range(9)]
    rows += [(TOUCH, 0, j, 0, t0 + 1000 * (j + 1)) for j in range(9)]
    rows += [(INSERT, 0, 10 + j, 10, t0 + 5000) for j in range(4)]
    rows += [(INSERT, 0, 20 + j, 10, t0 + 20_000) for j in range(8)]
    rows += [(TOUCH, 0, 20 + j, 0, t0 + 20_000) for j in (7, 3, 0)]
    rows += [(TOUCH, 0, 20 + j, 0, t0 + 21_000) for j in (2, 3, 4, 0)]
    rows += [(TOUCH, 0, j, 0, t0 + 9000) for j in range(9)]
    rows += [(TOUCH, 0, 20 + j, 0, t0 + 9000) for j in range(8)]
    rows += [(INSERT, 0, 30, 10, t0 + 9000), (TOUCH, 0, 9, 0, t0 + 9000), (TOUCH, 0, 30, 0, t0 + 9000)]
    # 1: lastUsed 0 (= now), entries in the future touched at `now` (moved back), keys that are not present
    caps.append(1_000_000)
    rows += [(INSERT, 1, 0, 5, 0), (INSERT, 1, 1, 5, now + 50_000), (INSERT, 1, 2, 5, now + 60_000), (INSERT, 1, 3, 5, now)]
    rows += [(TOUCH, 1, 1, 0, 0), (TOUCH, 1, 2, 0, now + 10_000), (TOUCH, 1, 0, 0, now - 5000), (INSERT, 1, 2, 99, 0)]
    rows += [(TOUCH, 1, 77, 0, 0), (RESIZE, 1, 77, 40, 0), (REMOVE, 1, 77, 0, 0), (TOUCH, 1, 3, 0, now + 60_000)]
    # 2: resize by 0, down, up, up past capacity (evicting older entries, then the resized one itself)
    caps.append(1000)
    rows += [(INSERT, 2, j, 100, t0 + 1000 * j) for j in range(8)]
    rows += [(RESIZE, 2, 3, 100, 0), (RESIZE, 2, 3, 40, 0), (RESIZE, 2, 3, 160, 0), (RESIZE, 2, 5, 400, 0),
             (RESIZE, 2, 6, 1001, 0)]
    # 3: an insert that evicts itself (older than everything), one larger than the capacity
    caps.append(10_000)
    rows += [(INSERT, 3, 0, 4000, now - 10), (INSERT, 3, 1, 4000, now - 5), (INSERT, 3, 2, 3000, now - 100_000),
             (INSERT, 3, 3, 10_001, 0), (INSERT, 3, 4, 2000, 0), (INSERT, 3, 5, 1, now - 1)]
    # 4: one insert that evicts hundreds of entries
    n4 = min(slots - 2, 500)
    caps.append(n4)
    rows += [(INSERT, 4, j, 1, t0 + (j // 3) * 1000) for j in range(n4)]
    rows += [(INSERT, 4, n4, n4 - 3, 0)]
    # 5: SET_CAPACITY to the weighted size, one below, below a single entry, growing, to 0; int64 accounting
    caps.append(2**62)
    rows += [(INSERT, 5, j, W_MAX, t0 + 1000 * j) for j in range(4)]
    rows += [(INSERT, 5, 4, 1, t0)]
    ws = 4 * W_MAX + 1
    rows += [(SETCAP, 5, 0, 0, ws), (SETCAP, 5, 0, 0, ws - 1), (SETCAP, 5, 0, 0, 2**62), (INSERT, 5, 6, W_MAX, 0),
             (SETCAP, 5, 0, 0, W_MAX - 1), (INSERT, 5, 7, 7, 0), (SETCAP, 5, 0, 0, 2**62), (SETCAP, 5, 0, 0, 0),
             (INSERT, 5, 8, W_MAX, now + 1), (SETCAP, 5, 0, 0, W_MAX)]
    # 6: an empty cache resized, then filled
    caps.append(0)
    rows += [(SETCAP, 6, 0, 0, 0), (INSERT, 6, 1, 1, 0), (SETCAP, 6, 0, 0, 1), (INSERT, 6, 1, 1, 0), (TOUCH, 6, 1, 0, 0)]
    return rows, caps


@pytest.mark.parametrize("slots", [1600, 1601])
@pytest.mark.parametrize("split", [False, True])
def test_lru_semantics_edges(product_lib, oracle_lib, slots, split):
    now = NOW0
    rows, caps = _semantics_scenario(slots, now)
    s = fleet(product_lib)
    s.lru_init(np.array(caps, dtype=np.int64), slots)
    ref = Ref(oracle_lib, caps)
    if split:
        for k, r in enumerate(rows):
            check(s, ref, events([r]), now, k)
    else:
        check(s, ref, events(rows), now)
    k0, t0, w0 = ref.lru[0].dump()
    assert len(k0) > 20 and len(set(t0.tolist())) < len(t0) - 10  # the tie scenario left runs of equal lastUsed values
    drain(s, ref, now + 1)


# ---------------------------------------------------------------------------------------------------------------------
# checked loads (MMP_LRU_LOAD) in batch
# ---------------------------------------------------------------------------------------------------------------------
def _load_scenarios(now):
    """(rows, caps, {event index: expected status}) -- every outcome, the guard's boundaries, and the stale oldestTime()
    a SET_CAPACITY leaves behind (N14)"""
    rows, caps, want = [], [], {}

    def inst(cap, setup, load, expect):
        i = len(caps)
        caps.append(cap)
        for r in setup:
            rows.append((r[0], i) + tuple(r[1:]))
        for ld, st in zip(load, expect):
            want[len(rows)] = st
            rows.append((LOAD, i) + tuple(ld))

    old = now - 1_200_000
    inst(10_000, [(INSERT, 1, 8000, now - 1000)], [(9, 100, 0)], [CHURN])
    inst(10_000, [(INSERT, 1, 8000, now - CHURN_AGE)], [(9, 100, 0)], [ACCEPTED])          # exactly min_churn_age old
    inst(10_000, [(INSERT, 1, 8000, now - CHURN_AGE + 1)], [(9, 100, 0)], [CHURN])
    inst(10_000, [(INSERT, 1, 10_000 - MIN_SPACE, now - 1)], [(9, 100, 0)], [ACCEPTED])    # exactly min_space free
    inst(10_000, [(INSERT, 1, 10_000 - MIN_SPACE + 1, now - 1)], [(9, 100, 0)], [CHURN])
    inst(10_000, [(INSERT, 1, 10_000, now - 1_000_000)], [(9, 100, now - 2_000_000)], [FALLTHRU])
    inst(10_000, [], [(9, 20_000, 0), (9, 10_001, now - 1)], [EARLY, EARLY])               # larger than the cache
    inst(10_000, [(INSERT, 1, 5000, now - 1_000_000), (INSERT, 2, 4000, now - 800_000)], [(9, 9000, now - 900_000)],
         [GROW_EVICTED])
    inst(10_000, [(INSERT, 1, 100, now - 5)], [(1, 9000, now - 1)], [EXISTS])
    inst(10_000, [], [(9, 100, 0), (10, 200, now - 3_000_000), (9, 50, 0)], [ACCEPTED, ACCEPTED, EXISTS])
    xy = [(INSERT, 1, 4000, old), (INSERT, 2, 4000, now - 1)]
    # SET_CAPACITY evicts X; oldestTime() still reports X, older than min_churn_age: the guard lets the load through
    inst(10_000, xy + [(SETCAP, 0, 0, 5000)], [(9, 100, 0)], [ACCEPTED])
    inst(10_000, xy + [(SETCAP, 0, 0, 9000), (SETCAP, 0, 0, 5000)], [(9, 100, 0)], [ACCEPTED])
    inst(10_000, xy + [(SETCAP, 0, 0, 5000), (SETCAP, 0, 0, 4000)], [(9, 100, 0)], [ACCEPTED])
    # ... until a step that refreshes the field: a read of a present key (even one that leaves its time as it is),
    inst(10_000, xy + [(SETCAP, 0, 0, 5000), (TOUCH, 2, 0, now - 1)], [(9, 100, 0)], [CHURN])
    inst(10_000, xy + [(SETCAP, 0, 0, 5000), (INSERT, 2, 7, 0)], [(9, 100, 0)], [CHURN])
    # a resize that changes the weight, a removal, an insert, the load's own placeholder
    inst(10_000, xy + [(SETCAP, 0, 0, 5000), (RESIZE, 2, 3999, 0)], [(9, 100, 0)], [CHURN])
    inst(10_000, xy + [(SETCAP, 0, 0, 5000), (INSERT, 3, 1, now - 2)], [(9, 100, 0)], [CHURN])
    inst(10_000, xy + [(INSERT, 3, 500, now - 2), (SETCAP, 0, 0, 5000), (REMOVE, 3, 0, 0)], [(9, 100, 0)], [CHURN])
    inst(10_000, xy + [(SETCAP, 0, 0, 5000)], [(9, 100, 0), (10, 100, 0)], [ACCEPTED, CHURN])
    # and not by steps that change nothing: an absent key, a resize to the same weight
    inst(10_000, xy + [(SETCAP, 0, 0, 5000), (TOUCH, 7, 0, 0), (REMOVE, 7, 0, 0), (RESIZE, 7, 5, 0), (RESIZE, 2, 4000, 0)],
         [(9, 100, 0)], [ACCEPTED])
    # a churn-rejected load changes nothing either
    inst(10_000, xy + [(SETCAP, 0, 0, 5000), (TOUCH, 2, 0, 0)], [(9, 100, 0), (10, 100, 0)], [CHURN, CHURN])
    # the field as a SET_CAPACITY of an empty cache leaves it (-1), and the stale value at the end of the call
    inst(10_000, [(SETCAP, 0, 0, 100)], [(9, 50, 0)], [ACCEPTED])
    inst(10_000, xy + [(SETCAP, 0, 0, 5000)], [], [])
    return rows, caps, want


@pytest.mark.parametrize("churn_age", [CHURN_AGE, 0])
def test_checked_loads_in_batch(product_lib, oracle_lib, churn_age):
    now = NOW0
    rows, caps, want = _load_scenarios(now)
    n_fixed = len(caps)
    rng = np.random.default_rng(77 + churn_age)
    n_rand = 40
    rcaps = rng.integers(20_000, 60_000, size=n_rand)
    s = fleet(product_lib, churn_age)
    s.lru_init(np.concatenate([np.array(caps, dtype=np.int64), rcaps]), 96)
    ref = Ref(oracle_lib, caps + [int(c) for c in rcaps], churn_age=churn_age)
    st = check(s, ref, events(rows), now, "scenarios")
    if churn_age:
        assert {k: int(st[k]) for k in want} == want
    else:
        assert CHURN not in st
    seen = set(int(x) for x in st)
    # loads interleaved with every other event on many caches, the clock moving across the guard's window
    # (80 keys: the 96 slots always have room)
    gen = Gen(rng, np.concatenate([np.array(caps), rcaps]), 80, np.zeros(n_fixed + n_rand, dtype=bool))
    for call in range(10):
        counts = [0] * n_fixed + [int(x) for x in rng.integers(0, 30, size=n_rand)]
        seen |= set(int(x) for x in check(s, ref, gen.batch(counts, now, p_load=0.5), now, call))
        now += int(rng.integers(1, 400_000))
    expect = {ACCEPTED, CHURN, FALLTHRU, EARLY, GROW_EVICTED, EXISTS} if churn_age else {ACCEPTED, FALLTHRU, EARLY, GROW_EVICTED, EXISTS}
    assert seen - {-1} == expect, seen
    drain(s, ref, now)


# ---------------------------------------------------------------------------------------------------------------------
# the C ABI's edges
# ---------------------------------------------------------------------------------------------------------------------
def _raw_apply(s, ev, now, cap):
    out = np.zeros(max(cap, 1), dtype=L.EVICTION)
    return s.lib.mmp_lru_apply(s.h, _ptr(ev), len(ev), now, _ptr(out), cap), out[:cap]


def test_lru_abi_edges(product_lib, oracle_lib):
    now = NOW0
    s = fleet(product_lib)
    ev = events([(INSERT, 0, 1, 10, 0)])
    assert _raw_apply(s, ev, now, 4)[0] == L.E_STATE  # before mmp_lru_init
    rng = np.random.default_rng(3)
    n_inst, slots = 9, 33
    caps = rng.integers(20_000, 60_000, size=n_inst)
    s.lru_init(caps, slots)
    ref = Ref(oracle_lib, caps)
    gen = Gen(rng, caps, slots, np.zeros(n_inst, dtype=bool))
    for call in range(3):
        check(s, ref, gen.batch([int(x) for x in rng.integers(0, 25, size=n_inst)], now), now, call)
    # an eviction buffer smaller than the evictions: the true total comes back, what was written is the oracle's, and
    # the events were applied whole
    ev = events([(SETCAP, i, 0, 0, int(c) // 4) for i, c in enumerate(caps)] + [(INSERT, 2, 500, 50_000, now - 1)])
    want, _ = ref.apply(ev, now)
    assert len(want) > 6
    n, out = _raw_apply(s, ev, now, 5)
    assert n == len(want)
    got = [tuple(int(x[k]) for k in ("instance", "model", "last_used", "weight", "event")) for x in out]
    assert set(got) <= set(want) and len(set(got)) == 5, (got, want)
    check_state(s, ref, "after a short buffer")
    check(s, ref, events([(INSERT, 0, 600, 10, 0), (INSERT, 1, 601, 10, 0), (INSERT, 1, 602, 10, 0)]), now)
    ev = events([(SETCAP, 0, 0, 0, 0), (SETCAP, 1, 0, 0, 0)])
    assert len(ref.apply(ev, now)[0]) >= 3
    with pytest.raises(MmpError):  # the wrapper does not return a truncated list
        s.lru_apply(ev, now, cap=1)
    check_state(s, ref, "after a short buffer through the wrapper")
    # malformed calls are refused whole: the state does not change
    before = s.lru_state()
    good = [(INSERT, 3, 7, 100, 0), (SETCAP, 4, 0, 0, 0), (TOUCH, 5, 1, 0, 0)]
    for bad in [(INSERT, n_inst, 1, 1, 0), (INSERT, -1, 1, 1, 0), (6, 3, 1, 1, 0), (-1, 3, 1, 1, 0), (TOUCH, 3, 1, 0, -1),
                (SETCAP, 3, 0, 0, -5), (INSERT, 3, -2, 1, 0)]:
        with pytest.raises(MmpError) as ei:
            s.lru_apply(events(good + [bad] + good), now)
        assert ei.value.code == L.E_ARG, bad
        after = s.lru_state()
        assert all(np.array_equal(a, b) for a, b in zip(before, after)), bad
    drain(s, ref, now, "after the refused calls")
    # more resident entries than slots: MMP_E_NOMEM (the state is unspecified afterwards)
    s.lru_init(np.full(n_inst, 2**62, dtype=np.int64), slots)
    with pytest.raises(MmpError) as ei:
        s.lru_apply(events([(INSERT, 4, k, 1, 0) for k in range(slots + 1)]), now)
    assert ei.value.code == L.E_NOMEM
    # a second mmp_lru_init with another slot count starts from empty caches (and an oldestTime() of -1)
    s.lru_init(caps, slots)
    check(s, Ref(oracle_lib, caps), events([(INSERT, 1, 1, 50_000, 0), (SETCAP, 1, 0, 0, 1000)]), now)
    s.lru_init(caps[:5], 7)
    ref = Ref(oracle_lib, caps[:5])
    check_state(s, ref, "re-initialised")
    gen = Gen(rng, caps[:5], 7, np.zeros(5, dtype=bool))
    for call in range(3):
        check(s, ref, gen.batch([11, 12, 13, 1, 0][call:] + [11, 12, 13, 1, 0][:call], now), now, call)
    drain(s, ref, now)


# ---------------------------------------------------------------------------------------------------------------------
# the closed loop with caches too large to stage: hot instances run the hooks on the unstaged path
# ---------------------------------------------------------------------------------------------------------------------
def test_closed_loop_unstaged_matches_oracle(product_lib, oracle_lib):
    from test_churn_gpu import run_small_closed_loop
    run_small_closed_loop(product_lib, False, 0.97, 6, slots=1601)
