"""The per-instance LRU caches of the tests on the oracle's side: events() builds an mmp_lru_event array, Ref holds every
instance's cache on ob.OracleLru (an MMP_LRU_LOAD event as loadLocal's literal sequence), check() runs one call through the
device and Ref and compares evictions, statuses and state, and Gen draws random events per cache."""
import numpy as np

from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet
from oracle import binding as ob

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
