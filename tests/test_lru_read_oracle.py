"""The read side of the oracle's time-ordered weighted LRU (orc_lru_read, orc_lru_last_used and orc_lru_weight of
tests/emul/lru_read_oracle.cpp) against orderedMap(false, MAX, usedSince) (CLHM:1226-1260), getLastUsedTime (CLHM:742-746)
and getWeight (CLHM:768-771) restated over the plain Python list of test_oracle_properties.py (itself pinned to the
oracle's deque there).

The device derives the walk from the (ts, seq) order of its slots instead of walking a deque: every entry with
ts >= used_since, and the entries with ts <= 0 only when no entry has 0 < ts < used_since.  Without forceSetLastUsedTime the
deque is ordered by lastUsed, so the literal walk must equal that derivation; the last test checks it on random streams."""
import numpy as np
import pytest

from lru_read_oracle import _read_oracle_so, lru_last_used, lru_read, lru_weight, read_oracle  # noqa: F401 (fixtures)
from oracle import binding as ob
from test_oracle_properties import BruteLru

pytestmark = pytest.mark.usefixtures("read_oracle")


def ordered_map(deque, used_since):
    """CLHM:1239-1250 over [key, weight, lastUsed] nodes, oldest first"""
    out = []
    for key, weight, last_used in reversed(deque):
        if last_used > 0 and last_used < used_since:
            break
        out.append((key, last_used, weight))
    return out


def derived(deque, used_since):
    """the device's rule, in deque order walked from the tail"""
    stops = any(0 < t < used_since for _, _, t in deque)
    return [(k, t, w) for k, w, t in reversed(deque) if t >= used_since or (t <= 0 and not stops)]


def cutoffs(deque, rng):
    ts = sorted({t for _, _, t in deque})
    picks = [0, -1, -(2**62), 2**62, 1]
    for t in rng.choice(ts, size=min(4, len(ts)), replace=False) if ts else []:
        picks += [int(t), int(t) + 1, int(t) - 1]
    if ts:
        picks += [ts[-1] + 1, ts[0]]
    return picks


def _stream(rng, n, now, force):
    ev = np.zeros(n, dtype=ob.LRU_EVENT)
    r = rng.uniform(size=n)
    ev["op"] = np.where(r < 0.45, 0, np.where(r < 0.72, 1, np.where(r < 0.85, 2, np.where(r < 0.94, 3, np.where(r < 0.97, 4, 5)))))
    if not force:
        ev["op"] = np.where(ev["op"] == 5, 1, ev["op"])
    ev["key"] = rng.integers(0, 120, size=n)
    ev["weight"] = np.where(ev["op"] == 4, rng.integers(15_000, 60_000, size=n), rng.integers(1, 6000, size=n))
    # coarse times (equal lastUsed values are common), 0 = now, and forced times of 0 and below
    lu = now - rng.integers(0, 50, size=n) * 10_000
    lu = np.where(rng.uniform(size=n) < 0.3, 0, lu)
    ev["last_used"] = np.where(ev["op"] == 5, np.where(rng.uniform(size=n) < 0.3, -rng.integers(0, 3, size=n), lu), lu)
    return ev


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("force", [False, True])
def test_read_matches_ordered_map(oracle_lib, seed, force):
    rng = np.random.default_rng(700 + seed + 50 * force)
    cap = int(rng.integers(20_000, 60_000))
    o, b = ob.OracleLru(cap), BruteLru(cap)
    now = 1_000_000
    stopped = full = 0
    for batch in range(8):
        n = 300
        ev = _stream(rng, n, now, force)
        o.apply(ev, now)
        sink = []
        for i in range(n):
            b.apply(int(ev["op"][i]), int(ev["key"][i]), int(ev["weight"][i]), int(ev["last_used"][i]), i, now, sink)
        for u in cutoffs(b.deque, rng):
            k, t, w = lru_read(o, u)
            want = ordered_map(b.deque, u)
            assert list(zip(k.tolist(), t.tolist(), w.tolist())) == want, (batch, u)
            stopped += len(want) < len(b.deque)
            full += len(want) == len(b.deque)
        for key in list(range(0, 130, 3)):
            node = b._find(key)
            assert lru_last_used(o, key) == (-1 if node is None or node[2] <= 0 else node[2]), (batch, key)
            assert lru_weight(o, key) == (-1 if node is None else node[1]), (batch, key)
        now += int(rng.integers(1, 200_000))
    assert stopped > 10 and full > 10


def test_entries_at_or_below_zero(oracle_lib):
    """lastUsed <= 0 never stops the walk; those entries are read only when nothing in (0, used_since) stops it first"""
    o, b = ob.OracleLru(1 << 40), BruteLru(1 << 40)
    rows = [(0, 1, 5, 0), (0, 2, 5, 0), (0, 3, 5, 700), (0, 4, 5, 900), (0, 5, 5, 0)]
    ev = np.array(rows, dtype=ob.LRU_EVENT)
    o.apply(ev, 0)  # now = 0: lastUsed 0 for keys 1, 2, 5
    sink = []
    for i, r in enumerate(rows):
        b.apply(*r, i, 0, sink)
    assert [n[2] for n in b.deque] == [0, 0, 0, 700, 900]
    assert lru_read(o, 800)[0].tolist() == [4]               # 700 stops the walk before the zeros
    assert lru_read(o, 700)[0].tolist() == [4, 3, 5, 2, 1]   # nothing in (0, 700): the zeros follow, newest first
    assert lru_read(o, 0)[0].tolist() == [4, 3, 5, 2, 1]
    assert lru_read(o, 10_000)[0].tolist() == []
    assert lru_last_used(o, 1) == -1 and lru_weight(o, 1) == 5 and lru_last_used(o, 4) == 900 and lru_weight(o, 99) == -1
    for u in (-5, 0, 1, 700, 701, 800, 900, 901):
        assert list(zip(*[x.tolist() for x in lru_read(o, u)])) == ordered_map(b.deque, u) == derived(b.deque, u), u


@pytest.mark.parametrize("seed", range(4))
def test_walk_equals_the_derivation_without_forced_times(oracle_lib, seed):
    rng = np.random.default_rng(900 + seed)
    o = ob.OracleLru(int(rng.integers(20_000, 60_000)))
    now = 0  # the first batch inserts at lastUsed 0 (= now) and below
    for batch in range(8):
        o.apply(_stream(rng, 300, now, False), now)
        kd, td, wd = o.dump()
        deque = [[int(x), int(y), int(z)] for x, y, z in zip(kd, wd, td)]
        for u in cutoffs(deque, rng):
            k, t, w = lru_read(o, u)
            assert list(zip(k.tolist(), t.tolist(), w.tolist())) == derived(deque, u), (batch, u)
        now += int(rng.integers(1, 200_000))
