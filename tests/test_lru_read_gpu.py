"""The read side of plug point 3 -- mmp_lru_read (descendingMapWithCutoff / descendingLruMap, CLHM:1226-1260, 1087-1116) and
mmp_lru_lookup (getLastUsedTime / getWeight, CLHM:742-771) -- against the oracle, whose walk follows its linked deque with the
literal break rule (tests/emul/lru_read_oracle.cpp, pinned in test_lru_read_oracle.py).  The standalone store is read after every apply call at cutoffs
around its timestamps, on shapes whose walks take the shared-memory path (up to 2048 entries) and the global-memory path;
the closed loop's caches are read after every window, with each copy's registration time."""
import ctypes as C
import threading
import time

import numpy as np
import pytest

from churn_harness import build, compare_window
from modelmesh_b200 import _lib as L
from lru_read_oracle import _read_oracle_so, lru_last_used, lru_read, lru_weight, read_oracle, sim_lru_read  # noqa: F401
from modelmesh_b200.fleet import MmpError, _ptr
from lru_ref import INSERT, NOW0, SETCAP, TOUCH, Gen, Ref, check, events, fleet

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("read_oracle")]

SMEM_WALK = 2048  # LRU_READ_SMEM: longer walks take the global-memory path


def want_read(ref, instances, used_since):
    """the oracle's walks, concatenated: (offsets, [(model, weight, last_used)])"""
    off, rows = [0], []
    for i in instances:
        k, t, w = lru_read(ref.lru[i], used_since)
        rows += list(zip(k.tolist(), w.tolist(), t.tolist()))
        off.append(len(rows))
    return off, rows


def as_rows(entries):
    return list(zip(entries["model"].tolist(), entries["weight"].tolist(), entries["last_used"].tolist()))


def cutoffs(s, rng):
    """0, a negative value, an existing timestamp, one above and one below it, above every timestamp"""
    _, e = s.lru_read()
    ts = np.unique(e["last_used"])
    picks = [0, -1, -(2**40)]
    if len(ts):
        for t in rng.choice(ts, size=min(3, len(ts)), replace=False):
            picks += [int(t), int(t) + 1, int(t) - 1]
        picks.append(int(ts[-1]) + 1)
    return picks


def check_read(s, ref, used_since, instances=None, tag=""):
    ids = list(range(len(ref.lru))) if instances is None else list(instances)
    off, e = s.lru_read(instances, used_since)
    want_off, want = want_read(ref, ids, used_since)
    assert off.tolist() == want_off, (tag, used_since)
    got = as_rows(e)
    if got != want:
        j = next(j for j, (a, b) in enumerate(zip(got, want)) if a != b)
        k = int(np.searchsorted(off, j, side="right")) - 1
        raise AssertionError((tag, used_since, "instance", ids[k], "position", j - int(off[k]), got[j:j + 3], want[j:j + 3]))
    assert (e["load_ts"] == -1).all(), tag  # the standalone store registers nothing
    return off


def check_lookup(s, ref, rng, keys, tag=""):
    n = 400
    inst = rng.integers(0, len(ref.lru), size=n).astype(np.int32)
    model = rng.integers(-2, keys + 20, size=n).astype(np.int32)
    lu, w, lt = s.lru_lookup(inst, model)
    for q in range(n):
        o = ref.lru[int(inst[q])]
        m = int(model[q])
        want_lu = -1 if m < 0 else lru_last_used(o, m)
        want_w = -1 if m < 0 else lru_weight(o, m)
        assert (int(lu[q]), int(w[q]), int(lt[q])) == (want_lu, want_w, -1), (tag, int(inst[q]), m)
    present = sum(int(w[q]) != -1 for q in range(n))
    return present


@pytest.mark.parametrize("slots,n_inst,hot", [(64, 64, False), (512, 64, True), (4096, 6, True)])
def test_standalone_reads_match_oracle(product_lib, oracle_lib, slots, n_inst, hot):
    rng = np.random.default_rng(slots + n_inst)
    caps = rng.integers(20_000, 60_000, size=n_inst).astype(np.int64)
    if hot:
        caps[1] = 2**40  # one cache that keeps every insert: its walk outgrows the shared-memory path on the last shape
    s = fleet(product_lib)
    s.lru_init(caps, slots)
    ref = Ref(oracle_lib, caps)
    keys = min(slots, 3500)
    gen = Gen(rng, caps, keys, np.zeros(n_inst, dtype=bool))
    now = NOW0
    if slots > SMEM_WALK:  # 2300 entries in runs of 50 equal times
        check(s, ref, events([(INSERT, 1, k, 1 + k % 7, now - (k // 50) * 1000) for k in range(2300)]), now, "fill")
    longest = present = 0
    for call in range(6):
        counts = [int(x) for x in rng.integers(0, 40, size=n_inst)]
        if hot:
            counts[1] = 600 if slots > SMEM_WALK else 200
        ev = gen.batch(counts, now)
        if hot:  # small weights and SET_CAPACITY events that keep the hot cache large
            mine = ev["instance"] == 1
            ev["weight"][mine] = rng.integers(1, 100, size=int(mine.sum()))
            ev["last_used"][mine & (ev["op"] == SETCAP)] = 2**40
        check(s, ref, ev, now, (slots, call))
        for u in cutoffs(s, rng):
            off = check_read(s, ref, u, tag=(slots, call))
            longest = max(longest, int(np.diff(off).max()))
        present += check_lookup(s, ref, rng, keys, (slots, call))
        now += int(rng.integers(1, 400_000))
    assert present > 50
    if slots > SMEM_WALK:
        assert longest > SMEM_WALK, longest
    ms = C.c_double()
    assert s.lib.mmp_last_timing(s.h, b"lru_read", C.byref(ms)) == 0 and ms.value > 0


def test_entries_at_or_below_zero(product_lib, oracle_lib):
    """entries touched at now_ms = 0 hold lastUsed 0: read only when nothing in (0, used_since) stops the walk"""
    s = fleet(product_lib)
    caps = np.full(3, 10**9, dtype=np.int64)
    s.lru_init(caps, 64)
    ref = Ref(oracle_lib, caps)
    check(s, ref, events([(INSERT, 0, 1, 5, 0), (INSERT, 0, 2, 5, 0), (INSERT, 1, 7, 5, 0), (INSERT, 2, 9, 5, 0)]), 0)
    check(s, ref, events([(INSERT, 0, 3, 5, 700), (INSERT, 0, 4, 5, 900), (INSERT, 0, 5, 5, 0), (TOUCH, 0, 1, 0, 0),
                          (INSERT, 2, 8, 5, 300)]), 0)
    for u in (-1, 0, 1, 300, 301, 700, 701, 900, 901):
        check_read(s, ref, u, tag=u)
    _, e = s.lru_read([0], 701)
    assert e["model"].tolist() == [4]                       # 700 stops the walk before the zeros
    _, e = s.lru_read([0], 700)
    assert e["model"].tolist() == [4, 3, 5, 2, 1]           # nothing in (0, 700): the zeros follow, newest first
    _, e = s.lru_read([1], 10**6)
    assert e["model"].tolist() == [7]                       # only zeros: nothing stops the walk
    lu, w, _ = s.lru_lookup([0, 0, 1], [1, 4, 7])
    assert lu.tolist() == [-1, 900, -1] and w.tolist() == [5, 5, 5]


def test_reads_do_not_change_the_caches(product_lib, oracle_lib):
    rng = np.random.default_rng(5)
    n_inst = 40
    caps = rng.integers(20_000, 60_000, size=n_inst).astype(np.int64)
    s = fleet(product_lib)
    s.lru_init(caps, 96)
    ref = Ref(oracle_lib, caps)
    gen = Gen(rng, caps, 80, np.zeros(n_inst, dtype=bool))
    now = NOW0
    for call in range(4):
        check(s, ref, gen.batch([int(x) for x in rng.integers(0, 30, size=n_inst)], now), now, call)
        now += 100_000
    before = s.lru_state()
    off, e = s.lru_read()
    s.lru_read(None, now - 50_000)
    s.lru_lookup(np.arange(n_inst), np.zeros(n_inst))
    after = s.lru_state()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    # a capacity-0 drain evicts each cache oldest first: the reversed read, entry for entry
    ev = s.lru_apply(events([(SETCAP, i, 0, 0, 0) for i in range(n_inst)]), now, cap=len(e) + 16)
    assert len(ev) == len(e) > 200
    for i in range(n_inst):
        mine = ev[ev["instance"] == i]
        walk = e[off[i]:off[i + 1]][::-1]
        assert mine["model"].tolist() == walk["model"].tolist() and mine["last_used"].tolist() == walk["last_used"].tolist(), i
        assert mine["weight"].tolist() == walk["weight"].tolist(), i
    off, e = s.lru_read()
    assert len(e) == 0 and not off.any()


def _raw_read(s, instances, n, used_since, cap, sentinel=0x5A):
    ids = None if instances is None else np.ascontiguousarray(instances, dtype=np.int32)
    off = np.full(n + 1, sentinel, dtype=np.int64)
    out = np.zeros(max(cap, 1) + 2, dtype=L.LRU_ENTRY)
    out.view(np.uint8)[:] = sentinel
    rc = s.lib.mmp_lru_read(s.h, _ptr(ids), n, used_since, _ptr(off), _ptr(out), cap)
    return rc, off, out


def test_read_abi_edges(product_lib, oracle_lib):
    s = fleet(product_lib)
    # before mmp_lru_init: MMP_E_STATE, nothing written
    rc, off, out = _raw_read(s, None, 2, 0, 4)
    assert rc == L.E_STATE and (off == 0x5A).all() and (out.view(np.uint8) == 0x5A).all()
    a = np.zeros(1, dtype=np.int64)
    assert s.lib.mmp_lru_lookup(s.h, 1, _ptr(np.zeros(1, np.int32)), _ptr(np.zeros(1, np.int32)), _ptr(a), _ptr(np.zeros(1, np.int32)),
                                _ptr(a)) == L.E_STATE
    rng = np.random.default_rng(9)
    n_inst = 12
    caps = rng.integers(20_000, 60_000, size=n_inst).astype(np.int64)
    s.lru_init(caps, 64)
    ref = Ref(oracle_lib, caps)
    gen = Gen(rng, caps, 64, np.zeros(n_inst, dtype=bool))
    counts = [int(x) for x in rng.integers(5, 30, size=n_inst)]
    counts[3] = counts[8] = 0  # empty caches
    check(s, ref, gen.batch(counts, NOW0), NOW0)
    full_off, full = s.lru_read()
    total = len(full)
    assert total > 50 and full_off[4] == full_off[3] and full_off[9] == full_off[8]
    # cap 0, 1, total - 1, total, total + 1: offsets whole, the first cap entries written, nothing past them
    for cap in (0, 1, total - 1, total, total + 1):
        rc, off, out = _raw_read(s, None, n_inst, 0, cap)
        assert rc == 0 and off.tolist() == full_off.tolist(), cap
        k = min(cap, total)
        assert as_rows(out[:k]) == as_rows(full[:k]), cap
        assert (out[k:].view(np.uint8) == 0x5A).all(), cap
    # subsets, repeated instances, NULL for all instances
    for ids in ([5], [3], [7, 2, 7, 7, 0], list(range(n_inst))[::-1], [8, 3]):
        check_read(s, ref, 0, ids, tag=ids)
        check_read(s, ref, NOW0 - 10_000, ids, tag=ids)
    rc, off, out = _raw_read(s, None, 4, 0, total)
    assert rc == 0 and off.tolist() == full_off[:5].tolist()
    rc, off, out = _raw_read(s, [], 0, 0, 0)
    assert rc == 0 and off.tolist() == [0]
    # errors: MMP_E_ARG, nothing written
    sentinel = lambda off, out: (off == 0x5A).all() and (out.view(np.uint8) == 0x5A).all()
    for ids, n, cap in (([0, -1], 2, 8), ([n_inst], 1, 8), (None, n_inst + 1, 8), ([1], 1, -1)):
        rc, off, out = _raw_read(s, ids, n, 0, cap)
        assert rc == L.E_ARG and sentinel(off, out), (ids, n, cap)
    out = np.zeros(4, dtype=L.LRU_ENTRY)
    assert s.lib.mmp_lru_read(s.h, None, 2, 0, None, _ptr(out), 4) == L.E_ARG            # offsets NULL
    off = np.full(3, 0x5A, dtype=np.int64)
    assert s.lib.mmp_lru_read(s.h, None, 2, 0, _ptr(off), None, 4) == L.E_ARG and (off == 0x5A).all()  # out NULL, cap > 0
    assert s.lib.mmp_lru_read(s.h, None, 2, 0, _ptr(off), None, 0) == 0 and off.tolist() == full_off[:3].tolist()
    # lookup errors
    i1, m1 = np.array([n_inst], np.int32), np.array([1], np.int32)
    lu, w, lt = np.full(1, 7, np.int64), np.full(1, 7, np.int32), np.full(1, 7, np.int64)
    assert s.lib.mmp_lru_lookup(s.h, 1, _ptr(i1), _ptr(m1), _ptr(lu), _ptr(w), _ptr(lt)) == L.E_ARG
    i1[0] = -1
    assert s.lib.mmp_lru_lookup(s.h, 1, _ptr(i1), _ptr(m1), _ptr(lu), _ptr(w), _ptr(lt)) == L.E_ARG
    i1[0] = 0
    assert s.lib.mmp_lru_lookup(s.h, 1, _ptr(i1), _ptr(m1), None, _ptr(w), _ptr(lt)) == L.E_ARG
    assert s.lib.mmp_lru_lookup(s.h, 1, None, _ptr(m1), _ptr(lu), _ptr(w), _ptr(lt)) == L.E_ARG
    assert lu[0] == 7 and w[0] == 7 and lt[0] == 7
    with pytest.raises(MmpError):
        s.lru_read([n_inst])


# ---------------------------------------------------------------------------------------------------------------------
# the closed loop: every cache after every window, with the registration time of each copy
# ---------------------------------------------------------------------------------------------------------------------
def _check_loop_caches(ep, sim, s, fl, pairs):
    off, e = s.lru_read()
    assert len(off) == fl.n_instances + 1
    for i in range(fl.n_instances):
        k, t, w, lt = sim_lru_read(sim, i)
        got = e[off[i]:off[i + 1]]
        assert got["model"].tolist() == k.tolist() and got["last_used"].tolist() == t.tolist(), (ep, i)
        assert got["weight"].tolist() == w.tolist() and got["load_ts"].tolist() == lt.tolist(), (ep, i)
    assert (e["load_ts"] >= 0).all(), ep  # every cached copy of the loop is registered
    u = int(np.median(e["last_used"])) if len(e) else 0
    off2, e2 = s.lru_read(None, u)
    for i in range(0, fl.n_instances, 7):
        assert e2[off2[i]:off2[i + 1]]["model"].tolist() == sim_lru_read(sim, i, u)[0].tolist(), (ep, i, u)
    if pairs:  # the (instance, model) pairs over all caches are the registry's loaded copies
        inst_of = np.repeat(np.arange(fl.n_instances), np.diff(off))
        cached = set(zip(inst_of.tolist(), e["model"].tolist()))
        loaded = set()
        for m in range(fl.n_models):
            row, ids = s.churn_model_ids(m)
            loaded |= {(int(x), m) for x in ids[:int(row["copy_count"])]}
        assert cached == loaded, (ep, sorted(cached ^ loaded)[:5])
        lu, w, lt = s.lru_lookup(inst_of[::5], e["model"][::5])
        assert lu.tolist() == [x if x > 0 else -1 for x in e["last_used"][::5].tolist()], ep
        assert w.tolist() == e["weight"][::5].tolist() and lt.tolist() == e["load_ts"][::5].tolist(), ep


@pytest.mark.parametrize("overflow", [False, True])
@pytest.mark.parametrize("with_types", [False, True])
def test_closed_loop_reads_match_oracle(product_lib, oracle_lib, overflow, with_types):
    from modelmesh_b200.synth import make_churn, make_churn_overflow
    seed = 4 + with_types
    w = make_churn(20_000, 200, seed, fill=0.90, with_types=with_types)
    if overflow:
        w = make_churn_overflow(w, 0.05, seed)
    fl = w.fleet
    o, sim, s = build(product_lib, w, slots=256)
    _check_loop_caches(-1, sim, s, fl, True)
    for ep in range(8):
        ev = w.events(ep, 2000, seed)
        now0 = fl.now_ms + ep * w.window_ms
        compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, seed * 100 + ep)
        _check_loop_caches(ep, sim, s, fl, ep in (3, 7))


# ---------------------------------------------------------------------------------------------------------------------
# reads concurrent with a writer see whole apply calls
# ---------------------------------------------------------------------------------------------------------------------
def test_concurrent_reads_see_whole_calls(product_lib, oracle_lib):
    rng = np.random.default_rng(21)
    n_inst, n_calls = 48, 24
    caps = rng.integers(20_000, 60_000, size=n_inst).astype(np.int64)
    s = fleet(product_lib)
    s.lru_init(caps, 128)
    ref = Ref(oracle_lib, caps)
    gen = Gen(rng, caps, 100, np.zeros(n_inst, dtype=bool))
    batches, states = [], [want_read(ref, range(n_inst), 0)]
    now = NOW0
    for call in range(n_calls):
        ev = gen.batch([int(x) for x in rng.integers(0, 40, size=n_inst)], now)
        ref.apply(ev, now)
        batches.append((ev, now))
        states.append(want_read(ref, range(n_inst), 0))
        now += int(rng.integers(1, 100_000))
    seen, errors, done = [], [], threading.Event()

    def writer():
        try:
            for ev, t in batches:
                time.sleep(0.005)  # (readers get in between the calls)
                s.lru_apply(ev, t, cap=4 * len(ev) + 100_000)
        except Exception as e:  # noqa: BLE001
            errors.append(e)
        finally:
            done.set()

    def reader():
        try:
            while not done.is_set():
                off, e = s.lru_read()
                seen.append((off.tolist(), as_rows(e)))
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=writer)] + [threading.Thread(target=reader) for _ in range(3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    index = {(tuple(off), tuple(rows)): j for j, (off, rows) in enumerate(states)}
    hits = [index.get((tuple(off), tuple(rows))) for off, rows in seen]
    assert None not in hits, hits.index(None)
    assert len(seen) > 10 and len(set(hits)) > 1, (len(seen), sorted(set(hits)))
    check_read(s, ref, 0, tag="after")
