"""The resident placement server's slots (one_mode 3, k_place_server): up to MMP_SERVER_SLOTS request threads at once each
get their answer from a slot and a warp of their own, without a launch; a call that finds every slot taken takes the graph
path.  Every answer equals mmp_place_batch with one_mode 0 on the same records, seed and ids, and the oracle on a sample;
mmp_server_stats shows which path answered.  The shapes are those of request threads calling getNext (MM:918-925,
1107-1110): kind 1 (one decision, unflagged or carrying its model's record with 0-4 ids and a fresh row inline) through
mmp_place_one, kind 2 (2-32 decisions through the slot's mapped tables) through mmp_place_batch."""
import copy
import ctypes as C
import threading
import time

import numpy as np
import pytest

from helpers import oracle_from_synth, oracle_inputs, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SplitMix, SynthDecisions, make_decisions, make_fleet
from request_model import hold_front, oracle_request, random_records

pytestmark = pytest.mark.gpu

SLOTS = 8  # MMP_SERVER_SLOTS
SEED = 31


def _pack(sd, rows):
    """Decisions rows of sd as one call of their own: extra[] slices and fresh rows copied into the call's own tables, in
    order (a request thread's shape: its decision's slice starts at 0, its fresh row is row 0)."""
    dec = np.ascontiguousarray(sd.dec[rows]).copy()
    ex, fr = [], []
    o = 0
    for j in range(len(dec)):
        a, n = int(dec["extra_off"][j]), int(dec["extra_n"][j])
        ex.append(sd.extra[a:a + n])
        dec["extra_off"][j] = o if n else 0
        o += n
        if dec["fresh"][j] >= 0:
            fr.append(sd.fresh[dec["fresh"][j]])
            dec["fresh"][j] = len(fr) - 1
    extra = np.ascontiguousarray(np.concatenate(ex), dtype=np.int32) if o else None
    fresh = np.ascontiguousarray(np.stack(fr), dtype=L.INSTANCE_ROW) if fr else None
    return dec, fresh, extra


class Call:
    """One mmp_place_one (kind 1) or mmp_place_batch (kind 2) call with its records and its own result buffer."""

    def __init__(self, sd, rows, one):
        self.dec, self.fresh, self.extra = _pack(sd, rows)
        self.one = one
        self.out = np.zeros(len(self.dec), dtype=L.DECISION_OUT)
        self.want = None

    def run(self, lib, h, now_ms, seed, out=None):
        out = self.out if out is None else out
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731
        if self.one:
            return lib.mmp_place_one(h, p(self.dec), p(self.fresh), p(self.extra), p(out), now_ms, seed)
        return lib.mmp_place_batch(h, p(self.dec), len(self.dec), p(self.fresh), 0 if self.fresh is None else len(self.fresh),
                                   p(self.extra), 0 if self.extra is None else len(self.extra), p(out), now_ms, seed)


@pytest.fixture(scope="module")
def world(product_lib, oracle_lib):
    """A C3 fleet, its oracle, and a pool of calls of both kinds with their one_mode 0 answers."""
    fl = make_fleet("C3", 3000, 10_000, 3)
    o = oracle_from_synth(fl)
    fl = hold_front(fl, o.cluster_order())
    ref = solver_from_synth(fl, product_lib)
    tid = {t: ref.type_id(t) for t in fl.type_names}
    names = list(fl.type_names)
    ids = [tid[t] for t in names]
    plain = make_decisions(fl, 400, 21)
    rq, k = random_records(fl, make_decisions(fl, 400, 22), ids, 22, sizes=(0, 1, 2, 3, 4))
    rq.dec["fresh"] = np.arange(len(rq.dec)) % len(rq.fresh)  # each with a fresh row of the caller's
    rng = SplitMix(23)
    calls = []
    for i in range(200):
        calls.append(Call(plain, [i], True))                                     # unflagged, its own extras and fresh row
        calls.append(Call(rq, [i], True))                                        # the model's record inline: 0-4 ids, fresh row
        n = int(rng.randint(1, 2, 33)[0])                                        # 2-32 decisions, both kinds mixed
        a = int(rng.randint(1, 0, 400 - n)[0])
        src = plain if i % 2 else rq
        calls.append(Call(src, list(range(a, a + n)), False))
    assert all(len(c.dec) == 1 and (c.extra is None or len(c.extra) <= 4) for c in calls if c.one)  # kind 1: inline
    ref._ck(product_lib.mmp_tune(ref.h, b"one_mode", 0))
    for c in calls:
        c.want = ref.place_batch(c.dec, fl.now_ms, SEED, fresh=c.fresh, extra=c.extra)
    ref.close()
    # the oracle on a sample of kind-1 calls of each shape (mmp_place_one numbers its decision 0); calls[3 i] is plain
    # decision i, calls[3 i + 1] request-model decision i
    o = oracle_from_synth(fl)
    none = np.zeros(0, dtype=np.int32)
    for i in range(0, 200, 5):
        c = calls[3 * i]
        sd1 = SynthDecisions(c.dec, c.fresh if c.fresh is not None else plain.fresh[:0], c.extra if c.extra is not None else none)
        od, off, idx = oracle_inputs(fl, sd1)
        got = o.get_next_batch(od, names, off, idx, fl.now_ms, SEED, fresh=c.fresh)
        assert (got["target"][0], got["n_candidates"][0]) == (c.want["target"][0], c.want["n_candidates"][0]), ("plain", i)
        c = calls[3 * i + 1]
        sd1 = SynthDecisions(c.dec, c.fresh, c.extra if c.extra is not None else none)
        got = oracle_request(o, names, k[[i]], sd1, fl.now_ms, SEED)
        assert (got["target"][0], got["n_candidates"][0]) == (c.want["target"][0], c.want["n_candidates"][0]), ("request", i)
    return fl, calls


def _fleet(lib, fl, **tune):
    s = solver_from_synth(fl, lib)
    s._ck(lib.mmp_tune(s.h, b"one_mode", 3))
    for key, v in tune.items():
        s._ck(lib.mmp_tune(s.h, key.encode(), v))
    return s


def _stats(s):
    st = s.server_stats()
    assert set(st) == {"answered", "fallbacks", "launches", "max_busy"}
    return st


def _threads(lib, s, fl, calls, n_threads, per_thread):
    """n_threads threads released together, each making per_thread calls from the pool; every answer checked."""
    barrier = threading.Barrier(n_threads)
    bad, errors = [], []

    def work(t):
        outs = [np.zeros(len(c.dec), dtype=L.DECISION_OUT) for c in calls]
        try:
            barrier.wait()
            for j in range(per_thread):
                q = (t * 97 + j * 7) % len(calls)
                c = calls[q]
                if c.run(lib, s.h, fl.now_ms, SEED, outs[q]) < 0:
                    raise RuntimeError(lib.mmp_last_error(s.h))
                if not np.array_equal(outs[q], c.want):
                    bad.append((t, j, q))
        except Exception as e:  # pragma: no cover
            errors.append(e)

    ts = [threading.Thread(target=work, args=(t,)) for t in range(n_threads)]
    for th in ts:
        th.start()
    for th in ts:
        th.join()
    assert not errors, errors[:2]
    assert not bad, (len(bad), bad[:5])
    return n_threads * per_thread


def test_eight_threads_each_get_a_slot(product_lib, world):
    fl, calls = world
    s = _fleet(product_lib, fl)
    n = _threads(product_lib, s, fl, calls, SLOTS, 300)
    st = _stats(s)
    # with at most MMP_SERVER_SLOTS callers a slot is always free: every call is the server's
    assert st["fallbacks"] == 0 and st["answered"] == n, st
    assert 2 <= st["max_busy"] <= SLOTS and st["launches"] >= 1, st
    s.close()


def test_sixteen_threads(product_lib, world):
    fl, calls = world
    s = _fleet(product_lib, fl)
    n = _threads(product_lib, s, fl, calls, 2 * SLOTS, 200)
    st = _stats(s)
    assert st["answered"] + st["fallbacks"] == n and st["max_busy"] <= SLOTS, st
    s.close()


def test_single_caller_launches_once_per_lifetime_or_epoch(product_lib, world):
    fl, calls = world
    life = 500_000  # (µs) longer than the calls below take: one launch serves them all
    s = _fleet(product_lib, fl, server_life_us=life, server_idle_us=life)
    t0 = time.monotonic()
    n = _threads(product_lib, s, fl, calls[:150], 1, 150)
    quick = time.monotonic() - t0 < 0.8 * life / 1e6  # (a host stall longer than the lifetime would end it: a relaunch)
    st = _stats(s)
    assert st["answered"] == n and st["fallbacks"] == 0 and st["max_busy"] == 1, st
    assert st["launches"] == 1 or not quick, st
    s.commit()  # a new epoch: the next call stops the block on the old view and launches one on the new
    t0 = time.monotonic()
    n += _threads(product_lib, s, fl, calls[:150], 1, 150)
    quick = time.monotonic() - t0 < 0.8 * life / 1e6
    st2 = _stats(s)
    assert st2["answered"] == n and st2["fallbacks"] == 0 and st2["max_busy"] == 1, st2
    assert st2["launches"] == st["launches"] + 1 or (not quick and st2["launches"] > st["launches"]), (st, st2)
    s.close()


def test_destroy_with_the_server_resident(product_lib, world):
    fl, calls = world
    s = _fleet(product_lib, fl, server_life_us=1_000_000, server_idle_us=1_000_000)
    _threads(product_lib, s, fl, calls[:30], 4, 30)
    assert _stats(s)["launches"] >= 1
    t0 = time.monotonic()
    s.close()  # the block is resident (1 s idle time): destroying the fleet makes it leave
    assert time.monotonic() - t0 < 0.9
    s2 = _fleet(product_lib, fl)
    _threads(product_lib, s2, fl, calls, 4, 100)
    assert _stats(s2)["answered"] == 400
    s2.close()


def _oracle_answers(fl, rows, sd, seed):
    """Per decision the oracle's target and count under instance rows `rows`, each decision a batch of one (id 0)."""
    fl2 = copy.copy(fl)
    fl2.inst_rows = rows
    o = oracle_from_synth(fl2)
    od, off, idx = oracle_inputs(fl2, sd)
    od["decision_id"] = 0
    res = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)
    return res["target"].copy(), res["n_candidates"].copy()


def test_commits_and_restarts_while_eight_threads_place(product_lib, oracle_lib):
    """A writer alternates device-path commits between two instance states and makes one structural commit while 8 readers
    place through the server, restarted often (200 µs life, 50 µs idle).  Every answer is the oracle's under one of the two
    states -- never a mixture -- and the block was launched again across epochs."""
    lib = product_lib
    fl = make_fleet("C3", 3000, 700, 3)
    sd = make_decisions(fl, 1024, 9)
    rows_a = fl.inst_rows.copy()
    rows_b = fl.inst_rows.copy()
    rng = np.random.default_rng(1)
    live = np.nonzero(rows_a["shutting_down"] == 0)[0]
    changed = rng.choice(live, size=150, replace=False)
    for i in changed:
        rows_b[i]["used"] = int(rng.integers(0, rows_b[i]["capacity"] + 1))
        rows_b[i]["count"] = int(rng.integers(0, 300))
        rows_b[i]["lru_time"] = int(fl.now_ms - rng.integers(1, 5_000_000))
    s = _fleet(lib, fl, server_life_us=200, server_idle_us=50)
    calls = [Call(sd, [i], True) for i in range(len(sd.dec))]
    results = np.zeros((3, len(calls)), dtype=L.DECISION_OUT)
    stop = threading.Event()
    errors, paths = [], []

    def writer():
        k = 0
        while not stop.is_set():
            rows = rows_b if k % 2 == 0 else rows_a
            try:
                for i in changed:
                    s.instance_update(int(i), rows[i])
                if k == 3:  # one structural (host-path) commit among the device-path ones
                    s._ck(lib.mmp_tune(s.h, b"commit_host_only", 1))
                s.commit()
                if k == 3:
                    s._ck(lib.mmp_tune(s.h, b"commit_host_only", 0))
                paths.append(s.commit_info()[0])
            except Exception as e:  # pragma: no cover
                errors.append(e)
                return
            k += 1

    barrier = threading.Barrier(SLOTS)

    def reader(t):
        out = np.zeros(1, dtype=L.DECISION_OUT)
        try:
            barrier.wait()
            for rep in range(3):
                for i in range(t, len(calls), SLOTS):
                    if calls[i].run(lib, s.h, fl.now_ms, SEED, out) < 0:
                        raise RuntimeError(lib.mmp_last_error(s.h))
                    results[rep, i] = out[0]
        except Exception as e:  # pragma: no cover
            errors.append(e)

    wt = threading.Thread(target=writer)
    wt.start()
    readers = [threading.Thread(target=reader, args=(t,)) for t in range(SLOTS)]
    for r in readers:
        r.start()
    for r in readers:
        r.join()
    stop.set()
    wt.join()
    assert not errors, errors[:2]
    st = _stats(s)
    assert st["answered"] == 3 * len(calls) and st["fallbacks"] == 0, st
    assert st["launches"] > 1, st
    assert 1 in paths and 2 in paths, paths[:20]  # a structural commit and device-path commits both happened
    ta, ca = _oracle_answers(fl, rows_a, sd, SEED)
    tb, cb = _oracle_answers(fl, rows_b, sd, SEED)
    ok_a = (results["target"] == ta) & (results["n_candidates"] == ca)
    ok_b = (results["target"] == tb) & (results["n_candidates"] == cb)
    bad = np.argwhere(~(ok_a | ok_b))
    assert len(bad) == 0, (len(bad), bad[:5])
    assert np.count_nonzero(ta != tb) > 20  # the two states really differ
    s.close()
