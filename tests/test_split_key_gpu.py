"""The per-model entry k_place_split reads (SplitKey: the model row's last_used, the lowest live rank of its inline edges,
its type slot and overflow mark), built by every commit path beside excl_ranks.  After each commit of a replayed
sequence a batch is placed with the two-pass path forced on (split = 1) and off (split = 0): the two must be byte
identical, and both equal the oracle.  The sequence moves every input of the entry: type changes (and request-model
decisions for a type id past the snapshot's type table), a model crossing between 4 and 5 edges, an excluded instance leaving the fleet, last_used
at its extremes and at the five-day line, a rolling upgrade, a churn window's commit, and placements on the old epoch
while a commit builds the new one."""
import threading

import numpy as np
import pytest

from churn_harness import build, compare_window
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthDecisions, make_churn, make_fleet
from oracle import binding as ob
from replay import GAP_TYPE, NUMERIC, STRUCTURAL, Replay, assert_same_results, oracle_batch
from upgrade import bump

pytestmark = pytest.mark.gpu

LONG_MIN, LONG_MAX = -(1 << 63), (1 << 63) - 1
FIVE_DAYS_MS = 5 * 86_400_000


def _place(rp, sd, seed, split):
    f = rp.f
    f._ck(rp.lib.mmp_tune(f.h, b"split", split))
    try:
        return f.place_batch(sd.dec, rp.now, seed, fresh=sd.fresh if len(sd.fresh) else None,
                             extra=sd.extra if len(sd.extra) else None)
    finally:
        f._ck(rp.lib.mmp_tune(f.h, b"split", 2))


def _sweep(rp, seed, flags=L.DF_MODEL_LAST_USED, last_used=None):
    """One decision per registry row (gap rows included), self drawn from the live set, a quarter favouring self."""
    rng = np.random.default_rng(seed)
    live = rp._live()
    n = rp.n_used
    dec = np.zeros(n, dtype=L.DECISION_IN)
    dec["model"] = np.arange(n)
    dec["self"] = live[rng.integers(0, len(live), size=n)]
    dec["flags"] = np.where(rng.uniform(size=n) < 0.25, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(flags)
    dec["fresh"] = -1
    if last_used is not None:
        dec["last_used"] = rng.choice(np.asarray(last_used, dtype=np.int64), size=n)
    return SynthDecisions(dec, np.zeros(0, dtype=L.INSTANCE_ROW), np.zeros(0, dtype=np.int32))


def _check(rp, seed, what, extra_batches=()):
    v, o = rp.view(), rp.oracle()
    for k, sd in enumerate((_sweep(rp, seed), rp.decisions(3000, seed + 1), rp.decisions(3000, seed + 2, plain=True)) + tuple(extra_batches)):
        on, off = _place(rp, sd, seed + k, 1), _place(rp, sd, seed + k, 0)
        assert on.tobytes() == off.tobytes(), (what, k, int(np.sum(on != off)))
        assert_same_results(on, oracle_batch(v, sd, o, seed + k), (what, k))


def _request_batch(rp, seed, n=2000):
    """Request-model decisions (MMP_DF_REQUEST_MODEL: the model field is a type id, no registry row is read), half of them
    for a type id past the snapshot's type table, which resolves as type 0, with the oracle's batch for them (no
    exclusions: no extras)."""
    rng = np.random.default_rng(seed)
    live = rp._live()
    name_of = {i: t for t, i in rp.tid.items()}
    known = np.asarray(sorted(name_of), dtype=np.int64)
    dec = np.zeros(n, dtype=L.DECISION_IN)
    dec["model"] = np.where(rng.uniform(size=n) < 0.5, 65534, known[rng.integers(0, len(known), size=n)])
    dec["self"] = live[rng.integers(0, len(live), size=n)]
    dec["flags"] = np.where(rng.uniform(size=n) < 0.3, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(L.DF_REQUEST_MODEL)
    dec["fresh"] = -1
    dec["last_used"] = rng.choice(np.asarray([LONG_MIN, LONG_MAX, rp.now - FIVE_DAYS_MS, rp.now], dtype=np.int64), size=n)
    od = np.zeros(n, dtype=ob.DECISION)
    gap = rp.o_names.index(GAP_TYPE)
    od["type_idx"] = [gap if m not in name_of else rp.o_names.index(name_of[m]) for m in dec["model"]]
    od["self"], od["fresh_idx"] = dec["self"], -1
    od["favour_self"] = (dec["flags"] & L.DF_FAVOUR_SELF) != 0
    od["last_used"] = dec["last_used"]
    od["decision_id"] = np.arange(n, dtype=np.uint64)
    return SynthDecisions(dec, np.zeros(0, dtype=L.INSTANCE_ROW), np.zeros(0, dtype=np.int32)), od


def _check_request(rp, seed, what):
    sd, od = _request_batch(rp, seed)
    on, off = _place(rp, sd, seed, 1), _place(rp, sd, seed, 0)
    assert on.tobytes() == off.tobytes(), (what, int(np.sum(on != off)))
    want = rp.oracle().get_next_batch(od, rp.o_names, np.zeros(len(od) + 1, dtype=np.int64), np.zeros(0, dtype=np.int32),
                                      rp.now, seed)
    assert_same_results(on, want, what)


def test_split_key_through_a_commit_sequence(product_lib, oracle_lib):
    rp = Replay(make_fleet("C3", 4000, 1300, 3), product_lib, 3)
    _check(rp, 1, "load")
    assert rp.numeric_window(n_inst=40, n_models=120) == 2
    _check(rp, 2, "device-path window")
    # type changes (a model row's type id is always one the snapshot knows: interning a name makes the next commit
    # structural), and request-model decisions for a known type and for a type id past the table
    front = [int(x) for x in rp.front[:6]]
    for m in range(10, 26):
        rp.upsert_model(m, front[:m % 5], tname=rp.type_names[(rp.mtype[m] + 1) % len(rp.type_names)])
    assert rp.commit(NUMERIC, 16) == 2
    _check(rp, 3, "type changes")
    _check_request(rp, 3, "request-model decisions")
    # a model crossing between 4 and 5 edges, all of them at the front of the order
    for k, ids in enumerate((front[:4], front[:5], front[:4], front[1:5])):
        rp.upsert_model(30, ids)
        rp.upsert_model(31, list(reversed(ids)))
        rp.commit(NUMERIC, 2)
        _check(rp, 4 + k, ("4/5 edges", len(ids)))
    # an excluded instance leaves the fleet: its edges have rank -1 in the new epoch
    gone = front[0]
    for m in range(40, 48):
        rp.upsert_model(m, [gone] + front[1:1 + m % 4])
    rp.commit(NUMERIC, 8)
    rp.remove(gone)
    assert rp.commit(STRUCTURAL, 0, ["remove"]) == 1
    _check(rp, 10, "excluded instance removed")
    # last_used at its extremes and around the five-day line, from the model row and from the decision
    lines = [LONG_MIN, LONG_MAX, rp.now - FIVE_DAYS_MS - 1, rp.now - FIVE_DAYS_MS, rp.now - FIVE_DAYS_MS + 1, 0]
    for m in range(50, 50 + 4 * len(lines)):
        rp.upsert_model(m, front[1:1 + m % 3], last_used=lines[m % len(lines)])
    assert rp.commit(NUMERIC, 4 * len(lines)) == 2
    _check(rp, 11, "last_used", (_sweep(rp, 12, flags=0, last_used=lines), _sweep(rp, 13, flags=L.DF_MODEL_LAST_USED, last_used=lines)))
    # a rolling upgrade: a third of the pods on the next version (host path), then all of them (device path again)
    live = rp._live()
    v0 = int(rp.rows["vers"][live[0]])
    bump(rp, live[::3], v0 + 1)
    assert rp.numeric_window(n_inst=20, n_models=60) == 1
    _check(rp, 14, "upgrade, mixed versions")
    bump(rp, rp._live(), v0 + 1)
    assert rp.numeric_window(n_inst=20, n_models=60) == 2
    _check(rp, 15, "upgrade done")
    rp.f.close()


def test_split_key_on_the_old_epoch_during_a_commit(product_lib, oracle_lib):
    """A thread places the same sweep through the two-pass path while the main thread edits models and commits: every
    result equals the one-pass result of the epoch before or of the epoch after the commit, byte for byte."""
    rp = Replay(make_fleet("C3", 20_000, 1300, 7), product_lib, 7)
    sd = _sweep(rp, 7)
    f = rp.f
    for rnd in range(3):
        before = _place(rp, sd, 7, 0)
        f._ck(rp.lib.mmp_tune(f.h, b"split", 1))
        got, stop = [], threading.Event()

        def worker():
            while not stop.is_set():
                got.append(f.place_batch(sd.dec, rp.now, 7))

        th = threading.Thread(target=worker)
        th.start()
        front = [int(x) for x in rp.front[:5]]
        for m in range(rnd * 500, rnd * 500 + 400):
            rp.upsert_model(m, front[:(m % 6)], last_used=rp.now - FIVE_DAYS_MS + (m % 3) - 1)
        rp.commit(NUMERIC, 400)
        stop.set()
        th.join()
        f._ck(rp.lib.mmp_tune(f.h, b"split", 2))
        after = _place(rp, sd, 7, 0)
        assert before.tobytes() != after.tobytes()
        assert got and all(g.tobytes() in (before.tobytes(), after.tobytes()) for g in got), rnd
        assert_same_results(after, oracle_batch(rp.view(), sd, rp.oracle(), 7), ("after", rnd))
    f.close()


def test_split_key_after_churn_windows(product_lib, oracle_lib):
    """The closed loop commits each window on the device from the registry it changed (loads, evictions): after each
    window (compared with the oracle's closed loop), a sweep over every model is placed with the two-pass path on and off,
    byte for byte."""
    w = make_churn(20_000, 200, 4, fill=0.9)
    fl = w.fleet
    o, sim, s = build(product_lib, w, slots=256)
    rng = np.random.default_rng(4)
    for ep in range(3):
        ev = w.events(ep, 2000, 4)
        now0 = fl.now_ms + ep * w.window_ms
        compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, 400 + ep)
        dec = np.zeros(fl.n_models, dtype=L.DECISION_IN)
        dec["model"] = np.arange(fl.n_models)
        dec["self"] = rng.integers(0, fl.n_instances, size=fl.n_models)
        dec["flags"] = np.where(rng.uniform(size=fl.n_models) < 0.3, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(L.DF_MODEL_LAST_USED)
        dec["fresh"] = -1
        res = []
        for split in (1, 0):
            s._ck(product_lib.mmp_tune(s.h, b"split", split))
            res.append(s.place_batch(dec, now0 + w.window_ms, 40 + ep))
        s._ck(product_lib.mmp_tune(s.h, b"split", 2))
        assert res[0].tobytes() == res[1].tobytes(), (ep, int(np.sum(res[0] != res[1])))
        assert np.count_nonzero(res[0]["target"] >= 0) > 0, ep
    s.close()
