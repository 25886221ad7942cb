"""Call-wide exclude sets (mmp_place_batch_excluding) on the H100 library: the derived slot tables (k_exclude_slots +
k_slot_lists) under every placement route -- k_place_direct in batch and slot order, the chunk pipeline, k_place_lanes,
the traced tile kernel, the B = 1 launches of every one_mode -- against the oracle with each decision's exclusion list
extended by the set, and against the same ids passed as every decision's extras."""
import threading

import numpy as np
import pytest

from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import MmpError
from modelmesh_b200.synth import SynthDecisions, load_into_fleet, make_decisions, make_fleet

from exclude_set import named_sets, oracle_excluding, random_set, rs_retry_type
from helpers import oracle_from_synth, solver_from_synth
from request_model import as_request_model
from test_direct_shapes_gpu import _overflow_heavy

pytestmark = pytest.mark.gpu

FLEETS = [("C2", 3000, 4000, 2), ("C3", 3000, 10_000, 3), ("C5", 3000, 10_000, 5), ("MIX", 500, 700, 41)]


def _kw(sd):
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def _compact(sd, n):
    """the first n decisions with only the fresh rows and extras they use (a small call's own side tables)"""
    dec = sd.dec[:n].copy()
    fr = dec["fresh"] >= 0
    fresh = sd.fresh[dec["fresh"][fr]] if len(sd.fresh) else sd.fresh[:0]
    dec["fresh"][fr] = np.arange(int(fr.sum()))
    slices = [sd.extra[a:a + b] for a, b in zip(dec["extra_off"], dec["extra_n"])]
    off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(x) for x in slices], out=off[1:])
    dec["extra_off"] = off[:-1]
    extra = np.concatenate(slices).astype(np.int32) if n else np.zeros(0, dtype=np.int32)
    return SynthDecisions(dec, fresh, extra)


def _with_extras(sd, xs):
    """the same decisions with xs appended to every decision's own extras (decisions that would exceed 16 are dropped)"""
    keep = sd.dec["extra_n"] + len(xs) <= L.MAX_EXTRA
    dec = sd.dec[keep].copy()
    slices = [np.concatenate([sd.extra[a:a + b], xs]) for a, b in zip(dec["extra_off"], dec["extra_n"])]
    off = np.zeros(len(slices) + 1, dtype=np.int64)
    np.cumsum([len(x) for x in slices], out=off[1:])
    dec["extra_off"], dec["extra_n"] = off[:-1], np.diff(off)
    return SynthDecisions(sd.dec[keep], sd.fresh, sd.extra), SynthDecisions(dec, sd.fresh, np.concatenate(slices).astype(np.int32))


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_small_set_equals_the_same_ids_as_extras(product_lib, config, nm, ni, seed):
    """<= 4 ids call-wide give out, trace and both mask planes byte-identical to mmp_place_batch_trace with the ids in every
    decision's extras; an empty set is byte-identical to mmp_place_batch / _trace."""
    fl = make_fleet(config, nm, ni, seed)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 3000, seed)
    order = s.cluster_order()
    for xs in (order[:1], order[[0, 2, 5, 40]], random_set(fl.n_instances, 4, seed)):
        xs = np.asarray(xs, dtype=np.int32)
        base, ext = _with_extras(sd, xs)
        a = s.place_batch(base.dec, fl.now_ms, seed, trace=True, masks=True, exclude=xs, **_kw(base))
        b = s.place_batch(ext.dec, fl.now_ms, seed, trace=True, masks=True, **_kw(ext))
        for x, y in zip(a, b):
            assert np.array_equal(x, y), (config, xs)
        _same(s.place_batch(base.dec, fl.now_ms, seed, exclude=xs, **_kw(base)), b[0], (config, "untraced", xs))
    empty = np.zeros(0, dtype=np.int32)
    assert np.array_equal(s.place_batch(sd.dec, fl.now_ms, 9, exclude=empty, **_kw(sd)), s.place_batch(sd.dec, fl.now_ms, 9, **_kw(sd)))
    a = s.place_batch(sd.dec, fl.now_ms, 9, trace=True, masks=True, exclude=empty, **_kw(sd))
    b = s.place_batch(sd.dec, fl.now_ms, 9, trace=True, masks=True, **_kw(sd))
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    s.close()


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_sets_equal_the_oracle(product_lib, oracle_lib, config, nm, ni, seed):
    """Sets of 1 / 17 / 200 / 2 000 ids, every candidate of one type, every instance, the batch's selves with their
    unconstrained answers, request-model decisions; not-live, never-upserted and duplicate ids are ignored."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 3000, seed)
    first = s.place_batch(sd.dec, fl.now_ms, seed, **_kw(sd))
    for name, xs in named_sets(s, fl, sd, first, seed):
        want = oracle_excluding(o, fl, sd, xs, seed)
        _same(s.place_batch(sd.dec, fl.now_ms, seed, exclude=xs, **_kw(sd)), want, (config, name))
        got, tr, _ = s.place_batch(sd.dec[:800], fl.now_ms, seed, trace=True, masks=True, exclude=xs, **_kw(sd))
        _same(got, want[:800], (config, name, "traced"))
        assert np.array_equal(tr["best"], want["best"][:800]), (config, name)
    # not-live ids (no rank), repeated ids: the same answers as without them
    order = np.asarray(s.cluster_order(), dtype=np.int32)
    dead = np.setdiff1d(np.arange(fl.n_instances, dtype=np.int32), order)[:30]
    xs = order[:12]
    noisy = np.concatenate([xs, dead, xs[::2], xs]).astype(np.int32)
    assert np.array_equal(s.place_batch(sd.dec, fl.now_ms, 4, exclude=noisy, **_kw(sd)), s.place_batch(sd.dec, fl.now_ms, 4, exclude=xs, **_kw(sd)))
    # request-model decisions keep their meaning under a set
    tid = {t: s.type_id(t) for t in fl.type_names}
    rq, flagged = as_request_model(fl, sd, tid)
    rq = SynthDecisions(rq.dec[flagged], rq.fresh, rq.extra)
    xs = random_set(fl.n_instances, 200, seed + 1)
    want = oracle_excluding(o, fl, rq, xs, seed, names=fl.type_names, type_idx=fl.model_type[sd.dec["model"][flagged]])
    _same(s.place_batch(rq.dec, fl.now_ms, seed, exclude=xs, **_kw(rq)), want, (config, "request-model"))
    s.close()


def test_never_upserted_ids_and_the_replicaset_retry(product_lib, oracle_lib):
    fl = make_fleet("C3", 3000, 4000, 33)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    big = s.max_instances
    # a second fleet with room for more instances than it holds: ids past the last upserted one are ignored
    from modelmesh_b200.fleet import Fleet
    roomy = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, big + 500, fl.n_models, lib=product_lib)
    load_into_fleet(fl, roomy)
    sd = make_decisions(fl, 3000, 34)
    xs = random_set(fl.n_instances, 200, 5)
    want = oracle_excluding(o, fl, sd, xs, 6)
    ghosts = np.arange(big, big + 500, 7, dtype=np.int32)
    _same(roomy.place_batch(sd.dec, fl.now_ms, 6, exclude=np.concatenate([xs, ghosts]), **_kw(sd)), want, "never upserted")
    roomy.close()
    # every unflagged candidate of a type excluded: the filter is retried without the replicaset rule
    t, free, flagged = rs_retry_type(s, fl)
    big_sd = make_decisions(fl, 20_000, 35)
    keep = fl.model_type[big_sd.dec["model"]] == fl.type_names.index(t)
    sub = SynthDecisions(big_sd.dec[keep], big_sd.fresh, big_sd.extra)
    want = oracle_excluding(o, fl, sub, free, 7)
    got, tr, _ = s.place_batch(sub.dec, fl.now_ms, 7, trace=True, exclude=free, **_kw(sub))
    _same(got, want, "rs retry traced")
    _same(s.place_batch(sub.dec, fl.now_ms, 7, exclude=free, **_kw(sub)), want, "rs retry")
    tgt = want["target"]
    assert (tgt >= 0).any() and np.isin(tgt[tgt >= 0], flagged).all()
    assert ((tr["flags"] & L.TF_RS_RETRY) != 0).mean() > 0.5
    s.close()


def test_malformed_sets_and_sharded_fleets(product_lib):
    fl = make_fleet("C3", 500, 1000, 3)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 50, 3)
    for xs in (np.asarray([3, fl.n_instances], dtype=np.int32), np.asarray([-1], dtype=np.int32)):
        out = np.full(len(sd.dec), -7, dtype=np.int64).view(L.DECISION_OUT)
        with pytest.raises(MmpError) as e:
            s.place_batch(sd.dec, fl.now_ms, 1, exclude=xs, out=out, **_kw(sd))
        assert e.value.code == L.E_ARG
        assert (out["target"] == -7).all() and (out["n_candidates"] == -1).all()  # untouched
    dec = np.ascontiguousarray(sd.dec, dtype=L.DECISION_IN)
    out = np.zeros(len(dec), dtype=L.DECISION_OUT)
    assert s.lib.mmp_place_batch_excluding(s.h, dec.ctypes.data, len(dec), None, 0, None, 0, None, 3, out.ctypes.data, None, None,
                                           fl.now_ms, 1) == L.E_ARG
    # a fleet that connected a communicator refuses a set; its unconnected twin answers
    twin = solver_from_synth(fl, product_lib)
    s.shard_connect(s.shard_unique_id())
    plain = SynthDecisions(sd.dec, sd.fresh, sd.extra)
    with pytest.raises(MmpError) as e:
        s.place_batch(plain.dec, fl.now_ms, 1, exclude=np.asarray([1, 2], dtype=np.int32), **_kw(plain))
    assert e.value.code == L.E_STATE
    twin.place_batch(plain.dec, fl.now_ms, 1, exclude=np.asarray([1, 2], dtype=np.int32), **_kw(plain))
    s.close()
    twin.close()


def test_routes(product_lib, oracle_lib):
    """B = 1 .. 32 in one_mode 0 .. 3, 8 193 and 12 000 decisions with and without the slot sort, more than 131 072
    decisions (the chunk pipeline), k_place_lanes (direct 0), lane budget 2: one answer, the oracle's."""
    fl = make_fleet("C5", 3000, 10_000, 5)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    xs = random_set(fl.n_instances, 500, 11)
    sd = make_decisions(fl, 12_000, 5)
    want = oracle_excluding(o, fl, sd, xs, 3)
    lib = product_lib
    for mode in (0, 1, 2, 3):
        s._ck(lib.mmp_tune(s.h, b"one_mode", mode))
        for n in (1, 2, 5, 17, 31, 32):
            part = _compact(sd, n)
            _same(s.place_batch(part.dec, fl.now_ms, 3, exclude=xs, **_kw(part)), want[:n], ("one_mode", mode, n))
    s._ck(lib.mmp_tune(s.h, b"one_mode", 3))
    for sort in (0, 1):
        s._ck(lib.mmp_tune(s.h, b"sort_slots", sort))
        for n in (8193, 12_000):
            part = SynthDecisions(sd.dec[:n], sd.fresh, sd.extra)
            _same(s.place_batch(part.dec, fl.now_ms, 3, exclude=xs, **_kw(part)), want[:n], ("sort", sort, n))
    s._ck(lib.mmp_tune(s.h, b"sort_slots", 2))
    s._ck(lib.mmp_tune(s.h, b"direct", 0))
    _same(s.place_batch(sd.dec, fl.now_ms, 3, exclude=xs, **_kw(sd)), want, "lanes")
    s._ck(lib.mmp_tune(s.h, b"direct", 1))
    s._ck(lib.mmp_tune(s.h, b"lane_budget", 2))
    _same(s.place_batch(sd.dec, fl.now_ms, 3, exclude=xs, **_kw(sd)), want, "lane budget 2")
    s._ck(lib.mmp_tune(s.h, b"lane_budget", 48))
    # the chunk pipeline: 140 000 decisions, a sample of them against the oracle at their places in the batch
    huge = make_decisions(fl, 140_000, 6)
    got = s.place_batch(huge.dec, fl.now_ms, 8, exclude=xs, **_kw(huge))
    pos = np.concatenate([np.arange(0, 1500), np.arange(131_000, 132_500), np.arange(138_500, 140_000)])
    sample = SynthDecisions(huge.dec[pos], huge.fresh, huge.extra)
    _same(got[pos], oracle_excluding(o, fl, sample, xs, 8, positions=pos), "chunks")
    s.close()


def test_overflow_heavy_fleet(product_lib, oracle_lib):
    fl, order, edges = _overflow_heavy(10_000, 6000, 41)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 6000, 41)
    for xs in (np.asarray(order[[0, 31, 32, 383, 384, 385]], dtype=np.int32), random_set(fl.n_instances, 2000, 42)):
        want = oracle_excluding(o, fl, sd, xs, 3)
        for sort in (0, 1):
            s._ck(product_lib.mmp_tune(s.h, b"sort_slots", sort))
            _same(s.place_batch(sd.dec, fl.now_ms, 3, exclude=xs, **_kw(sd)), want, ("overflow-heavy", sort, len(xs)))
    s._ck(product_lib.mmp_tune(s.h, b"sort_slots", 2))
    s.close()


def test_isolation_threads_and_commits(product_lib, oracle_lib):
    """A call with a set leaves the snapshot's tables alone; 8 threads with 8 sets each get their own answers; a numeric
    and a structural commit between calls: each epoch's answers are the oracle's on that epoch."""
    fl = make_fleet("C3", 3000, 10_000, 3)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 4000, 3)
    before = s.place_batch(sd.dec, fl.now_ms, 5, **_kw(sd))
    one = _compact(sd, 1)
    before1 = s.place_batch(one.dec, fl.now_ms, 5, **_kw(one))
    s.place_batch(sd.dec, fl.now_ms, 5, exclude=np.arange(fl.n_instances, dtype=np.int32), **_kw(sd))
    s.place_batch(one.dec, fl.now_ms, 5, exclude=np.arange(fl.n_instances, dtype=np.int32), **_kw(one))
    assert np.array_equal(s.place_batch(sd.dec, fl.now_ms, 5, **_kw(sd)), before)
    assert np.array_equal(s.place_batch(one.dec, fl.now_ms, 5, **_kw(one)), before1)
    sets = [random_set(fl.n_instances, 50 + 300 * t, 100 + t) for t in range(8)]
    wants = [oracle_excluding(o, fl, sd, x, 5) for x in sets]
    errors = []

    def worker(t):
        try:
            for _ in range(3):
                _same(s.place_batch(sd.dec, fl.now_ms, 5, exclude=sets[t], **_kw(sd)), wants[t], ("thread", t))
                part = _compact(sd, 4)
                _same(s.place_batch(part.dec, fl.now_ms, 5, exclude=sets[t], **_kw(part)), wants[t][:4], ("thread B=4", t))
        except Exception as e:  # reported below
            errors.append(e)

    ths = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    assert not errors, errors[0]
    # a numeric commit (the device path), then a structural one (the first instance of PLACEMENT_ORDER shutting down)
    xs = sets[3]
    rows = fl.inst_rows.copy()
    for i in np.random.default_rng(3).choice(fl.n_instances, 400, replace=False):
        rows[i]["count"] += 3
        rows[i]["used"] = max(0, int(rows[i]["used"]) - 1000)
        s.instance_update(int(i), rows[i])
    s.commit()
    assert s.commit_info()[0] == 2
    fl.inst_rows = rows
    _same(s.place_batch(sd.dec, fl.now_ms, 5, exclude=xs, **_kw(sd)), oracle_excluding(oracle_from_synth(fl), fl, sd, xs, 5), "numeric commit")
    gone = int(np.asarray(s.cluster_order())[0])
    rows[gone]["shutting_down"] = 1
    s.instance_update(gone, rows[gone])
    s.commit()
    assert s.commit_info()[0] == 1
    fl.inst_rows = rows
    _same(s.place_batch(sd.dec, fl.now_ms, 5, exclude=xs, **_kw(sd)), oracle_excluding(oracle_from_synth(fl), fl, sd, xs, 5), "structural commit")
    s.close()
