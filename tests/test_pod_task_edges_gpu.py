"""mmp_janitor_run, mmp_rate_run, mmp_shutdown_run and mmp_evict_run on the device at their edges (tests/pod_task_edges.py),
against the restatements exactly -- out, loads, edits and report:
  * every hand-built case of tests/test_{janitor,rate,shutdown,evict}_run_oracle.py, whose known answers those files check
    on the restatement; every PLACED entry also against mmp_place_batch on the same record (MMP_DF_OWN_ID, extra {pod}),
    and a rate run's round-0 loads against mmp_place_batch / mmp_place_batch_excluding;
  * both sides of every edge pair: the rebalance gate where its long arithmetic wraps and per type set on a
    type-constrained fleet (a set at 20 * free / cap == 1, one at 0, a type without constraints), 2 x load_timeout_ms wrapping,
    registration times at Long.MIN_VALUE / MAX_VALUE, an odd failure expiry, the pod loaded and failed on one model,
    extreme lastUsed values, the shutdown cutoff wrapping, lru_t = Long.MIN_VALUE, found_other with one ranked instance,
    the heavy-set bound, an unranked pod's rpm, chains of 16 / 17 / 18, a chain going on from a SELF answer with and
    without a fresh row, the janitor's budget, an odd adjusted capacity,
    quirk N15 keeping a model that does not remove, a Long.MAX_VALUE candidate key, and the saturation line itself;
  * a model whose copy count is saturated (280 loaded + 20 failed loads) with the pod at loaded positions 10 and 270 and as
    the failed load at 290: undecided in every task;
  * one fleet of 3 200 models at n = 255, 256, 257, 511, 512, 513, 1 025 and 3 000 entries (several blocks of k_*_plan and
    k_*_index, several 512-entry tiles of k_rate_plan with chains in each), two entries of one model in different blocks
    and tiles refused with nothing written, and the four calls interleaved with refused ones, each answering as alone."""
import numpy as np
import pytest

import pod_task_edges as pe
import rate_run_oracle as rro
from common import EXPIRY, HOUR
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import MmpError
from modelmesh_b200.synth import make_fleet
from pod_tasks import (IT, busiest_pod, composed_evict, composed_shutdown, cross_check_rate, evict_params, ids, janitor_params, rate_params,
                       report_dict, same_out, shutdown_params, timed_solver)

pytestmark = pytest.mark.gpu
SIZES = (255, 256, 257, 511, 512, 513, 1025, 3000)


def _device(s, c):
    """c on the device, in the restatement's shape"""
    if c.task == "janitor":
        edits, r = s.janitor_run(c.pod, c.entries, c.params)
        return [(int(e["model"]), int(e["what"]), int(e["last_used"]), int(e["last_unload_time"])) for e in edits], report_dict(r)
    if c.task == "rate":
        out, loads, r = s.rate_run(c.pod, c.entries, c.params, c.seed, fresh_self=c.fresh)
        return out, [tuple(int(x) for x in ld) for ld in loads], {k: getattr(r, k) for k in c.want[2]}
    if c.task == "shutdown":
        out, r = s.shutdown_run(c.pod, c.entries, c.params, c.seed, fresh_self=c.fresh)
        return out, report_dict(r)
    out, r = s.evict_run(c.pod, c.entries, c.params, c.seed, fresh_self=c.fresh)
    return out, report_dict(r)


def _same(c, got):
    w = c.want
    if c.task == "janitor":
        return got[0] == w[0] and got[1] == w[1]
    if c.task == "rate":
        return same_out(got[0], w[0]) and got[1] == w[1] and got[2] == w[2]
    return got[0].tobytes() == w[0].tobytes() and got[1] == w[1]


def _check(s, c, o=None):
    """the device equals the restatement, and every placed decision equals the placement call's on the same record"""
    got = _device(s, c)
    assert _same(c, got), (c.name, got, c.want)
    if c.task == "shutdown":
        assert composed_shutdown(s, c.pod, c.entries, got[0], c.params, c.seed, c.fresh) == got[1]["n_placed"]
    elif c.task == "evict":
        assert composed_evict(s, c.pod, c.entries, got[0], c.params, c.seed, c.fresh) == got[1]["n_placed"]
    elif c.task == "rate" and got[2]["gate"] == L.RATE_RAN:
        own = o is None
        o = oracle_from_synth(c.fl) if own else o
        heavy = rro.heavy_set(o, c.fl, c.pod, int(c.params["scale"]["scale_up_rpm_threshold"][0]))
        if own:
            o.close()
        cross_check_rate(s, c.fl, c.ts, c.pod, c.entries, c.params, c.seed, got[0], got[1], heavy, c.fresh)
    return got


def _run_all(lib, cases):
    fleets = {}
    try:
        for c in cases:
            k = c.fleet_key()
            if k not in fleets:
                fleets[k] = timed_solver(lib, c.fl, c.ts, c.lul)
            _check(fleets[k], c)
    finally:
        for s in fleets.values():
            s.close()


def test_hand_built_cases_on_the_device(product_lib, oracle_lib):
    cases = pe.hand_cases(oracle_lib)
    assert {c.name for c in cases} == {f"{m}::{t}" for m, ts in pe.HAND_BUILT.items() for t in ts}
    _run_all(product_lib, cases)


def test_edge_pairs_on_the_device(product_lib, oracle_lib):
    pairs = pe.all_pairs()
    for name, a, b, sig in pairs:
        assert sig(a.want) != sig(b.want), name
    _run_all(product_lib, [c for _, a, b, _ in pairs for c in (a, b)])


def test_saturated_records_on_the_device(product_lib, oracle_lib):
    cases = pe.saturated_cases()
    assert [int(w) for w in cases[0].want[0]["what"][:3]] == [L.SD_UNDECIDED] * 3
    assert [int(w) for w in cases[1].want[0]["what"][:3]] == [L.EV_UNDECIDED] * 3
    _run_all(product_lib, cases)


# ------------------------------------------------------------------------------------------------------------- shapes

def _shape_fleet():
    """C3, 3 200 models x 400 instances, a time for every registration (30 % recent), the pod the instance with the most
    registrations"""
    fl = make_fleet("C3", 3200, 400, 11)
    rng = np.random.default_rng(11)
    n, now = len(fl.edge_inst), fl.now_ms
    ts = np.where(rng.uniform(size=n) < 0.3, now - rng.integers(0, EXPIRY, size=n),
                  now - rng.integers(EXPIRY, 4 * HOUR, size=n)).astype(np.int64)
    lul = np.where(rng.uniform(size=fl.n_models) < 0.3, now - rng.integers(0, 200_000, size=fl.n_models), 0).astype(np.int64)
    S = busiest_pod(fl)
    return fl, ts, lul, S


def _shape_entries(fl, ts, S, n_max):
    """one entry array per task over the same n_max models in a random order (most of them not the pod's)"""
    rng = np.random.default_rng(5)
    now = fl.now_ms
    models = rng.permutation(fl.n_models)[:n_max]
    first_ts = []
    for m in models:
        a, b = int(fl.edge_off[m]), int(fl.edge_off[m + 1])
        hit = [q for q in range(a, b) if fl.edge_inst[q] == S]
        first_ts.append(int(ts[hit[0]]) if hit else int(rng.integers(1, now)))
    first_ts = np.array(first_ts, dtype=np.int64)
    n = len(models)
    u = rng.uniform(size=n)
    ev = np.zeros(n, dtype=L.EVICT_ENTRY)
    ev["model"], ev["load_ts"], ev["load_complete_ts"] = models, first_ts, first_ts
    ev["last_used"] = np.where(u < 0.1, 0, now - rng.integers(1, HOUR, size=n))
    sd = np.zeros(n, dtype=L.SHUTDOWN_ENTRY)
    sd["model"] = models
    sd["lru_t"] = np.where(u < 0.6, now - rng.integers(0, HOUR, size=n), now - rng.integers(HOUR, 6 * HOUR, size=n))
    sd["last_used"] = now - rng.integers(1, 3 * HOUR, size=n)
    ra = np.zeros(n, dtype=L.SCALE_IN)
    ra["instance"], ra["model"] = S, models
    ra["count"] = np.where(u < 0.25, rng.integers(2000, 20_000, size=n), rng.integers(0, 200, size=n))
    ra["last_used"] = now - rng.integers(0, HOUR, size=n)
    ra["i1"] = IT - rng.integers(0, 400, size=n)
    ra["i2"] = np.minimum(IT, ra["i1"] + rng.integers(0, 300, size=n))
    ja = np.zeros(n, dtype=L.JANITOR_ENTRY)
    ja["model"], ja["weight"], ja["load_ts"] = models, rng.integers(1, 400, size=n), first_ts
    ja["last_used"] = now - rng.integers(1, 40 * HOUR, size=n)
    ja["flags"] = np.where(rng.uniform(size=n) < 0.1, L.JANITOR_FAILED, 0)
    return dict(evict=ev, shutdown=sd, rate=ra, janitor=ja)


def _shape_case(fl, ts, lul, S, task, entries):
    now = fl.now_ms
    params = dict(evict=evict_params(now), shutdown=shutdown_params(now), rate=rate_params(now, 1000),
                  janitor=janitor_params(now, 1 << 40))[task]
    return pe.solved(pe.Case(task, fl, ts, lul, S, np.ascontiguousarray(entries), params, 23, None, f"shape/{task}/{len(entries)}"))


def test_shapes_duplicates_and_interleaving(product_lib, oracle_lib):
    fl, ts, lul, S = _shape_fleet()
    ents = _shape_entries(fl, ts, S, max(SIZES))
    o = oracle_from_synth(fl)
    s = timed_solver(product_lib, fl, ts, lul)
    alone = {}
    for n in SIZES:
        for task in pe.TASKS:
            c = _shape_case(fl, ts, lul, S, task, ents[task][:n])
            alone[(task, n)] = (c, _check(s, c, o))
    # the rate runs draw past one tile: chains in at least two 512-entry tiles, decision ids of 512 and more
    c, (out, loads, _) = alone[("rate", max(SIZES))]
    first = ids(fl, ts, c.entries, out, c.params)
    chain_rows = np.nonzero((first >= 0) & (out["action"] == 2))[0]
    assert len(set(chain_rows // 512)) >= 2 and first.max() >= 512 and any(ld[2] > 0 for ld in loads)
    # the shutdown and evict plans decide and place entries in their first block and in later ones (256 threads each)
    for task, bit in (("shutdown", L.SD_PLACED), ("evict", L.EV_PLACED)):
        placed = np.nonzero(alone[(task, max(SIZES))][1][0]["what"] & bit)[0]
        assert placed.min() < 256 and len(set(placed // 256)) >= 3, (task, placed)

    def refused(task, n, pair):
        e = ents[task][:n].copy()
        e["model"][pair[1]] = e["model"][pair[0]]
        p = alone[(task, n)][0].params
        if task in ("shutdown", "evict"):
            out = np.zeros(n, dtype=L.SHUTDOWN_ACTION if task == "shutdown" else L.EVICT_ACTION)
            before = out.tobytes()
            with pytest.raises(MmpError) as err:
                getattr(s, task + "_run")(S, e, p, 23, out=out)
            assert out.tobytes() == before
        elif task == "rate":
            with pytest.raises(MmpError) as err:
                s.rate_run(S, e, p, 23)
        else:
            with pytest.raises(MmpError) as err:
                s.janitor_run(S, e, p)
        assert err.value.code == L.E_ARG, (task, n, pair)

    # two entries of one model in different blocks (3, 300) and tiles (3, 600)
    for task in pe.TASKS:
        for pair in ((3, 300), (3, 600)):
            refused(task, 1025, pair)
    # the four calls interleaved with refused ones: each answers as it did alone (the shared slot array is left clean)
    rng = np.random.default_rng(3)
    for step in range(24):
        task, n = pe.TASKS[step % 4], SIZES[int(rng.integers(0, len(SIZES)))]
        if step % 3 == 1:
            refused(pe.TASKS[(step + 1) % 4], 1025, (3, 300 if step % 2 else 600))
        c, first = alone[(task, n)]
        assert _same(c, _device(s, c)), (step, task, n)
    s.close()
    o.close()
