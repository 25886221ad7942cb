"""ClusterStats (k_stats), the type-set stats built from its per-partition sums (k_type_stats, k_churn_type_ok) and the
reaper's selection against the oracle, where the ordinary synthetic fleets never go:
  A. more than STATS_SMEM_PARTS (511) prohibited-type-set partitions (TCM:557-579), so k_stats adds every instance straight
     into global memory: mmp_stats, its cap contract, mmp_reaper_select over every partition, mmp_scale_eval and the closed
     loop's reload-elsewhere rule (a12);
  B. instance values the synthetic rows never take: Long.MAX_VALUE / 0 lru times (ISST:57-61), free space at the isFull edge
     (MM:4640-4642), copy counts and capacities that wrap, no live instance, and a fleet large enough that every thread of
     k_stats' grid-stride loop takes more than one instance;
  C. the reaper's bounded most-recently-used selection (MM:6675-6719, N12) at runs of equal lastUsed, lastUsed exactly at the
     cutoff and at globalLru, total_count around the number of unique candidates, a cap below the selection, registry sizes at
     the edges of the select / radix-sort calls, and a size estimate of 0 (MM:6651)."""
import copy
import ctypes as C

import numpy as np
import pytest

from churn_harness import build, compare_window
from common import LONG_MAX, vp
from helpers import oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import MmpError
from modelmesh_b200.synth import SplitMix, make_churn, make_fleet
from oracle import binding as ob
from scan_checks import converged_oracle, partition_maps

pytestmark = pytest.mark.gpu

FIELDS = ("total_capacity", "total_free", "global_lru", "instance_count", "model_copy_count")
SMEM_PARTS = 511  # STATS_SMEM_PARTS (scan_kernels.cuh): past it k_stats accumulates in global memory


def _partition_heavy(fl, seed):
    """Ten more labels req-0..9, each instance holding a uniformly random subset of them, and the types
    ty<k> (requires req-k), tz<k> (requires req-k and req-(k+3)%10, prefers req-(k+1)%10) and one unconstrained type.
    An instance's prohibited-type set is then its subset of req-*: up to 1024 partitions."""
    rng = SplitMix(seed ^ 0x5EED)
    req = [f"req-{k}" for k in range(10)]
    bits = rng.randint(fl.n_instances, 0, 1024)
    fl.inst_labels = [sorted(set(fl.inst_labels[i]) | {req[k] for k in range(10) if (int(bits[i]) >> k) & 1})
                      for i in range(fl.n_instances)]
    cfg = {}
    for k in range(10):
        cfg[f"ty{k}"] = {"required": [req[k]]}
    for k in range(10):
        cfg[f"tz{k}"] = {"required": sorted({req[k], req[(k + 3) % 10]}), "preferred": [req[(k + 1) % 10]]}
    fl.type_config = cfg
    fl.type_names = list(cfg) + ["free"]
    fl.model_type = rng.randint(fl.n_models, 0, len(fl.type_names)).astype(np.int32)
    return fl


def _check_stats(fl, o, s):
    """mmp_stats against orc_cluster_stats / orc_partition_stats: every field of every partition (ids mapped through instance
    membership), the number of entries, and the PARTITION_STATS_COMP order (TCM:264-271).  Partitions that tie exactly keep
    the reference's HashMap order (TCM:264-292), so the oracle is matched by id, not by position.  Returns the product's
    (stats, ids) and the oracle's partition count."""
    st, ids = s.stats(cap=fl.n_instances + 2)
    g = o.cluster_stats()
    assert [int(st[0][k]) for k in FIELDS] == [int(g[k]) for k in FIELDS], (st[0], g)
    if fl.type_config is None:
        assert len(st) == 1
        return st, ids, 0
    ost, oids = o.partition_stats(cap=fl.n_instances + 2)
    live = ost["instance_count"] > 0
    by_o = {int(i): x for i, x in zip(oids[live], ost[live])}
    assert len(st) - 1 == len(by_o), (len(st) - 1, len(by_o))
    pmap = partition_maps(fl, o, s)
    assert len(set(int(p) for p in ids[1:])) == len(ids) - 1
    for x, pid in zip(st[1:], ids[1:]):
        y = by_o[pmap[int(pid)]]
        assert [int(x[k]) for k in FIELDS] == [int(y[k]) for k in FIELDS], (int(pid), x, y)
    key = lambda x: (-int(x["total_free"]), int(x["global_lru"]), -int(x["total_capacity"]))
    keys = [key(x) for x in st[1:]]
    assert keys == sorted(keys)
    assert keys == [key(y) for y in ost[live]]  # the same sequence of sort keys: only exact ties may be ordered differently
    return st, ids, len(by_o)


def _om(fl):
    om = np.zeros(fl.n_models, dtype=ob.MODEL)
    om["last_used"], om["type_idx"], om["n_loaded"], om["n_failed"] = fl.model_last_used, fl.model_type, fl.n_loaded, fl.n_failed
    return om


def _reaper_cluster(fl, o, s):
    """one cluster-wide pass (no type exclusion) from an empty `taken`; returns the selection"""
    om = _om(fl)
    taken_o, taken_s = np.zeros(fl.n_models, np.uint8), np.zeros(fl.n_models, np.uint8)
    a = o.reaper_select(om, fl.type_names, -1, fl.now_ms, taken=taken_o)
    b = s.reaper_select(-1, fl.now_ms, taken=taken_s)
    assert np.array_equal(a, b), (a[:8], b[:8], len(a), len(b))
    assert np.array_equal(taken_o, taken_s)
    return a


def _reaper_partitions(fl, o, s, ids):
    """every partition in the product's stats order, `taken` carried from one to the next (MM:6473-6489);
    returns the selection of each call"""
    om = _om(fl)
    pmap = partition_maps(fl, o, s)
    taken_o, taken_s = np.zeros(fl.n_models, np.uint8), np.zeros(fl.n_models, np.uint8)
    sel = []
    for pid in ids[1:]:
        a = o.reaper_select(om, fl.type_names, pmap[int(pid)], fl.now_ms, taken=taken_o)
        b = s.reaper_select(int(pid), fl.now_ms, taken=taken_s)
        assert np.array_equal(a, b), (int(pid), a[:8], b[:8], len(a), len(b))
        assert np.array_equal(taken_o, taken_s), int(pid)
        sel.append(a)
    return sel


# ---------------------------------------------------------------------------------------------------------------
# A. more than 511 partitions
# ---------------------------------------------------------------------------------------------------------------
def _keep_four_with_times(fl, rng):
    """at most 4 registrations per model, each with a load / failure time, and a lastUnloadTime per model (the record recipe
    of test_registry_scans_gpu.py)"""
    nm = fl.n_models
    keep = np.minimum(fl.edge_off[1:] - fl.edge_off[:-1], 4)
    off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(keep, out=off[1:])
    inst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m] + keep[m]] for m in range(nm)])
    fl.n_loaded = np.minimum(fl.n_loaded, keep).astype(np.int32)
    fl.n_failed = (keep - fl.n_loaded).astype(np.int32)
    fl.edge_off, fl.edge_inst = off, inst.astype(np.int32)
    ts = (fl.now_ms - rng.integers(0, 4 * 3_600_000, size=len(inst))).astype(np.int64)
    ts = np.where(rng.uniform(size=len(inst)) < 0.3, fl.now_ms - rng.integers(0, 120_000, size=len(inst)), ts).astype(np.int64)
    lul = np.where(rng.uniform(size=nm) < 0.3, fl.now_ms - rng.integers(0, 200_000, size=nm), 0).astype(np.int64)
    return ts, lul


@pytest.fixture(scope="module")
def heavy(product_lib, oracle_lib):
    """C3 rows at 3 000 instances under the req-* scheme (~980 partitions, 1.2e10 units of capacity)"""
    rng = np.random.default_rng(1)
    fl = _partition_heavy(make_fleet("C3", 4000, 3000, 1), 1)
    ts, lul = _keep_four_with_times(fl, rng)
    s = solver_from_synth(fl, product_lib)
    for m in range(fl.n_models):
        e = np.ascontiguousarray(ts[fl.edge_off[m]:fl.edge_off[m + 1]])
        s._ck(product_lib.mmp_model_times(s.h, m, vp(e), len(e), int(lul[m])))
    s.commit()
    o = oracle_from_synth(fl, bulk=True)  # bulk_add is the converged state (N10)
    return fl, o, s, ts, lul


def test_partition_heavy_stats_match_oracle(heavy):
    fl, o, s, _, _ = heavy
    st, ids, n_o = _check_stats(fl, o, s)
    print(f"partitions: product {len(st) - 1}, oracle {n_o}")
    assert len(st) - 1 > SMEM_PARTS and n_o > SMEM_PARTS
    # the cluster's capacity - free does not fit an int: the reaper's (int) average-size cast truncates (MM:6624-6627)
    assert int(st[0]["total_capacity"]) - int(st[0]["total_free"]) > (1 << 31)


def test_partition_heavy_stats_cap_contract(heavy):
    """mmp_stats returns the full count whatever cap is, and writes exactly the first cap entries of the full call"""
    fl, o, s, _, _ = heavy
    full, fids = s.stats(cap=fl.n_instances + 2)
    assert len(full) > SMEM_PARTS + 1
    for cap in (1, 100):
        out = np.zeros(cap + 4, dtype=L.CLUSTER_STATS)
        out["total_capacity"] = -7
        ids = np.full(cap + 4, -7, dtype=np.int32)
        n = s._ck(s.lib.mmp_stats(s.h, vp(out), vp(ids), cap))
        assert n == len(full)
        assert np.array_equal(out[:cap], full[:cap]) and np.array_equal(ids[:cap], fids[:cap])
        assert (out["total_capacity"][cap:] == -7).all() and (ids[cap:] == -7).all()


def test_partition_heavy_reaper_matches_oracle(heavy):
    fl, o, s, _, _ = heavy
    st, ids = s.stats(cap=fl.n_instances + 2)
    assert len(ids) - 1 > SMEM_PARTS
    # both branches of triggerProactiveLoadsForInstanceSubset: partitions with room above the 1/8 reserve on some instance
    # that may load (free-space count > 0), and partitions without (only models used after the cutoff qualify)
    rows = fl.inst_rows
    room = ((rows["capacity"] - rows["used"]) - rows["capacity"] // 8 > 0) & (rows["l_threads"] * 50 - rows["l_in_prog"] > 0)
    part_room = {}
    for i in range(fl.n_instances):
        p = s.instance_partition(i)
        if p >= 0:
            part_room[p] = part_room.get(p, False) or bool(room[i])
    assert any(part_room.values()) and not all(part_room.values())
    sel = _reaper_partitions(fl, o, s, ids)
    n_sel = sum(len(a) for a in sel)
    print(f"reaper: {sum(1 for a in sel if len(a))} of {len(sel)} partitions selected {n_sel} models")
    assert n_sel > 0
    # the cluster-wide pass: the size estimate from the truncated (int) average
    _reaper_cluster(fl, o, s)


def test_partition_heavy_scale_eval_matches_oracle(heavy, product_lib, oracle_lib):
    """rateTrackingTask / removeModelCopies (test_registry_scans_gpu.py's recipe): every type's set spans hundreds of
    partitions in k_type_stats"""
    fl, o, s, ts, lul = heavy
    lib = product_lib
    nm, ni = fl.n_models, fl.n_instances
    rng = np.random.default_rng(3)
    n = 6000
    rec = np.zeros(n, dtype=L.SCALE_IN)
    models = rng.integers(0, nm, size=n)
    rec["model"] = models
    for r in range(n):
        m = int(models[r])
        k = int(fl.n_loaded[m])
        rec["instance"][r] = int(fl.edge_inst[fl.edge_off[m] + rng.integers(0, k)]) if k and rng.uniform() < 0.9 else int(rng.integers(0, ni))
    rec["count"] = np.where(rng.uniform(size=n) < 0.5, rng.integers(0, 50, size=n), rng.integers(0, 20_000, size=n))
    rec["last_used"] = np.where(rng.uniform(size=n) < 0.05, 0, fl.now_ms - rng.integers(0, 40 * 3_600_000, size=n))
    rec["last_heavy"] = np.where(rng.uniform(size=n) < 0.4, 0, fl.now_ms - rng.integers(0, 30 * 3_600_000, size=n))
    rec["flags"] = (rng.uniform(size=n) < 0.15).astype(np.int32)
    it = 5000
    rec["i1"] = it - rng.integers(0, 400, size=n)
    rec["i2"] = np.minimum(it, rec["i1"] + rng.integers(0, 300, size=n))
    m64 = models.astype(np.int64)
    deg = (fl.edge_off[m64 + 1] - fl.edge_off[m64]).astype(np.int64)
    eoff = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=eoff[1:])
    einst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64]).astype(np.int32)
    ets = np.concatenate([ts[fl.edge_off[m]:fl.edge_off[m + 1]] for m in m64]).astype(np.int64)
    nl = fl.n_loaded[m64].astype(np.int32)
    tidx = fl.model_type[m64].astype(np.int32)
    lulr = lul[m64].astype(np.int64)
    orec = np.zeros(n, dtype=ob.SCALE_IN)
    for k in ("instance", "model", "count", "last_used", "last_heavy", "i1", "i2", "flags"):
        orec[k] = rec[k]
    names = (C.c_char_p * len(fl.type_names))(*[t.encode() for t in fl.type_names])
    acted = 0
    for thr, can_remove, lru_thr in ((2000, 1, 6 * 3_600_000), (300, 1, 1000), (5, 0, 6 * 3_600_000)):
        p = np.zeros(1, dtype=L.SCALE_PARAMS)
        p["now"], p["last_check_time"], p["iteration"], p["scale_up_rpm_threshold"] = fl.now_ms, fl.now_ms - 10_000, it, thr
        p["second_copy_min_age_iters"], p["second_copy_max_age_iters"], p["second_copy_lru_threshold_ms"] = 42, 240, lru_thr
        p["rate_check_interval_ms"], p["assume_completed_ms"], p["second_copy_remove_max_age_ms"], p["can_remove"] = 10_000, 30_000, 36_000_000, can_remove
        out = np.zeros(n, dtype=L.SCALE_OUT)
        s._ck(lib.mmp_scale_eval(s.h, vp(rec), n, vp(p), vp(out)))
        op = np.zeros(1, dtype=ob.SCALE_PARAMS)
        for k in op.dtype.names:
            if k != "pad":
                op[k] = p[k]
        up = np.zeros(n, dtype=ob.SCALE_OUT)
        down = np.zeros(n, dtype=ob.SCALE_OUT)
        assert oracle_lib.orc_rate_task_eval(o.h, n, vp(orec), vp(op), names, len(fl.type_names), vp(tidx), vp(eoff), vp(einst),
                                             vp(ets), vp(nl), vp(up)) == 0
        assert oracle_lib.orc_janitor_eval(o.h, n, vp(orec), vp(op), vp(eoff), vp(einst), vp(ets), vp(nl), vp(lulr), vp(down)) == 0
        for k in ("action", "copies_to_load", "load_last_used", "rpm", "i1", "i2", "set_heavy"):
            bad = np.nonzero(out[k] != up[k])[0]
            assert len(bad) == 0, (thr, k, len(bad), bad[:5], out[bad[:5]], up[bad[:5]], rec[bad[:5]])
        bad = np.nonzero(out["remove"] != down["remove"])[0]
        assert len(bad) == 0, (thr, "remove", len(bad), bad[:5], rec[bad[:5]])
        acted += int(np.count_nonzero(out["action"] > 0))
    assert acted > 0


def test_partition_heavy_closed_loop_matches_oracle(product_lib, oracle_lib):
    """the closed loop with ~780 partitions: the reload-elsewhere rule's "type set < 95 % full" test (MM:2918-2920) sums
    hundreds of k_stats partitions per type in k_churn_type_ok"""
    seed = 8
    w = make_churn(30_000, 1_500, seed, fill=0.90)
    _partition_heavy(w.fleet, seed)
    fl = w.fleet
    o, sim, s = build(product_lib, w, slots=256)
    n_p = len(s.stats(cap=fl.n_instances + 2)[0]) - 1
    ost, _ = o.partition_stats(cap=fl.n_instances + 2)
    n_o = int(np.count_nonzero(ost["instance_count"] > 0))
    print(f"partitions: product {n_p}, oracle {n_o}")
    assert n_p > SMEM_PARTS and n_o > SMEM_PARTS
    totals = dict(dec=0, acc=0, evict=0, reload=0)
    for ep in range(6):
        ev = w.events(ep, 3000, seed)
        now0 = fl.now_ms + ep * w.window_ms
        dec, evi, rep = compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, seed * 100 + ep)
        totals["dec"] += len(dec); totals["acc"] += int(np.count_nonzero(dec["status"] == ob.SIM_ACCEPTED))
        totals["evict"] += len(evi); totals["reload"] += int(evi["reload"].sum())
    print(totals)
    assert totals["acc"] > 0 and totals["evict"] > 0 and totals["reload"] > 0, totals


# ---------------------------------------------------------------------------------------------------------------
# B. boundary instance values
# ---------------------------------------------------------------------------------------------------------------
def _boundary_fleet(case, seed=31):
    fl = make_fleet("C3", 600, 240, seed)
    rows = fl.inst_rows
    ni = fl.n_instances
    rng = np.random.default_rng(seed)
    ms = fl.min_space_units
    if case == "lru_max":
        rows["lru_time"] = LONG_MAX
    elif case == "lru_mix":
        r = rng.uniform(size=ni)
        rows["lru_time"] = np.where(r < 0.4, 0, np.where(r < 0.8, LONG_MAX, rows["lru_time"]))
    elif case == "is_full_edge":
        k = np.arange(ni)
        rem = ms - 1 + k % 3  # min_space - 1, min_space, min_space + 1
        rows["used"] = np.where(k % 10 == 9, rows["capacity"] + 1 + k, rows["capacity"] - rem)  # and some used > capacity
    elif case == "count_wrap":
        # four instances in one partition at the validated maximum: the int copy count wraps there and in the cluster
        rows["count"][:4] = 1_000_000_000
        rows["shutting_down"][:4] = 0
        for i in range(1, 4):
            fl.inst_labels[i] = list(fl.inst_labels[0])
    elif case == "capacity_wrap":
        rows["shutting_down"][:3] = 0
        rows["capacity"][:3] = (1 << 62) + 12345
        rows["used"][:3] = 1000
    elif case == "all_down":
        rows["shutting_down"] = 1
    return fl


@pytest.mark.parametrize("case", ["lru_max", "lru_mix", "is_full_edge", "count_wrap", "capacity_wrap", "all_down"])
def test_boundary_stats_match_oracle(product_lib, oracle_lib, case):
    fl = _boundary_fleet(case)
    o = converged_oracle(fl)
    s = solver_from_synth(fl, product_lib)
    st, ids, n_o = _check_stats(fl, o, s)
    g = st[0]
    if case == "lru_max":
        assert int(g["global_lru"]) == LONG_MAX and (st["global_lru"] == LONG_MAX).all()
    elif case == "is_full_edge":
        rem = np.maximum(0, fl.inst_rows["capacity"] - fl.inst_rows["used"])
        live = fl.inst_rows["shutting_down"] == 0
        assert int(g["total_free"]) == int(rem[live & (rem >= fl.min_space_units)].sum())
    elif case == "count_wrap":
        assert int(g["model_copy_count"]) < 0 and (st["model_copy_count"][1:] < 0).any()
    elif case == "capacity_wrap":
        assert int(g["total_capacity"]) < 0
    elif case == "all_down":
        assert len(st) == 1 and int(g["instance_count"]) == 0 and int(g["global_lru"]) == LONG_MAX
    sel_c = _reaper_cluster(fl, o, s)
    sel_p = _reaper_partitions(fl, o, s, ids)
    if case in ("capacity_wrap", "all_down"):  # totalCapacity <= 0: the reaper returns before the sweep (MM:6458)
        assert len(sel_c) == 0 and all(len(a) == 0 for a in sel_p)


@pytest.mark.parametrize("config", ["C3", "C5"])
def test_stats_match_oracle_65536_instances(product_lib, oracle_lib, config):
    """more instances than k_stats has threads on an H100 (132 blocks x 256): the grid-stride loop takes several per thread"""
    fl = make_fleet(config, 2000, 65_536, 5)
    o = oracle_from_synth(fl)  # bulk
    s = solver_from_synth(fl, product_lib)
    st, _, n_o = _check_stats(fl, o, s)
    assert int(st[0]["instance_count"]) == int(np.count_nonzero(fl.inst_rows["shutting_down"] == 0)) > 132 * 256
    print(f"{config}: {n_o} partitions")


# ---------------------------------------------------------------------------------------------------------------
# C. the reaper's selection at its edges
# ---------------------------------------------------------------------------------------------------------------
_EDGE_FLEETS = {}


def _edge_fleet(regime):
    """160 C3 instances.  free: the synthetic rows (room on most instances); cutoff: every instance between min_space and the
    1/8 reserve, so the free-space count is 0 and only models used after the cutoff qualify; wrapped: three instances whose
    free space wraps the cluster's totalFree negative, so globalLru is the cluster's LRU (MM:6460) while the other partitions
    still have room."""
    if regime not in _EDGE_FLEETS:
        fl = make_fleet("C3", 10, 160, 11)
        rows = fl.inst_rows
        rng = np.random.default_rng(11)
        if regime == "cutoff":
            rows["used"] = rows["capacity"] - rng.integers(fl.min_space_units, rows["capacity"] // 8, size=fl.n_instances)
        elif regime == "wrapped":
            rows["shutting_down"][:3] = 0
            rows["capacity"][:3] = 3 << 61  # three of them: the capacity sum wraps past zero (positive), the free sum negative
            rows["used"][:3] = 1 << 61
            for i in range(3):
                fl.inst_labels[i] = ["lbl-00", "lbl-01", "lbl-02", "lbl-03"]
        _EDGE_FLEETS[regime] = (fl, converged_oracle(fl))
    return _EDGE_FLEETS[regime]


def _with_registry(fl, last_used, n_loaded, n_failed, model_type):
    f = copy.copy(fl)
    n = len(last_used)
    f.model_last_used = np.asarray(last_used, dtype=np.int64)
    f.n_loaded, f.n_failed = np.asarray(n_loaded, dtype=np.int32), np.asarray(n_failed, dtype=np.int32)
    f.model_type = np.asarray(model_type, dtype=np.int32)
    f.model_size = np.full(n, 6400, dtype=np.int32)
    f.model_rpm = np.zeros(n, dtype=np.int32)
    deg = (f.n_loaded + f.n_failed).astype(np.int64)
    f.edge_off = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=f.edge_off[1:])
    owner = np.repeat(np.arange(n, dtype=np.int64), deg)
    j = np.arange(int(f.edge_off[-1]), dtype=np.int64) - f.edge_off[owner]
    f.edge_inst = ((owner * 7 + j * 13) % fl.n_instances).astype(np.int32)  # distinct per model (deg <= 3)
    return f


def _times(o, now):
    g = o.cluster_stats()
    glru = int(g["global_lru"])  # every subset's LRU is the cluster's (N10): one cutoff for every call
    cutoff = glru + max((now - glru) // 3, 1_200_000)
    return glru, cutoff


@pytest.mark.parametrize("n", [1, 255, 256, 257, 4097, 100_003])
@pytest.mark.parametrize("regime", ["free", "cutoff", "wrapped"])
def test_reaper_selection_edges(product_lib, oracle_lib, regime, n):
    fl0, o = _edge_fleet(regime)
    now = fl0.now_ms
    glru, cutoff = _times(o, now)
    g = o.cluster_stats()
    assert (int(g["total_free"]) <= 0) == (regime == "wrapped")
    rng = np.random.default_rng(n)
    # a handful of values, so that runs of equal lastUsed are long, among them the boundaries of both strict rules
    vals = np.array([0, glru - 1, glru, glru + 1, cutoff - 1, cutoff, cutoff + 1, cutoff + 7, (cutoff + now) // 2, now - 1000, now])
    lu = vals[rng.integers(0, len(vals), size=n)]
    lu = np.where(rng.uniform(size=n) < 0.2, now - rng.integers(0, 40 * 3_600_000, size=n), lu)
    n_loaded = np.where(rng.uniform(size=n) < 0.25, rng.integers(1, 3, size=n), 0)
    r = rng.uniform(size=n)
    n_failed = np.where(r < 0.8, 0, np.where(r < 0.9, 1, 2))
    mt = rng.integers(0, len(fl0.type_names), size=n)
    if n == 1:
        lu[0], n_loaded[0], n_failed[0], mt[0] = cutoff + 1, 0, 0, fl0.type_names.index("untyped")
    fl = _with_registry(fl0, lu, n_loaded, n_failed, mt)
    s = solver_from_synth(fl, product_lib)
    st, ids = s.stats(cap=fl.n_instances + 2)
    sel_c = _reaper_cluster(fl, o, s)
    sel_p = _reaper_partitions(fl, o, s, ids)
    total = len(sel_c) + sum(len(a) for a in sel_p)
    assert total > 0
    # a cap below the selection: the full count comes back, the first `cap` ids are written, every selected model is taken
    pmap = partition_maps(fl, o, s)
    om = _om(fl)
    for pid in [-1] + [int(p) for p in ids[1:]]:
        taken_o = np.zeros(n, np.uint8)
        a = o.reaper_select(om, fl.type_names, pid if pid < 0 else pmap[pid], now, taken=taken_o)
        if len(a) < 2:
            continue
        cap = len(a) // 2
        out = np.full(cap + 4, -7, dtype=np.int32)
        taken_s = np.zeros(n, np.uint8)
        k = s._ck(product_lib.mmp_reaper_select(s.h, pid, now, vp(taken_s), vp(out), cap))
        assert k == len(a) and np.array_equal(out[:cap], a[:cap]) and (out[cap:] == -7).all(), (pid, k, len(a))
        assert np.array_equal(taken_s, taken_o) and int(taken_s.sum()) == len(a)
        break
    else:
        assert n == 1, "no call selected two models"


@pytest.mark.parametrize("regime", ["free", "cutoff", "wrapped"])
def test_reaper_total_count_edges(product_lib, oracle_lib, regime):
    """total_count one below, at and one above the number of unique candidates.  total_count depends on the stats alone; a
    registry of distinct lastUsed values all after the cutoff finds it (the oracle selects min(unique, total_count))."""
    fl0, o = _edge_fleet(regime)
    now = fl0.now_ms
    glru, cutoff = _times(o, now)
    untyped = fl0.type_names.index("untyped")
    n_probe = 20_000
    probe = _with_registry(fl0, cutoff + 1 + np.arange(n_probe), np.zeros(n_probe), np.zeros(n_probe), np.full(n_probe, untyped))
    s = solver_from_synth(probe, product_lib)
    st, ids = s.stats(cap=fl0.n_instances + 2)
    pmap = partition_maps(probe, o, s)
    target = None
    for pid in [-1] + [int(p) for p in ids[1:]]:
        a = o.reaper_select(_om(probe), probe.type_names, pid if pid < 0 else pmap[pid], now)
        b = s.reaper_select(pid, now)
        assert np.array_equal(a, b), pid
        if 2 <= len(a) < n_probe:
            target, t_count = pid, len(a)
            break
    assert target is not None
    rng = np.random.default_rng(7)
    for u in (t_count - 1, t_count, t_count + 1):
        # u unique candidate times, each repeated by later models (runs of equal lastUsed), and as many non-candidates
        base = cutoff + 1 + rng.permutation(4 * u)[:u]
        lu = np.concatenate([base, base[rng.integers(0, u, size=u)], base[rng.integers(0, u, size=u)]])
        nl = np.concatenate([np.zeros(2 * u), np.ones(u)])
        nf = np.concatenate([np.zeros(u), rng.integers(0, 2, size=u), np.zeros(u)])
        f = _with_registry(fl0, lu, nl, nf, np.full(len(lu), untyped))
        s2 = solver_from_synth(f, product_lib)
        st2, ids2 = s2.stats(cap=fl0.n_instances + 2)
        pid = target
        if pid >= 0:  # the same partition in this fleet's numbering
            want = pmap[pid]
            pid = next(int(p) for p, q in partition_maps(f, o, s2).items() if q == want)
        taken_o, taken_s = np.zeros(len(lu), np.uint8), np.zeros(len(lu), np.uint8)
        a = o.reaper_select(_om(f), f.type_names, target if target < 0 else pmap[target], now, taken=taken_o)
        b = s2.reaper_select(pid, now, taken=taken_s)
        assert np.array_equal(a, b) and np.array_equal(taken_o, taken_s), (u, len(a), len(b))
        assert len(a) == min(u, t_count), (u, t_count, len(a))


def _zero_estimate_fleet(with_candidates):
    """Instances report copies but use no space: capacity - free = 0 with more than 10 copies, so the size estimate is 0"""
    fl = make_fleet("C2", 10, 40, 2)
    fl.inst_rows["used"] = 0
    fl.inst_rows["count"] = 5
    n = 300
    rng = np.random.default_rng(2)
    lu = fl.now_ms - rng.integers(0, 3_600_000, size=n)
    if with_candidates:
        nl, nf = np.where(np.arange(n) % 3 == 0, 0, 1), np.zeros(n)
    else:  # every model has a copy, or has failed twice: none passes the candidate rule (MM:6574-6577)
        nl, nf = np.where(np.arange(n) % 2 == 0, 1, 0), np.where(np.arange(n) % 2 == 0, 0, 2)
    return _with_registry(fl, lu, nl, nf, rng.integers(0, len(fl.type_names), size=n))


@pytest.mark.parametrize("with_candidates", [True, False])
def test_reaper_zero_size_estimate(product_lib, oracle_lib, with_candidates):
    fl = _zero_estimate_fleet(with_candidates)
    o = converged_oracle(fl)
    s = solver_from_synth(fl, product_lib)
    g = o.cluster_stats()
    assert int(g["total_capacity"]) == int(g["total_free"]) > 0 and int(g["model_copy_count"]) > 10
    om = _om(fl)
    out = np.zeros(fl.n_models, dtype=np.int32)
    names = (C.c_char_p * len(fl.type_names))(*[t.encode() for t in fl.type_names])
    rc = oracle_lib.orc_reaper_select(o.h, fl.n_models, vp(om), names, len(fl.type_names), -1, fl.now_ms, None, vp(out), len(out))
    if with_candidates:
        assert rc == -4  # the reference's ArithmeticException (MM:6651)
        with pytest.raises(MmpError) as e:
            s.reaper_select(-1, fl.now_ms)
        assert e.value.code == L.E_ARG
    else:  # an empty candidate list never reaches the division (MM:6470)
        assert rc == 0
        assert len(s.reaper_select(-1, fl.now_ms)) == 0
