"""mmp_scale_eval (k_scale_eval: rateTrackingTask MM:5684-5806, getExcludeSet MM:5835-5856, loadedSince MM:5858-5870,
removeModelCopies MM:6197-6310, removeSecondModelCopy MM:6314-6335) and the registry prune (k_registry_prune:
pruneMissingInstances MM:6752-6784) against orc_rate_task_eval / orc_janitor_eval / orc_prune_missing at the values random
records never take: every strict or non-strict comparison as a PAIR of cases, one on each side of its line, and the Java
int / long arithmetic where it wraps.

The fleets are built by hand: 48 instances whose id order differs from their index order, one shutting down (SHUT) and one
not in the instance table (GONE), and variants of the free space, the LRU times, the versions (quirk N1) and the type
constraints.  Each boundary case names its fleet, its parameters and one cache entry on a model of its own.  The CPU test
runs the oracle alone and checks that the two sides of every pair answer differently, so a case that misses its line fails
there rather than passing silently on the GPU."""
import ctypes as C

import numpy as np
import pytest

from helpers import oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import LONG_MAX, NOW_MS, SynthFleet
from oracle import binding as ob
from test_fleet_scans_edges_gpu import _converged_oracle
from test_oracle_properties import brute_compare
from test_registry_overflow_gpu import GONE_MS, HOUR, _oracle_prune, _oracle_scale, _params, _scale

NOW = NOW_MS
INT_MAX, INT_MIN = (1 << 31) - 1, -(1 << 31)
NI, CAP, MIN_SPACE, CHURN = 48, 1_000_000, 10_000, 600_000
SHUT, GONE = 47, 46                     # shutting down (in the table, not live); deleted from the table
H, A, B = 5, 6, 7                       # published rpm 7000, 9000, 8999 (every other instance: 100)
FEW, ONE, TWO, THREE, ZCAP = range(5, 15), (15,), (16, 17), (18, 19, 20), (40, 41)
FREE = (0, 1, 2, 3, 42, 43, 44, 45)     # the only instances that are not full (when the fleet has free space)
P_, Q_, S_ = 10, 0, 11                  # the N1 cycle on fleet "n1"
LIVE_CAP = (NI - 2) * CAP               # capacity of the live instances
GLRU = NOW - 6 * HOUR                   # the LRU time of instance 0, the fleets' globalLru
OLD = NOW - 2 * HOUR
TD = 60_000                             # now - last_check_time: rpm == count
CUTOFF = NOW - (TD + 10_000 + 2 * 30_000)   # loadedSince's cutoff under the default parameters
TYPES = ("plain", "few", "one", "two", "three", "zcap")
DEFAULT_P = dict(now=NOW, last_check_time=NOW - TD, iteration=5000, scale_up_rpm_threshold=1000, second_copy_min_age_iters=42,
                 second_copy_max_age_iters=240, second_copy_lru_threshold_ms=100 * HOUR, rate_check_interval_ms=10_000,
                 assume_completed_ms=30_000, second_copy_remove_max_age_ms=36 * HOUR, can_remove=1)
LOWER, UPPER = 5000 - 240, 5000 - 42     # the second-copy window under the default parameters
COUNT_WRAP = (1 << 63) // 60_000 + 1    # count * 60 000 wraps a long

# fleet name -> total free space of the live instances (spread over FREE) and variants
FLEETS = {
    "tight": dict(free=LIVE_CAP * 5 // 100),        # totalFree * 100 / totalCapacity == 5: the janitor may remove
    "tight6": dict(free=LIVE_CAP * 6 // 100),       # == 6: it may not
    "free10": dict(free=LIVE_CAP // 10),            # 10 * totalFree / totalCapacity == 1: a second copy may load
    "free10m": dict(free=LIVE_CAP // 10 - 1),       # == 0
    "cap0": dict(free=0, cap0=True),                # totalCapacity == 0
    "wrap": dict(free=0, wrap=True),                # totalFree and totalCapacity wrap (three instances of 3 * 2^61)
    "empty": dict(free=LIVE_CAP * 5 // 100, lru=LONG_MAX),     # every cache empty: globalLru = Long.MAX_VALUE
    "glru_small": dict(free=LIVE_CAP * 5 // 100, glru=1),      # minAgeMs below 600 000
    "glru_mid": dict(free=LIVE_CAP * 5 // 100, glru=100_000_000),   # minAgeMs between the bounds: 3 104 000
    "n1": dict(free=LIVE_CAP * 5 // 100, n1=True),
    "tc": dict(free=0, tc=True),
    "live0": dict(free=0, live=0), "live1": dict(free=0, live=1), "live2": dict(free=0, live=2),
}
MIN_AGE_MID = (3 * 100_000_000 + 10_400_000) // 100


def _instances(spec):
    rows = np.zeros(NI, dtype=L.INSTANCE_ROW)
    rows["capacity"], rows["used"] = CAP, CAP
    rows["lru_time"] = GLRU + np.arange(NI) * 1000
    rows["start_time"], rows["vers"], rows["count"], rows["l_threads"], rows["rpm"], rows["active"] = NOW - 86_400_000, 7, 10, 8, 100, 1
    rows["rpm"][[H, A, B]] = 7000, 9000, 8999
    free = spec["free"]
    for k, i in enumerate(FREE):
        rows["used"][i] = CAP - (free // len(FREE) + (free % len(FREE) if k == 0 else 0))
    if spec.get("cap0"):
        rows["capacity"], rows["used"] = 0, 0
    if spec.get("wrap"):
        rows["capacity"][:3], rows["used"][:3] = 3 << 61, 1 << 61
    if "lru" in spec:
        rows["lru_time"] = spec["lru"]
    if "glru" in spec:
        rows["lru_time"][39] = spec["glru"]
    if spec.get("n1"):
        rows["vers"] = 1
        rows["vers"][[P_, S_]] = 2
        rows["lru_time"][S_] = 2 * CHURN
    rows["shutting_down"][SHUT] = 1
    if "live" in spec:
        rows["shutting_down"][spec["live"]:] = 1
    labels = [[] for _ in range(NI)]
    cfg = None
    if spec.get("tc"):
        for name, members in zip(TYPES[1:], (FEW, ONE, TWO, THREE, ZCAP)):
            for i in members:
                labels[i].append(name)
        rows["capacity"][list(ZCAP)], rows["used"][list(ZCAP)] = 0, 0
        cfg = {t: {"required": [t]} for t in TYPES[1:]}
    assert (rows["used"] >= 0).all() and (rows["capacity"] >= 0).all()  # what mmp_instance_upsert accepts
    return rows, labels, cfg


def pt(fleet="tight", p=None, loaded=((20, OLD), (10, OLD)), failed=(), lul=0, ty="plain", **rec):
    """One cache entry on a model of its own: its registrations [(instance, load / failure time)] and its entry fields
    (default: the pod holding the first copy, used 40 h ago, never heavy, outside the second-copy window)."""
    r = dict(instance=loaded[0][0] if loaded else 20, count=0, last_used=NOW - 40 * HOUR, last_heavy=0, i1=4000, i2=4000, flags=0)
    r.update(rec)
    return dict(fleet=fleet, p=dict(p or {}), loaded=list(loaded), failed=list(failed), lul=lul, ty=ty, rec=r)


def _n1(holder, other):
    return pt("n1", loaded=((holder, OLD), (other, OLD)))


def _few(instance, loaded, failed=(), count=5000):
    return pt("tc", loaded=[(i, OLD) for i in loaded], failed=[(i, OLD) for i in failed], ty="few", instance=instance, count=count)


THREE_COPIES = ((20, OLD), (21, OLD), (22, OLD))
SIX_COPIES = tuple((20 + k, OLD) for k in range(6))
IN_WINDOW = dict(i1=LOWER, i2=LOWER)
NO_EXCL = dict(scale_up_rpm_threshold=2500)   # maxRpm 10 000: nobody is excluded

# (name, side a, side b): the two sides must answer differently
PAIRS = [
    # ---- rateTrackingTask: the rate, the heavy line, the threshold ----
    ("time_delta_1ms", pt(p=dict(last_check_time=NOW - 1), count=1), pt(p=dict(last_check_time=NOW - 2), count=1)),
    ("time_delta_huge", pt(p=dict(last_check_time=NOW - (1 << 61)), count=1 << 46), pt(p=dict(last_check_time=NOW - (1 << 62)), count=1 << 46)),
    ("count_60000_wraps", pt(count=COUNT_WRAP), pt(count=COUNT_WRAP - 1)),
    ("int_cast_wraps", pt(count=1 << 31), pt(count=(1 << 31) - 1)),
    ("rpm_at_thr", pt(count=999), pt(count=1000)),
    ("rpm_above_thr", pt(count=1000), pt(count=1001)),
    ("heavy_line", pt(count=750), pt(count=751)),
    ("heavy_line_below", pt(count=749), pt(count=750)),
    ("thr_int_max_heavy", pt(p=dict(scale_up_rpm_threshold=INT_MAX), count=536_870_911), pt(p=dict(scale_up_rpm_threshold=INT_MAX), count=536_870_912)),
    ("thr_int_max_scale", pt(p=dict(scale_up_rpm_threshold=INT_MAX), count=INT_MAX), pt(p=dict(scale_up_rpm_threshold=INT_MAX), count=INT_MAX - 1)),
    ("thr_2pow29_exclude", pt(p=dict(scale_up_rpm_threshold=1 << 29), count=1 << 29), pt(p=dict(scale_up_rpm_threshold=(1 << 29) - 1), count=1 << 29)),
    # ---- the second-copy window (one copy; free10: the space rule holds) ----
    ("window_lower", pt("free10", loaded=((20, OLD),), i1=LOWER - 1, i2=LOWER - 1), pt("free10", loaded=((20, OLD),), i1=LOWER, i2=LOWER)),
    ("window_upper", pt("free10", loaded=((20, OLD),), i1=UPPER, i2=UPPER), pt("free10", loaded=((20, OLD),), i1=UPPER + 1, i2=UPPER + 1)),
    ("window_i2_upper", pt("free10", loaded=((20, OLD),), i1=4000, i2=UPPER), pt("free10", loaded=((20, OLD),), i1=4000, i2=UPPER + 1)),
    ("window_i1_lower", pt("free10", loaded=((20, OLD),), i1=LOWER, i2=5000), pt("free10", loaded=((20, OLD),), i1=LOWER - 1, i2=5000)),
    ("window_wraps_int_min", pt("free10", p=dict(iteration=INT_MIN + 100), loaded=((20, OLD),), i1=INT_MIN + 60, i2=INT_MIN + 60),
     pt("free10", p=dict(iteration=INT_MIN + 240), loaded=((20, OLD),), i1=INT_MIN + 60, i2=INT_MIN + 60)),
    ("window_int_max", pt("free10", p=dict(iteration=INT_MAX), loaded=((20, OLD),), i1=INT_MAX - 42, i2=INT_MAX - 42),
     pt("free10", p=dict(iteration=INT_MAX), loaded=((20, OLD),), i1=INT_MAX - 41, i2=INT_MAX - 41)),
    # ---- the second copy's space rule ----
    ("free_tenth", pt("free10", loaded=((20, OLD),), **IN_WINDOW), pt("free10m", loaded=((20, OLD),), **IN_WINDOW)),
    ("free_negative", pt("free10", loaded=((20, OLD),), **IN_WINDOW), pt("wrap", loaded=((20, OLD),), **IN_WINDOW)),
    ("type_set_cap0", pt("tc", loaded=((ZCAP[0], OLD),), ty="zcap", p=dict(second_copy_lru_threshold_ms=0), count=5000, **IN_WINDOW),
     pt("tc", loaded=((TWO[0], OLD),), ty="two", p=dict(second_copy_lru_threshold_ms=0), count=5000, **IN_WINDOW)),
    ("lru_threshold", pt(loaded=((20, OLD),), p=dict(second_copy_lru_threshold_ms=NOW - GLRU), **IN_WINDOW),
     pt(loaded=((20, OLD),), p=dict(second_copy_lru_threshold_ms=NOW - GLRU - 1), **IN_WINDOW)),
    ("lru_long_max", pt("empty", loaded=((20, OLD),), p=dict(second_copy_lru_threshold_ms=NOW - LONG_MAX), **IN_WINDOW),
     pt("empty", loaded=((20, OLD),), p=dict(second_copy_lru_threshold_ms=NOW - LONG_MAX - 1), **IN_WINDOW)),
    # ---- loadedSince ----
    ("loaded_at_cutoff", pt(loaded=((20, OLD), (10, CUTOFF)), count=2000), pt(loaded=((20, OLD), (10, CUTOFF + 1)), count=2000)),
    ("loaded_time_unknown", pt(loaded=((20, OLD), (10, 0)), count=2000), pt(loaded=((20, OLD), (10, CUTOFF + 1)), count=2000)),
    ("loaded_by_self", pt(loaded=((20, NOW), (10, OLD)), count=2000), pt(loaded=((20, NOW), (10, OLD)), instance=30, count=2000)),
    ("loaded_at_position_5", pt(loaded=SIX_COPIES[:5] + ((25, CUTOFF),), count=2000), pt(loaded=SIX_COPIES[:5] + ((25, CUTOFF + 1),), count=2000)),
    # ---- the exclude set (type "few": ten instances, H, A and B among them) ----
    ("max_rpm_self_branch", _few(A, (A, B, 8, 9, 10)), _few(B, (A, B, 8, 9, 10))),   # maxRpm = ourRpm - 2 thr: 7000 vs 6999 (H)
    ("self_not_live", _few(A, (8, 9)), _few(SHUT, (8, 9))),
    ("excluded_holds_failed_pos5", _few(B, (8, 9, 10, 11, 12), (H,)), _few(B, (8, 9, 10, 11, 12), (13,))),   # candidates 1 / 0
    ("excluded_holds_loaded_pos4", _few(B, (8, 9, 10, 11, H)), _few(B, (8, 9, 10, 11, 12))),
    ("excluded_holds_loaded_inline", _few(B, (A, 8, 9, 10)), _few(B, (11, 8, 9, 10))),
    # ---- the copies cap and the suitable instances ----
    ("copies_cap", pt(count=14_000), pt(count=16_000)),                 # suitable / 3 = 15
    ("copies_cap_few", dict(_few(8, (8, 9), count=5000), p=dict(scale_up_rpm_threshold=2500)),
     dict(_few(8, (8, 9), count=10_000), p=dict(scale_up_rpm_threshold=2500))),
    ("suitable_1_2", pt("tc", loaded=((ONE[0], OLD),), ty="one", count=5000, p=NO_EXCL), pt("tc", loaded=((TWO[0], OLD),), ty="two", count=5000, p=NO_EXCL)),
    ("suitable_2_3", pt("tc", loaded=((TWO[0], OLD),), ty="two", count=5000, p=NO_EXCL), pt("tc", loaded=((THREE[0], OLD),), ty="three", count=5000, p=NO_EXCL)),
    ("unconfigured_type", _few(A, (A, B, 8, 9, 10)), dict(_few(A, (A, B, 8, 9, 10)), ty="plain")),
    ("n_ranks_1_2", pt("live1", loaded=((0, OLD),), instance=0, count=5000), pt("live2", loaded=((0, OLD),), instance=0, count=5000)),
    ("n_ranks_0_2", pt("live0", loaded=((0, OLD),), instance=0, count=5000), pt("live2", loaded=((0, OLD),), instance=0, count=5000)),
    # ---- removeModelCopies: the space rule, the entry, the other valid instance ----
    ("janitor_free_5_6", pt(), pt("tight6")),
    ("janitor_cap0", pt(), pt("cap0")),
    ("janitor_free_negative", pt("wrap"), pt("tight6")),
    ("janitor_no_local_stats_tc", pt("tc", flags=0), pt("tc", flags=1)),
    ("janitor_last_used_0", pt(), pt(last_used=0)),
    ("janitor_one_copy", pt(), pt(loaded=((20, OLD),))),
    ("janitor_other_shut", pt(), pt(loaded=((20, OLD), (SHUT, OLD)))),
    ("janitor_other_gone", pt(), pt(loaded=((20, OLD), (GONE, OLD)))),
    ("janitor_others_invalid", pt(loaded=THREE_COPIES), pt(loaded=((20, OLD), (SHUT, OLD), (GONE, OLD)))),
    # ---- two copies ----
    ("scale_down_age", pt(last_used=NOW - (NOW - GLRU) // 10), pt(last_used=NOW - (NOW - GLRU) // 10 - 1)),
    ("last_heavy_cache_age_5", pt(p=dict(second_copy_remove_max_age_ms=600_000), last_used=NOW - 20 * 60_000, last_heavy=NOW - (NOW - GLRU) // 5 + 1),
     pt(p=dict(second_copy_remove_max_age_ms=600_000), last_used=NOW - 20 * 60_000, last_heavy=NOW - (NOW - GLRU) // 5)),
    ("last_heavy_0", pt(p=dict(second_copy_remove_max_age_ms=600_000), last_used=NOW - 20 * 60_000, last_heavy=0),
     pt(p=dict(second_copy_remove_max_age_ms=600_000), last_used=NOW - 20 * 60_000, last_heavy=NOW - (NOW - GLRU) // 5 - 1)),
    ("remove_max_age", pt(p=dict(second_copy_remove_max_age_ms=(NOW - GLRU) // 10 - 1), last_used=NOW - (NOW - GLRU) // 10),
     pt(p=dict(second_copy_remove_max_age_ms=(NOW - GLRU) // 10 + 1), last_used=NOW - (NOW - GLRU) // 10)),
    ("self_not_live_two_copies", pt(), pt(loaded=((SHUT, OLD), (10, OLD)))),
    ("placement_order", pt(), pt(loaded=((10, OLD), (20, OLD)))),
    ("n1_pq", _n1(P_, Q_), _n1(Q_, P_)),
    ("n1_qs", _n1(Q_, S_), _n1(S_, Q_)),
    ("n1_sp", _n1(S_, P_), _n1(P_, S_)),
    # ---- three or more copies ----
    ("last_unload", pt(loaded=THREE_COPIES, lul=NOW - 80_000), pt(loaded=THREE_COPIES, lul=NOW - 79_999)),
    ("last_unload_0", pt(loaded=THREE_COPIES, lul=0), pt(loaded=THREE_COPIES, lul=NOW - 1)),
    ("last_unload_negative", pt(loaded=THREE_COPIES, lul=-5), pt(loaded=THREE_COPIES, lul=NOW - 1)),
    ("recent_load_30min", pt(loaded=THREE_COPIES[:2] + ((22, NOW - 1_800_000),)), pt(loaded=THREE_COPIES[:2] + ((22, NOW - 1_799_999),))),
    ("recent_load_position_5", pt(loaded=SIX_COPIES[:5] + ((25, NOW - 1_800_000),)), pt(loaded=SIX_COPIES[:5] + ((25, NOW - 1_799_999),))),
    ("min_age_above", pt(loaded=THREE_COPIES, last_heavy=NOW - 18_000_000), pt(loaded=THREE_COPIES, last_heavy=NOW - 18_000_000 + 1)),
    ("min_age_below", pt("glru_small", loaded=THREE_COPIES, last_heavy=NOW - 600_000), pt("glru_small", loaded=THREE_COPIES, last_heavy=NOW - 600_000 + 1)),
    ("min_age_between", pt("glru_mid", loaded=THREE_COPIES, last_heavy=NOW - MIN_AGE_MID), pt("glru_mid", loaded=THREE_COPIES, last_heavy=NOW - MIN_AGE_MID + 1)),
    ("min_age_wraps", pt("empty", loaded=THREE_COPIES, last_heavy=NOW - 600_000), pt("empty", loaded=THREE_COPIES, last_heavy=NOW - 600_000 + 1)),
    ("since_interval_10", pt(p=dict(last_check_time=NOW - 1000), loaded=THREE_COPIES), pt(p=dict(last_check_time=NOW - 999), loaded=THREE_COPIES)),
    ("rpm_two_thirds", pt(loaded=THREE_COPIES, count=666), pt(loaded=THREE_COPIES, count=667)),
    ("rpm_two_thirds_below", pt(loaded=THREE_COPIES, count=665), pt(loaded=THREE_COPIES, count=667)),
    ("janitor_count_wraps", pt(loaded=THREE_COPIES, count=COUNT_WRAP), pt(loaded=THREE_COPIES, count=COUNT_WRAP - 1)),
]
# cases without a line of their own: still compared field by field
SINGLES = [
    ("no_local_stats_without_tc", pt(flags=1)),
    ("thr_at_rpm", pt(count=1000, p=dict(scale_up_rpm_threshold=1000))),
    ("five_copies", pt(loaded=SIX_COPIES[:5])),
    ("six_copies_self_at_5", pt(loaded=SIX_COPIES, instance=25)),
    ("unconfigured_type_window", pt("tc", loaded=((8, OLD),), ty="plain", **IN_WINDOW)),
]


def _points():
    pts = []
    for name, a, b in PAIRS:
        pts += [(name + "/a", a), (name + "/b", b)]
    return pts + SINGLES


def _fleet(name, pts):
    """The fleet `name` with one model per case: (SynthFleet, times, lastUnloadTimes, model of each case)"""
    rows, labels, cfg = _instances(FLEETS[name])
    nm = len(pts)
    deg = [len(x["loaded"]) + len(x["failed"]) for _, x in pts]
    off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(deg, out=off[1:])
    regs = [r for _, x in pts for r in x["loaded"] + x["failed"]]
    fl = SynthFleet(name, NOW, MIN_SPACE, CHURN, 6400, rows, [f"pod-{(i * 29) % NI:02d}" for i in range(NI)], [None] * NI, [None] * NI,
                    labels, cfg, list(TYPES), np.array([TYPES.index(x["ty"]) for _, x in pts], dtype=np.int32),
                    np.full(nm, NOW - HOUR, dtype=np.int64), np.full(nm, 6400, dtype=np.int32), np.zeros(nm, dtype=np.int32), off,
                    np.array([i for i, _ in regs], dtype=np.int32), np.array([len(x["loaded"]) for _, x in pts], dtype=np.int32),
                    np.array([len(x["failed"]) for _, x in pts], dtype=np.int32))
    ts = np.array([t for _, t in regs], dtype=np.int64)
    lul = np.array([x["lul"] for _, x in pts], dtype=np.int64)
    return fl, ts, lul


def _oracle(fl):
    o = _converged_oracle(fl) if fl.type_config is not None else oracle_from_synth(fl)
    o.instance_event(ob.DELETED, GONE, None, fl.inst_ids[GONE], now_ms=NOW)
    return o


def _product(fl, ts, lul, lib):
    s = solver_from_synth(fl, lib)
    for m in range(fl.n_models):
        s.model_times(m, ts[fl.edge_off[m]:fl.edge_off[m + 1]], int(lul[m]))
    s.instance_remove(GONE)
    s.commit()
    return s


def _groups():
    """cases grouped by (fleet, parameters): one batch per group"""
    g = {}
    for name, x in _points():
        g.setdefault((x["fleet"], tuple(sorted(x["p"].items()))), []).append((name, x))
    return g


def _batch(pts, p_over, model0=0):
    rec = np.zeros(len(pts), dtype=L.SCALE_IN)
    for r, (_, x) in enumerate(pts):
        for k, v in x["rec"].items():
            rec[k][r] = v
        rec["model"][r] = model0 + r
    p = _params(NOW, 1000, 1, 0)
    for k, v in dict(DEFAULT_P, **dict(p_over)).items():
        p[k] = v
    return rec, p


def _run(oracle_lib, product_lib=None):
    """{case: (product outputs or None, oracle outputs)} over every group"""
    res = {}
    fleets = {}
    for (fname, p_over), pts in _groups().items():
        fleets.setdefault(fname, []).append((p_over, pts))
    for fname, groups in fleets.items():
        every = [x for _, pts in groups for x in pts]
        fl, ts, lul = _fleet(fname, every)
        o = _oracle(fl)
        s = _product(fl, ts, lul, product_lib) if product_lib is not None else None
        m0 = 0
        for p_over, pts in groups:
            rec, p = _batch(pts, p_over, m0)
            up, down = _oracle_scale(oracle_lib, o, fl, ts, lul, rec, p)
            out = _scale(product_lib, s, rec, p) if s is not None else None
            for r, (name, _) in enumerate(pts):
                want = tuple(int(up[k][r]) for k in ("action", "copies_to_load", "load_last_used", "rpm", "i1", "i2", "set_heavy")) + (int(down["remove"][r]),)
                got = None if out is None else tuple(int(out[k][r]) for k in ("action", "copies_to_load", "load_last_used", "rpm", "i1", "i2", "set_heavy", "remove"))
                res[name] = (got, want)
            m0 += len(pts)
        o.close()
        if s is not None:
            s.close()
    return res


def test_n1_fleet_is_a_cycle_under_the_comparator(oracle_lib):
    """P < Q, Q < S and S < P under PLACEMENT_ORDER re-derived from the Java text and under the oracle's comparator"""
    fl, _, _ = _fleet("n1", [("x", _n1(P_, Q_))])
    rows, ids = fl.inst_rows, fl.inst_ids
    cmp = lambda a, b: brute_compare(rows[a], ids[a], None, None, [], rows[b], ids[b], None, None, [], MIN_SPACE, CHURN)
    assert cmp(P_, Q_) < 0 and cmp(Q_, S_) < 0 and cmp(S_, P_) < 0
    o = _oracle(fl)
    assert o.compare(P_, Q_) < 0 and o.compare(Q_, S_) < 0 and o.compare(S_, P_) < 0
    o.close()


def test_boundary_pairs_straddle_their_line(oracle_lib):
    """the oracle alone: the two sides of every pair answer differently"""
    res = _run(oracle_lib)
    same = [name for name, _, _ in PAIRS if res[name + "/a"][1] == res[name + "/b"][1]]
    assert not same, [(n, res[n + "/a"][1]) for n in same]


@pytest.mark.gpu
def test_scale_eval_boundaries_match_oracle(product_lib, oracle_lib):
    res = _run(oracle_lib, product_lib)
    bad = {name: r for name, r in res.items() if r[0] != r[1]}
    assert not bad, bad
    # the N1 cycle: with a linear order of P, Q and S, one of the three pairs would answer against the comparator
    assert [res[f"n1_{k}/{s}"][1][7] for k in ("pq", "qs", "sp") for s in "ab"] == [0, 1, 0, 1, 0, 1]


# ---------------------------------------------------------------------------------------------------------------
# the registry prune
# ---------------------------------------------------------------------------------------------------------------
MISSING_TS = (40, 41, 42)       # not in the table, missing since before the pass (40, 42) / exactly GONE_MS before it (41)
WIDE, BACK, SELF2 = 43, 44, 45  # missing for the first time on ~3000 models; re-added between passes; the other self
NM = 6000


def _prune_fleet():
    rows, labels, cfg = _instances(FLEETS["tight"])
    rng = np.random.default_rng(45)
    common = np.setdiff1d(np.arange(NI), [40, 41, 42, WIDE, BACK, SELF2, GONE])
    edges, ts = [], []
    for m in range(NM):
        k = int(rng.integers(1, 7))
        inst = list(rng.choice(common, size=k, replace=False))
        t = list(NOW - rng.integers(HOUR, 4 * HOUR, size=k))
        if m < 8:   # the time edges on 40: now - ts = GONE_MS - 1, GONE_MS, GONE_MS + 1 and ts = 0; then 41 and 42
            inst[0] = (40, 40, 40, 40, 41, 42, 40, 42)[m]
            t[0] = (NOW - GONE_MS + 1, NOW - GONE_MS, NOW - GONE_MS - 1, 0, OLD, OLD, OLD, OLD)[m]
        elif m % 2 == 0:  # WIDE at every position, BACK and SELF2 now and then, the rest spread over the registry
            inst[int(rng.integers(0, k))] = WIDE
            if m % 10 == 0 and k > 1:
                inst[(inst.index(WIDE) + 1) % k] = BACK if m % 20 == 0 else SELF2
        elif m % 7 == 1:
            inst[int(rng.integers(0, k))] = int(rng.choice(MISSING_TS))
        edges.append(inst)
        ts += t
    off = np.zeros(NM + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=off[1:])
    nl = np.array([max(1, len(e) - 1) for e in edges], dtype=np.int32)
    fl = SynthFleet("prune", NOW, MIN_SPACE, CHURN, 6400, rows, [f"pod-{(i * 29) % NI:02d}" for i in range(NI)], [None] * NI, [None] * NI,
                    labels, cfg, list(TYPES), np.zeros(NM, dtype=np.int32), np.full(NM, NOW - HOUR, dtype=np.int64),
                    np.full(NM, 6400, dtype=np.int32), np.zeros(NM, dtype=np.int32), off, np.concatenate(edges).astype(np.int32), nl,
                    (np.diff(off) - nl).astype(np.int32))
    return fl, np.array(ts, dtype=np.int64)


def _missing():
    miss = np.zeros(NI, dtype=np.int64)
    miss[[40, 42, SELF2]] = NOW - GONE_MS - 1
    miss[41] = NOW - GONE_MS
    return miss


def test_prune_boundary_pairs_straddle_their_line(oracle_lib):
    """orc_prune_missing on one registration of a missing instance: now - ts and now - missing_since at their lines"""
    fl, _ = _prune_fleet()
    o = oracle_from_synth(fl)
    for i in (40, 41, 42, WIDE, BACK, SELF2, GONE):
        o.instance_event(ob.DELETED, i, None, fl.inst_ids[i], now_ms=NOW)

    def pruned(ts, since):
        miss = np.zeros(NI, dtype=np.int64)
        miss[40] = since
        out = np.zeros(1, dtype=np.uint8)
        return oracle_lib.orc_prune_missing(o.h, 0, np.array([40], np.int32).ctypes.data_as(C.c_void_p), np.array([ts], np.int64).ctypes.data_as(C.c_void_p),
                                            1, NOW, GONE_MS, miss.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
    old = NOW - GONE_MS - 1
    assert pruned(NOW - GONE_MS + 1, old) == 0 and pruned(NOW - GONE_MS, old) == 1 and pruned(NOW - GONE_MS - 1, old) == 1 and pruned(0, old) == 1
    assert pruned(OLD, NOW - GONE_MS) == 0 and pruned(OLD, NOW - GONE_MS - 1) == 1 and pruned(OLD, 0) == 0
    o.close()


@pytest.mark.gpu
def test_registry_prune_boundaries_match_oracle(product_lib, oracle_lib):
    fl, ts = _prune_fleet()
    s = solver_from_synth(fl, product_lib)
    for m in range(NM):
        s.model_times(m, ts[fl.edge_off[m]:fl.edge_off[m + 1]])
    o = oracle_from_synth(fl)
    for i in (40, 41, 42, WIDE, BACK, SELF2, GONE):
        s.instance_remove(i)
        o.instance_event(ob.DELETED, i, None, fl.inst_ids[i], now_ms=NOW)
    s.commit()
    vp = lambda a: a.ctypes.data_as(C.c_void_p)
    views = {"ids": (_missing(), _missing()), "four": (_missing(), _missing())}
    deg = np.diff(fl.edge_off)
    on = lambda i: {m for m in range(NM) if i in fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]]}
    for rnd, now in enumerate((NOW, NOW + GONE_MS + 1)):
        if rnd == 1:  # BACK rejoins the table between the passes
            s.instance_upsert(BACK, fl.inst_rows[BACK], fl.inst_ids[BACK])
            s.commit()
            o.instance_event(ob.ADDED, BACK, fl.inst_rows[BACK], fl.inst_ids[BACK], now_ms=now)
        mp, mo = views["ids"]
        before = mp.copy()
        n, pm, pi = s.registry_prune_ids(0, now, GONE_MS, mp, 1 << 20)
        want, _ = _oracle_prune(oracle_lib, o, fl, ts, 0, now, mo)
        got = list(zip(pm.tolist(), pi.tolist()))
        assert n == len(want) and got == want, (rnd, n, len(want))
        assert np.array_equal(mp, mo), rnd
        for cap in (0, 1, n - 1, n, n + 1):
            k, cm, ci = s.registry_prune_ids(0, now, GONE_MS, before.copy(), max(cap, 0))
            assert k == n and list(zip(cm.tolist(), ci.tolist())) == want[:cap], (rnd, cap)
        fp, fo = views["four"]
        before4 = fp.copy()
        outm, outk = np.zeros(NM, dtype=np.int32), np.zeros(NM, dtype=np.uint8)
        k4 = s._ck(product_lib.mmp_registry_prune(s.h, 0, now, GONE_MS, vp(fp), vp(outm), vp(outk), NM))
        _, masks = _oracle_prune(oracle_lib, o, fl, ts, 0, now, fo, first=4)
        assert k4 == len(masks) and list(zip(outm[:k4].tolist(), outk[:k4].tolist())) == sorted(masks.items()), rnd
        assert np.array_equal(fp, fo), rnd
        # a cap below the count: the first cap models in model order (the pruned models spread over every block)
        ordered = sorted(masks.items())
        assert k4 > 200 and ordered[-1][0] - ordered[0][0] > 20 * 256
        for cap in (0, 1, k4 - 1, k4, k4 + 1):
            cm = np.full(cap + 2, -7, dtype=np.int32)
            ck = np.full(cap + 2, 0xEE, dtype=np.uint8)
            assert s._ck(product_lib.mmp_registry_prune(s.h, 0, now, GONE_MS, vp(before4.copy()), vp(cm), vp(ck), cap)) == k4, (rnd, cap)
            n_w = min(cap, k4)
            assert list(zip(cm[:n_w].tolist(), ck[:n_w].tolist())) == ordered[:cap] and (cm[n_w:] == -7).all(), (rnd, cap)
        pruned_inst = set(pi.tolist())
        assert SELF2 in pruned_inst and 0 not in pruned_inst
        if rnd == 0:
            # the time edges on instance 40 and the missing-since edges on 41 / 42
            first = {m: i for m, i in want if m < 8}
            assert sorted(first) == [1, 2, 3, 5, 6, 7], first
            # WIDE: stamped by this pass on every model it is registered on, pruned on none
            assert mp[WIDE] == now and mp[BACK] == now and WIDE not in pruned_inst and BACK not in pruned_inst
        else:
            wide = {m for m, i in want if i == WIDE}
            assert len(wide) > 2500 and wide == on(WIDE), (len(wide), len(on(WIDE)))
            assert BACK not in pruned_inst and (deg[sorted(wide)] > 4).any()
    # the other pod prunes the first: SELF2's own registrations stay
    m2 = _missing()
    mo2 = _missing()
    n, pm, pi = s.registry_prune_ids(SELF2, NOW, GONE_MS, m2, 1 << 20)
    want, _ = _oracle_prune(oracle_lib, o, fl, ts, SELF2, NOW, mo2)
    assert list(zip(pm.tolist(), pi.tolist())) == want and np.array_equal(m2, mo2) and SELF2 not in set(pi.tolist())
    o.close()
    s.close()
