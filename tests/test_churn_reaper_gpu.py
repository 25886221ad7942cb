"""The reaper's proactive loads in the device closed loop (MMP_CHURN_REAPER events of mmp_churn_step):
  * a one-event window [REAPER(caller, t)] decides exactly what mmp_reaper_select selects, partition by partition in
    mmp_stats order with one shared `taken` array, in the same order -- on free fleets (free-space count), full ones (the
    lastUsed cutoff), with and without type constraints, equal-lastUsed runs, 0/1/2 failed loads, a partition whose count is
    0, a fleet without candidates and a size estimate of 0;
  * multi-window traces mixing REQUEST, REMOVE and REAPER equal the oracle's closed loop (oracle/mm_sim.inc, stepped with
    the REAPER event of tests/emul/reaper_sim.cpp) event for event, as test_churn_gpu.py compares them: coalescing both
    ways, two REAPER events in one window, churn- or early-rejected loads, a fleet with overflow registrations, an
    out-of-range caller;
  * a window without REAPER events reports the same bytes and launches the same kernels after a REAPER window as on a fleet
    that never saw one;
  * C4 at full size (500k models x 2 500 instances) with one REAPER event per window."""
import numpy as np
import pytest

from churn_harness import build as _build_churn, compare_window, device_selection, recent_unloaded, reaper_workload, with_failed
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import make_churn, make_churn_overflow
from oracle import binding as ob
from reaper_oracle import _reaper_oracle_so, reaper_oracle, with_reaper  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("reaper_oracle")]


def _build(product_lib, w, slots):
    """churn_harness.build's fleet, oracle and device loop, the oracle's loop stepping with REAPER events (reaper_oracle.py)"""
    o, sim, s = _build_churn(product_lib, w, slots)
    return o, with_reaper(sim, w.fleet.n_models), s


def reaper_event(caller: int, t: int) -> np.ndarray:
    e = np.zeros(1, dtype=L.CHURN_EVENT)
    e["type"], e["caller"], e["t"] = L.CHURN_REAPER, caller, t
    return e


def request_event(model: int, caller: int, t: int) -> np.ndarray:
    e = np.zeros(1, dtype=L.CHURN_EVENT)
    e["type"], e["model"], e["caller"], e["t"] = L.CHURN_REQUEST, model, caller, t
    return e


@pytest.mark.parametrize("case,seed", [("free", 3), ("free_tc", 4), ("cutoff", 5), ("cutoff_tc", 6), ("full", 7), ("ties", 8),
                                       ("none", 9), ("zero", 10), ("part0_tc", 11)])
def test_reaper_window_decides_the_selection(product_lib, oracle_lib, case, seed):
    w = reaper_workload(case, seed)
    fl = w.fleet
    o, sim, s = _build(product_lib, w, slots=256)
    t = fl.now_ms + 500
    want = device_selection(s, t)
    ev = reaper_event(17, t)
    dec, _, _ = compare_window(0, o, sim, s, ev, fl.now_ms, fl.now_ms + w.window_ms, seed)
    assert [int(m) for m in dec["model"]] == want, (case, len(dec), len(want))
    assert np.all(dec["event"] == 0) and np.all(dec["self"] == 17)
    if case in ("free", "free_tc", "cutoff", "cutoff_tc", "ties", "part0_tc"):
        assert len(want) > 10, (case, len(want))
    if case in ("none", "zero"):
        assert not want, (case, len(want))
    if case.startswith("cutoff"):  # candidates on both sides of the cutoff: the walk stopped before the list's end
        assert len(want) < int(np.count_nonzero(fl.n_loaded == 0)), len(want)
    if case == "ties":
        lu = fl.model_last_used[want]
        assert len(set(lu.tolist())) == len(lu)  # one model per lastUsed
        assert not set(want) & set(int(m) for m in w.unloaded_models if fl.n_failed[m] >= 2)
def _compare_malformed_window(ep, o, sim, s, ev, now0, now1, seed):
    """compare_window for a window whose REAPER caller is no instance: its malformed decisions name no target on either side
    (the oracle answers getNext's null, the device MMP_TARGET_INVALID, as for a REQUEST of that caller)"""
    dec_o, evi_o, rows_o, npub_o, carry_o = sim.step(ev, now0, now1, seed)
    dec_p, evi_p, rows_p, rep = s.churn_step(ev, now0, now1, seed)
    assert len(dec_p) == len(dec_o), (ep, len(dec_p), len(dec_o))
    keep = dec_o["status"] != ob.SIM_SKIPPED
    named = keep & (dec_o["status"] != ob.SIM_INVALID)
    for k in ("event", "status", "model", "self", "target", "n_candidates"):
        m = named if k in ("target", "n_candidates") else keep if k == "model" else slice(None)
        a, b = dec_p[k][m], dec_o[k][m]
        assert np.array_equal(a, b), (ep, k)
    assert np.all(dec_p["target"][dec_o["status"] == ob.SIM_INVALID] == -3)
    for k in ("instance", "model", "last_used", "weight", "order", "reload"):
        assert np.array_equal(evi_p[k], evi_o[k]), (ep, k)
    for k in ("lru_time", "capacity", "used", "count", "l_in_prog", "rpm", "l_threads"):
        assert np.array_equal(rows_p[k], rows_o[k]), (ep, k)
    assert rep.n_published == npub_o and rep.n_carry == carry_o
    assert np.array_equal(s.cluster_order(), o.cluster_order()), ep
    return dec_o, evi_o, rep


def _run_trace(product_lib, w, windows, seed, build_events):
    fl = w.fleet
    o, sim, s = _build(product_lib, w, slots=256)
    out = []
    for ep in range(windows):
        now0 = fl.now_ms + ep * w.window_ms
        ev = build_events(ep, now0)
        co0 = sim.coalesced()
        bad = np.any((ev["type"] == L.CHURN_REAPER) & ((ev["caller"] < 0) | (ev["caller"] >= fl.n_instances)))
        dec, evi, rep = (_compare_malformed_window if bad else compare_window)(ep, o, sim, s, ev, now0, now0 + w.window_ms, seed * 100 + ep)
        assert rep.n_coalesced == sim.coalesced() - co0, (ep, rep.n_coalesced, sim.coalesced() - co0)
        reaper = np.isin(dec["event"], np.nonzero(ev["type"] == L.CHURN_REAPER)[0])
        out.append((ev, dec, reaper, rep))
    for m in range(0, fl.n_models, 41):
        copies, lu = sim.model_copies(m)
        row, ids = s.churn_model_ids(m)
        assert int(row["copy_count"]) == len(copies) and list(ids[:len(copies)]) == list(copies) and int(row["last_used"]) == lu, m
    return out


def test_reaper_trace_coalescing_and_malformed_caller(product_lib, oracle_lib):
    w = make_churn(20_000, 200, 21, fill=0.5)
    fl = w.fleet
    top = [int(m) for m in recent_unloaded(w, 4)]  # surely selected by the first REAPER (free space: the most recent first)

    def events(ep, now0):
        base = w.events(ep, 2000, 21)
        base = base[~np.isin(base["model"], top)]
        if ep == 0:  # a miss of top[0] before the REAPER, one of top[1] after it
            return np.concatenate([base[:300], request_event(top[0], 3, now0 + 400), base[300:900], reaper_event(9, now0 + 900),
                                   base[900:1200], request_event(top[1], 4, now0 + 1300), base[1200:]])
        if ep == 1:  # two REAPER events in one window
            return np.concatenate([base[:500], reaper_event(2, now0 + 500), base[500:1500], reaper_event(50, now0 + 1500), base[1500:]])
        if ep == 2:  # a leader that is not an instance: its decisions are malformed
            return np.concatenate([base[:1000], reaper_event(fl.n_instances + 7, now0 + 1000), base[1000:]])
        return np.concatenate([base, reaper_event(ep, now0 + 1999)])

    out = _run_trace(product_lib, w, 5, 21, events)
    ev0, dec0, r0, rep0 = out[0]
    assert top[0] not in set(dec0["model"][r0].tolist()) and top[1] in set(dec0["model"][r0].tolist())
    assert rep0.n_coalesced >= 2 and rep0.ms_reaper > 0
    ev1, dec1, r1, rep1 = out[1]  # the second run reads the same snapshot: what it selects again the first one decided
    first, second = np.nonzero(ev1["type"] == L.CHURN_REAPER)[0]
    n1 = np.count_nonzero(dec1["event"] == first)
    assert n1 > 10 and np.count_nonzero(dec1["event"] == second) < n1 and rep1.n_coalesced >= n1
    _, dec2, r2, _ = out[2]
    assert np.count_nonzero(r2) > 10 and np.all(dec2["status"][r2] == ob.SIM_INVALID)
    assert sum(int(np.count_nonzero(d["status"][r] == ob.SIM_ACCEPTED)) for _, d, r, _ in out) > 100


def test_reaper_loads_rejected_on_full_caches(product_lib, oracle_lib):
    """published records at half the caches' real use: the reaper sees free space and sends stale models to full caches,
    where loadLocal's churn guard (MM:3872-3884) or early reject (MM:5185-5190) turns them away"""
    w = make_churn(20_000, 200, 23, fill=0.97, with_types=True)
    w.fleet.inst_rows["used"] //= 2
    out = _run_trace(product_lib, w, 4, 23, lambda ep, now0: np.concatenate([w.events(ep, 2000, 23), reaper_event(ep + 1, now0 + 1999)]))
    st = np.concatenate([d["status"][r] for _, d, r, _ in out])
    assert np.count_nonzero((st == ob.SIM_EARLY) | (st == ob.SIM_CHURN)) > 0, np.bincount(st)


def test_reaper_on_overflow_registrations(product_lib, oracle_lib):
    w = make_churn_overflow(make_churn(20_000, 200, 25, fill=0.6), 0.05, 25)
    out = _run_trace(product_lib, w, 4, 25, lambda ep, now0: np.concatenate([w.events(ep, 2000, 25)[:1000], reaper_event(ep + 3, now0 + 1000),
                                                                              w.events(ep, 2000, 25)[1000:]]))
    assert sum(int(np.count_nonzero(d["status"][r] == ob.SIM_ACCEPTED)) for _, d, r, _ in out) > 50


def test_window_without_reaper_unchanged(product_lib, oracle_lib):
    """Fleets a and b from one workload without reaper candidates; b's first window carries a REAPER event at its end (which
    selects nothing).  Every window's reports are the same bytes, and every later window launches the same kernels."""
    w = make_churn(20_000, 200, 27, fill=0.9)
    w = with_failed(w, {int(m): 2 for m in w.unloaded_models})
    fl = w.fleet
    _, _, a = _build(product_lib, w, slots=256)
    _, _, b = _build(product_lib, w, slots=256)
    for ep in range(4):
        now0 = fl.now_ms + ep * w.window_ms
        ev = w.events(ep, 2000, 27)
        eb = np.concatenate([ev, reaper_event(5, now0 + 1999)]) if ep == 0 else ev
        la, lb = a.kernel_launches(), b.kernel_launches()
        ra = a.churn_step(ev, now0, now0 + w.window_ms, 300 + ep)
        rb = b.churn_step(eb, now0, now0 + w.window_ms, 300 + ep)
        for x, y in zip(ra[:3], rb[:3]):  # every field (an eviction record's 4 bytes of padding are not written)
            assert all(x[k].tobytes() == y[k].tobytes() for k in x.dtype.names), ep
        for k in ("n_published", "n_carry", "n_coalesced", "n_lru_events"):
            assert getattr(ra[3], k) == getattr(rb[3], k), (ep, k)
        assert ra[3].ms_reaper == 0
        if ep == 0:
            assert rb[3].ms_reaper > 0 and b.kernel_launches() - lb > a.kernel_launches() - la
        else:
            assert b.kernel_launches() - lb == a.kernel_launches() - la and rb[3].ms_reaper == 0, ep
    assert np.array_equal(a.cluster_order(), b.cluster_order())


def test_reaper_c4_full_size(product_lib, oracle_lib):
    """C4 (500k models x 2 500 instances, 97 % fill) with 100 instances publishing 30 % less than their caches hold, so that the
    reaper has free space to fill and stale copies to displace: 20 000 events and one REAPER event per 2 s window, against
    the oracle"""
    w = make_churn(500_000, 2_500, 4)
    fl = w.fleet
    fl.inst_rows["used"][:100] = fl.inst_rows["used"][:100] * 7 // 10
    o, sim, s = _build(product_lib, w, slots=512)
    picked = 0
    for ep in range(3):
        now0 = fl.now_ms + ep * w.window_ms
        base = w.events(ep, 20_000, 4)
        ev = np.concatenate([base[:10_000], reaper_event(ep * 7, now0 + 1000), base[10_000:]])
        dec, _, rep = compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, 400 + ep)
        picked += int(np.count_nonzero(dec["event"] == 10_000))
    assert picked > 1000, picked
