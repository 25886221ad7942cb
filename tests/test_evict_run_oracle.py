"""The restatement of one pod's eviction listener (tests/evict_run_oracle.py), checked without a GPU on small hand-built
fleets with known answers, one edge each: the registration's age at exactly 2 x loadTimeoutMs and one ms past it, a failed
entry, a loadTimestamp that does not match, the pod only in failedIn, no registration of the pod, 20 * free / capacity at 1
and at 0, a one-instance cluster and zero capacity, another copy on a ranked instance and on one gone from the table, 2 and
3 recent failures with and without the pod's own dropped one, updateLastUsed with 0 and an older value,
updateLastUnloadTime with 2 and 3 copies left, the pod past its fourth registration and a model with 20 registrations."""
import numpy as np

import evict_run_oracle as ero
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import NOW_MS
from common import EXPIRY, HOUR
from pod_task_edges import hand_fleet
from pod_tasks import HAND_TIMEOUT, evict_params

POD = 0
OLD = NOW_MS - 2 * HAND_TIMEOUT - 1   # a registration time that reloads
RECENT_FAIL = NOW_MS - EXPIRY // 2 + 1
UR = L.EV_UNREGISTER | L.EV_RELOAD

def ents(*rows):
    """rows of (model, last_used, load_ts, load_complete_ts, flags)"""
    e = np.zeros(len(rows), dtype=L.EVICT_ENTRY)
    for r, (m, lu, lt, lct, fl) in enumerate(rows):
        e[r] = (m, fl, lu, lt, lct)
    return e


def run(regs, ni, rows, seed=5, lul=None, edit=None, **kw):
    """(fleet, out, report, the type set's stats); edit(fl): changes to the fleet's instance rows before the oracle is built"""
    fl, ts, o = hand_fleet(regs, ni, seed=seed, **kw)
    assert fl.now_ms == NOW_MS
    if edit is not None:
        o.close()
        edit(fl)
        o = oracle_from_synth(fl)
    lul = np.zeros(len(regs), dtype=np.int64) if lul is None else np.asarray(lul, dtype=np.int64)
    out, rep = ero.evict_run(o, fl, ts, lul, POD, ents(*rows), evict_params(fl.now_ms, HAND_TIMEOUT), seed)
    stats = o.type_stats(fl.type_names[0])
    o.close()
    return fl, out, rep, stats


def report(**nonzero):
    return {**{k: 0 for k in ero.REPORT_KEYS + ("n_none",)}, **nonzero}


def test_reload_needs_an_age_past_twice_the_timeout(oracle_lib):
    now = NOW_MS
    t0, t1 = now - 2 * HAND_TIMEOUT, now - 2 * HAND_TIMEOUT - 1
    fl, out, rep, _ = run([([(POD, t0)], []), ([(POD, t1)], [])], 12, [(0, now - 5000, t0, 0, 0), (1, now - 5000, t1, 0, 0)])
    assert list(out["what"]) == [L.EV_UNREGISTER, UR | L.EV_PLACED]
    assert out["target"][0] == L.TARGET_INVALID and out["n_candidates"][0] == 0
    assert out["target"][1] >= 1 and out["n_candidates"][1] > 0
    assert list(out["last_used"]) == [now - 5000] * 2 and list(out["last_unload_time"]) == [0, 0]
    assert rep == report(n_unregister=2, n_reload=1, n_placed=1)


def test_failed_entry_is_deregistered_and_not_reloaded(oracle_lib):
    """model 0: a loaded copy whose entry is a cached failure; model 1: the pod's failure record, its entry failed"""
    fl, out, rep, _ = run([([(POD, OLD)], []), ([(1, OLD)], [(POD, OLD)])], 12,
                          [(0, NOW_MS - 10, OLD, 0, L.EV_ENTRY_FAILED), (1, NOW_MS - 10, 0, OLD, L.EV_ENTRY_FAILED)])
    assert list(out["what"]) == [L.EV_UNREGISTER, L.EV_DROP_FAILURE]
    assert list(out["last_used"]) == [NOW_MS - 10] * 2
    assert list(out["target"]) == [L.TARGET_INVALID] * 2
    assert rep == report(n_unregister=1, n_drop_failure=1)


def test_load_ts_that_does_not_match_writes_nothing_but_still_reloads(oracle_lib):
    lul = [NOW_MS - 7]
    fl, out, rep, _ = run([([(POD, OLD)], [])], 12, [(0, NOW_MS - 10, OLD + 1, OLD, 0)], lul=lul)
    assert out["what"][0] == L.EV_RELOAD | L.EV_PLACED and out["target"][0] >= 1
    assert out["last_used"][0] == NOW_MS - HOUR and out["last_unload_time"][0] == NOW_MS - 7   # the record's own
    assert rep == report(n_reload=1, n_placed=1)


def test_pod_only_in_failed_in_reloads_from_the_failure_time(oracle_lib):
    """model 0: an old failure record; model 1: a failure 2 x timeout ago, too young to reload"""
    young = NOW_MS - 2 * HAND_TIMEOUT
    fl, out, rep, _ = run([([], [(POD, OLD)]), ([], [(POD, young)])], 12, [(0, 0, 5, OLD, 0), (1, 0, 5, young, 0)])
    assert list(out["what"]) == [L.EV_DROP_FAILURE | L.EV_RELOAD | L.EV_PLACED, L.EV_DROP_FAILURE]
    assert list(out["last_used"]) == [NOW_MS] * 2   # updateLastUsed(0) is now
    assert list(out["last_unload_time"]) == [0, 0]  # not unregistered: the record's own
    assert rep == report(n_drop_failure=2, n_reload=1, n_placed=1)


def test_no_registration_of_the_pod(oracle_lib):
    fl, out, rep, _ = run([([(1, OLD)], [(2, OLD)]), ([], [])], 12, [(0, NOW_MS - 10, OLD, OLD, 0), (1, NOW_MS - 10, OLD, OLD, 0)],
                          lul=[NOW_MS - 3, 0])
    assert list(out["what"]) == [0, 0]
    assert list(out["last_used"]) == [NOW_MS - HOUR] * 2 and list(out["last_unload_time"]) == [NOW_MS - 3, 0]
    assert rep == report()


def _rows(cap, free_on=None, free=0):
    """every instance `cap` units with nothing free but instance free_on, which has `free` units free"""
    def edit(fl):
        fl.inst_rows["capacity"] = cap
        fl.inst_rows["used"] = cap
        if free_on is not None:
            fl.inst_rows["used"][free_on] = cap - free
    return edit


def test_rebalance_gate_at_its_edges(oracle_lib):
    regs, row = [([(POD, OLD)], [])], [(0, NOW_MS - 10, OLD, 0, 0)]
    ni, cap = 10, 200_000   # the type set holds 2 000 000 units: a twentieth is 100 000
    _, out, rep, st = run(regs, ni, row, edit=_rows(cap, 3, 100_000))
    assert (int(st["total_capacity"]), int(st["total_free"]), int(st["instance_count"])) == (2_000_000, 100_000, 10)
    assert out["what"][0] == UR | L.EV_PLACED and out["target"][0] == 3
    _, out, rep, st = run(regs, ni, row, edit=_rows(cap, 3, 99_999))
    assert int(st["total_free"]) == 99_999
    assert out["what"][0] == UR | L.EV_CLUSTER_FULL and out["target"][0] == L.TARGET_INVALID
    assert rep == report(n_unregister=1, n_reload=1, n_cluster_full=1)
    _, out, _, st = run(regs, 1, row)
    assert int(st["instance_count"]) == 1 and int(st["total_capacity"]) > 0 and int(st["total_free"]) > 0
    assert out["what"][0] == UR | L.EV_CLUSTER_FULL
    _, out, _, st = run(regs, ni, row, edit=_rows(0))
    assert int(st["total_capacity"]) == 0 and int(st["instance_count"]) == ni
    assert out["what"][0] == UR | L.EV_CLUSTER_FULL


def test_a_live_copy_elsewhere_is_a_forward_and_a_gone_one_is_not(oracle_lib):
    """model 0 has a second copy on instance 1; model 1 on instance 5, which is shutting down (out of the table)"""
    def edit(fl):
        fl.inst_rows["shutting_down"][5] = 1
    fl, out, rep, _ = run([([(POD, OLD), (1, OLD)], []), ([(POD, OLD), (5, OLD)], [])], 12,
                          [(0, NOW_MS - 10, OLD, 0, 0), (1, NOW_MS - 10, OLD, 0, 0)], edit=edit)
    assert list(out["what"]) == [UR | L.EV_LOADED_ELSEWHERE, UR | L.EV_PLACED]
    assert out["target"][0] == L.TARGET_INVALID and out["target"][1] not in (POD, 1, 5) and out["target"][1] >= 0
    assert rep == report(n_unregister=2, n_reload=2, n_loaded_elsewhere=1, n_placed=1)


def test_failure_count_after_the_edit(oracle_lib):
    """models 0 / 1: 2 / 3 recent failures elsewhere; 2: the pod's own recent failure dropped + 2 others; 3: the same + 3
    others; 4: the pod's recent failure not dropped (load_complete_ts differs) + 2 others"""
    f = RECENT_FAIL
    mine = NOW_MS - 200_000   # recent, and old enough to reload
    regs = [([(POD, OLD)], [(2, f), (3, f), (4, f - 1)]),
            ([(POD, OLD)], [(2, f), (3, f), (4, f)]),
            ([], [(POD, mine), (2, f), (3, f)]),
            ([], [(POD, mine), (2, f), (3, f), (4, f)]),
            ([], [(POD, mine), (2, f), (3, f)])]
    rows = [(0, NOW_MS - 10, OLD, 0, 0), (1, NOW_MS - 10, OLD, 0, 0), (2, NOW_MS - 10, 0, mine, 0), (3, NOW_MS - 10, 0, mine, 0),
            (4, NOW_MS - 10, 0, mine + 1, 0)]
    fl, out, rep, _ = run(regs, 20, rows)
    D = L.EV_DROP_FAILURE | L.EV_RELOAD
    assert list(out["what"]) == [UR | L.EV_PLACED, UR | L.EV_REFUSED, D | L.EV_PLACED, D | L.EV_REFUSED, L.EV_RELOAD | L.EV_REFUSED]
    assert out["target"][0] >= 5 and out["target"][2] >= 4
    assert rep == report(n_unregister=2, n_drop_failure=2, n_reload=5, n_refused=3, n_placed=2)


def test_update_last_used_and_last_unload_time(oracle_lib):
    """model 0: lastUsed 0 (now); 1: an older lastUsed than the record's; 2 / 3: 3 / 4 loaded copies, 2 / 3 left; 4: only a
    failure record dropped, lastUnloadTime untouched"""
    young = NOW_MS - 1000   # no reload: the arithmetic alone
    regs = [([(POD, young)], []), ([(POD, young)], []), ([(POD, young), (1, young), (2, young)], []),
            ([(POD, young), (1, young), (2, young), (3, young)], []), ([(1, young), (2, young), (3, young)], [(POD, young)])]
    rows = [(0, 0, young, 0, 0), (1, NOW_MS - 2 * HOUR, young, 0, 0), (2, NOW_MS - 10, young, 0, 0), (3, NOW_MS - 10, young, 0, 0),
            (4, NOW_MS - 10, 0, young, 0)]
    fl, out, rep, _ = run(regs, 12, rows, lul=[5, 5, 5, 5, 5])
    assert list(out["what"]) == [L.EV_UNREGISTER] * 4 + [L.EV_DROP_FAILURE]
    assert list(out["last_used"]) == [NOW_MS, NOW_MS - HOUR, NOW_MS - 10, NOW_MS - 10, NOW_MS - 10]
    assert list(out["last_unload_time"]) == [0, 0, 0, NOW_MS, 5]


def test_registrations_past_the_fourth(oracle_lib):
    """model 0: the pod the sixth loaded copy, the others gone from the table; model 1: 20 registrations, the pod the 17th
    loaded; model 2: 20 registrations, the pod the last failed one"""
    ni = 40
    gone = (1, 2, 3, 4, 5)

    def edit(fl):
        fl.inst_rows["shutting_down"][list(gone)] = 1
    regs = [([(i, OLD) for i in gone] + [(POD, OLD)], []),
            ([(i, OLD) for i in range(6, 22)] + [(POD, OLD)], [(i, OLD) for i in (22, 23, 24)]),
            ([(i, OLD) for i in range(6, 23)], [(23, OLD), (24, OLD), (POD, OLD)])]
    rows = [(0, NOW_MS - 10, OLD, 0, 0), (1, NOW_MS - 10, OLD, 0, 0), (2, NOW_MS - 10, 0, OLD, 0)]
    fl, out, rep, _ = run(regs, ni, rows, edit=edit)
    assert list(out["what"]) == [UR | L.EV_PLACED, UR | L.EV_LOADED_ELSEWHERE, L.EV_DROP_FAILURE | L.EV_RELOAD | L.EV_LOADED_ELSEWHERE]
    assert out["target"][0] >= 6
    assert list(out["last_unload_time"]) == [NOW_MS, NOW_MS, 0]
