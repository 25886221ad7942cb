"""The oracle composition of the janitor's registry loop (tests/janitor_run_oracle.py), checked without a GPU:
  * on hand-built records with known answers: failure expiry at and one past its age, the in-use expiry at now - lastUsed of
    179 999 and 180 000, a failure without an entry, a failed entry on a loaded registration, equal-lastUsed candidates (N15),
    the budget (a first removal over it allowed, a later heavy one refused, a later light one allowed), a registration time
    that is not the entry's loadTimestamp, and Long.MAX_VALUE as an entry's lastUsed;
  * its removeModelCopies part (orc_janitor_eval) against brute_janitor_entry of tests/brute.py."""
import numpy as np

import janitor_run_oracle as jro
from common import EXPIRY, HOUR, LONG_MAX
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import make_fleet
from pod_task_edges import janitor_hand_fleet as hand_fleet
from pod_tasks import janitor_params
from brute import brute_janitor_entry

def entry(model, last_used, weight=10, load_ts=0, failed=False, last_heavy=0, count=0):
    e = np.zeros(1, dtype=L.JANITOR_ENTRY)
    e["model"], e["weight"], e["last_used"], e["load_ts"], e["flags"] = model, weight, last_used, load_ts, L.JANITOR_FAILED if failed else 0
    e["last_heavy"], e["count"] = last_heavy, count
    return e


def known_case():
    """(fleet, times, lastUnloadTime, self, entries, the oracle fleet): model k of the records below"""
    fl0 = make_fleet("C3", 1, 24, 3)
    fl0.inst_rows["used"] = fl0.inst_rows["capacity"] - fl0.inst_rows["capacity"] // 50
    o0 = oracle_from_synth(fl0)
    order = [int(x) for x in o0.cluster_order()]
    o0.close()
    S, A, B, C = order[-1], order[0], order[1], order[2]  # self is the least desirable pod: it drops the second copies
    now = fl0.now_ms
    old = now - 2 * HOUR
    regs = [
        ([], [(S, now - EXPIRY)]),                       # 0  failure at exactly the expiry, no entry: kept
        ([], [(S, now - EXPIRY - 1)]),                   # 1  one past it, no entry: dropped
        ([], [(S, now - EXPIRY // 2 - 1)]),              # 2  failed entry used 179 999 ms ago: the in-use expiry, dropped + local
        ([], [(S, now - EXPIRY // 2 - 1)]),              # 3  ... used 180 000 ms ago: the full expiry, kept
        ([(A, old), (S, old)], []),                      # 4  failed entry on a loaded registration: unregistered, lul 0
        ([(A, old), (B, old), (C, old), (S, old)], []),  # 5  loaded, no entry: unregistered, three remain: lul = now
        ([(A, old), (S, old + 6)], []),                  # 6  candidate at lastUsed T ...
        ([(A, old), (S, old + 7)], []),                  # 7  ... and another at T: dropped by the TreeSet (N15)
        ([(A, old), (S, old + 8)], []),                  # 8  load_ts mismatch: not removed, not counted
        ([(A, old), (S, old + 9)], []),                  # 9  first removal, weight 60
        ([(A, old), (S, old + 10)], []),                 # 10 heavy (50): over what is left of the budget
        ([(A, old), (S, old + 11)], []),                 # 11 light (30): within it
        ([(A, old), (S, old + 12)], [(S, now - 1000)]),  # 12 Long.MAX_VALUE lastUsed, and a fresh failure beside the copy
        ([(A, old), (S, old + 13)], []),                 # 13 not in the pod's cache at all
    ]
    fl, ts = hand_fleet(regs)
    lul = np.zeros(fl.n_models, dtype=np.int64)
    T = now - 50_000
    ents = np.concatenate([
        entry(2, now - 179_999, failed=True), entry(3, now - 180_000, failed=True), entry(4, now - 5000, failed=True),
        entry(6, T, weight=5, load_ts=old + 6), entry(7, T, weight=5, load_ts=old + 7),
        entry(8, now - 40_000, weight=10, load_ts=old + 1), entry(9, now - 30_000, weight=60, load_ts=old + 9),
        entry(10, now - 20_000, weight=50, load_ts=old + 10), entry(11, now - 10_000, weight=30, load_ts=old + 11),
        entry(12, LONG_MAX, weight=5, load_ts=old + 12)])
    return fl, ts, lul, S, ents, oracle_from_synth(fl)


def test_known_answers(oracle_lib):
    fl, ts, lul, S, ents, o = known_case()
    now = fl.now_ms
    rec_lu = now - HOUR
    # budget 100: model 6 (5, first removal), 9 (60), 10 refused (50 > 35), 11 (30)
    edits, rep = jro.janitor_run(o, fl, ts, lul, S, ents, janitor_params(now, 2000))
    got = {m: (w, lu, ul) for m, w, lu, ul in edits}
    assert got[1] == (L.JE_DROP_FAILURE, rec_lu, 0)
    assert got[2] == (L.JE_DROP_FAILURE | L.JE_REMOVE_LOCAL, now - 179_999, 0)
    assert got[4] == (L.JE_UNREGISTER, now - 5000, 0)
    assert got[5] == (L.JE_UNREGISTER, rec_lu, now)
    assert got[6] == (L.JE_SCALE_DOWN, now - 50_000, 0)
    assert got[9] == (L.JE_SCALE_DOWN, now - 30_000, 0) and got[11] == (L.JE_SCALE_DOWN, now - 10_000, 0)
    assert got[12] == (L.JE_DROP_FAILURE, LONG_MAX, 0)   # the entry is present and not failed: its failure record goes
    assert got[13] == (L.JE_UNREGISTER, rec_lu, 0)
    assert set(got) == {1, 2, 4, 5, 6, 9, 11, 12, 13}   # 0, 3 kept; 7 dropped by N15; 8 load_ts; 10 over the budget
    assert rep == dict(n_referencing=14, n_edits=9, n_candidates=6, n_removed=3, weight_removed=95)
    # budget 50: model 6 (5), then 9 (60 > 45) refused, 10 (50) refused, 11 (30) allowed
    edits, rep = jro.janitor_run(o, fl, ts, lul, S, ents, janitor_params(now, 1000))
    assert [m for m, w, _, _ in edits if w & L.JE_SCALE_DOWN] == [6, 11] and rep["weight_removed"] == 35
    # without models 6 and 7 the first removal (60) exceeds the budget of 50 and is allowed; nothing fits after it
    edits, rep = jro.janitor_run(o, fl, ts, lul, S, ents[~np.isin(ents["model"], [6, 7])], janitor_params(now, 1000))
    assert [m for m, w, _, _ in edits if w & L.JE_SCALE_DOWN] == [9] and rep["n_removed"] == 1
    # every candidate removable but the mismatched load_ts with the budget out of the way
    assert jro.remove_model_copies(o, fl, ts, lul, S, 8, ents[ents["model"] == 8][0], janitor_params(now, 1000)[0], 1) == 1
    assert jro.remove_model_copies(o, fl, ts, lul, S, 7, ents[ents["model"] == 7][0], janitor_params(now, 1000)[0], 1) == 1
    assert jro.remove_model_copies(o, fl, ts, lul, S, 12, ents[ents["model"] == 12][0], janitor_params(now, 1000)[0], 1) == 0
    o.close()


def test_remove_model_copies_matches_brute_force(oracle_lib):
    rng = np.random.default_rng(7)
    fl = make_fleet("C3", 1500, 120, 7)
    fl.inst_rows["used"] = fl.inst_rows["capacity"] - fl.inst_rows["capacity"] // 50
    ts = np.where(rng.uniform(size=len(fl.edge_inst)) < 0.3, fl.now_ms - rng.integers(0, 120_000, size=len(fl.edge_inst)),
                  fl.now_ms - rng.integers(0, 4 * HOUR, size=len(fl.edge_inst))).astype(np.int64)
    lul = np.where(rng.uniform(size=fl.n_models) < 0.3, fl.now_ms - rng.integers(0, 200_000, size=fl.n_models), 0).astype(np.int64)
    o = oracle_from_synth(fl)
    order = [int(x) for x in o.cluster_order()]
    pos = {i: k for k, i in enumerate(order)}
    for i in range(fl.n_instances):
        pos.setdefault(i, 1 << 30)
    st = o.cluster_stats()
    gst = {k: int(st[k]) for k in ("total_capacity", "total_free", "global_lru")}
    sd = [bool(x) for x in fl.inst_rows["shutting_down"]]
    have_tc = fl.type_config is not None
    ps, pids = o.partition_stats()
    pst = {int(pid): {k: int(x[k]) for k in gst} for x, pid in zip(ps, pids)}
    n = removed = 0
    for S in range(fl.n_instances):
        S = int(S)
        local = pst.get(o.instance_partition(S)) if have_tc else gst   # instanceSetStats() of the pod
        p = janitor_params(fl.now_ms, 10_000)[0]
        p["scale"]["second_copy_remove_max_age_ms"] = 36 * HOUR
        for m in range(fl.n_models):
            a, k = int(fl.edge_off[m]), int(fl.n_loaded[m])
            loaded = [(int(fl.edge_inst[q]), int(ts[q])) for q in range(a, a + k)]
            if S not in [i for i, _ in loaded]:
                continue
            ce = entry(m, fl.now_ms - int(rng.integers(1, 40 * HOUR)), last_heavy=int(rng.choice([0, fl.now_ms - int(rng.integers(0, 30 * HOUR))])),
                       count=int(rng.integers(0, 50)))[0]
            for can in (0, 1):
                e = dict(instance=S, last_used=int(ce["last_used"]), last_heavy=int(ce["last_heavy"]), count=int(ce["count"]))
                pd = {k2: int(p["scale"][k2]) for k2 in ("now", "last_check_time", "scale_up_rpm_threshold", "rate_check_interval_ms",
                                                          "second_copy_remove_max_age_ms")}
                pd["can_remove"] = can
                want = brute_janitor_entry(e, pd, have_tc, local, loaded, int(lul[m]), fl.inst_ids, sd, pos)
                got = jro.remove_model_copies(o, fl, ts, lul, S, m, ce, p, can)
                assert got == want, (S, m, can, got, want)
                n += 1
                removed += got
    assert n > 200 and removed > 10, (n, removed)
    o.close()
