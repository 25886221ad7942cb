"""The oracle composition of the leader's reaper task (tests/reaper_run_oracle.py), checked without a GPU:
  * without anything to prune or repair it selects what the closed-loop oracle's REAPER event decides
    (tests/emul/reaper_sim.cpp), with and without type constraints, on free and full fleets;
  * its prune, repair, candidates and `missings` cleanup equal a plain restatement of pruneModelRegistry's loop body
    (MM:6536-6590, pruneMissingInstances MM:6752-6784) on small fleets with pods gone."""
import numpy as np
import pytest

import reaper_run_oracle as rro
from helpers import oracle_from_synth
from oracle import binding as ob
from churn_harness import with_failed
from common import GONE_MS
from modelmesh_b200.synth import make_churn
from reaper_oracle import _reaper_oracle_so, reaper_event, reaper_oracle, reaper_sim  # noqa: F401


@pytest.mark.usefixtures("reaper_oracle")
@pytest.mark.parametrize("with_types,fill,seed", [(False, 0.5, 31), (True, 0.5, 32), (False, 0.9, 33), (True, 0.97, 34)])
def test_composition_selects_what_the_reaper_event_decides(oracle_lib, with_types, fill, seed):
    w = make_churn(6000, 48, seed, fill=fill, with_types=with_types)
    fl = w.fleet
    o, sim = reaper_sim(w)
    t = fl.now_ms + 500
    missing = np.zeros(fl.n_instances, dtype=np.int64)
    got = rro.reaper_run(o, fl, np.full(len(fl.edge_inst), fl.now_ms - rro.HOUR, dtype=np.int64), 5, t, GONE_MS, missing,
                         np.ones(fl.n_instances, dtype=bool), seed)  # (before the window: the sim's step changes the fleet)
    dec, _, _, _, _ = sim.step(reaper_event(5, t), fl.now_ms, fl.now_ms + w.window_ms, seed)
    want = [int(m) for m in dec["model"][dec["event"] == 0]]
    assert not got["pairs"] and not got["repaired"] and got["stopped"] == -1
    assert [m for m, _, _, _ in got["loads"]] == want
    assert len(want) > 10
    assert all(lu == int(fl.model_last_used[m]) for m, _, _, lu in got["loads"])


def _restated(fl, ts, present, leader, now, gone_ms, missings: dict, last_used, global_lru):
    """pruneModelRegistry's loop body per record (MM:6553-6578) over dict records, then the cleanup (MM:6601-6607)"""
    pairs, repaired, cands = [], [], []
    not_found = set()
    for m in range(fl.n_models):
        a, k, b = int(fl.edge_off[m]), int(fl.n_loaded[m]), int(fl.edge_off[m + 1])
        insts = {int(fl.edge_inst[j]): int(ts[j]) for j in range(a, a + k)}
        fail_insts = {int(fl.edge_inst[j]): int(ts[j]) for j in range(a + k, b)}
        for mp in (insts, fail_insts):  # pruneMissingInstances
            for iid, t in list(mp.items()):
                if now - t < gone_ms or iid == leader:
                    continue
                if iid not in not_found:
                    if present[iid]:
                        continue
                    not_found.add(iid)
                since = missings.setdefault(iid, now) if iid not in missings else missings[iid]
                if iid in missings and since != now and now - since > gone_ms:
                    del mp[iid]
                    pairs.append((m, iid))
        lu = int(last_used[m])
        if lu == rro.LONG_MAX:  # repairLastUsedTimeIfNeeded
            lu = now - rro.REPAIR_AGE_MS
            repaired.append(m)
        if not insts and len(fail_insts) < 2 and (global_lru == 0 or lu > global_lru):
            cands.append(m)
    for iid in [i for i, v in missings.items() if now - v > gone_ms or present[i]]:
        del missings[iid]
    return pairs, repaired, cands


@pytest.mark.parametrize("seed", [41, 42, 43])
def test_composition_prunes_as_the_reference_loop(oracle_lib, seed):
    w = make_churn(3000, 40, seed, fill=0.5)
    w = with_failed(w, {int(m): 2 for m in w.unloaded_models[:200]})  # failed loads on instances 0 and 1
    fl = w.fleet
    rng = np.random.default_rng(seed)
    fl.model_last_used[rng.choice(fl.n_models, size=30, replace=False)] = rro.LONG_MAX
    o = oracle_from_synth(fl, bulk=False)
    gone = np.asarray([0, 1] + list(rng.choice(np.arange(2, 40), size=5, replace=False)))
    for i in gone:
        o.instance_event(ob.DELETED, int(i), None, fl.inst_ids[int(i)], now_ms=fl.now_ms)
    present = ~np.isin(np.arange(fl.n_instances), gone)
    leader = int(gone[-1])  # the leader's own registrations: never pruned, though its pod is gone from the table
    ts = np.where(rng.uniform(size=len(fl.edge_inst)) < 0.3, fl.now_ms - rng.integers(0, GONE_MS, size=len(fl.edge_inst)),
                  fl.now_ms - rng.integers(GONE_MS, 4 * rro.HOUR, size=len(fl.edge_inst))).astype(np.int64)
    missing = np.zeros(fl.n_instances, dtype=np.int64)
    missing[gone[:4]] = fl.now_ms - 660_000     # first seen missing 11 minutes ago
    missing[gone[4]] = fl.now_ms - 60_000       # ... one minute ago
    missing[np.nonzero(present)[0][:3]] = fl.now_ms - 900_000  # stale entries of instances back in the table
    now = fl.now_ms
    ref = {int(i): int(v) for i, v in enumerate(missing) if v}
    pr = rro.prune(o, fl, ts, leader, now, GONE_MS, missing)
    lu, repaired = rro.repair(fl.model_last_used, now)
    rro.cleanup(missing, present, now, GONE_MS)
    cs = o.cluster_stats()
    glru = 0 if cs["total_free"] > 0 else int(cs["global_lru"])
    pairs, rep, cands = _restated(fl, ts, present, leader, now, GONE_MS, ref, fl.model_last_used, glru)
    assert pr.pairs == pairs and repaired == rep and len(pairs) > 20 and len(rep) == 30
    assert {i: int(v) for i, v in enumerate(missing) if v} == ref
    mine = [m for m in range(fl.n_models) if pr.n_loaded[m] == 0 and pr.n_failed[m] < 2 and (glru == 0 or lu[m] > glru)]
    assert mine == cands
    assert not any(i == leader for _, i in pairs)
    # pruning made candidates: models whose only copies, or one of two failed loads, were on gone pods
    assert any(fl.n_loaded[m] > 0 for m in cands) and any(fl.n_failed[m] == 2 for m in cands)
