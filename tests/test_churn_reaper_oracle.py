"""The reaper's proactive loads in the oracle's closed loop (the REAPER event of tests/emul/reaper_sim.cpp, which steps
oracle/mm_sim.inc's loop with it), without a GPU:
  * a window's REAPER decisions are the concatenation of orc_reaper_select over the partitions in getPartitionStats order
    with one `taken` set (the whole cluster without type constraints), read from the registry and fleet of the window's start;
  * the closed loop's invariants (registry == caches, capacities) hold after every window of traces with REAPER events."""
import numpy as np
import pytest

from helpers import oracle_from_synth
from modelmesh_b200._lib import CHURN_REAPER
from modelmesh_b200.synth import make_churn
from oracle import binding as ob
from reaper_oracle import _reaper_oracle_so, reaper_oracle, with_reaper  # noqa: F401

pytestmark = pytest.mark.usefixtures("reaper_oracle")


def _sim(w):
    fl = w.fleet
    o = oracle_from_synth(fl, bulk=False)
    models = np.zeros(fl.n_models, dtype=ob.SIM_MODEL)
    models["last_used"], models["type_idx"], models["size_units"] = fl.model_last_used, fl.model_type, fl.model_size
    sim = with_reaper(ob.OracleSim(o, models, fl.type_names, fl.edge_off, fl.edge_inst, fl.n_loaded, w.capacity, w.load_timeout_ms,
                                   fl.now_ms - 60_000), fl.n_models)
    order = np.argsort(w.seed_instance, kind="stable")
    bounds = np.searchsorted(w.seed_instance[order], np.arange(fl.n_instances + 1))
    for i in range(fl.n_instances):
        sel = order[bounds[i]:bounds[i + 1]]
        if len(sel):
            sim.seed(i, w.seed_model[sel], w.seed_last_used[sel], w.seed_weight[sel], w.seed_load_ts[sel], fl.now_ms)
    return o, sim


def reaper_event(caller: int, t: int) -> np.ndarray:
    e = np.zeros(1, dtype=ob.SIM_EVENT)
    e["type"], e["caller"], e["t"] = CHURN_REAPER, caller, t
    return e


def expected_selection(o, sim, fl, t):
    """orc_reaper_select partition by partition over the sim's registry as it stands"""
    om = np.zeros(fl.n_models, dtype=ob.MODEL)
    for m in range(fl.n_models):
        copies, lu = sim.model_copies(m)
        om[m]["n_loaded"], om[m]["last_used"] = len(copies), lu
    om["type_idx"], om["n_failed"] = fl.model_type, fl.n_failed
    parts = [-1] if fl.type_config is None else [int(p) for p in o.partition_stats()[1]]
    taken = np.zeros(fl.n_models, dtype=np.uint8)
    sel = []
    for p in parts:
        sel += [int(x) for x in o.reaper_select(om, fl.type_names, p, t, taken=taken)]
    return sel


@pytest.mark.parametrize("with_types,fill,seed", [(False, 0.5, 3), (True, 0.5, 4), (False, 0.9, 5), (True, 0.9, 6)])
def test_sim_reaper_decisions_are_the_partition_selections(oracle_lib, with_types, fill, seed):
    w = make_churn(6000, 48, seed, fill=fill, with_types=with_types)
    fl = w.fleet
    o, sim = _sim(w)
    picked = 0
    for ep in range(3):
        now0 = fl.now_ms + ep * w.window_ms
        t = now0 + 700
        want = expected_selection(o, sim, fl, t)
        ev = reaper_event(5 + ep, t)
        if ep == 2:  # behind a window of ordinary traffic: only first decisions of a model count
            ev = np.concatenate([w.events(ep, 600, seed).astype(ob.SIM_EVENT), ev])
        before = sim.coalesced()
        dec, _, _, _, _ = sim.step(ev, now0, now0 + w.window_ms, 100 + ep)
        mine = dec[dec["event"] == len(ev) - 1]
        assert np.all(mine["self"] == 5 + ep)
        decided_before = set(int(m) for m in dec["model"][dec["event"] != len(ev) - 1])
        assert [int(m) for m in mine["model"]] == [m for m in want if m not in decided_before], ep
        assert sim.coalesced() - before >= sum(m in decided_before for m in want)
        picked += len(mine)
    assert picked > 20, picked


@pytest.mark.parametrize("with_types,fill,seed", [(False, 0.6, 4), (True, 0.9, 5), (False, 0.99, 6)])
def test_closed_loop_with_reaper_conserves_copies_and_capacity(oracle_lib, with_types, fill, seed):
    w = make_churn(8000, 60, seed, fill=fill, with_types=with_types)
    fl = w.fleet
    o, sim = _sim(w)
    accepted = 0
    for ep in range(6):
        now0 = fl.now_ms + ep * w.window_ms
        ev = w.events(ep, 1200, seed).astype(ob.SIM_EVENT)
        ev = np.concatenate([ev[:400], reaper_event(ep, now0 + 900), ev[400:]] + ([reaper_event(1, now0 + 1500)] if ep % 2 else []))
        before = {m: set(int(x) for x in sim.model_copies(m)[0]) for m in range(fl.n_models)}
        dec, evi, rows, npub, carry = sim.step(ev, now0, now0 + w.window_ms, 400 + ep)
        after = {m: set(int(x) for x in sim.model_copies(m)[0]) for m in range(fl.n_models)}
        resident = sum(sim.lru_state(i)[2] for i in range(fl.n_instances))
        assert resident == sum(len(v) for v in after.values()), ep
        for i in range(fl.n_instances):
            assert sim.lru_state(i)[1] <= int(w.capacity[i]), (ep, i)
        for d in dec[dec["status"] == ob.SIM_ACCEPTED]:
            t = int(d["self"]) if int(d["target"]) == ob.SELF else int(d["target"])
            assert 0 <= t < fl.n_instances and t not in before[int(d["model"])], (ep, d)
        reaper = dec[np.isin(dec["event"], np.nonzero(ev["type"] == CHURN_REAPER)[0])]
        assert len(set(int(m) for m in dec["model"][dec["status"] != ob.SIM_SKIPPED])) == np.count_nonzero(dec["status"] != ob.SIM_SKIPPED)
        accepted += int(np.count_nonzero(reaper["status"] == ob.SIM_ACCEPTED))
    if fill < 0.95:
        assert accepted > 0


def test_reaper_step_without_reaper_events_is_the_oracle_step(oracle_lib):
    """orc_sim_step_reaper restates orc_sim_step: on a trace without REAPER events the two sims report the same"""
    w = make_churn(6000, 48, 7, fill=0.9, with_types=True)
    fl = w.fleet
    _, a = _sim(w)
    o = oracle_from_synth(fl, bulk=False)
    models = np.zeros(fl.n_models, dtype=ob.SIM_MODEL)
    models["last_used"], models["type_idx"], models["size_units"] = fl.model_last_used, fl.model_type, fl.model_size
    b = ob.OracleSim(o, models, fl.type_names, fl.edge_off, fl.edge_inst, fl.n_loaded, w.capacity, w.load_timeout_ms, fl.now_ms - 60_000)
    order = np.argsort(w.seed_instance, kind="stable")
    bounds = np.searchsorted(w.seed_instance[order], np.arange(fl.n_instances + 1))
    for i in range(fl.n_instances):
        sel = order[bounds[i]:bounds[i + 1]]
        if len(sel):
            b.seed(i, w.seed_model[sel], w.seed_last_used[sel], w.seed_weight[sel], w.seed_load_ts[sel], fl.now_ms)
    for ep in range(5):
        now0 = fl.now_ms + ep * w.window_ms
        ev = w.events(ep, 1000, 7)
        ra, rb = a.step(ev, now0, now0 + w.window_ms, 50 + ep), b.step(ev, now0, now0 + w.window_ms, 50 + ep)
        for x, y in zip(ra[:3], rb[:3]):
            assert all(np.array_equal(x[k], y[k]) for k in x.dtype.names), ep
        assert ra[3:] == rb[3:] and a.coalesced() == b.coalesced()
