"""GPU parity for the batch scans: ClusterStats reductions, reaper selection, per-instance LRU (C ABI vs oracle)."""
import numpy as np
import pytest

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SplitMix, make_fleet
from oracle import binding as ob

from helpers import oracle_from_synth, solver_from_synth
from scan_checks import partition_maps

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 2000, 500, 2), ("C3", 3000, 3000, 3), ("C5", 3000, 2500, 5),
                                               ("MIX", 800, 300, 4), ("MIX", 800, 160, 8)])
def test_stats_match_oracle(product_lib, oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    # one UPDATED event per instance so that every subset's LRU has been recomputed over the final fleet (N10)
    for i in range(fl.n_instances):
        if not fl.inst_rows["shutting_down"][i]:
            r = fl.inst_rows[i].copy()
            r["l_in_prog"] += 1
            o.instance_event(ob.UPDATED, i, r, fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i], fl.now_ms)
            o.instance_event(ob.UPDATED, i, fl.inst_rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i], fl.now_ms)
    s = solver_from_synth(fl, product_lib)
    st, ids = s.stats()
    g = o.cluster_stats()
    for k in ("total_capacity", "total_free", "global_lru", "instance_count", "model_copy_count"):
        assert int(st[0][k]) == int(g[k]), k
    if fl.type_config is None:
        assert len(st) == 1
        return
    pmap = partition_maps(fl, o, s)
    ost, oids = o.partition_stats()
    by_o = {int(i): x for i, x in zip(oids, ost) if x["instance_count"] > 0}
    assert len(st) - 1 == len(by_o)
    for x, pid in zip(st[1:], ids[1:]):
        y = by_o[pmap[int(pid)]]
        for k in ("total_capacity", "total_free", "global_lru", "instance_count", "model_copy_count"):
            assert int(x[k]) == int(y[k]), (k, pid)
    # TCM.getPartitionStats order (TCM:264-271): free desc, lru asc, capacity desc
    keys = [(-int(x["total_free"]), int(x["global_lru"]), -int(x["total_capacity"])) for x in st[1:]]
    assert keys == sorted(keys)


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 20000, 300, 2), ("C3", 30000, 1000, 3), ("C5", 30000, 800, 5),
                                               ("MIX", 5000, 200, 4), ("MIX", 5000, 97, 9), ("MIX", 3000, 64, 21)])
def test_reaper_select_matches_oracle(product_lib, oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    if config == "C5":  # leave some room so that the free-space branch is taken too
        fl.inst_rows["used"][::3] = fl.inst_rows["capacity"][::3] // 2
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    om = np.zeros(nm, dtype=ob.MODEL)
    om["last_used"], om["type_idx"], om["n_loaded"], om["n_failed"] = fl.model_last_used, fl.model_type, fl.n_loaded, fl.n_failed
    if fl.type_config is None:
        a = o.reaper_select(om, fl.type_names, -1, fl.now_ms)
        b = s.reaper_select(-1, fl.now_ms)
        assert len(a) > 0 and np.array_equal(a, b)
        return
    pmap = partition_maps(fl, o, s)
    st, ids = s.stats()
    taken_o = np.zeros(nm, dtype=np.uint8)
    taken_s = np.zeros(nm, dtype=np.uint8)
    total = 0
    for pid in ids[1:]:  # partitions in getPartitionStats order, `taken` carried from one to the next (MM:6473-6489)
        a = o.reaper_select(om, fl.type_names, pmap[int(pid)], fl.now_ms, taken=taken_o)
        b = s.reaper_select(int(pid), fl.now_ms, taken=taken_s)
        assert np.array_equal(a, b), (pid, a[:5], b[:5])
        assert np.array_equal(taken_o, taken_s)
        total += len(a)
    assert total > 0 or config == "MIX"  # some regime-randomised fleets have nothing to load proactively


@pytest.mark.parametrize("seed", range(6))
def test_lru_matches_oracle_cached_oldest_time(product_lib, oracle_lib, seed):
    """evictions, weightedSize(), size() and oldestTime() -- the field CLHM caches, which a setCapacity leaves stale
    (N14) -- against the oracle's LRU after every batch"""
    rng = SplitMix(1000 + seed)
    n_inst, slots = 37, 96
    caps = rng.randint(n_inst, 20_000, 60_000)
    fl = make_fleet("C1", 10, 16, 1)
    s = solver_from_synth(fl, product_lib)
    s.lru_init(caps, slots)
    oracles = [ob.OracleLru(int(c)) for c in caps]
    now = 1_000_000
    n_models = 300
    for batch in range(12):
        n = 900
        ev = np.zeros(n, dtype=L.LRU_EVENT)
        r = rng.uniform(n)
        ev["op"] = np.where(r < 0.45, L_INSERT, np.where(r < 0.75, L_TOUCH, np.where(r < 0.88, L_RESIZE, np.where(r < 0.97, L_REMOVE, L_SETCAP))))
        ev["instance"] = rng.randint(n, 0, n_inst)
        ev["model"] = rng.randint(n, 0, n_models)
        ev["weight"] = rng.randint(n, 1, 9000)
        # coarse timestamps so that equal lastUsed values (the tie rules of LinkedDeque.insert/reposition) are common
        ts = now + (rng.randint(n, -40, 40) * 1000)
        ev["last_used"] = np.where(rng.uniform(n) < 0.2, 0, ts)
        setcap = ev["op"] == L_SETCAP
        ev["last_used"] = np.where(setcap, rng.randint(n, 15_000, 70_000), ev["last_used"])
        got = s.lru_apply(ev, now)
        want = []
        for i in range(n_inst):
            sel = np.nonzero(ev["instance"] == i)[0]
            oe = np.zeros(len(sel), dtype=ob.LRU_EVENT)
            oe["op"] = ev["op"][sel]
            oe["key"] = ev["model"][sel]
            oe["weight"] = np.where(ev["op"][sel] == L_SETCAP, ev["last_used"][sel], ev["weight"][sel])
            oe["last_used"] = np.where(ev["op"][sel] == L_SETCAP, 0, ev["last_used"][sel])
            for x in oracles[i].apply(oe, now):
                want.append((i, int(x["key"]), int(x["last_used"]), int(x["weight"]), int(sel[x["event"]])))
        got_l = [(int(x["instance"]), int(x["model"]), int(x["last_used"]), int(x["weight"]), int(x["event"])) for x in got]
        assert got_l == want, (batch, got_l[:5], want[:5])
        oldest, weighted, count = s.lru_state()
        assert [int(x) for x in weighted] == [o.weighted_size() for o in oracles]
        assert [int(x) for x in count] == [o.size() for o in oracles]
        # oldestTime() as CLHM caches it: stale after a setCapacity's evictions (N14)
        assert [int(x) for x in oldest] == [o.oldest_time() for o in oracles]
        now += 7_000


L_INSERT, L_TOUCH, L_RESIZE, L_REMOVE, L_SETCAP = 0, 1, 2, 3, 4
