"""k_place_direct launch shapes against the oracle: sweeps and mixed batches on C3 and C5, batch sizes around the warp,
block and slot-sort edges with and without the slot sort, and an overflow-heavy fleet whose inline edges sit at the word
edges and the edge of the 12-word window, decided by pods that hold the model beyond that window (self's word from
RowRanks)."""
import numpy as np
import pytest

from helpers import compare_decisions, oracle_from_synth, oracle_inputs_fast, solver_from_synth
from modelmesh_b200.synth import SynthDecisions, make_decisions, make_fleet

pytestmark = pytest.mark.gpu


def _oracle(fl, sd, o, seed):
    od, off, idx = oracle_inputs_fast(fl, sd)
    return o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def _kw(sd):
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


@pytest.mark.parametrize("config,seed", [("C3", 3), ("C5", 5)])
def test_sweep_and_mixed_batches_match_oracle(product_lib, oracle_lib, config, seed):
    fl = make_fleet(config, 3000, 10_000, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    for sd in (make_decisions(fl, 20_000, seed, sweep=True, plain=True), make_decisions(fl, 20_000, seed + 1)):
        _same(s.place_batch(sd.dec, fl.now_ms, seed, **_kw(sd)), _oracle(fl, sd, o, seed), config)
    s.close()


def test_batch_sizes_at_warp_block_and_sort_edges(product_lib, oracle_lib):
    fl = make_fleet("C5", 4000, 10_000, 37)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 8193, 37)
    want = _oracle(fl, sd, o, 9)
    for sort in (0, 1):
        s._ck(product_lib.mmp_tune(s.h, b"sort_slots", sort))
        for n in (1, 31, 33, 127, 129, 8191, 8192, 8193):
            part = SynthDecisions(sd.dec[:n], sd.fresh, sd.extra)
            _same(s.place_batch(part.dec, fl.now_ms, 9, **_kw(part)), want[:n], (sort, n))
    s._ck(product_lib.mmp_tune(s.h, b"sort_slots", 2))


def _overflow_heavy(ni: int, nm: int, seed: int):
    """C3 with about a quarter of the models holding 5-12 instances; the first (inline) edges of every model are the
    instances at ranks 0, 31, 32 (word edge), 383, 384, 385 (edge of the 12-word window) and n_ranks-1."""
    fl = make_fleet("C3", nm, ni, seed)
    # the placement order depends on the instance rows only: take it from the oracle
    order = oracle_from_synth(fl).cluster_order()
    nr = len(order)
    special = order[[0, 31, 32, 383, 384, 385, nr - 1]]
    rng = np.random.default_rng(seed)
    deg = np.where(rng.uniform(size=nm) < 0.25, rng.integers(5, 13, size=nm), rng.integers(0, 5, size=nm))
    edges = []
    for m in range(nm):
        inl = list(rng.choice(special, size=min(4, deg[m]), replace=False))
        rest = [int(x) for x in rng.choice(ni, size=deg[m] + 8, replace=False) if x not in inl][:max(0, deg[m] - 4)]
        edges.append([int(x) for x in inl] + rest)
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([x for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    return fl, order, edges


def test_overflow_heavy_fleet_at_word_and_window_edges(product_lib, oracle_lib):
    fl, order, edges = _overflow_heavy(10_000, 6000, 41)
    rank = np.full(fl.n_instances, -1, dtype=np.int64)
    rank[order] = np.arange(len(order))
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    assert np.array_equal(s.cluster_order(), order)
    assert np.mean([len(e) > 4 for e in edges]) > 0.2
    # decisions by a pod that holds the model beyond the window (ranks 384, 385, n_ranks-1), and ordinary ones
    rng = np.random.default_rng(41)
    sd = make_decisions(fl, 12_000, 41)
    held = [(m, i) for m, e in enumerate(edges) for i in e[:4] if rank[i] >= 384]
    pick = rng.choice(len(held), size=6000, replace=False)
    sd.dec["model"][:6000] = [held[k][0] for k in pick]
    sd.dec["self"][:6000] = [held[k][1] for k in pick]
    sd.dec["fresh"][:6000] = -1
    assert (rank[sd.dec["self"]] >= 0).all()
    for sort in (0, 1):
        s._ck(product_lib.mmp_tune(s.h, b"sort_slots", sort))
        _same(s.place_batch(sd.dec, fl.now_ms, 3, **_kw(sd)), _oracle(fl, sd, o, 3), ("overflow-heavy", sort))
    s._ck(product_lib.mmp_tune(s.h, b"sort_slots", 2))
    sweep = make_decisions(fl, fl.n_models, 42, sweep=True, plain=True)
    _same(s.place_batch(sweep.dec, fl.now_ms, 4), _oracle(fl, sweep, o, 4), "overflow-heavy sweep")
    small = SynthDecisions(sd.dec[:1500], sd.fresh, sd.extra)
    compare_decisions(fl, small, o, s, seed=6, full_lists=False)
