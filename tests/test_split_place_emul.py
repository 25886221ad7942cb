"""CPU checks of the two-pass placement path: the per-slot summaries (slot_summary, both values of c_self) and the
answer they give a decision clear of its slot's reach (split_answer), compiled by g++ from place_core.cuh.

The tests/emul/split_place.cpp harness resolves a batch as k_place_direct does, then answers from the summaries every
decision k_place_split would answer, and counts the answers that differ from the walk."""
import numpy as np
import pytest

from modelmesh_b200._lib import DF_FAVOUR_SELF
from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import oracle_from_synth, solver_from_synth
from split_place import oracle_same, place_split, split_lib  # noqa: F401  (split_lib: module fixture)


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 3000, 1300, 33), ("C5", 1500, 500, 5), ("MIX", 800, 300, 14),
                                               ("MIX", 800, 700, 41), ("C2", 2000, 400, 2)])
def test_summary_answers_equal_the_walk(split_lib, oracle_lib, config, nm, ni, seed):
    """Plain sweeps (most decisions answered from the summaries), favour_self sweeps, and mixed batches (fresh records,
    extras, request-model decisions): every answer from a summary equals the decision's walk, and the walk the oracle."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, split_lib)
    sweep = make_decisions(fl, 3000, seed, sweep=True, plain=True)
    fav = make_decisions(fl, 2000, seed + 3, sweep=True, plain=True)
    fav.dec["flags"] |= DF_FAVOUR_SELF
    answered = 0
    for k, sd in enumerate((sweep, fav, make_decisions(fl, 2000, seed + 1))):
        out, counts = place_split(split_lib, s, sd, fl.now_ms, seed + k)
        assert counts[1] == 0, (config, k, counts)
        oracle_same(o, fl, sd, out, seed + k)
        answered += counts[0]
    assert answered > 0
    s.close()


def test_reach_edges_on_a_front_loaded_fleet(split_lib, oracle_lib):
    """Every model's inline edges and every self among the first 64 ranks: exclusions and selves at, just before and just
    past best, the shortlist and its cut."""
    fl = make_fleet("C3", 3000, 1500, 21)
    order = oracle_from_synth(fl).cluster_order()
    rng = np.random.default_rng(21)
    nm = fl.n_models
    front = order[:64]
    edges = [list(rng.choice(front, size=rng.integers(0, 5), replace=False)) for _ in range(nm)]
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([int(x) for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, split_lib)
    sd = make_decisions(fl, 3000, 21, sweep=True, plain=True)
    sd.dec["self"] = rng.choice(front, size=len(sd.dec))
    for k in range(2):
        out, counts = place_split(split_lib, s, sd, fl.now_ms, 21 + k)
        assert counts[1] == 0, counts
        oracle_same(o, fl, sd, out, 21 + k)
        sd.dec["flags"] |= DF_FAVOUR_SELF
    s.close()
