"""The two-pass path of large k_place_direct batches (mmp_tune "split"): per-slot summaries, the pass that answers
decisions clear of their slot's reach, the walk over the rest and the one-warp-per-decision pass over models with
overflow ids.  Every batch is placed with the path forced on (split = 1) and off (split = 0) and must equal both the
other path and the oracle, byte for byte."""
import numpy as np
import pytest

from exclude_set import oracle_excluding
from helpers import oracle_from_synth, oracle_inputs_fast, solver_from_synth
from modelmesh_b200._lib import DF_FAVOUR_SELF
from modelmesh_b200.synth import SynthDecisions, make_decisions, make_fleet

pytestmark = pytest.mark.gpu


def _oracle(fl, sd, o, seed, exclude=None):
    if exclude is not None:
        return oracle_excluding(o, fl, sd, exclude, seed)
    od, off, idx = oracle_inputs_fast(fl, sd)
    return o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)


def _kw(sd):
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


def _place(lib, s, fl, sd, seed, split, **kw):
    s._ck(lib.mmp_tune(s.h, b"split", split))
    try:
        return s.place_batch(sd.dec, fl.now_ms, seed, **_kw(sd), **kw)
    finally:
        s._ck(lib.mmp_tune(s.h, b"split", 2))


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def _check(lib, fl, s, o, sd, seed, what, exclude=None):
    kw = {} if exclude is None else dict(exclude=exclude)
    on = _place(lib, s, fl, sd, seed, 1, **kw)
    off = _place(lib, s, fl, sd, seed, 0, **kw)
    assert on.tobytes() == off.tobytes(), (what, int(np.sum(on != off)))
    _same(on, _oracle(fl, sd, o, seed, exclude), what)


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 20_000, 10_000, 3), ("C5", 20_000, 10_000, 5), ("MIX", 6000, 3000, 14),
                                               ("MIX", 6000, 700, 41), ("MIX", 4000, 1500, 7)])
def test_split_equals_walk_and_oracle(product_lib, oracle_lib, config, nm, ni, seed):
    """Plain sweeps (most decisions answered from the summaries) and mixed batches (fresh records, extra excludes,
    favour_self, request-model decisions: most of them walked)."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    _check(product_lib, fl, s, o, make_decisions(fl, 40_000, seed, sweep=True, plain=True), seed, (config, "sweep"))
    _check(product_lib, fl, s, o, make_decisions(fl, 30_000, seed + 1), seed + 2, (config, "mixed"))
    s.close()


def test_split_under_a_call_wide_exclude_set(product_lib, oracle_lib):
    """The summaries come from the call's own view: an exclude set that takes out the front of the order moves every
    slot's best and reach."""
    fl = make_fleet("C3", 8000, 4000, 33)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    order = o.cluster_order()
    sd = make_decisions(fl, 20_000, 33, sweep=True, plain=True)
    for ex in (order[:3], order[[0, 5, 40, 41, 300]], order[:40]):
        _check(product_lib, fl, s, o, sd, 5, ("exclude", len(ex)), exclude=np.asarray(ex, dtype=np.int32))
    s.close()


def test_split_edges_of_the_reach(product_lib, oracle_lib):
    """Decisions whose model's inline edges and self sit at every rank around the front of the order -- best, the
    shortlist, its cut and just past them -- with and without favour_self: the summary's reach must send every one that
    could differ to the walk."""
    fl = make_fleet("C3", 6000, 3000, 21)
    o = oracle_from_synth(fl)
    order = o.cluster_order()
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
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 30_000, 21, sweep=True, plain=True)
    sd.dec["self"] = rng.choice(np.concatenate([front, order[:8]]), size=len(sd.dec))
    _check(product_lib, fl, s, o, sd, 21, "front")
    sd.dec["flags"] |= DF_FAVOUR_SELF
    _check(product_lib, fl, s, o, sd, 22, "front, favour_self")
    s.close()


def test_split_batches_of_overflow_models_and_sizes(product_lib, oracle_lib):
    """A fleet where every model holds 5-8 instances (every decision goes to the one-warp-per-decision pass), and batch
    sizes around warp, block and the default threshold of the path."""
    fl = make_fleet("C3", 3000, 2000, 8)
    rng = np.random.default_rng(8)
    nm = fl.n_models
    edges = [list(rng.choice(fl.n_instances, size=rng.integers(5, 9), replace=False)) for _ in range(nm)]
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([int(x) for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    _check(product_lib, fl, s, o, make_decisions(fl, 9000, 8, sweep=True, plain=True), 8, "all overflow")
    s.close()
    fl = make_fleet("C3", 300_000, 2500, 9)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, (1 << 18) + 33, 9, sweep=True, plain=True)
    for n in (1000, 1025, 8191, (1 << 17) + 1, (1 << 18) - 1, (1 << 18) + 33):
        part = SynthDecisions(sd.dec[:n], sd.fresh, sd.extra)
        on, off = _place(product_lib, s, fl, part, 9, 1), _place(product_lib, s, fl, part, 9, 0)
        dflt = s.place_batch(part.dec, fl.now_ms, 9)
        assert on.tobytes() == off.tobytes() == dflt.tobytes(), n
    _same(dflt, _oracle(fl, sd, o, 9), "threshold")
    s.close()
