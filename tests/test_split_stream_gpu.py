"""The two-pass path's launches at their batch-size and work-list edges: k_place_split's blocks and waves, and
k_place_tail, the persistent launch whose warps take the walk tiles and the overflow decisions from one device-side
counter.  Every batch is placed with the path forced on (split = 1) and off (split = 0), byte for byte, and against the
oracle."""
import ctypes as C

import numpy as np
import pytest

from helpers import oracle_from_synth, oracle_inputs_fast, solver_from_synth
from modelmesh_b200._lib import DECISION_OUT
from modelmesh_b200.synth import make_decisions, make_fleet

pytestmark = pytest.mark.gpu

SEED = 77


def _oracle(fl, sd, o, seed):
    od, off, idx = oracle_inputs_fast(fl, sd)
    return o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=None)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


class _DeviceBatch:
    """The records of a batch in device memory, placed whole (mmp_place_batch_device: no chunks) or by prefix"""

    def __init__(self, s, dec):
        self.s, self.lib = s, s.lib
        dec = np.ascontiguousarray(dec)
        self.n = len(dec)
        self.d_in, self.d_out = C.c_void_p(), C.c_void_p()
        s._ck(self.lib.mmp_device_alloc(s.h, dec.nbytes, C.byref(self.d_in)))
        s._ck(self.lib.mmp_device_alloc(s.h, self.n * DECISION_OUT.itemsize, C.byref(self.d_out)))
        s._ck(self.lib.mmp_device_upload(s.h, self.d_in, dec.ctypes.data_as(C.c_void_p), dec.nbytes))

    def place(self, n, now_ms, split):
        s, lib = self.s, self.lib
        s._ck(lib.mmp_tune(s.h, b"split", split))
        try:
            ms = C.c_float()
            s._ck(lib.mmp_place_batch_device(s.h, self.d_in, n, self.d_out, now_ms, SEED, C.byref(ms)))
        finally:
            s._ck(lib.mmp_tune(s.h, b"split", 2))
        got = np.zeros(n, dtype=DECISION_OUT)
        s._ck(lib.mmp_device_download(s.h, got.ctypes.data_as(C.c_void_p), self.d_out, got.nbytes))
        return got

    def close(self):
        self.s._ck(self.lib.mmp_device_free(self.s.h, self.d_in))
        self.s._ck(self.lib.mmp_device_free(self.s.h, self.d_out))


def _with_edges(fl, edges):
    nm = fl.n_models
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([int(x) for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)
    return fl


def test_split_stream_batch_size_edges(product_lib, oracle_lib):
    """Batch sizes just under, at and just over a full wave of k_place_split's 256-thread blocks (for every count of
    resident blocks per SM), and one tile plus 1, 31 and 33 decisions past several such waves, on a small fleet so the
    2^18+ batches wrap its registry many times."""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    fl = make_fleet("C3", 4000, 2000, 12)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sizes = set()
    for b in range(1, 9):  # resident blocks per SM
        g = sm * b * 256   # decisions in one wave: a tile of 32 per resident warp
        sizes |= {g - 1, g, g + 1}
    for b in (4, 8):
        sizes |= {3 * sm * b * 256 + 32 + r for r in (1, 31, 33)}
    big = max(sizes)
    sd = make_decisions(fl, big, 12, sweep=True, plain=True)
    db = _DeviceBatch(s, sd.dec)
    try:
        off = db.place(big, fl.now_ms, 0)
        _same(off, _oracle(fl, sd, o, SEED), "split = 0 against the oracle")
        for n in sorted(sizes):
            on = db.place(n, fl.now_ms, 1)
            assert on.tobytes() == off[:n].tobytes(), (n, int(np.sum(on != off[:n])))
    finally:
        db.close()
        s.close()


def _work_counter_fleet(kind, seed):
    """kind: "none" (no model has an edge and every self lies at the back of the order: the summaries answer every
    decision), "walk" (the models' edges and the selves sit in the front of the order), "ovf" (every model holds 5-8
    instances) or "both" (overflow models and walked decisions interleaved within every warp's tiles)"""
    fl = make_fleet("C3", 3000, 2000, seed)
    o = oracle_from_synth(fl)
    order = np.asarray(o.cluster_order())
    rng = np.random.default_rng(seed)
    nm = fl.n_models
    front, back = order[:48], order[-600:]
    if kind == "none":
        edges = [[] for _ in range(nm)]
    elif kind == "walk":
        edges = [list(rng.choice(front, size=rng.integers(1, 5), replace=False)) for _ in range(nm)]
    elif kind == "ovf":
        edges = [list(rng.choice(fl.n_instances, size=rng.integers(5, 9), replace=False)) for _ in range(nm)]
    else:
        edges = [list(rng.choice(fl.n_instances, size=rng.integers(5, 9), replace=False)) if m % 3 == 0 else
                 list(rng.choice(front, size=rng.integers(0, 3), replace=False)) for m in range(nm)]
    fl = _with_edges(fl, edges)
    n = (1 << 18) + 45
    sd = make_decisions(fl, n, seed, sweep=True, plain=True)
    if kind == "none":
        sd.dec["self"] = rng.choice(back, size=n)
    elif kind == "walk":
        sd.dec["self"] = rng.choice(front, size=n)
    elif kind == "both":
        sd.dec["self"] = np.where(np.arange(n) % 2 == 0, rng.choice(front, size=n), rng.choice(back, size=n))
    return fl, sd


@pytest.mark.parametrize("kind,seed", [("none", 31), ("walk", 32), ("ovf", 33), ("both", 34)])
def test_split_tail_work_counter(product_lib, oracle_lib, kind, seed):
    """Batches with no walked and no overflow decision, walked decisions only, overflow decisions only, and both
    interleaved in one warp's tiles: k_place_tail's walk tiles and overflow items, taken from one counter."""
    fl, sd = _work_counter_fleet(kind, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    db = _DeviceBatch(s, sd.dec)
    try:
        for n in (db.n, db.n - 13, 8191):
            on, off = db.place(n, fl.now_ms, 1), db.place(n, fl.now_ms, 0)
            assert on.tobytes() == off.tobytes(), (kind, n, int(np.sum(on != off)))
        _same(db.place(db.n, fl.now_ms, 1), _oracle(fl, sd, o, SEED), kind)
    finally:
        db.close()
        s.close()


def test_split_sparse_snapshot_sorted_walk(product_lib, oracle_lib):
    """A C5 batch (sparse candidate sets: the default keeps it on one launch) forced through the two passes: the split
    pass writes the slot-order keys and k_place_tail walks the sorted perm."""
    fl = make_fleet("C5", 20_000, 10_000, 5)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, (1 << 18) + 7, 5, sweep=True, plain=True)
    db = _DeviceBatch(s, sd.dec)
    try:
        on, off = db.place(db.n, fl.now_ms, 1), db.place(db.n, fl.now_ms, 0)
        assert on.tobytes() == off.tobytes(), int(np.sum(on != off))
        _same(on, _oracle(fl, sd, o, SEED), "C5")
    finally:
        db.close()
        s.close()
