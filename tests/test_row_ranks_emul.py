"""CPU checks of k_place_direct's row access: decide_stream reading a decision's exclusion row through RowRanks, the
model's excluded ranks (SnapshotView::excl_ranks), instead of through its bitmap row.

The tests/emul/row_ranks.cpp harness resolves a batch as the kernel does (window, self's row word and every word beyond
the window from the ranks; models with overflow ids and whatever the lane routine declines go to the general routine on
the bitmap row), walks every decision the ranks resolve through the bitmap row as well, and counts disagreements.
"""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from modelmesh_b200 import _lib
from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import oracle_from_synth, oracle_inputs, solver_from_synth

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def ranks_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("row_ranks") / "libmmplace_emul_ranks.so")
    subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wl,-Bsymbolic", "-shared", "-o", so,
                           os.path.join(HERE, "emul", "row_ranks.cpp")])
    lib = _lib.load(so, require_all=False)
    lib.mmp_emul_place_ranks.restype = C.c_int32
    lib.mmp_emul_place_ranks.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32,
                                         C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_uint64, C.c_void_p]
    return lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def place_ranks(lib, s, sd, now_ms, seed, window, budget):
    dec = np.ascontiguousarray(sd.dec, dtype=_lib.DECISION_IN)
    fresh = np.ascontiguousarray(sd.fresh, dtype=_lib.INSTANCE_ROW) if len(sd.fresh) else None
    extra = np.ascontiguousarray(sd.extra, dtype=np.int32) if len(sd.extra) else None
    out = np.zeros(len(dec), dtype=_lib.DECISION_OUT)
    counts = np.zeros(4, dtype=np.int64)
    s._ck(lib.mmp_emul_place_ranks(s.h, _ptr(dec), len(dec), _ptr(fresh), 0 if fresh is None else len(fresh), _ptr(extra),
                                   0 if extra is None else len(extra), window, budget, _ptr(out), now_ms, seed, _ptr(counts)))
    return out, counts


@pytest.mark.parametrize("window,budget", [(12, 192), (5, 64), (1, 64), (0, 400)])
@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 2000, 1300, 33), ("C5", 1500, 500, 5), ("MIX", 500, 300, 14),
                                               ("MIX", 500, 700, 41), ("C5", 900, 10000, 5)])
def test_rank_rows_equal_bitmap_rows(ranks_lib, oracle_lib, config, nm, ni, seed, window, budget):
    """Every decision the lane routine resolves from the model's excluded ranks equals its walk on the bitmap row, field for
    field; models with more than 4 ids (0.2 % of the C3 / C5 models, 3 % of MIX) are declined and resolved from their row;
    the batch's results equal the oracle's."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, ranks_lib)
    for k, sd in enumerate((make_decisions(fl, 2000, seed), make_decisions(fl, 1500, seed + 1, sweep=True, plain=True))):
        out, counts = place_ranks(ranks_lib, s, sd, fl.now_ms, seed + k, window, budget)
        mismatch, ovf, resolved, declined = (int(x) for x in counts)
        assert mismatch == 0
        assert resolved > declined
        if k == 1:
            assert ovf > 0  # the sweep covers the registry: its overflow models went through the row
        od, off, idx = oracle_inputs(fl, sd)
        ores = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed + k, fresh=sd.fresh if len(sd.fresh) else None)
        assert np.array_equal(out["target"], ores["target"])
        assert np.array_equal(out["n_candidates"], ores["n_candidates"])
