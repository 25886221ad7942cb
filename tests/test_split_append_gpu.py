"""The worklists of k_place_split on the device (DESIGN.md §5.2.1): each block appends its walked and overflow-id decisions
to sub-list blockIdx % SPLIT_LISTS of each list with one atomic per list, k_place_tail maps its work items onto the
sub-lists' tiles and entries.  Every batch is placed with the two
passes forced on (split = 1) and off (split = 0); the two must be byte identical and equal the oracle.  The result
buffer is filled with a sentinel before each call, so a walked decision that no list held would show.

Batch sizes sit at the edges of a warp (n = 1, 31 mod 32), of a block (255, 257 mod 256), of the last sub-list's last
block (partial for SPLIT_LISTS = 32) and of the size the default takes the two passes from (2^18 - 1, 2^18 + 1); the
contents: every decision walked (each carries an extra exclude, so every block fills its sub-lists), none walked
(decisions the slot summaries answer), a mix of walked and overflow-id decisions, the C3 and C5 sweeps (C5 walks its
list in slot order), a call-wide exclude set and mmp_place_sweep."""
import ctypes as C

import numpy as np
import pytest

from exclude_set import oracle_excluding, random_set
from helpers import oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthDecisions, make_decisions, make_fleet
from replay import assert_same_results, oracle_batch
from split_widen import GROUPS, front_cases

pytestmark = pytest.mark.gpu

SENTINEL = 0x7EADBEEF


def _device_place(s, lib, sd, now, seed, split, offset):
    """mmp_place_batch_device with split forced, the records `offset` bytes past a fresh allocation's base and the
    results pre-filled with SENTINEL; the launches it took"""
    dec = np.ascontiguousarray(sd.dec)
    assert not len(sd.fresh) and not len(sd.extra)
    sent = np.zeros(len(dec), dtype=L.DECISION_OUT)
    sent["target"] = SENTINEL
    sent["n_candidates"] = SENTINEL
    d_in, d_out = C.c_void_p(), C.c_void_p()
    s._ck(lib.mmp_device_alloc(s.h, dec.nbytes + offset, C.byref(d_in)))
    s._ck(lib.mmp_device_alloc(s.h, sent.nbytes, C.byref(d_out)))
    try:
        rec = C.c_void_p(d_in.value + offset)
        s._ck(lib.mmp_device_upload(s.h, rec, dec.ctypes.data_as(C.c_void_p), dec.nbytes))
        s._ck(lib.mmp_device_upload(s.h, d_out, sent.ctypes.data_as(C.c_void_p), sent.nbytes))
        s._ck(lib.mmp_tune(s.h, b"split", split))
        k0 = s.kernel_launches()
        ms = C.c_float()
        s._ck(lib.mmp_place_batch_device(s.h, rec, len(dec), d_out, now, seed, C.byref(ms)))
        launches = s.kernel_launches() - k0
        out = np.zeros(len(dec), dtype=L.DECISION_OUT)
        s._ck(lib.mmp_device_download(s.h, out.ctypes.data_as(C.c_void_p), d_out, out.nbytes))
    finally:
        s._ck(lib.mmp_tune(s.h, b"split", 2))
        s._ck(lib.mmp_device_free(s.h, d_in))
        s._ck(lib.mmp_device_free(s.h, d_out))
    assert not np.any(out["target"] == SENTINEL), int(np.sum(out["target"] == SENTINEL))
    return out, launches


def _on_off(s, lib, sd, now, seed, what, offset=0):
    on, n_on = _device_place(s, lib, sd, now, seed, 1, offset)
    off, n_off = _device_place(s, lib, sd, now, seed, 0, offset)
    assert n_on >= 3 and n_on > n_off, (what, n_on, n_off)
    assert on.tobytes() == off.tobytes(), (what, int(np.sum(on != off)))
    return on


@pytest.fixture(scope="module")
def c3(product_lib, oracle_lib):
    fl = make_fleet("C3", 3000, 1300, 33)
    s = solver_from_synth(fl, product_lib)
    yield fl, oracle_from_synth(fl), s
    s.close()


# n = 1, 31 (mod 32); 255, 257 (mod 256); the last block of sub-list 31 of 32 partial; 2^18 -+ 1
SIZES = [1025, 2079, 4351, 4353, 32 * 256 * 2 - 100, (1 << 18) - 1, (1 << 18) + 1]


@pytest.mark.parametrize("n", SIZES)
def test_batch_sizes(c3, product_lib, n):
    fl, o, s = c3
    sd = make_decisions(fl, n, 7, plain=True)
    on = _on_off(s, product_lib, sd, fl.now_ms, 7, n, offset=16 if n & 1 else 0)
    assert_same_results(on, oracle_batch(fl, sd, o, 7), n)


def _host_on_off(s, lib, sd, now, seed, what, **kw):
    """mmp_place_batch (or mmp_place_batch_excluding) with split forced on and off: byte identical, two passes taken"""
    got, launches = {}, {}
    for split in (1, 0):
        s._ck(lib.mmp_tune(s.h, b"split", split))
        try:
            k0 = s.kernel_launches()
            got[split] = s.place_batch(sd.dec, now, seed, fresh=sd.fresh if len(sd.fresh) else None,
                                       extra=sd.extra if len(sd.extra) else None, **kw)
            launches[split] = s.kernel_launches() - k0
        finally:
            s._ck(lib.mmp_tune(s.h, b"split", 2))
    assert launches[1] >= 3 and launches[1] > launches[0], (what, launches)
    assert got[1].tobytes() == got[0].tobytes(), (what, int(np.sum(got[1] != got[0])))
    return got[1]


def test_every_decision_walked(c3, product_lib):
    """each decision carries one extra exclude, which the summaries never answer: every block fills its walk sub-list
    to the block's size"""
    fl, o, s = c3
    n = 8 * 256 * 3 + 40
    sd = make_decisions(fl, n, 9, plain=True)
    sd.dec["extra_off"] = np.arange(n, dtype=np.int32)
    sd.dec["extra_n"] = 1
    sd = SynthDecisions(sd.dec, sd.fresh, random_set(fl.n_instances, n, 9))
    on = _host_on_off(s, product_lib, sd, fl.now_ms, 9, "walked")
    assert_same_results(on, oracle_batch(fl, sd, o, 9), "walked")


@pytest.fixture(scope="module")
def front(product_lib, oracle_lib):
    fl, sd, group, rank, allowed = front_cases()
    s = solver_from_synth(fl, product_lib)
    yield fl, oracle_from_synth(fl), s, sd, group
    s.close()


@pytest.mark.parametrize("groups,n", [("ACDFG", 8 * 256 * 2 + 33), ("BE", 3 * 256 + 45), ("ABCDEFG", 8 * 256 * 4 + 77),
                                      ("EC", 4097)])
def test_walked_and_overflow_lists(front, product_lib, groups, n):
    """hand-built decisions: groups A, C, D, F and G are answered from the summaries (nothing listed), B is walked and
    E (a model with overflow ids) goes on the overflow list; each mix is tiled to n, so the sub-lists' lengths are not
    multiples of 32"""
    fl, o, s, sd, group = front
    pick = np.isin(np.asarray([GROUPS[g] for g in group]), list(groups))
    base = sd.dec[pick]
    tsd = SynthDecisions(np.resize(base, n), sd.fresh, sd.extra)
    for offset in (0, 16):
        on = _on_off(s, product_lib, tsd, fl.now_ms, 5, (groups, offset), offset)
        assert_same_results(on, oracle_batch(fl, tsd, o, 5), (groups, offset))


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 3000, 1300, 33), ("C5", 1500, 500, 5)])
def test_sweeps_exclude_set_and_sweep_entry(product_lib, oracle_lib, config, nm, ni, seed):
    """the bench's sweep (C5: the walk list sorted into slot order), the same batch under a call-wide exclude set, and
    mmp_place_sweep; the first call on the fleet is mmp_slot_summaries, so the counters are first sized there"""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    try:
        assert s._ck(product_lib.mmp_slot_summaries(s.h, C.c_int64(fl.now_ms), None, None, 0)) > 0
        sd = make_decisions(fl, 4 * nm + 3, seed, sweep=True, plain=True)
        on = _on_off(s, product_lib, sd, fl.now_ms, seed, config, offset=16)
        assert_same_results(on, oracle_batch(fl, sd, o, seed), config)
        xs = np.concatenate([s.cluster_order()[:3], random_set(fl.n_instances, 40, seed)]).astype(np.int32)
        ex = _host_on_off(s, product_lib, sd, fl.now_ms, seed, (config, "exclude"), exclude=xs)
        assert_same_results(ex, oracle_excluding(o, fl, sd, xs, seed), (config, "exclude"))
        selfs = sd.dec["self"][:nm]
        sw = {}
        for split in (1, 0):
            s._ck(product_lib.mmp_tune(s.h, b"split", split))
            try:
                k0 = s.kernel_launches()
                sw[split] = (s.place_sweep(0, nm, selfs, fl.now_ms, seed + 1), s.kernel_launches() - k0)
            finally:
                s._ck(product_lib.mmp_tune(s.h, b"split", 2))
        assert sw[1][1] > sw[0][1], (sw[1][1], sw[0][1])
        assert sw[1][0].tobytes() == sw[0][0].tobytes()
    finally:
        s.close()
