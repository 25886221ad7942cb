"""GPU parity tests proper: the CUDA library (through the C ABI) against the oracle on the same seeded inputs."""
import numpy as np
import pytest

from modelmesh_b200.synth import make_decisions, make_fleet

from helpers import compare_decisions, oracle_from_synth, solver_from_synth

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("config,nm,ni,seed", [
    ("C1", 1000, 16, 1), ("C2", 5000, 1000, 2), ("C2", 3000, 2000, 12), ("C3", 5000, 3000, 3), ("C5", 5000, 4000, 5),
    ("C3", 3000, 10000, 33), ("C5", 2000, 10000, 55), ("C3", 1000, 7000, 7), ("C5", 1000, 12345, 9),
    ("C3", 500, 20000, 11), ("C5", 300, 40000, 13), ("C3", 300, 65536, 17),
])
def test_decisions_match_oracle(product_lib, oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    assert np.array_equal(s.cluster_order(), o.cluster_order())
    nd = 3000 if ni <= 4000 else 1200
    sd = make_decisions(fl, nd, seed)
    compare_decisions(fl, sd, o, s, seed=seed * 7919)
    sd = make_decisions(fl, 1000, seed + 1, sweep=True, plain=True)
    compare_decisions(fl, sd, o, s, seed=seed)


@pytest.mark.parametrize("seed", range(60))
def test_mixed_regimes_match_oracle(product_lib, oracle_lib, seed):
    ni = [33, 64, 97, 160, 300, 1000, 1025, 2100, 4200][seed % 9]
    fl = make_fleet("MIX", 600, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    assert np.array_equal(s.cluster_order(), o.cluster_order())
    sd = make_decisions(fl, 1500, seed)
    compare_decisions(fl, sd, o, s, seed=seed + 99)


@pytest.mark.parametrize("kernel,tile,ring_k", [("lanes", 16, 4), ("tile", 16, 4)])
@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 4000, 10000, 3), ("C5", 3000, 5000, 5), ("MIX", 600, 300, 14), ("C2", 3000, 1000, 2),
                                               ("C3", 2000, 16000, 7)])
def test_kernel_variants_match_oracle(product_lib, oracle_lib, monkeypatch, kernel, tile, ring_k, config, nm, ni, seed):
    """k_place_lanes (one decision per lane) and the untraced cooperative k_place give the same, oracle-identical
    answers.  On these fleets' rows of <= 2 KiB k_place runs tiles of 16 lanes and a ring of 4 rows per warp: `tile` and
    `ring_k` record that shape in the test ids."""
    monkeypatch.setenv("MMP_KERNEL", kernel)
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 2500, seed)
    compare_decisions(fl, sd, o, s, seed=seed * 17, full_lists=False)
    sd = make_decisions(fl, 2500, seed + 1, sweep=True, plain=True)
    compare_decisions(fl, sd, o, s, seed=seed, full_lists=False)


def _oracle_results(fl, sd, oracle, seed, ids=None):
    from helpers import oracle_inputs_fast
    od, off, idx = oracle_inputs_fast(fl, sd)
    if ids is not None:
        od["decision_id"] = ids
    return oracle.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 100_000, 1_000, 2), ("C5", 100_000, 10_000, 5), ("C3", 150_000, 10_000, 3)])
def test_baseline_sized_fleets_match_oracle(product_lib, oracle_lib, config, nm, ni, seed):
    """BASELINE.json configurations at (C2) or near (C3/C5: 10k instances, a 100-150k slice of the registry) their full
    size: every decision of a registry sweep and of a mixed batch equals the oracle's (target, n_candidates).
    C5 is the adversarial fleet: 70 % of its walks leave the lane routine's window and are redone cooperatively."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    for plain in (True, False):
        sd = make_decisions(fl, min(nm, 100_000), seed, sweep=plain, plain=plain)
        want = _oracle_results(fl, sd, o, seed)
        got = s.place_batch(sd.dec, fl.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
        bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
        assert len(bad) == 0, (config, plain, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def test_batch_properties(product_lib, oracle_lib):
    """Size-independent properties of the batched entry points on a 10k-instance fleet: a batch is idempotent; a batch
    equals its slices placed separately with mmp_fleet_set_id_base (what a registry shard does), also when it is large
    enough to be pipelined in chunks and carries fresh rows and extra excludes; the device-resident
    entry point equals the host one; a one-decision call equals the batch's entry."""
    import ctypes as C
    from modelmesh_b200._lib import DECISION_OUT
    fl = make_fleet("C3", 60_000, 10_000, 3)
    s = solver_from_synth(fl, product_lib)
    lib = product_lib
    sd = make_decisions(fl, 60_000, 9, sweep=True, plain=True)
    a = s.place_batch(sd.dec, fl.now_ms, 5)
    b = s.place_batch(sd.dec, fl.now_ms, 5)
    assert np.array_equal(a, b)
    # slices with their id base
    cuts = [0, 1, 31, 32, 33, 20_000, 20_007, 60_000]
    parts = []
    for lo, hi in zip(cuts[:-1], cuts[1:]):
        s._ck(lib.mmp_fleet_set_id_base(s.h, lo))
        parts.append(s.place_batch(sd.dec[lo:hi], fl.now_ms, 5))
    s._ck(lib.mmp_fleet_set_id_base(s.h, 0))
    assert np.array_equal(np.concatenate(parts), a)
    # a batch with fresh rows and extra excludes that spans two pipelined chunks (131 072 decisions each) equals its slices
    big = make_decisions(fl, 200_000, 10)
    kw = dict(fresh=big.fresh, extra=big.extra)
    whole = s.place_batch(big.dec, fl.now_ms, 5, **kw)
    parts = []
    for lo, hi in ((0, 70_000), (70_000, 131_077), (131_077, 200_000)):
        s._ck(lib.mmp_fleet_set_id_base(s.h, lo))
        parts.append(s.place_batch(big.dec[lo:hi], fl.now_ms, 5, **kw))
    s._ck(lib.mmp_fleet_set_id_base(s.h, 0))
    assert len(big.fresh) and len(big.extra) and (whole["target"] >= 0).any()
    assert np.array_equal(np.concatenate(parts), whole)
    # device-resident entry point
    d_in, d_out = C.c_void_p(), C.c_void_p()
    dec = np.ascontiguousarray(sd.dec)
    s._ck(lib.mmp_device_alloc(s.h, dec.nbytes, C.byref(d_in)))
    s._ck(lib.mmp_device_alloc(s.h, len(dec) * DECISION_OUT.itemsize, C.byref(d_out)))
    s._ck(lib.mmp_device_upload(s.h, d_in, dec.ctypes.data_as(C.c_void_p), dec.nbytes))
    ms = C.c_float()
    s._ck(lib.mmp_place_batch_device(s.h, d_in, len(dec), d_out, fl.now_ms, 5, C.byref(ms)))
    dev = np.zeros(len(dec), dtype=DECISION_OUT)
    s._ck(lib.mmp_device_download(s.h, dev.ctypes.data_as(C.c_void_p), d_out, dev.nbytes))
    assert np.array_equal(dev, a) and ms.value > 0
    s._ck(lib.mmp_device_free(s.h, d_in)); s._ck(lib.mmp_device_free(s.h, d_out))
    # single-decision calls (decision id 0 of their own batch)
    for i in (0, 17, 59_999):
        s._ck(lib.mmp_fleet_set_id_base(s.h, i))
        one = s.place_one(sd.dec[i], fl.now_ms, 5)
        assert (one["target"], one["n_candidates"]) == (a[i]["target"], a[i]["n_candidates"])
    s._ck(lib.mmp_fleet_set_id_base(s.h, 0))
    # and the whole thing against the oracle
    want = _oracle_results(fl, sd, oracle_from_synth(fl), 5)
    assert np.array_equal(a["target"], want["target"]) and np.array_equal(a["n_candidates"], want["n_candidates"])


def test_registry_sweep_entry_point(product_lib, oracle_lib):
    """mmp_place_sweep on the GPU (records built on the device, results streamed back chunk by chunk) = mmp_place_batch."""
    from modelmesh_b200._lib import DF_FAVOUR_SELF
    fl = make_fleet("C3", 300_000, 10_000, 3)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 300_000, 4, sweep=True, plain=True)
    whole = s.place_batch(sd.dec, fl.now_ms, 5)
    fav = (sd.dec["flags"] & DF_FAVOUR_SELF) != 0
    assert np.array_equal(s.place_sweep(0, 300_000, sd.dec["self"], fl.now_ms, 5, favour=fav), whole)
    s._ck(product_lib.mmp_fleet_set_id_base(s.h, 1000))
    assert np.array_equal(s.place_sweep(1000, 777, sd.dec["self"][1000:1777], fl.now_ms, 5, favour=fav[1000:1777]), whole[1000:1777])
    s._ck(product_lib.mmp_fleet_set_id_base(s.h, 0))
    leader = int(sd.dec["self"][0])
    d2 = sd.dec.copy()
    d2["self"] = leader
    d2["flags"] &= ~np.uint32(DF_FAVOUR_SELF)
    assert np.array_equal(s.place_sweep(0, 300_000, leader, fl.now_ms, 5), s.place_batch(d2, fl.now_ms, 5))


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 3000, 1300, 3), ("C5", 2500, 700, 5), ("MIX", 800, 300, 14)])
def test_latency_paths_equal_the_batch(product_lib, oracle_lib, config, nm, ni, seed):
    """Tiny batches (B = 1 .. 32: one getNext on a request thread) through the four launch paths -- a request to the resident
    k_place_server, k_place_small replayed as a CUDA graph (default), k_place_small as a stream launch, the streaming kernel -- give what the same decisions give inside a
    large batch, fresh rows and extra excludes included; between commits the graph is re-captured for the new epoch."""
    import ctypes as C
    fl = make_fleet(config, nm, ni, seed)
    s = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 700, seed)
    fresh = sd.fresh if len(sd.fresh) else None
    extra = sd.extra if len(sd.extra) else None
    for rnd in range(2):
        whole = s.place_batch(sd.dec, fl.now_ms, 11, fresh=fresh, extra=extra)
        for mode in (3, 2, 1, 0):  # 3: requests to the resident server kernel (restarted for the new epoch in round 2)
            s._ck(product_lib.mmp_tune(s.h, b"one_mode", mode))
            for lo, cnt in ((0, 1), (1, 1), (5, 7), (40, 32), (100, 33), (200, 300)):
                s._ck(product_lib.mmp_fleet_set_id_base(s.h, lo))
                got = s.place_batch(sd.dec[lo:lo + cnt], fl.now_ms, 11, fresh=fresh, extra=extra)
                assert np.array_equal(got, whole[lo:lo + cnt]), (rnd, mode, lo, cnt)
            s._ck(product_lib.mmp_fleet_set_id_base(s.h, 0))
            for i in (3, 77, 311):
                d = sd.dec[i:i + 1].copy()
                s._ck(product_lib.mmp_fleet_set_id_base(s.h, i))
                one = s.place_one(d, fl.now_ms, 11, fresh=fresh, extra=extra)
                assert int(one["target"]) == int(whole["target"][i]) and int(one["n_candidates"]) == int(whole["n_candidates"][i]), (rnd, mode, i)
            s._ck(product_lib.mmp_fleet_set_id_base(s.h, 0))
        s._ck(product_lib.mmp_tune(s.h, b"one_mode", 3))
        # a new epoch (numeric update -> device-path commit): the next round replays a re-captured graph
        r = fl.inst_rows[int(np.nonzero(fl.inst_rows["shutting_down"] == 0)[0][0])].copy()
        r["count"] = int(r["count"]) + 50
        s.instance_update(int(np.nonzero(fl.inst_rows["shutting_down"] == 0)[0][0]), r)
        s.commit()


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 20000, 10000, 3), ("C5", 9000, 5000, 5), ("MIX", 9000, 300, 14), ("C2", 5000, 1000, 2)])
def test_direct_kernel_equals_the_streaming_kernel(product_lib, config, nm, ni, seed):
    """k_place_direct (rows read straight from memory: the window by three 16-byte loads, the rest through the word list) against
    k_place_lanes (whole rows through TMA landing stages) on the same batches, fresh rows / extra excludes included, and with a
    lane budget so small that many decisions go to the cooperative routine."""
    fl = make_fleet(config, nm, ni, seed)
    s = solver_from_synth(fl, product_lib)
    for plain in (True, False):
        sd = make_decisions(fl, min(nm, 20000), seed, sweep=plain, plain=plain)
        kw = dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
        s._ck(product_lib.mmp_tune(s.h, b"direct", 0))
        want = s.place_batch(sd.dec, fl.now_ms, 21, **kw)
        for budget, sort in ((192, 0), (192, 1), (6, 1), (6, 0)):  # sort 1: batches of >= 8192 decisions resolved in type-slot order
            s._ck(product_lib.mmp_tune(s.h, b"lane_budget", budget))
            s._ck(product_lib.mmp_tune(s.h, b"sort_slots", sort))
            s._ck(product_lib.mmp_tune(s.h, b"direct", 1))
            got = s.place_batch(sd.dec, fl.now_ms, 21, **kw)
            s._ck(product_lib.mmp_tune(s.h, b"direct", 0))
            assert np.array_equal(got, want), (plain, budget, sort, np.nonzero(got != want)[0][:5])
        s._ck(product_lib.mmp_tune(s.h, b"sort_slots", 2))
        s._ck(product_lib.mmp_tune(s.h, b"direct", 1))
        s._ck(product_lib.mmp_tune(s.h, b"lane_budget", 192))
    s.close()
