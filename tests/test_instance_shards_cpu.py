"""Instance-sharded placement (SURVEY.md §8e) on CPU: each shard resolves every decision over its own rank range and
publishes one 64-bit key; the minimum over shards is the answer of the shard holding the globally first entry under
PLACEMENT_ORDER (min-loc), or "open" when that shard's walk ran past its range (resolved by the row-gather pass).
Checked against the unsharded solver (which the other parity tests pin to the oracle).  tests/emul stands in for the
CUDA library; the gloo test runs the same exchange with torch.distributed all_reduce(MIN) on two processes."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import free_port
from modelmesh_b200 import _lib
from modelmesh_b200.fleet import Fleet
from modelmesh_b200.sharding import combine_shard_keys, decode_shard_keys
from modelmesh_b200.synth import load_into_fleet, make_decisions, make_fleet


def shard_keys(lib, fl, sd, rank, world, shape):
    f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models,
              shard_rank=rank, shard_count=world, lib=lib)
    load_into_fleet(fl, f)
    keys = np.zeros(len(sd.dec), dtype=np.uint64)
    lib.mmp_emul_set_keys(f.h, keys.ctypes.data_as(C.c_void_p))
    lib.mmp_emul_set_window(shape)
    try:
        f.place_batch(sd.dec, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
    finally:
        lib.mmp_emul_set_window(32)
        lib.mmp_emul_set_keys(f.h, None)
    f.close()
    return keys


@pytest.mark.parametrize("shape", [32, 2])
@pytest.mark.parametrize("config,nm,ni,seed,world", [("C3", 1500, 4000, 3, 2), ("C3", 1500, 4000, 3, 8), ("C5", 1200, 3000, 5, 4),
                                                      ("MIX", 500, 700, 8, 3), ("MIX", 500, 300, 14, 2), ("MIX", 500, 520, 21, 4),
                                                      ("C2", 1500, 1000, 2, 8)])
def test_min_loc_combine_matches_unsharded(emul_lib, config, nm, ni, seed, world, shape):
    lib = emul_lib
    lib.mmp_emul_set_keys.argtypes = [C.c_void_p, C.c_void_p]
    fl = make_fleet(config, nm, ni, seed)
    for plain in (True, False):
        sd = make_decisions(fl, 1500, seed, sweep=plain, plain=plain)
        ref_f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=lib)
        load_into_fleet(fl, ref_f)
        ref = ref_f.place_batch(sd.dec, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None,
                                extra=sd.extra if len(sd.extra) else None)
        keys = np.stack([shard_keys(lib, fl, sd, r, world, shape) for r in range(world)])
        best = combine_shard_keys(keys)
        target, ncand, is_open = decode_shard_keys(best)
        closed = ~is_open
        assert np.array_equal(target[closed], ref["target"][closed])
        assert np.array_equal(ncand[closed], ref["n_candidates"][closed])
        # a single shard is the unsharded problem: nothing may be left open
        if world == 1:
            assert not is_open.any()
        # the open ones are exactly those whose winning shard could not finish inside its range; the gather pass gives
        # them whole rows, i.e. the unsharded answer -- here we only require that they are a minority on these fleets
        assert is_open.mean() < 0.9
    # world == 1 degenerates to the unsharded solver
    k1 = shard_keys(lib, fl, sd, 0, 1, shape)
    t1, c1, o1 = decode_shard_keys(k1)
    assert not o1.any() and np.array_equal(t1, ref["target"]) and np.array_equal(c1, ref["n_candidates"])


def _worker(rank, world, port, so_path, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lib = _lib.load(so_path, require_all=False)
        lib.mmp_emul_set_keys.argtypes = [C.c_void_p, C.c_void_p]
        fl = make_fleet("C3", 1200, 2500, 3)
        sd = make_decisions(fl, 1200, 3, sweep=True, plain=True)
        keys = shard_keys(lib, fl, sd, rank, world, 2)
        # all_reduce(MIN) over unsigned keys: gloo has no uint64, so flip the sign bit (order-preserving map to int64)
        t = torch.from_numpy((keys ^ np.uint64(1 << 63)).view(np.int64).copy())
        dist.all_reduce(t, op=dist.ReduceOp.MIN)
        best = t.numpy().view(np.uint64) ^ np.uint64(1 << 63)
        if rank == 0:
            q.put(best.copy())
    finally:
        dist.destroy_process_group()


def test_two_process_gloo_exchange(emul_lib):
    import torch.multiprocessing as mp
    so = emul_lib._name
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, so, q)) for r in range(2)]
    for p in procs:
        p.start()
    best = q.get(timeout=300)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    fl = make_fleet("C3", 1200, 2500, 3)
    sd = make_decisions(fl, 1200, 3, sweep=True, plain=True)
    ref_f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=emul_lib)
    load_into_fleet(fl, ref_f)
    ref = ref_f.place_batch(sd.dec, fl.now_ms, 77)
    target, ncand, is_open = decode_shard_keys(best)
    assert not is_open.any()
    assert np.array_equal(target, ref["target"]) and np.array_equal(ncand, ref["n_candidates"])
