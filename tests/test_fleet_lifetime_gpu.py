"""A fleet's CUDA resources end with the fleet: one that has used every kind it owns -- the placement contexts' streams,
events, pinned buffers and slot-sort scratch, a call-wide exclude set, the captured graph and the resident server of
B <= 32 batches, the closed loop's state and step events -- is destroyed, and a fresh fleet on the same device, three
times over, gives the oracle's answers again.  The instance-shard peer path (IPC mappings, peer buffers and events) does
the same on two GPUs; skipped on a single-GPU box."""
import os

import numpy as np
import pytest

from exclude_set import oracle_excluding, random_set
from helpers import compare_decisions, oracle_from_synth
from modelmesh_b200.synth import SynthDecisions, load_into_fleet, make_churn, make_decisions, make_fleet
from test_churn_gpu import _build, _compare_window
from test_exclude_set_gpu import _compact, _kw, _same
from test_instance_shards_gpu import _free_port

pytestmark = pytest.mark.gpu

ROUNDS = 3
NONE = np.zeros(0, dtype=np.int32)


def test_fresh_fleets_after_destroy_match_the_oracle(product_lib, oracle_lib):
    lib = product_lib
    for rnd in range(ROUNDS):
        seed = 4 + rnd
        w = make_churn(20_000, 200, seed, fill=0.9, with_types=True)
        fl = w.fleet
        o, sim, s = _build(product_lib, w, slots=256)
        sd = make_decisions(fl, 9000, seed)
        # a batch large enough for the slot sort, in slot order, against the oracle
        s._ck(lib.mmp_tune(s.h, b"sort_slots", 1))
        compare_decisions(fl, sd, o, s, seed, full_lists=False)
        s._ck(lib.mmp_tune(s.h, b"sort_slots", 2))
        want = oracle_excluding(o, fl, sd, NONE, seed)
        # a call-wide exclude set: the call's own slot tables
        xs = random_set(fl.n_instances, 24, seed)
        _same(s.place_batch(sd.dec, fl.now_ms, seed, exclude=xs, **_kw(sd)), oracle_excluding(o, fl, sd, xs, seed), (rnd, "exclude"))
        # B <= 32 through the captured graph (one_mode 2) and the resident server (3)
        part = _compact(sd, 32)
        for mode in (2, 3):
            s._ck(lib.mmp_tune(s.h, b"one_mode", mode))
            for n in (1, 32):
                small = SynthDecisions(part.dec[:n], part.fresh, part.extra)
                _same(s.place_batch(small.dec, fl.now_ms, seed, **_kw(small)), want[:n], (rnd, "one_mode", mode, n))
        # the closed loop: two windows, each ending in a device-path commit
        for ep in range(2):
            now0 = fl.now_ms + ep * w.window_ms
            _compare_window((rnd, ep), o, sim, s, w.events(ep, 2000, seed), now0, now0 + w.window_ms, seed * 100 + ep)
        s.close()


def _peer_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from modelmesh_b200 import _lib
        from modelmesh_b200.fleet import Fleet
        lib = _lib.load_product()
        fl = make_fleet("C5", 2000, 5000, 5)
        sd = make_decisions(fl, 4000, 5)
        results = []
        for _ in range(ROUNDS):
            f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models,
                      device=rank, shard_rank=rank, shard_count=world, lib=lib)
            load_into_fleet(fl, f)
            uid = [f.shard_unique_id() if rank == 0 else None]
            dist.broadcast_object_list(uid, src=0)
            f.shard_connect(uid[0])
            blobs = [None] * world
            dist.all_gather_object(blobs, f.shard_ipc_export(8192))
            f.shard_ipc_import(blobs)
            dist.barrier()
            results.append(f.place_batch(sd.dec, fl.now_ms, 77, **_kw(sd)).copy())
            results.append(int(f.shard_peer_stats()["batches"]))
            dist.barrier()
            f.close()
        q.put((rank, results))
    except BaseException:  # the parent must not wait for a worker that died
        import traceback
        q.put((rank, "worker failed:\n" + traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def test_fresh_sharded_fleets_after_destroy_match_the_oracle(product_lib, oracle_lib):
    import torch
    world = 2
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_peer_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        r, res = q.get(timeout=600)
        if isinstance(res, str):
            for p in procs:
                p.kill()
            pytest.fail(f"rank {r}: {res}")
        got[r] = res
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    fl = make_fleet("C5", 2000, 5000, 5)
    sd = make_decisions(fl, 4000, 5)
    want = oracle_excluding(oracle_from_synth(fl), fl, sd, NONE, 77)
    for r in range(world):
        for k in range(ROUNDS):
            _same(got[r][2 * k], want, ("rank", r, "round", k))
            assert got[r][2 * k + 1] == 1, (r, k)  # the batch went through the peer path
