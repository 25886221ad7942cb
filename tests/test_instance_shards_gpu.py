"""Instance-sharded placement on real GPUs, one process per GPU, both exchange paths: the collective one (NCCL
all-reduce(min) of the shard keys + row-gather pass) and the peer-access one (decisions dealt across the shards, rows read
from / results stored to peers' memory through CUDA IPC mappings, k_place_dealt): every shard must return exactly what the
unsharded solver returns.  Needs >= 2 GPUs; skipped on
a single-GPU box.  The protocol itself is covered on CPU by test_instance_shards_cpu.py."""
import os
import socket

import numpy as np
import pytest

from modelmesh_b200.synth import load_into_fleet, make_decisions, make_fleet

CASES = [("C3", 3000, 10000, 3), ("C5", 2000, 5000, 5), ("MIX", 500, 700, 8), ("MIX", 500, 300, 14), ("C2", 3000, 1000, 2)]


def _worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from modelmesh_b200 import _lib
        from modelmesh_b200.fleet import Fleet
        lib = _lib.load_product()
        results = []
        for config, nm, ni, seed in CASES:
            fl = make_fleet(config, nm, ni, seed)
            f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models,
                      device=rank, shard_rank=rank, shard_count=world, lib=lib)
            load_into_fleet(fl, f)
            uid = [f.shard_unique_id() if rank == 0 else None]
            dist.broadcast_object_list(uid, src=0)
            f.shard_connect(uid[0])
            for plain in (True, False):
                sd = make_decisions(fl, 4000, seed, sweep=plain, plain=plain)
                out = f.place_batch(sd.dec, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None,
                                    extra=sd.extra if len(sd.extra) else None)
                results.append(out.copy())
            results.append(np.asarray([f.shard_open_decisions()], dtype=np.int64))
            # ---- the peer-access path: blobs exchanged through the process group, the same batches dealt across the shards ----
            blobs = [None] * world
            dist.all_gather_object(blobs, f.shard_ipc_export(8192))
            f.shard_ipc_import(blobs)
            dist.barrier()
            for rnd in range(2):
                for plain in (True, False):
                    sd = make_decisions(fl, 4000, seed, sweep=plain, plain=plain)
                    out = f.place_batch(sd.dec, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None,
                                        extra=sd.extra if len(sd.extra) else None)
                    results.append(out.copy())
                if rnd == 0:  # a new epoch: the other snapshot's column blocks, through the pointers mapped at import
                    row = fl.inst_rows[1].copy()
                    row["used"] = row["capacity"] // 3
                    row["count"] = 5
                    f.instance_update(1, row)
                    f.commit()
            st = f.shard_peer_stats()
            results.append(np.asarray([st["batches"], st["remote_row_words"], st["result_bytes_to_peers"], int(st["active"])], dtype=np.int64))
            dist.barrier()
            f.close()
        q.put((rank, results))
    except BaseException:  # the parent must not wait for a worker that died
        import traceback
        q.put((rank, "worker failed:\n" + traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_matches_unsharded(product_lib, world):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    import torch.multiprocessing as mp
    from modelmesh_b200.fleet import Fleet
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
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
    k = 0
    total_open = 0
    peer_words = 0
    for config, nm, ni, seed in CASES:
        fl = make_fleet(config, nm, ni, seed)
        ref_f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
        load_into_fleet(fl, ref_f)
        for plain in (True, False):
            sd = make_decisions(fl, 4000, seed, sweep=plain, plain=plain)
            ref = ref_f.place_batch(sd.dec, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None,
                                    extra=sd.extra if len(sd.extra) else None)
            for r in range(world):
                out = got[r][k]
                bad = np.nonzero((out["target"] != ref["target"]) | (out["n_candidates"] != ref["n_candidates"]))[0]
                assert len(bad) == 0, (config, plain, r, len(bad), bad[:5], out[bad[:5]], ref[bad[:5]])
            k += 1
        total_open += int(got[0][k][0])
        k += 1
        for rnd in range(2):
            for plain in (True, False):
                sd = make_decisions(fl, 4000, seed, sweep=plain, plain=plain)
                ref = ref_f.place_batch(sd.dec, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None,
                                        extra=sd.extra if len(sd.extra) else None)
                for r in range(world):
                    out = got[r][k]
                    bad = np.nonzero((out["target"] != ref["target"]) | (out["n_candidates"] != ref["n_candidates"]))[0]
                    assert len(bad) == 0, ("peers", config, rnd, plain, r, len(bad), bad[:5], out[bad[:5]], ref[bad[:5]])
                k += 1
            if rnd == 0:
                row = fl.inst_rows[1].copy()
                row["used"] = row["capacity"] // 3
                row["count"] = 5
                ref_f.instance_update(1, row)
                ref_f.commit()
        for r in range(world):
            st = got[r][k]
            assert st[0] == 4 and st[3] == 1, (config, r, st)  # all four batches went through the peer path
            peer_words += int(st[1])
        k += 1
        ref_f.close()
    assert total_open > 0  # the row-gather pass was exercised (C5 / MIX walks cross shard boundaries)
    assert peer_words > 0  # ... and so were reads from peers' column blocks


def _place_batch_device(fleet, dec, now_ms):
    """mmp_place_batch_device on records uploaded to device memory, seed 77"""
    import ctypes as C
    from modelmesh_b200._lib import DECISION_OUT
    lib = fleet.lib
    dec = np.ascontiguousarray(dec)
    d_in, d_out = C.c_void_p(), C.c_void_p()
    fleet._ck(lib.mmp_device_alloc(fleet.h, dec.nbytes, C.byref(d_in)))
    fleet._ck(lib.mmp_device_alloc(fleet.h, len(dec) * DECISION_OUT.itemsize, C.byref(d_out)))
    try:
        fleet._ck(lib.mmp_device_upload(fleet.h, d_in, dec.ctypes.data_as(C.c_void_p), dec.nbytes))
        ms = C.c_float()
        fleet._ck(lib.mmp_place_batch_device(fleet.h, d_in, len(dec), d_out, now_ms, 77, C.byref(ms)))
        got = np.zeros(len(dec), dtype=DECISION_OUT)
        fleet._ck(lib.mmp_device_download(fleet.h, got.ctypes.data_as(C.c_void_p), d_out, got.nbytes))
        return got
    finally:
        fleet._ck(lib.mmp_device_free(fleet.h, d_in)); fleet._ck(lib.mmp_device_free(fleet.h, d_out))


@pytest.mark.gpu
def test_single_shard_takes_the_collective_path(product_lib, oracle_lib):
    """One GPU: a fleet of ONE shard that connects (ncclCommInitRank with one rank) sends its batches through the same
    keys -> ncclAllReduce(min) -> decode path as a sharded fleet, over whole rows, from each of the three batch entry
    points (mmp_place_batch, mmp_place_sweep, mmp_place_batch_device).  Results must equal the plain path's (and the
    oracle's), including decisions the lane routine hands to the cooperative routine."""
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from helpers import oracle_from_synth, oracle_inputs_fast
    from modelmesh_b200._lib import DF_FAVOUR_SELF
    from modelmesh_b200.fleet import Fleet

    for config, nm, ni, seed in [("C3", 40_000, 10_000, 3), ("C5", 3000, 5000, 5), ("MIX", 500, 300, 14)]:
        fl = make_fleet(config, nm, ni, seed)
        plain_f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
        load_into_fleet(fl, plain_f)
        f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
        load_into_fleet(fl, f)
        f.shard_connect(f.shard_unique_id())
        for plain in (True, False):
            sd = make_decisions(fl, min(nm, 40_000), seed, sweep=plain, plain=plain)
            kw = dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
            want = plain_f.place_batch(sd.dec, fl.now_ms, 77, **kw)
            got = f.place_batch(sd.dec, fl.now_ms, 77, **kw)
            assert np.array_equal(got, want)
            if plain:  # a registry sweep, and records that are already on the device
                fav = (sd.dec["flags"] & DF_FAVOUR_SELF) != 0
                assert np.array_equal(f.place_sweep(0, len(sd.dec), sd.dec["self"], fl.now_ms, 77, favour=fav),
                                      plain_f.place_sweep(0, len(sd.dec), sd.dec["self"], fl.now_ms, 77, favour=fav))
                assert np.array_equal(_place_batch_device(f, sd.dec, fl.now_ms), want)
                assert np.array_equal(_place_batch_device(plain_f, sd.dec, fl.now_ms), want)
        assert f.shard_open_decisions() == 0  # a single shard's range is the whole row: no walk can leave it
        o = oracle_from_synth(fl)
        od, off, idx = oracle_inputs_fast(fl, sd)
        res = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None)
        assert np.array_equal(got["target"], res["target"]) and np.array_equal(got["n_candidates"], res["n_candidates"])
        f.close(); plain_f.close()


@pytest.mark.gpu
def test_collective_path_refuses_rows_it_cannot_stage(product_lib, oracle_lib):
    """One GPU: the collective path's key and gather passes run on k_place_lanes, whose landing stages hold rows of at most
    580 words: rows of 576 words, fleets of up to 18 432 instances.  A connected one-shard fleet of 18 432 instances places like its
    unconnected twin and the oracle from all three batch entry points; at 18 433 instances (rows of 608 words) all three
    refuse with MMP_E_STATE, and the unconnected twin still places the batch as the oracle does."""
    import sys
    sys.path.insert(0, os.path.dirname(__file__))
    from helpers import oracle_from_synth, oracle_inputs_fast
    from modelmesh_b200._lib import DF_FAVOUR_SELF, E_STATE
    from modelmesh_b200.fleet import Fleet, MmpError

    for ni in (18_432, 18_433):
        fl = make_fleet("C3", 3000, ni, 3)
        plain_f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
        load_into_fleet(fl, plain_f)
        f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
        load_into_fleet(fl, f)
        f.shard_connect(f.shard_unique_id())
        sd = make_decisions(fl, fl.n_models, 3, sweep=True, plain=True)
        fav = (sd.dec["flags"] & DF_FAVOUR_SELF) != 0
        want = plain_f.place_batch(sd.dec, fl.now_ms, 77)
        od, off, idx = oracle_inputs_fast(fl, sd)
        res = oracle_from_synth(fl).get_next_batch(od, fl.type_names, off, idx, fl.now_ms, 77)
        assert np.array_equal(want["target"], res["target"]) and np.array_equal(want["n_candidates"], res["n_candidates"])
        calls = {"batch": lambda: f.place_batch(sd.dec, fl.now_ms, 77),
                 "sweep": lambda: f.place_sweep(0, len(sd.dec), sd.dec["self"], fl.now_ms, 77, favour=fav),
                 "device": lambda: _place_batch_device(f, sd.dec, fl.now_ms)}
        if ni == 18_432:
            assert np.array_equal(calls["batch"](), want)
            assert np.array_equal(calls["sweep"](), plain_f.place_sweep(0, len(sd.dec), sd.dec["self"], fl.now_ms, 77, favour=fav))
            assert np.array_equal(calls["device"](), want)
        else:
            for name, call in calls.items():
                with pytest.raises(MmpError, match="rows of 608 words are wider than the 580 words the collective path can stage") as e:
                    call()
                assert e.value.code == E_STATE, name
        f.close(); plain_f.close()
