"""world_size-2 (and 3) gloo tests of the N>1 host logic: registry sharding, gather of per-shard results, max-over-ranks
timing reduction — on CPU, with the tests/emul harness standing in for the CUDA library."""
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from helpers import free_port
from modelmesh_b200.sharding import localize_decisions, owner_of, shard_range


def test_shard_range_and_owner():
    for n in (1, 7, 10, 1000, 1_000_003):
        for w in (1, 2, 3, 4, 8):
            covered = 0
            for r in range(w):
                lo, hi = shard_range(r, w, n)
                assert lo == covered and hi >= lo
                covered = hi
            assert covered == n
            idx = np.unique(np.concatenate([np.arange(min(n, 50)), np.arange(max(0, n - 50), n), np.arange(0, n, max(1, n // 97))]))
            own = owner_of(idx, w, n)
            for i, o in zip(idx, own):
                lo, hi = shard_range(int(o), w, n)
                assert lo <= i < hi


def _worker(rank, world, port, so_path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from modelmesh_b200 import _lib
        from modelmesh_b200._lib import DECISION_OUT, MODEL_ROW
        from modelmesh_b200.fleet import Fleet
        from modelmesh_b200.synth import make_decisions, make_fleet
        lib = _lib.load(so_path, require_all=False)
        fl = make_fleet("C3", 3000, 700, 3)
        sd = make_decisions(fl, 3000, 3, sweep=True, plain=True)
        lo, hi = shard_range(rank, world, fl.n_models)
        # this rank's registry shard: instance table replicated, models [lo, hi)
        f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, hi - lo, lib=lib)
        f.types_set_json(fl.type_json())
        tid = {t: f.type_id(t) for t in fl.type_names}
        f.replicasets_set(fl.replaced_replicasets)
        for i in range(fl.n_instances):
            f.instance_upsert(i, fl.inst_rows[i], fl.inst_ids[i], fl.inst_locs[i], fl.inst_zones[i], fl.inst_labels[i])
        rows = np.zeros(hi - lo, dtype=MODEL_ROW)
        rows["last_used"] = fl.model_last_used[lo:hi]
        rows["type_id"] = np.asarray([tid[t] for t in fl.type_names], dtype=np.uint16)[fl.model_type[lo:hi]]
        rows["copy_count"] = np.minimum(255, fl.n_loaded[lo:hi])
        rows["fail_count"] = np.minimum(255, fl.n_failed[lo:hi])
        f.models_bulk(0, rows, fl.edge_off[lo:hi + 1] - fl.edge_off[lo], fl.edge_inst[fl.edge_off[lo]:fl.edge_off[hi]])
        f.commit()
        mine = localize_decisions(sd.dec, lo, hi)
        out = f.place_batch(mine, fl.now_ms, seed=77)
        # gather (target, n_candidates) of every shard on every rank
        t = torch.from_numpy(out.view(np.int32).reshape(-1, 2).copy())
        sizes = [torch.zeros(1, dtype=torch.int64) for _ in range(world)]
        dist.all_gather(sizes, torch.tensor([t.shape[0]], dtype=torch.int64))
        mx = int(max(int(s_) for s_ in sizes))
        pad = torch.zeros((mx, 2), dtype=torch.int32)
        pad[: t.shape[0]] = t
        parts = [torch.zeros((mx, 2), dtype=torch.int32) for _ in range(world)]
        dist.all_gather(parts, pad)
        # max-over-ranks timing reduction used by bench.py
        tm = torch.tensor([float(rank + 1)], dtype=torch.float64)
        dist.all_reduce(tm, op=dist.ReduceOp.MAX)
        assert float(tm) == float(world)
        if rank == 0:
            merged = np.concatenate([p[: int(s_)].numpy() for p, s_ in zip(parts, sizes)])
            q.put((merged, int(f.row_words())))
    finally:
        dist.barrier()
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_registry_sharded_placement_matches_unsharded(emul_lib, world):
    from modelmesh_b200.synth import make_decisions, make_fleet
    from helpers import solver_from_synth
    so = emul_lib._name
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, so, q)) for r in range(world)]
    for p in procs:
        p.start()
    merged, _ = q.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    fl = make_fleet("C3", 3000, 700, 3)
    sd = make_decisions(fl, 3000, 3, sweep=True, plain=True)
    s = solver_from_synth(fl, emul_lib)
    # unsharded reference: the sweep is ordered by model, so shard r's decisions are the contiguous slice [lo, hi);
    # the pick hash uses the position inside the call, hence compare shard by shard
    got = merged
    pos = 0
    for r in range(world):
        lo, hi = shard_range(r, world, fl.n_models)
        ref = s.place_batch(sd.dec[lo:hi], fl.now_ms, seed=77)
        assert np.array_equal(got[pos:pos + (hi - lo)], ref.view(np.int32).reshape(-1, 2)), r
        pos += hi - lo
    assert pos == len(got)
