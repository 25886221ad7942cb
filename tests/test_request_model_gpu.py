"""Request-model decisions (MMP_DF_REQUEST_MODEL) on every placement path of the H100 library: k_place_direct in batch
and in slot order, k_place_lanes, the traced tile kernel, the B = 1 paths (k_place_small
as a launch and as a graph, k_place_server with its inline extras and with the mapped tables), the micro-batcher, mixed
batches; a model registered or changed after the last commit; instance-sharded fleets (>= 2 GPUs).

(a) a decision carrying its model's committed record equals the one reading it from the registry, (b) decisions on
records the snapshot has never seen equal the oracle on the same records."""
import ctypes as C
import os
import socket

import numpy as np
import pytest

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthDecisions, load_into_fleet, make_decisions, make_fleet

from helpers import oracle_from_synth, solver_from_synth
from request_model import as_request_model, hold_front, oracle_request, random_records

pytestmark = pytest.mark.gpu


def _kw(sd):
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def _setup(lib, config, nm, ni, seed, n_random=6000):
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl)
    fl = hold_front(fl, o.cluster_order())
    s = solver_from_synth(fl, lib)
    tid = {t: s.type_id(t) for t in fl.type_names}
    sd = make_decisions(fl, fl.n_models, seed, sweep=True)
    rq, flagged = as_request_model(fl, sd, tid)
    new = ["late-type"]
    names = list(fl.type_names) + new
    ids = [tid[t] for t in fl.type_names] + [s.type_id(t) for t in new]
    rnd, k = random_records(fl, make_decisions(fl, n_random, seed + 3), ids, seed)
    return fl, s, o, sd, rq, flagged, (rnd, oracle_request(o, names, k, rnd, fl.now_ms, seed)), seed


def _check(s, fl, sd, rq, rnd_want, seed, what):
    _same(s.place_batch(rq.dec, fl.now_ms, seed, **_kw(rq)), s.place_batch(sd.dec, fl.now_ms, seed, **_kw(sd)), ("(a)",) + what)
    rnd, want = rnd_want
    _same(s.place_batch(rnd.dec, fl.now_ms, seed, **_kw(rnd)), want, ("(b)",) + what)


FLEETS = [("C3", 3000, 10_000, 3), ("C5", 3000, 10_000, 5), ("MIX", 500, 700, 41)]


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_direct_each_minb_lanes_and_slot_order(product_lib, oracle_lib, config, nm, ni, seed):
    fl, s, o, sd, rq, flagged, rw, seed = _setup(product_lib, config, nm, ni, seed)
    assert flagged.mean() > 0.95
    tid = {t: s.type_id(t) for t in fl.type_names}
    _check(s, fl, sd, rq, rw, seed, (config, "direct"))
    # slot-sorted launches (>= 8192 decisions): the sort key of a request-model decision is its own type id
    big = make_decisions(fl, 9000, seed + 9)
    brq, _ = as_request_model(fl, big, tid)
    for sort in (0, 1):
        s._ck(product_lib.mmp_tune(s.h, b"sort_slots", sort))
        _same(s.place_batch(brq.dec, fl.now_ms, 2, **_kw(brq)), s.place_batch(big.dec, fl.now_ms, 2, **_kw(big)), ("sorted (a)", sort))
    rnd, want = rw
    rep = SynthDecisions(np.concatenate([rnd.dec, rnd.dec]), rnd.fresh, rnd.extra)  # 12 000 decisions: sorted too
    s._ck(product_lib.mmp_tune(s.h, b"sort_slots", 1))
    got = s.place_batch(rep.dec, fl.now_ms, seed, **_kw(rep))
    _same(got[:len(rnd.dec)], want, ("sorted (b)", config))
    s._ck(product_lib.mmp_tune(s.h, b"sort_slots", 2))
    s._ck(product_lib.mmp_tune(s.h, b"direct", 0))  # k_place_lanes: the rows through the TMA landing stages
    _check(s, fl, sd, rq, rw, seed, (config, "lanes"))
    s._ck(product_lib.mmp_tune(s.h, b"direct", 1))
    s.close()


@pytest.mark.parametrize("config,nm,ni,seed", FLEETS)
def test_traced_tile_kernel(product_lib, oracle_lib, config, nm, ni, seed):
    fl, s, o, sd, rq, flagged, (rnd, want), seed = _setup(product_lib, config, nm, ni, seed, n_random=2000)
    part = slice(0, 1500)
    a = SynthDecisions(sd.dec[part], sd.fresh, sd.extra)
    b = SynthDecisions(rq.dec[part], rq.fresh, rq.extra)
    oa, ta, ma = s.place_batch(a.dec, fl.now_ms, seed, trace=True, masks=True, **_kw(a))
    ob_, tb, mb = s.place_batch(b.dec, fl.now_ms, seed, trace=True, masks=True, **_kw(b))
    assert np.array_equal(oa, ob_) and np.array_equal(ta, tb) and np.array_equal(ma, mb)
    oa, ta, _ = s.place_batch(a.dec, fl.now_ms, seed, trace=True, **_kw(a))
    ob_, tb, _ = s.place_batch(b.dec, fl.now_ms, seed, trace=True, **_kw(b))
    assert np.array_equal(oa, ob_)
    for k in ("best", "n_remaining", "pick_index", "cut_rank", "best_rank"):
        assert np.array_equal(ta[k], tb[k]), k
    assert np.array_equal(ta["flags"] & 255, tb["flags"] & 255)
    got, tr, _ = s.place_batch(rnd.dec, fl.now_ms, seed, trace=True, masks=True, **_kw(rnd))
    _same(got, want, ("traced (b)", config))
    assert np.array_equal(tr["best"], want["best"])


def _one_by_one(lib, s, sd, fl, seed, idx):
    out = np.zeros(1, dtype=L.DECISION_OUT)
    res = np.zeros(len(idx), dtype=L.DECISION_OUT)
    fresh = np.ascontiguousarray(sd.fresh, dtype=L.INSTANCE_ROW) if len(sd.fresh) else None
    for j, i in enumerate(idx):
        d = np.ascontiguousarray(sd.dec[i:i + 1])
        x = sd.extra[d["extra_off"][0]:d["extra_off"][0] + d["extra_n"][0]].astype(np.int32)
        d["extra_off"] = 0  # a request thread's own extra[]: the slice starts the table (the server's kind 1 shape)
        fp = d.copy()
        if fresh is not None and d["fresh"][0] >= 0:  # its own fresh row, at index 0
            f1, fp["fresh"] = fresh[d["fresh"][0]:d["fresh"][0] + 1], 0
        else:
            f1, fp["fresh"] = None, -1
        s._ck(lib.mmp_place_one(s.h, fp.ctypes.data_as(C.c_void_p), None if f1 is None else f1.ctypes.data_as(C.c_void_p),
                                x.ctypes.data_as(C.c_void_p) if len(x) else None, out.ctypes.data_as(C.c_void_p), fl.now_ms, seed))
        res[j] = out[0]
    return res


def _oracle_one(o, names, k, sd, fl, seed, idx):
    """the oracle on each decision as a batch of one (decision id 0, as mmp_place_one numbers it)"""
    return np.concatenate([oracle_request(o, names, k[[i]], SynthDecisions(sd.dec[[i]], sd.fresh, sd.extra), fl.now_ms, seed)
                           for i in idx])


@pytest.mark.parametrize("one_mode", [1, 2, 3])
def test_single_decisions_each_one_mode(product_lib, oracle_lib, one_mode):
    """mmp_place_one: k_place_small as a launch (1) and as a graph (2), k_place_server (3): kind 1 carries 1-4 extras
    inline, kind 2 (5 and 16) reads the mapped tables.  Each call is a batch of one: decision id 0."""
    fl = make_fleet("C3", 3000, 10_000, 3)
    o = oracle_from_synth(fl)
    fl = hold_front(fl, o.cluster_order())
    s = solver_from_synth(fl, product_lib)
    tid = {t: s.type_id(t) for t in fl.type_names}
    s._ck(product_lib.mmp_tune(s.h, b"one_mode", one_mode))
    sd = make_decisions(fl, 400, 11)
    rq, flagged = as_request_model(fl, sd, tid)
    idx = np.nonzero(flagged)[0][:300]
    got = _one_by_one(product_lib, s, rq, fl, 5, idx)
    want = _one_by_one(product_lib, s, sd, fl, 5, idx)
    _same(got, want, ("(a)", one_mode))
    names = list(fl.type_names) + ["late-type"]
    ids = [tid[t] for t in fl.type_names] + [s.type_id("late-type")]
    rnd, k = random_records(fl, make_decisions(fl, 300, 12), ids, 12, sizes=(0, 1, 2, 3, 4, 5, 16))
    idx = np.arange(300)
    got = _one_by_one(product_lib, s, rnd, fl, 5, idx)
    _same(got, _oracle_one(o, names, k, rnd, fl, 5, idx), ("(b)", one_mode))


def test_batcher_and_mixed_batches(product_lib, oracle_lib):
    fl = make_fleet("MIX", 500, 700, 14)
    o = oracle_from_synth(fl)
    fl = hold_front(fl, o.cluster_order())
    s = solver_from_synth(fl, product_lib)
    tid = {t: s.type_id(t) for t in fl.type_names}
    names = list(fl.type_names) + ["late-type"]
    ids = [tid[t] for t in fl.type_names] + [s.type_id("late-type")]
    rnd, k = random_records(fl, make_decisions(fl, 400, 15), ids, 15)
    # the micro-batcher: each decision's result is that of a batch of one hashed with the batcher's own id for it
    bt = C.c_void_p()
    s._ck(product_lib.mmp_batcher_create(s.h, 64, 50, 99, C.byref(bt)))
    try:
        fresh = np.ascontiguousarray(rnd.fresh, dtype=L.INSTANCE_ROW)
        extra = np.ascontiguousarray(rnd.extra, dtype=np.int32)
        out = np.zeros(1, dtype=L.DECISION_OUT)
        did = C.c_uint32()
        got = np.zeros(len(rnd.dec), dtype=L.DECISION_OUT)
        dids = np.zeros(len(rnd.dec), dtype=np.uint64)
        for i in range(len(rnd.dec)):
            d = np.ascontiguousarray(rnd.dec[i:i + 1])
            s._ck(product_lib.mmp_place_submit(bt, d.ctypes.data_as(C.c_void_p), fresh.ctypes.data_as(C.c_void_p),
                                               extra.ctypes.data_as(C.c_void_p), fl.now_ms, out.ctypes.data_as(C.c_void_p), C.byref(did)))
            got[i], dids[i] = out[0], did.value
    finally:
        product_lib.mmp_batcher_destroy(bt)
    from request_model import oracle_inputs_request
    od, off, idx = oracle_inputs_request(k, rnd)
    od["decision_id"] = dids
    want = o.get_next_batch(od, names, off, idx, fl.now_ms, 99, fresh=rnd.fresh)
    _same(got, want, "batcher")
    # mixed batches: flagged and unflagged decisions in one launch, every path
    sd = make_decisions(fl, 3000, 16)
    rq, flagged = as_request_model(fl, sd, tid)
    mixed = rq.dec.copy()
    mixed[::3] = sd.dec[::3]
    mixed["extra_off"][::3] += len(rq.extra)
    mb = SynthDecisions(mixed, sd.fresh, np.concatenate([rq.extra, sd.extra]).astype(np.int32))
    assert ((mixed["flags"] & L.DF_REQUEST_MODEL) != 0).mean() > 0.5
    want = s.place_batch(sd.dec, fl.now_ms, 8, **_kw(sd))
    for direct in (1, 0):
        s._ck(product_lib.mmp_tune(s.h, b"direct", direct))
        _same(s.place_batch(mb.dec, fl.now_ms, 8, **_kw(mb)), want, ("mixed", direct))
    s._ck(product_lib.mmp_tune(s.h, b"direct", 1))
    got, _, _ = s.place_batch(mb.dec, fl.now_ms, 8, trace=True, masks=True, **_kw(mb))
    _same(got, want, "mixed traced")


def test_model_registered_or_changed_since_the_commit(product_lib, oracle_lib):
    """Commit; upsert a new model and change another's record without committing.  Request-model decisions on the new
    records equal the oracle on them while the unflagged decision for the new index is still MMP_TARGET_INVALID; after
    the commit, flagged and unflagged decisions agree."""
    fl = make_fleet("C3", 3000, 10_000, 21)
    o = oracle_from_synth(fl)
    nm = fl.n_models
    s = solver_from_synth(fl, product_lib, max_models=nm + 1)
    tid = {t: s.type_id(t) for t in fl.type_names}
    new_type = s.type_id("registered-later")  # a type name first seen after the commit
    live = np.nonzero(fl.inst_rows["shutting_down"] == 0)[0]
    rows = np.zeros(2, dtype=L.MODEL_ROW)
    rows["last_used"] = fl.now_ms - 1000
    rows["size_units"] = 100
    rows["type_id"] = [new_type, tid[fl.type_names[0]]]
    rows["copy_count"] = [2, 3]
    rec_new = [int(live[0]), int(live[5])]
    rec_edit = [int(live[1]), int(live[2]), int(live[3]), int(live[9])]
    s.model_upsert(nm, rows[0], rec_new)       # registered (registerModel with loadNow) -- not committed
    s.model_upsert(7, rows[1], rec_edit)       # model 7's record changed -- not committed
    names = list(fl.type_names) + ["registered-later"]
    sd = make_decisions(fl, 64, 22)
    dec = sd.dec.copy()
    dec["flags"] = (dec["flags"] & np.uint32(L.DF_FAVOUR_SELF)) | np.uint32(L.DF_REQUEST_MODEL)
    dec["last_used"] = fl.now_ms - 1000
    k = np.where(np.arange(64) % 2 == 0, len(names) - 1, 0).astype(np.int32)
    dec["model"] = np.where(k == len(names) - 1, new_type, tid[fl.type_names[0]])
    recs = [rec_new if i % 2 == 0 else rec_edit for i in range(64)]
    extra = np.asarray([x for r in recs for x in r], dtype=np.int32)
    dec["extra_n"] = [len(r) for r in recs]
    dec["extra_off"] = np.concatenate([[0], np.cumsum(dec["extra_n"])[:-1]])
    rq = SynthDecisions(dec, sd.fresh, extra)
    want = oracle_request(o, names, k, rq, fl.now_ms, 4)
    for direct in (1, 0):
        s._ck(product_lib.mmp_tune(s.h, b"direct", direct))
        _same(s.place_batch(rq.dec, fl.now_ms, 4, **_kw(rq)), want, ("before commit", direct))
    idx = np.arange(8)
    _same(_one_by_one(product_lib, s, rq, fl, 4, idx), _oracle_one(o, names, k, rq, fl, 4, idx), "before commit, one by one")
    un = sd.dec.copy()
    un["model"] = np.where(np.arange(64) % 2 == 0, nm, 7)
    un["flags"] &= np.uint32(L.DF_FAVOUR_SELF)
    un["last_used"] = fl.now_ms - 1000
    un["extra_n"] = 0
    out = s.place_batch(un, fl.now_ms, 4, fresh=sd.fresh)
    assert (out["target"][::2] == L.TARGET_INVALID).all()  # the new index is past the committed registry
    s.commit()
    _same(s.place_batch(rq.dec, fl.now_ms, 4, **_kw(rq)), s.place_batch(un, fl.now_ms, 4, fresh=sd.fresh), "after commit")
    _same(s.place_batch(rq.dec, fl.now_ms, 4, **_kw(rq)), want, "after commit vs oracle")


# ---- instance-sharded fleets: both exchange paths answer every request-model decision MMP_TARGET_INVALID ----
def _shard_worker(rank, world, port, q):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from modelmesh_b200.fleet import Fleet
        lib = L.load_product()
        fl = make_fleet("C3", 3000, 10_000, 3)
        f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models,
                  device=rank, shard_rank=rank, shard_count=world, lib=lib)
        tid = load_into_fleet(fl, f)
        sd = make_decisions(fl, 4000, 3)
        rq, _ = as_request_model(fl, sd, tid)
        mixed = rq.dec.copy()
        mixed[::2] = sd.dec[::2]
        mixed["extra_off"][::2] += len(rq.extra)
        extra = np.concatenate([rq.extra, sd.extra]).astype(np.int32)
        uid = [f.shard_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(uid, src=0)
        f.shard_connect(uid[0])
        res = [f.place_batch(mixed, fl.now_ms, 77, fresh=sd.fresh, extra=extra).copy()]
        blobs = [None] * world
        dist.all_gather_object(blobs, f.shard_ipc_export(8192))
        f.shard_ipc_import(blobs)
        dist.barrier()
        res.append(f.place_batch(mixed, fl.now_ms, 77, fresh=sd.fresh, extra=extra).copy())
        res.append(np.asarray([int(f.shard_peer_stats()["active"])]))
        dist.barrier()
        f.close()
        q.put((rank, res))
    except BaseException:
        import traceback
        q.put((rank, "worker failed:\n" + traceback.format_exc()))
        raise
    finally:
        dist.destroy_process_group()


def test_instance_sharded_fleets_refuse_request_model_decisions(product_lib):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs (the CPU shard harness covers the rule: test_request_model_emul.py)")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = [ctx.Process(target=_shard_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(2):
        r, res = q.get(timeout=600)
        if isinstance(res, str):
            for p in procs:
                p.kill()
            pytest.fail(f"rank {r}: {res}")
        got[r] = res
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    fl = make_fleet("C3", 3000, 10_000, 3)
    ref = solver_from_synth(fl, product_lib)
    sd = make_decisions(fl, 4000, 3)
    want = ref.place_batch(sd.dec, fl.now_ms, 77, **_kw(sd))
    for r in range(2):
        assert got[r][2][0] == 1  # the peer path was taken
        for out in got[r][:2]:
            assert (out["target"][1::2] == L.TARGET_INVALID).all()
            _same(out[::2], want[::2], ("sharded unflagged", r))
