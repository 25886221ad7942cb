"""The peer-memory instance-shard path (mmp_shard_ipc_export / _import, k_place_dealt, k_dealt_wait) on ONE GPU: G shard
fleets of one process on device 0, each called from a thread of its own, use each other's memory directly.  Every shard's
results must equal those of one unsharded fleet given the same call (and, on the first epoch, the oracle's), at the path's
edges: the replicated front (the first SHARD_FRONT_WORDS = 16 row words) and the column blocks around it, empty last
shards, G = 2 ... 16 (MAX_SHARDS: the widest DealtPeers), the deal of warp batches (wb % G, the tail warp included), both result-buffer halves, both snapshots' exported blocks, the
shared-memory redo of declined lanes, the three batch entry points and the max_batch bound.

Rows are stored in whole 32-word units (HostState::row_words), so every fleet has column blocks past the front: a fleet of
fewer than 513 live instances keeps every rank in the front, and its blocks past it hold only padding.

A shard that synchronised the device (a buffer that grows, a commit, fleet destruction) while a peer waits in
k_dealt_wait would wait for that peer in turn: every buffer is sized before the import, and commits, device allocations and
close() run on the main thread between steps."""
import concurrent.futures as cf
import ctypes as C
import threading

import numpy as np
import pytest

from helpers import oracle_from_synth, oracle_inputs_fast
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet, MmpError
from modelmesh_b200.synth import SynthDecisions, load_into_fleet, make_decisions, make_fleet

FRONT_WORDS = 16      # SHARD_FRONT_WORDS: row words replicated on every shard
MAX_BATCH = 8250      # the max_batch every shard exports (258 warp batches, the last one of 26 decisions)
LANE_BUDGET = 192     # the default walk budget of a lane; 2 sends many decisions to the warp's shared-memory redo
STEP_TIMEOUT_S = 60   # a step that does not finish fails the test (k_dealt_wait itself gives up after 4 s)


def _overflow_fleet():
    """The front-edge fleet with a quarter of its models holding 5-12 registrations: the four inline ones anywhere, the
    overflow ones half in the front and half in word 16 (ranks 512-539), so that k_build_bitmap_ovf writes both the
    replicated front and a column block past it."""
    fl = make_fleet("C5", 800, 540, 7)
    order = oracle_from_synth(fl).cluster_order()
    front, past = order[:512], order[512:]
    rng = np.random.default_rng(11)
    edges = []
    for m in range(fl.n_models):
        k = int(rng.integers(5, 13)) if rng.uniform() < 0.25 else int(rng.integers(0, 5))
        inl = [int(x) for x in rng.choice(order, size=min(4, k), replace=False)]
        n_ovf = k - len(inl)
        ovf = [int(x) for x in rng.permutation(past) if x not in inl][:(n_ovf + 1) // 2]
        ovf += [int(x) for x in rng.permutation(front) if x not in inl][:n_ovf - len(ovf)]
        edges.append(inl + ovf)
    fl.edge_off = np.zeros(fl.n_models + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([x for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(fl.n_models, dtype=np.int32)
    return fl


# name -> (builder, row words, what it is for)
FLEETS = {
    "front_only": (lambda: make_fleet("MIX", 500, 300, 14), 32),   # fewer than 513 ranks: every walk ends in the front
    "front_edge": (lambda: make_fleet("C5", 800, 540, 7), 32),     # first entries and cuts in word 16, the only live word past the front
    "self_past": (lambda: make_fleet("C3", 2000, 1000, 3), 32),    # walks end in the front, selves lie past it
    "overflow": (_overflow_fleet, 32),                             # overflow registrations in the front and past it
    "c5": (lambda: make_fleet("C5", 2000, 5000, 5), 160),          # long walks across several blocks
    "c3": (lambda: make_fleet("C3", 3000, 10000, 3), 320),         # the flagship shape
}
# (front_only at G = 16: shards 8-15 hold no row word; front_edge at G = 8: shard 4 holds word 16, the only live word past
# the front, and shards 5-7 hold only padding)
CASES = [("front_only", 2), ("front_only", 16), ("front_edge", 3), ("front_edge", 8), ("self_past", 2), ("self_past", 4),
         ("overflow", 3), ("c5", 2), ("c5", 3), ("c5", 4), ("c5", 8), ("c3", 4), ("c3", 8), ("c3", 16)]
# fleets whose decisions end (first entry or cut) in every column block past the front that holds live ranks
DEEP = {"front_edge", "overflow", "c5"}


def _blocks(rw, g):
    """[(lo, hi)] row words of every shard: HostState::shard_words, restated"""
    block = ((rw + g - 1) // g + 3) // 4 * 4
    return [(min(rw, r * block), min(rw, min(rw, r * block) + block)) for r in range(g)]


def _dealt(n, g):
    """decisions of a batch of n dealt to each shard: warp batch wb (32 decisions, the last one short) to shard wb % G"""
    out = [0] * g
    for wb in range((n + 31) // 32):
        out[wb % g] += min(32, n - 32 * wb)
    return out


def _batch(fl, order, n, seed, g, plain):
    """n decisions: a plain registry sweep, or mixed ones (fresh rows, extra excludes, favourSelf) with, mixed in, selves
    ranked past the front, decisions of 6 extra excludes (more than a lane takes: the warp's redo), malformed ones and
    request-model ones.  Returns (decisions, positions to hold MMP_TARGET_INVALID whatever the unsharded fleet says,
    positions the oracle cannot take)."""
    sd = make_decisions(fl, n, seed + 1000 * g, sweep=plain, plain=plain)
    none = np.zeros(0, dtype=np.int64)
    if plain:
        return sd, none, none
    dec, extra = sd.dec, list(sd.extra)
    i = np.arange(n)
    past = order[FRONT_WORDS * 32:]
    if len(past):
        k = i[i % 5 == 2]
        dec["self"][k] = past[(k * 7919) % len(past)]
    for j in i[i % 13 == 6]:  # six extra excludes
        dec["extra_off"][j], dec["extra_n"][j] = len(extra), 6
        extra += [int(order[(j * 31 + t * 97) % len(order)]) for t in range(6)]
    bad = i[i % 97 == 40]
    for t, j in enumerate(bad):
        if t % 3 == 0:
            dec["model"][j] = fl.n_models
        elif t % 3 == 1:
            dec["self"][j] = fl.n_instances
        else:
            dec["extra_off"][j], dec["extra_n"][j] = len(extra) + 5, 2
    req = i[i % 89 == 17]
    dec["flags"][req] = (dec["flags"][req] & ~np.uint32(L.DF_MODEL_LAST_USED)) | np.uint32(L.DF_REQUEST_MODEL)
    dec["model"][req] = 0
    dec["extra_n"][req] = 0
    return SynthDecisions(dec, sd.fresh, np.asarray(extra, dtype=np.int32)), req, np.union1d(bad, req)


def _kw(sd):
    return dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)


def _same(got, want, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


# ---------------------------------------------------------------------------------------------------------------
# the batches of one (fleet, G): epoch 0 steps, the lane-budget steps, and the steps after each commit
# ---------------------------------------------------------------------------------------------------------------
def _sizes(g):
    return [1, 31, 32, 33, 32 * g - 1, 32 * g, 32 * g + 1, 8193, MAX_BATCH]


def _epoch0_batches(fl, order, g):
    return [(n, plain, _batch(fl, order, n, 17 * n + k, g, plain)) for k, n in enumerate(_sizes(g)) for plain in (False, True)]


def _later_batches(fl, order, g):
    """{epoch: the three batches placed after that epoch's commit}"""
    return {epoch: [_batch(fl, order, n, 31 * epoch + k, g, plain)
                    for k, (n, plain) in enumerate(((8193, False), (MAX_BATCH, True), (32 * g + 1, False)))]
            for epoch in (1, 2)}


# ---------------------------------------------------------------------------------------------------------------
# CPU: the chosen fleets keep the properties the GPU test relies on
# ---------------------------------------------------------------------------------------------------------------
def test_fleets_reach_the_path_edges(emul_lib, oracle_lib):
    """Row widths and shard layouts of the chosen fleets, and (on the CPU harness, unsharded, traced) where their decisions
    end: on the deep fleets every column block past the front that holds live ranks holds the first entry or the cut of
    some decision of the test's batches; on the others selves lie past the front; on the front-only fleet nothing does."""
    layouts = {(32, 2): [(0, 16), (16, 32)], (32, 3): [(0, 12), (12, 24), (24, 32)], (32, 4): [(0, 8), (8, 16), (16, 24), (24, 32)],
               (32, 8): [(4 * r, 4 * r + 4) for r in range(8)],
               (32, 16): [(4 * r, 4 * r + 4) for r in range(8)] + [(32, 32)] * 8}  # shards 8-15 empty
    for name, g in CASES:
        fl = FLEETS[name][0]()
        rw = FLEETS[name][1]
        f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=emul_lib)
        load_into_fleet(fl, f)
        assert f.row_words() == rw, (name, f.row_words())
        got = _blocks(rw, g)  # (the GPU test checks mmp_shard_words against it)
        if (rw, g) in layouts:
            assert got == layouts[(rw, g)], (name, g, got)
        order = f.cluster_order()
        n_live = len(order)
        ends, selves_past = [], 0
        for n, plain, (sd, req, skip) in _epoch0_batches(fl, order, g):
            if n < 8193:
                continue
            _, tr, _ = f.place_batch(sd.dec, fl.now_ms, 77, trace=True, **_kw(sd))
            ok = np.ones(len(sd.dec), dtype=bool)
            ok[skip] = False
            for k in ("best_rank", "cut_rank"):
                v = tr[k][ok]
                ends.append(v[(v >= 0) & (v < n_live)])
            rank_of = np.full(fl.n_instances, -1, dtype=np.int64)
            rank_of[order] = np.arange(n_live)
            s_ok = (sd.dec["self"] >= 0) & (sd.dec["self"] < fl.n_instances)
            selves_past += int(np.count_nonzero(rank_of[sd.dec["self"][s_ok]] >= FRONT_WORDS * 32))
        words = np.unique(np.concatenate(ends) >> 5)
        live_words = set(range((n_live + 31) // 32))
        f.close()
        if name == "front_only":
            assert n_live <= FRONT_WORDS * 32 and selves_past == 0
            continue
        assert selves_past > 0, name
        if name in DEEP:
            for r, (lo, hi) in enumerate(got):
                held = [w for w in range(max(lo, FRONT_WORDS), hi) if w in live_words]
                if held:
                    assert any(w in words for w in held), (name, g, r, lo, hi, words[words >= FRONT_WORDS][:20])
        if name in ("front_edge", "overflow"):
            assert n_live > FRONT_WORDS * 32 and max(live_words) == FRONT_WORDS  # word 16: the only live word past the front


# ---------------------------------------------------------------------------------------------------------------
# GPU: G shard fleets of one process on device 0
# ---------------------------------------------------------------------------------------------------------------
class _Shards:
    """G shard fleets of one SynthFleet on device 0, one worker thread per shard; a step hands every shard the same call,
    and the threads start it together."""

    def __init__(self, fl, g, lib):
        self.g = g
        self.fleets = []
        for r in range(g):
            f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models,
                      device=0, shard_rank=r, shard_count=g, lib=lib)
            load_into_fleet(fl, f)
            assert f.shard_words() == _blocks(f.row_words(), g)[r] + (_blocks(f.row_words(), g)[0][1],), r
            self.fleets.append(f)
        self.pool = cf.ThreadPoolExecutor(max_workers=g)
        self.dealt = [0] * g
        self.steps = 0

    def run(self, call):
        """call(fleet) on every shard at once; returns the G results"""
        gate = threading.Barrier(self.g)

        def one(f):
            gate.wait(timeout=STEP_TIMEOUT_S)
            return call(f)
        futs = [self.pool.submit(one, f) for f in self.fleets]
        return [fu.result(timeout=STEP_TIMEOUT_S) for fu in futs]

    def step(self, n, call):
        """a dealt step of n decisions"""
        outs = self.run(call)
        self.steps += 1
        for r, k in enumerate(_dealt(n, self.g)):
            self.dealt[r] += k
        return outs

    def close(self):
        self.pool.shutdown(wait=True)
        for f in self.fleets:
            f.close()


def _device_place(fleet, bufs, dec, now_ms):
    """mmp_place_batch_device from records already uploaded to bufs = (d_in, d_out); seed 77"""
    ms = C.c_float()
    fleet._ck(fleet.lib.mmp_place_batch_device(fleet.h, bufs[0], len(dec), bufs[1], now_ms, 77, C.byref(ms)))


def _run_case(name, g, product_lib, report):
    fl = FLEETS[name][0]()
    ref = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, fl.n_instances, fl.n_models, lib=product_lib)
    load_into_fleet(fl, ref)
    order = ref.cluster_order()
    oracle = oracle_from_synth(fl)
    sh = _Shards(fl, g, product_lib)
    lib = product_lib
    dev = []
    try:
        epoch0 = _epoch0_batches(fl, order, g)
        later = _later_batches(fl, order, g)
        # ---- size every placement buffer now, for every batch the case places: a buffer that grew during a step would
        # synchronise the device ----
        every = [sd for _, _, (sd, _, _) in epoch0] + [sd for bs in later.values() for sd, _, _ in bs]
        n_fresh = max(len(sd.fresh) for sd in every)
        n_extra = max(len(sd.extra) for sd in every)
        big = make_decisions(fl, MAX_BATCH + 1, 5, sweep=True, plain=True).dec
        fresh = fl.inst_rows[np.arange(n_fresh) % fl.n_instances].copy()
        fresh["shutting_down"] = 0
        extra = np.zeros(n_extra, dtype=np.int32)
        for f in sh.fleets:
            with pytest.raises(MmpError, match="not connected") as e:
                f.place_batch(big, fl.now_ms, 77, fresh=fresh, extra=extra)
            assert e.value.code == L.E_STATE
            with pytest.raises(MmpError, match="not connected") as e:
                f.place_sweep(0, fl.n_models, np.zeros(fl.n_models, dtype=np.int32) + int(order[0]), fl.now_ms, 77,
                              favour=np.ones(fl.n_models, dtype=bool))
            assert e.value.code == L.E_STATE
            d_in, d_out = C.c_void_p(), C.c_void_p()
            f._ck(lib.mmp_device_alloc(f.h, MAX_BATCH * L.DECISION_IN.itemsize, C.byref(d_in)))
            f._ck(lib.mmp_device_alloc(f.h, MAX_BATCH * L.DECISION_OUT.itemsize, C.byref(d_out)))
            dev.append((d_in, d_out))
        # ---- the exchange: every shard imports every blob ----
        blobs = [f.shard_ipc_export(MAX_BATCH) for f in sh.fleets]
        for f in sh.fleets:
            f.shard_ipc_import(blobs)
            assert f.shard_peer_stats()["active"]

        def batch_step(sd, req, skip, what, with_oracle):
            n = len(sd.dec)
            assert n <= MAX_BATCH and len(sd.fresh) <= n_fresh and len(sd.extra) <= n_extra, what  # (sized above)
            want = ref.place_batch(sd.dec, fl.now_ms, 77, **_kw(sd))
            if with_oracle:
                clean = sd.dec.copy()
                clean["model"][skip] = 0
                clean["self"][skip] = int(order[0])
                clean["extra_n"][skip] = 0
                clean["flags"][skip] &= ~np.uint32(L.DF_REQUEST_MODEL)
                od, off, idx = oracle_inputs_fast(fl, SynthDecisions(clean, sd.fresh, sd.extra))
                res = oracle.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, 77, fresh=sd.fresh if len(sd.fresh) else None)
                keep = np.ones(n, dtype=bool)
                keep[skip] = False
                _same(want[keep], res[keep], ("oracle", what))
            want = want.copy()
            want["target"][req] = L.TARGET_INVALID  # a request-model decision is malformed on an instance-sharded fleet
            want["n_candidates"][req] = 0
            outs = sh.step(n, lambda f: f.place_batch(sd.dec, fl.now_ms, 77, **_kw(sd)))
            for r, o in enumerate(outs):
                _same(o, want, (what, "shard", r))
            return n

        decided = 0
        # ---- epoch 0: every batch size, plain and mixed, against the unsharded fleet and the oracle ----
        for n, plain, (sd, req, skip) in epoch0:
            decided += batch_step(sd, req, skip, (name, g, "epoch0", n, plain), True)
        # the registry sweep, one self per decision and one self for all
        selves = order[(np.arange(fl.n_models) * 37) % len(order)].astype(np.int32)
        fav = (np.arange(fl.n_models) % 3) == 0
        for self_idx in (selves, int(order[-1])):
            want = ref.place_sweep(0, fl.n_models, self_idx, fl.now_ms, 77, favour=fav)
            outs = sh.step(fl.n_models, lambda f: f.place_sweep(0, fl.n_models, self_idx, fl.now_ms, 77, favour=fav))
            for r, o in enumerate(outs):
                _same(o, want, (name, g, "sweep", np.isscalar(self_idx), r))
            decided += fl.n_models
        # records already on the device
        sd = make_decisions(fl, 8193, 99, sweep=False, plain=True)
        want = ref.place_batch(sd.dec, fl.now_ms, 77)
        for f, b in zip(sh.fleets, dev):
            f._ck(lib.mmp_device_upload(f.h, b[0], sd.dec.ctypes.data_as(C.c_void_p), sd.dec.nbytes))
        sh.step(len(sd.dec), lambda f: _device_place(f, dev[sh.fleets.index(f)], sd.dec, fl.now_ms))
        for r, (f, b) in enumerate(zip(sh.fleets, dev)):
            got = np.zeros(len(sd.dec), dtype=L.DECISION_OUT)
            f._ck(lib.mmp_device_download(f.h, got.ctypes.data_as(C.c_void_p), b[1], got.nbytes))
            _same(got, want, (name, g, "device", r))
        decided += len(sd.dec)
        # one decision more than max_batch: refused on every shard, without a step; the next step is right
        over = make_decisions(fl, MAX_BATCH + 1, 3, sweep=True, plain=True).dec
        for r, f in enumerate(sh.fleets):
            with pytest.raises(MmpError, match="max_batch") as e:
                f.place_batch(over, fl.now_ms, 77)
            assert e.value.code == L.E_ARG, r
            assert f.shard_peer_stats()["batches"] == sh.steps, r
        # a walk budget of 2 steps: most decisions take the warp's redo over the row assembled in shared memory
        for f in sh.fleets:
            f._ck(lib.mmp_tune(f.h, b"lane_budget", 2))
        for n, plain, (sd, req, skip) in epoch0:
            if n in (33, 32 * g + 1, 8193):
                decided += batch_step(sd, req, skip, (name, g, "budget2", n, plain), False)
        for f in sh.fleets:
            f._ck(lib.mmp_tune(f.h, b"lane_budget", LANE_BUDGET))
        # ---- a device-path commit (a numeric update), then a host-path commit (a removed instance): three steps each,
        # through the other snapshot's exported blocks and back ----
        victim = int(order[len(order) // 2])
        gone = int(order[0])
        for epoch, edit, path in ((1, lambda f: f.instance_update(victim, _busier(fl.inst_rows[victim])), 2),
                                  (2, lambda f: f.instance_remove(gone), 1)):
            for f in [ref] + sh.fleets:
                edit(f)
                f.commit()
                assert f.commit_info()[0] == path, (name, g, epoch)
            for sd, req, skip in later[epoch]:
                decided += batch_step(sd, req, skip, (name, g, "epoch", epoch, len(sd.dec)), False)
        # ---- counters ----
        rw = FLEETS[name][1]
        owners = {w: r for r, (lo, hi) in enumerate(_blocks(rw, g)) for w in range(lo, hi)}
        remote = []
        for r, f in enumerate(sh.fleets):
            st = f.shard_peer_stats()
            assert st["active"], (name, g, r)
            assert st["batches"] == sh.steps, (name, g, r, st)
            assert st["result_bytes_to_peers"] == 8 * (g - 1) * sh.dealt[r], (name, g, r, st, sh.dealt[r])
            # every shard's deal holds decisions of 6 extras, redone over the whole row: it reads every word past the
            # front that another shard owns, and no other
            if any(owners[w] != r for w in range(FRONT_WORDS, rw)):
                assert st["remote_row_words"] > 0, (name, g, r, st)
            else:
                assert st["remote_row_words"] == 0, (name, g, r, st)
            remote.append(st["remote_row_words"])
        report.append(f"{name} G={g}: {decided} decisions in {sh.steps} steps; remote_row_words per shard {remote}")
    finally:
        for f, (d_in, d_out) in zip(sh.fleets, dev):
            f._ck(lib.mmp_device_free(f.h, d_in))
            f._ck(lib.mmp_device_free(f.h, d_out))
        sh.close()
        ref.close()


def _busier(row):
    row = row.copy()
    row["used"] = row["capacity"] // 3
    row["count"] = 5
    return row


@pytest.mark.gpu
@pytest.mark.parametrize("name,g", CASES, ids=[f"{n}-G{g}" for n, g in CASES])
def test_shard_fleets_on_one_gpu_match_unsharded(product_lib, oracle_lib, name, g):
    """G shard fleets on one GPU place every batch as one unsharded fleet does (and as the oracle does on the first
    epoch), from all three entry points, at both lane budgets, across a device-path and a host-path commit; max_batch + 1
    is refused without a step; the peer counters add up to the deal."""
    report = []
    _run_case(name, g, product_lib, report)
    print("\n".join(report))
