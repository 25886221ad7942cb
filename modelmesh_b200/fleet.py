"""Thin numpy-friendly wrapper over the libmmplace C ABI (include/mmplace.h).

``Fleet`` owns one ``mmp_fleet*``.  It is used by the tests and by bench.py; a Java host binds the same entry points
through JNI (INTEGRATION.md).  ``Fleet(cfg)`` uses the CUDA library; tests that run without a GPU pass ``lib=`` with the
CPU harness built from tests/emul (same symbols, single-lane shape of the same decision routine).
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import (CHURN_DECISION, CHURN_EVENT, CHURN_EVICTION, CHURN_REAPER, CLUSTER_STATS, DECISION_IN, DECISION_OUT,
                   DECISION_TRACE, EVICT_ACTION, EVICT_ENTRY, EVICT_PARAMS, EVICTION, INSTANCE_ROW, JANITOR_CACHE_ACTION, JANITOR_EDIT,
                   JANITOR_ENTRY, JANITOR_PARAMS, JANITOR_TASK_ENTRY, JANITOR_TASK_PARAMS, LRU_ENTRY, LRU_EVENT, MODEL_ROW, RATE_LOAD,
                   RATE_PARAMS, REAPER_LOAD, SCALE_IN, SCALE_OUT, SHUTDOWN_ACTION, SHUTDOWN_ENTRY, SHUTDOWN_PARAMS, ChurnConfig,
                   ChurnReport, EvictReport, JanitorReport, JanitorTaskReport, MmpConfig, RateReport, ReaperReport, ShutdownReport)


class MmpError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"libmmplace error {code}: {msg}")
        self.code = code


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _strs(items: Sequence[str]):
    arr = (C.c_char_p * max(1, len(items)))()
    for i, s in enumerate(items):
        arr[i] = s.encode("utf-8")
    return arr


class Fleet:
    def __init__(self, min_space_units: int, min_churn_age_ms: int, default_model_size_units: int, max_instances: int,
                 max_models: int, device: int = 0, shard_rank: int = 0, shard_count: int = 1, lib=None):
        self.lib = lib if lib is not None else _lib.load_product()
        cfg = MmpConfig(min_space_units, min_churn_age_ms, default_model_size_units, max_instances, max_models, device,
                        shard_rank, shard_count, 0, 0)
        self.max_instances, self.max_models = max_instances, max_models
        h = C.c_void_p()
        rc = self.lib.mmp_fleet_create(C.byref(cfg), C.byref(h))
        if rc < 0:
            raise MmpError(rc, (self.lib.mmp_last_error(None) or b"").decode())
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.mmp_fleet_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc: int) -> int:
        if rc < 0:
            raise MmpError(rc, (self.lib.mmp_last_error(self.h) or b"").decode())
        return rc

    # ---- ingest ----
    def instance_upsert(self, idx: int, row: np.ndarray, iid: str, loc: Optional[str] = None, zone: Optional[str] = None,
                        labels: Iterable[str] = ()):
        labels = list(labels)
        row = np.ascontiguousarray(row, dtype=INSTANCE_ROW).reshape(1)
        self._ck(self.lib.mmp_instance_upsert(self.h, idx, _ptr(row), iid.encode(), None if loc is None else loc.encode(),
                                              None if zone is None else zone.encode(), _strs(labels), len(labels)))

    def instance_update(self, idx: int, row: np.ndarray):
        row = np.ascontiguousarray(row, dtype=INSTANCE_ROW).reshape(1)
        self._ck(self.lib.mmp_instance_update(self.h, idx, _ptr(row)))

    def instance_remove(self, idx: int):
        self._ck(self.lib.mmp_instance_remove(self.h, idx))

    def types_set_json(self, js: Optional[str]):
        self._ck(self.lib.mmp_types_set_json(self.h, None if js is None else js.encode()))

    def type_id(self, name: str) -> int:
        return self._ck(self.lib.mmp_type_id(self.h, name.encode()))

    def replicasets_set(self, prefixes: Sequence[str]):
        self._ck(self.lib.mmp_replicasets_set(self.h, _strs(prefixes), len(prefixes)))

    def model_upsert(self, m: int, row: np.ndarray, instance_ids: Sequence[int] = ()):
        row = np.ascontiguousarray(row, dtype=MODEL_ROW).reshape(1)
        ids = np.ascontiguousarray(instance_ids, dtype=np.int32)
        self._ck(self.lib.mmp_model_upsert(self.h, m, _ptr(row), _ptr(ids), len(ids)))

    def models_bulk(self, first: int, rows: np.ndarray, edge_off: np.ndarray, edge_inst: np.ndarray):
        rows = np.ascontiguousarray(rows, dtype=MODEL_ROW)
        edge_off = np.ascontiguousarray(edge_off, dtype=np.int64)
        edge_inst = np.ascontiguousarray(edge_inst, dtype=np.int32)
        assert len(edge_off) == len(rows) + 1
        self._ck(self.lib.mmp_models_bulk(self.h, first, len(rows), _ptr(rows), _ptr(edge_off), _ptr(edge_inst)))

    def commit(self) -> int:
        return self._ck(self.lib.mmp_fleet_commit(self.h))

    # ---- placement ----
    def place_batch(self, dec: np.ndarray, now_ms: int, seed: int, fresh: Optional[np.ndarray] = None,
                    extra: Optional[np.ndarray] = None, trace: bool = False, masks: bool = False,
                    out: Optional[np.ndarray] = None, exclude: Optional[np.ndarray] = None):
        """exclude: a call-wide exclude set (instance indices, any length) added to every decision's exclusions
        (mmp_place_batch_excluding); None keeps the plain call, an array -- even an empty one -- takes that entry point."""
        dec = np.ascontiguousarray(dec, dtype=DECISION_IN)
        n = len(dec)
        if out is None:
            out = np.zeros(n, dtype=DECISION_OUT)
        fresh_a = None if fresh is None else np.ascontiguousarray(fresh, dtype=INSTANCE_ROW)
        extra_a = None if extra is None else np.ascontiguousarray(extra, dtype=np.int32)
        nf = 0 if fresh_a is None else len(fresh_a)
        ne = 0 if extra_a is None else len(extra_a)
        if exclude is not None:
            xs = np.ascontiguousarray(exclude, dtype=np.int32)
            tr = np.zeros(n, dtype=DECISION_TRACE) if trace or masks else None
            cm = np.zeros((n, 2, self.row_words()), dtype=np.uint32) if masks else None
            self._ck(self.lib.mmp_place_batch_excluding(self.h, _ptr(dec), n, _ptr(fresh_a), nf, _ptr(extra_a), ne, _ptr(xs), len(xs),
                                                        _ptr(out), _ptr(tr), _ptr(cm), now_ms, seed))
            return out if tr is None else (out, tr, cm)
        if not trace and not masks:
            self._ck(self.lib.mmp_place_batch(self.h, _ptr(dec), n, _ptr(fresh_a), nf, _ptr(extra_a), ne, _ptr(out),
                                              now_ms, seed))
            return out
        tr = np.zeros(n, dtype=DECISION_TRACE)
        cm = np.zeros((n, 2, self.row_words()), dtype=np.uint32) if masks else None
        self._ck(self.lib.mmp_place_batch_trace(self.h, _ptr(dec), n, _ptr(fresh_a), nf, _ptr(extra_a), ne, _ptr(out),
                                                _ptr(tr), _ptr(cm), now_ms, seed))
        return out, tr, cm

    def place_sweep(self, first_model: int, n: int, self_idx, now_ms: int, seed: int, favour: Optional[np.ndarray] = None):
        """Registry sweep (the reaper's batch, MM:6616-6735): model first_model + i on behalf of self_idx[i] (or one
        instance for all when self_idx is an int); favour = optional bool[n] of favourSelf flags."""
        out = np.zeros(n, dtype=DECISION_OUT)
        if np.isscalar(self_idx):
            sa, stride = np.asarray([self_idx], dtype=np.int32), 0
        else:
            sa, stride = np.ascontiguousarray(self_idx, dtype=np.int32), 1
            assert len(sa) == n
        bits = None
        if favour is not None:
            bits = np.packbits(np.asarray(favour, dtype=bool), bitorder="little")
            bits = np.concatenate([bits, np.zeros((-len(bits)) % 4, dtype=np.uint8)]).view(np.uint32)
        self._ck(self.lib.mmp_place_sweep(self.h, first_model, n, _ptr(sa), stride, _ptr(bits), _ptr(out), now_ms, seed))
        return out

    def place_one(self, dec: np.ndarray, now_ms: int, seed: int, fresh: Optional[np.ndarray] = None,
                  extra: Optional[np.ndarray] = None):
        dec = np.ascontiguousarray(dec, dtype=DECISION_IN).reshape(1)
        out = np.zeros(1, dtype=DECISION_OUT)
        fresh_a = None if fresh is None else np.ascontiguousarray(fresh, dtype=INSTANCE_ROW)
        extra_a = None if extra is None else np.ascontiguousarray(extra, dtype=np.int32)
        self._ck(self.lib.mmp_place_one(self.h, _ptr(dec), _ptr(fresh_a), _ptr(extra_a), _ptr(out), now_ms, seed))
        return out[0]

    # ---- instance-sharded multi-GPU ----
    def shard_unique_id(self) -> bytes:
        """Shard 0: the 128-byte NCCL id the host hands to its peers (any transport)."""
        buf = C.create_string_buffer(128)
        self._ck(self.lib.mmp_shard_unique_id(buf))
        return buf.raw

    def shard_connect(self, uid: bytes):
        assert len(uid) == 128
        self._ck(self.lib.mmp_shard_connect(self.h, C.c_char_p(uid)))

    def shard_words(self):
        lo, hi = C.c_int32(), C.c_int32()
        stride = self._ck(self.lib.mmp_shard_words(self.h, C.byref(lo), C.byref(hi)))
        return lo.value, hi.value, stride

    def shard_ipc_export(self, max_batch: int) -> bytes:
        """This shard's blob for the peer-access path (mmp_shard_ipc_export): exchange by any means, then shard_ipc_import."""
        buf = C.create_string_buffer(_lib.SHARD_IPC_BYTES)
        self._ck(self.lib.mmp_shard_ipc_export(self.h, int(max_batch), buf))
        return buf.raw

    def shard_ipc_import(self, blobs: Sequence[bytes]):
        """All shards' blobs ordered by shard rank (this shard's own included)."""
        raw = b"".join(blobs)
        assert len(raw) == _lib.SHARD_IPC_BYTES * len(blobs)
        self._ck(self.lib.mmp_shard_ipc_import(self.h, C.c_char_p(raw)))

    def shard_peer_stats(self):
        """{batches, remote_row_words, result_bytes_to_peers, active} of the peer-access path."""
        out = np.zeros(4, dtype=np.int64)
        self._ck(self.lib.mmp_shard_peer_stats(self.h, out.ctypes.data_as(C.c_void_p)))
        return {"batches": int(out[0]), "remote_row_words": int(out[1]), "result_bytes_to_peers": int(out[2]), "active": bool(out[3])}

    def shard_open_decisions(self) -> int:
        return int(self.lib.mmp_shard_open_decisions(self.h))

    # ---- introspection ----
    def row_words(self) -> int:
        return self._ck(self.lib.mmp_row_words(self.h))

    def live_instances(self) -> int:
        return self._ck(self.lib.mmp_live_instances(self.h))

    def cluster_order(self) -> np.ndarray:
        buf = np.zeros(self.max_instances, dtype=np.int32)
        n = self._ck(self.lib.mmp_cluster_order(self.h, _ptr(buf), len(buf)))
        return buf[:n].copy()

    def type_sets(self, type_id: int, n_idx: int):
        a = np.zeros(n_idx, dtype=np.uint8)
        p = np.zeros(n_idx, dtype=np.uint8)
        an, pn = C.c_int32(), C.c_int32()
        self._ck(self.lib.mmp_type_sets(self.h, type_id, n_idx, _ptr(a), C.byref(an), _ptr(p), C.byref(pn)))
        return (None if an.value else a.astype(bool)), (None if pn.value else p.astype(bool))

    def kernel_launches(self) -> int:
        return int(self.lib.mmp_kernel_launches(self.h))

    def instance_partition(self, idx: int) -> int:
        return int(self.lib.mmp_instance_partition(self.h, idx))

    def stats(self, cap: int = 256):
        out = np.zeros(cap, dtype=CLUSTER_STATS)
        ids = np.zeros(cap, dtype=np.int32)
        n = self._ck(self.lib.mmp_stats(self.h, _ptr(out), _ptr(ids), cap))
        return out[:n].copy(), ids[:n].copy()

    def reaper_select(self, partition: int, now_ms: int, taken: Optional[np.ndarray] = None, cap: Optional[int] = None):
        cap = cap or self.max_models
        out = np.zeros(cap, dtype=np.int32)
        n = self._ck(self.lib.mmp_reaper_select(self.h, partition, now_ms, _ptr(taken), _ptr(out), cap))
        return out[:n].copy()

    # ---- LRU ----
    def lru_init(self, capacity: np.ndarray, slots_per_instance: int):
        capacity = np.ascontiguousarray(capacity, dtype=np.int64)
        self._ck(self.lib.mmp_lru_init(self.h, len(capacity), _ptr(capacity), slots_per_instance))
        self._lru_n = len(capacity)

    def lru_apply(self, events: np.ndarray, now_ms: int, cap: Optional[int] = None) -> np.ndarray:
        events = np.ascontiguousarray(events, dtype=LRU_EVENT)
        cap = cap or max(16, 4 * len(events))
        out = np.zeros(cap, dtype=EVICTION)
        n = self._ck(self.lib.mmp_lru_apply(self.h, _ptr(events), len(events), now_ms, _ptr(out), cap))
        if n > cap:
            raise MmpError(-1, f"eviction buffer too small ({n} > {cap})")
        return out[:n].copy()

    def lru_apply_status(self, events: np.ndarray, now_ms: int, cap: Optional[int] = None):
        """mmp_lru_apply + the outcome of every MMP_LRU_LOAD event (loadLocal's admission rules)."""
        events = np.ascontiguousarray(events, dtype=LRU_EVENT)
        cap = cap or max(16, 4 * len(events))
        out = np.zeros(cap, dtype=EVICTION)
        status = np.zeros(len(events), dtype=np.int32)
        n = self._ck(self.lib.mmp_lru_apply_status(self.h, _ptr(events), len(events), now_ms, _ptr(out), cap, _ptr(status)))
        if n > cap:
            raise MmpError(-1, f"eviction buffer too small ({n} > {cap})")
        return out[:n].copy(), status

    def lru_read(self, instances: Optional[Sequence[int]] = None, used_since: int = 0):
        """mmp_lru_read: descendingMapWithCutoff(used_since) of each listed cache (None: every cache), as (offsets, entries):
        cache k's walk is entries[offsets[k]:offsets[k + 1]], most recently used first (LRU_ENTRY records)."""
        ids = None if instances is None else np.ascontiguousarray(instances, dtype=np.int32)
        n = self._lru_n if ids is None else len(ids)
        offsets = np.zeros(n + 1, dtype=np.int64)
        cap = getattr(self, "_lru_read_cap", 1024)
        while True:  # one call unless the caches grew past the last read's total
            out = np.zeros(max(cap, 1), dtype=LRU_ENTRY)
            self._ck(self.lib.mmp_lru_read(self.h, _ptr(ids), n, used_since, _ptr(offsets), _ptr(out), cap))
            if offsets[n] <= cap:
                return offsets, out[:offsets[n]].copy()
            cap = self._lru_read_cap = int(offsets[n])

    def lru_lookup(self, instance, model):
        """mmp_lru_lookup: getLastUsedTime / getWeight and the copy's load_ts for (instance, model) pairs; -1 where absent"""
        inst = np.ascontiguousarray(instance, dtype=np.int32)
        mod = np.ascontiguousarray(model, dtype=np.int32)
        assert inst.shape == mod.shape
        n = len(inst)
        last_used, weight, load_ts = np.zeros(n, dtype=np.int64), np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int64)
        self._ck(self.lib.mmp_lru_lookup(self.h, n, _ptr(inst), _ptr(mod), _ptr(last_used), _ptr(weight), _ptr(load_ts)))
        return last_used, weight, load_ts

    # ---- the closed loop (churn) ----
    def churn_init(self, load_timeout_ms: int, last_published_ms: int, slots_per_instance: int):
        cfg = ChurnConfig(load_timeout_ms, last_published_ms, slots_per_instance, 0)
        self._ck(self.lib.mmp_churn_init(self.h, C.byref(cfg)))
        self._lru_n = self.max_instances

    def churn_seed(self, instance, model, last_used, weight, load_ts, now_ms: int):
        a = [np.ascontiguousarray(instance, dtype=np.int32), np.ascontiguousarray(model, dtype=np.int32),
             np.ascontiguousarray(last_used, dtype=np.int64), np.ascontiguousarray(weight, dtype=np.int32),
             np.ascontiguousarray(load_ts, dtype=np.int64)]
        self._ck(self.lib.mmp_churn_seed(self.h, len(a[0]), _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), _ptr(a[3]), _ptr(a[4]), now_ms))

    def churn_step(self, events: np.ndarray, now0: int, now1: int, seed: int, want_rows: bool = True):
        ev = np.ascontiguousarray(events, dtype=CHURN_EVENT)
        # (a CHURN_REAPER event decides up to one load per model)
        n_rp = int(np.count_nonzero(ev["type"] == CHURN_REAPER)) * self.max_models
        cap_d = len(ev) + 65536 + n_rp
        cap_e = 4 * (len(ev) + n_rp) + 65536
        dec = np.zeros(cap_d, dtype=CHURN_DECISION)
        evi = np.zeros(cap_e, dtype=CHURN_EVICTION)
        rows = np.zeros(self.max_instances, dtype=INSTANCE_ROW) if want_rows else None
        nd, ne = C.c_int32(), C.c_int32()
        rep = ChurnReport()
        self._ck(self.lib.mmp_churn_step(self.h, _ptr(ev), len(ev), now0, now1, seed, _ptr(dec), cap_d, C.byref(nd), _ptr(evi), cap_e,
                                         C.byref(ne), _ptr(rows), C.byref(rep)))
        if nd.value > cap_d or ne.value > cap_e:
            raise MmpError(-1, "churn report buffers too small")
        return dec[:nd.value].copy(), evi[:ne.value].copy(), rows, rep

    def churn_model(self, model: int):
        row = np.zeros(1, dtype=MODEL_ROW)
        inst = np.zeros(4, dtype=np.int32)
        self._ck(self.lib.mmp_churn_model(self.h, model, _ptr(row), _ptr(inst)))
        return row[0], inst

    def churn_model_ids(self, model: int):
        """mmp_churn_model_ids: (row, every registration's instance index: the first copy_count loaded, then the failed loads)"""
        row = np.zeros(1, dtype=MODEL_ROW)
        ids = np.zeros(16, dtype=np.int32)
        n = self._ck(self.lib.mmp_churn_model_ids(self.h, model, _ptr(row), _ptr(ids), len(ids)))
        if n > len(ids):
            ids = np.zeros(n, dtype=np.int32)
            n = self._ck(self.lib.mmp_churn_model_ids(self.h, model, _ptr(row), _ptr(ids), len(ids)))
        return row[0], ids[:n].copy()

    def model_times(self, m: int, edge_ts: np.ndarray, last_unload_time: int = 0):
        ts = np.ascontiguousarray(edge_ts, dtype=np.int64)
        self._ck(self.lib.mmp_model_times(self.h, m, _ptr(ts), len(ts), int(last_unload_time)))

    def registry_prune_ids(self, self_idx: int, now_ms: int, assume_gone_ms: int, missing_since: np.ndarray, cap: int):
        """mmp_registry_prune_ids: (total, models, instances) of the first min(total, cap) pruned registrations.
        missing_since (int64[max_instances]) is updated in place."""
        assert missing_since.dtype == np.int64 and missing_since.flags.c_contiguous
        models = np.zeros(max(cap, 1), dtype=np.int32)
        inst = np.zeros(max(cap, 1), dtype=np.int32)
        n = self._ck(self.lib.mmp_registry_prune_ids(self.h, self_idx, now_ms, assume_gone_ms, _ptr(missing_since), _ptr(models),
                                                     _ptr(inst), cap))
        k = min(n, cap)
        return n, models[:k], inst[:k]

    def reaper_run(self, leader: int, now_ms: int, assume_gone_ms: int, missing_since: np.ndarray, seed: int,
                   pruned_cap: Optional[int] = None, repaired_cap: Optional[int] = None, loads_cap: Optional[int] = None):
        """mmp_reaper_run, one run of the leader's reaper task: ((models, instances) of the pruned registrations, repaired model
        ids, loads (REAPER_LOAD records), report).  Each list holds the first min(total, cap) entries; the caps default to
        room for every entry.  missing_since (int64[max_instances]) is updated in place, cleaned up as the reaper does."""
        assert missing_since.dtype == np.int64 and missing_since.flags.c_contiguous
        caps = [self.max_models * 4 if pruned_cap is None else pruned_cap, self.max_models if repaired_cap is None else repaired_cap,
                self.max_models if loads_cap is None else loads_cap]
        pm, pi = np.zeros(max(caps[0], 1), dtype=np.int32), np.zeros(max(caps[0], 1), dtype=np.int32)
        rep = np.zeros(max(caps[1], 1), dtype=np.int32)
        loads = np.zeros(max(caps[2], 1), dtype=REAPER_LOAD)
        r = ReaperReport()
        self._ck(self.lib.mmp_reaper_run(self.h, leader, now_ms, assume_gone_ms, _ptr(missing_since), seed, _ptr(pm), _ptr(pi), caps[0],
                                         _ptr(rep), caps[1], _ptr(loads), caps[2], C.byref(r)))
        k = min(r.n_pruned, caps[0])
        return (pm[:k].copy(), pi[:k].copy()), rep[:min(r.n_repaired, caps[1])].copy(), loads[:min(r.n_loads, caps[2])].copy(), r

    def janitor_run(self, self_idx: int, entries: np.ndarray, params: np.ndarray, cap: Optional[int] = None):
        """mmp_janitor_run, the registry loop of one pod's janitor task: (edits (JANITOR_EDIT records, model order), report).
        entries: JANITOR_ENTRY records of the pod's cache; params: one JANITOR_PARAMS record.  The edits hold the first
        min(n_edits, cap); without a cap every edit (a second call when they outnumber 2 x entries + 1024)."""
        assert entries.dtype == JANITOR_ENTRY and params.dtype == JANITOR_PARAMS and entries.flags.c_contiguous
        room = 2 * len(entries) + 1024 if cap is None else cap
        while True:
            edits = np.zeros(max(room, 1), dtype=JANITOR_EDIT)
            r = JanitorReport()
            self._ck(self.lib.mmp_janitor_run(self.h, self_idx, _ptr(entries), len(entries), _ptr(params), _ptr(edits), room, C.byref(r)))
            if cap is not None or r.n_edits <= room:
                return edits[:min(r.n_edits, room)].copy(), r
            room = r.n_edits

    def janitor_task(self, self_idx: int, entries: np.ndarray, params: np.ndarray, cap: Optional[int] = None):
        """mmp_janitor_task, one run of one pod's whole janitor task: (out (JANITOR_CACHE_ACTION per entry), edits
        (JANITOR_EDIT records, model order), report).  entries: JANITOR_TASK_ENTRY records of the pod's cache, most recently used
        first; params: one JANITOR_TASK_PARAMS record.  The edits hold the first min(n_edits, cap); without a cap every edit."""
        assert entries.dtype == JANITOR_TASK_ENTRY and params.dtype == JANITOR_TASK_PARAMS and entries.flags.c_contiguous
        room = 2 * len(entries) + 1024 if cap is None else cap
        while True:
            out = np.zeros(len(entries), dtype=JANITOR_CACHE_ACTION)
            edits = np.zeros(max(room, 1), dtype=JANITOR_EDIT)
            r = JanitorTaskReport()
            self._ck(self.lib.mmp_janitor_task(self.h, self_idx, _ptr(entries), len(entries), _ptr(params), _ptr(out), _ptr(edits), room,
                                               C.byref(r)))
            if cap is not None or r.registry.n_edits <= room:
                return out, edits[:min(r.registry.n_edits, room)].copy(), r
            room = r.registry.n_edits

    def rate_run(self, self_idx: int, entries: np.ndarray, params: np.ndarray, seed: int, fresh_self: Optional[np.ndarray] = None,
                 loads_cap: Optional[int] = None):
        """mmp_rate_run, one run of one pod's rate-tracking task: (out (SCALE_OUT per entry), loads (RATE_LOAD records in
        (entry, chain_pos) order), report).  entries: SCALE_IN records of the pod's cache; params: one RATE_PARAMS record;
        fresh_self: the pod's own INSTANCE_ROW or None.  The loads hold the first min(n_loads, loads_cap); without a cap
        every load (a second call when they outnumber 2 x entries + 64)."""
        assert entries.dtype == SCALE_IN and params.dtype == RATE_PARAMS and entries.flags.c_contiguous
        fr = None if fresh_self is None else np.ascontiguousarray(fresh_self, dtype=INSTANCE_ROW).reshape(1)
        room = 2 * len(entries) + 64 if loads_cap is None else loads_cap
        while True:
            out = np.zeros(len(entries), dtype=SCALE_OUT)
            loads = np.zeros(max(room, 1), dtype=RATE_LOAD)
            r = RateReport()
            self._ck(self.lib.mmp_rate_run(self.h, self_idx, _ptr(entries), len(entries), _ptr(params), _ptr(fr), seed, _ptr(out),
                                           _ptr(loads), room, C.byref(r)))
            if loads_cap is not None or r.n_loads <= room:
                return out, loads[:min(r.n_loads, room)].copy(), r
            room = r.n_loads

    def shutdown_run(self, self_idx: int, entries: np.ndarray, params: np.ndarray, seed: int, fresh_self: Optional[np.ndarray] = None,
                     out: Optional[np.ndarray] = None):
        """mmp_shutdown_run, one pod's pre-shutdown migration: (out (SHUTDOWN_ACTION per entry, entry order), report).
        entries: SHUTDOWN_ENTRY records of runtimeCache.descendingLruMap(); params: one SHUTDOWN_PARAMS record; fresh_self: the
        pod's own INSTANCE_ROW or None.  out: a caller-allocated SHUTDOWN_ACTION array of len(entries) to write into (one is
        allocated when None); a caller that runs the call often allocates it once."""
        assert entries.dtype == SHUTDOWN_ENTRY and params.dtype == SHUTDOWN_PARAMS and entries.flags.c_contiguous
        if out is None:
            out = np.zeros(len(entries), dtype=SHUTDOWN_ACTION)
        assert out.dtype == SHUTDOWN_ACTION and len(out) == len(entries) and out.flags.c_contiguous
        fr = None if fresh_self is None else np.ascontiguousarray(fresh_self, dtype=INSTANCE_ROW).reshape(1)
        r = ShutdownReport()
        self._ck(self.lib.mmp_shutdown_run(self.h, self_idx, _ptr(entries), len(entries), _ptr(params), _ptr(fr), seed, _ptr(out),
                                           C.byref(r)))
        return out, r

    def evict_run(self, self_idx: int, entries: np.ndarray, params: np.ndarray, seed: int, fresh_self: Optional[np.ndarray] = None,
                  out: Optional[np.ndarray] = None):
        """mmp_evict_run, one pod's eviction listener over a burst of evictions: (out (EVICT_ACTION per entry, entry order),
        report).  entries: EVICT_ENTRY records in listener order; params: one EVICT_PARAMS record; fresh_self: the pod's own
        INSTANCE_ROW or None.  out: a caller-allocated EVICT_ACTION array of len(entries) to write into (one is allocated when
        None); a caller that runs the call often allocates it once."""
        assert entries.dtype == EVICT_ENTRY and params.dtype == EVICT_PARAMS and entries.flags.c_contiguous
        if out is None:
            out = np.zeros(len(entries), dtype=EVICT_ACTION)
        assert out.dtype == EVICT_ACTION and len(out) == len(entries) and out.flags.c_contiguous
        fr = None if fresh_self is None else np.ascontiguousarray(fresh_self, dtype=INSTANCE_ROW).reshape(1)
        r = EvictReport()
        self._ck(self.lib.mmp_evict_run(self.h, self_idx, _ptr(entries), len(entries), _ptr(params), _ptr(fr), seed, _ptr(out),
                                        C.byref(r)))
        return out, r

    def commit_info(self):
        path, ms = C.c_int32(), C.c_double()
        self._ck(self.lib.mmp_commit_info(self.h, C.byref(path), C.byref(ms)))
        return int(path.value), float(ms.value)

    def server_stats(self):
        """The resident server (one_mode 3) since the fleet was created: {"answered": requests it answered, "fallbacks": calls
        that found every one of its MMP_SERVER_SLOTS slots taken and took the graph path, "launches": its launches,
        "max_busy": the most slots busy at once}."""
        out = np.zeros(4, dtype=np.int64)
        self._ck(self.lib.mmp_server_stats(self.h, _ptr(out)))
        return dict(zip(("answered", "fallbacks", "launches", "max_busy"), (int(v) for v in out)))

    def lru_state(self):
        n = self._lru_n
        oldest = np.zeros(n, dtype=np.int64)
        weighted = np.zeros(n, dtype=np.int64)
        count = np.zeros(n, dtype=np.int32)
        self._ck(self.lib.mmp_lru_state(self.h, n, _ptr(oldest), _ptr(weighted), _ptr(count)))
        return oldest, weighted, count


def candidates_from_masks(order: np.ndarray, best: int, mask_row: np.ndarray, include_best: bool) -> list:
    """Expand a rank-space candidate mask into the ordered list of instance indices (PLACEMENT_ORDER order)."""
    bits = np.unpackbits(mask_row.view(np.uint8), bitorder="little")
    ranks = np.nonzero(bits)[0]
    lst = [int(order[r]) for r in ranks]
    return ([int(best)] + lst) if include_best else lst
