"""ctypes binding of the CPU oracle (oracle/mm_oracle.h).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from typing import Optional, Sequence

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "_build", "libmm_oracle.so")

INST = np.dtype([("lru_time", "<i8"), ("capacity", "<i8"), ("used", "<i8"), ("start_time", "<i8"), ("vers", "<i8"),
                 ("count", "<i4"), ("l_threads", "<i4"), ("l_in_prog", "<i4"), ("rpm", "<i4"), ("shutting_down", "<i4"),
                 ("active", "<i4")], align=True)
STATS = np.dtype([("total_capacity", "<i8"), ("total_free", "<i8"), ("global_lru", "<i8"), ("instance_count", "<i4"),
                  ("model_copy_count", "<i4")], align=True)
DECISION = np.dtype([("type_idx", "<i4"), ("self", "<i4"), ("fresh_idx", "<i4"), ("favour_self", "<i4"),
                     ("last_used", "<i8"), ("decision_id", "<u8")], align=True)
RESULT = np.dtype([("target", "<i4"), ("n_candidates", "<i4"), ("n_remaining", "<i4"), ("pick_index", "<i4"),
                   ("best", "<i4"), ("flags", "<i4")], align=True)
LRU_EVENT = np.dtype([("op", "<i4"), ("key", "<i4"), ("weight", "<i8"), ("last_used", "<i8")], align=True)
EVICTION = np.dtype([("key", "<i4"), ("event", "<i4"), ("last_used", "<i8"), ("weight", "<i8")], align=True)
MODEL = np.dtype([("last_used", "<i8"), ("type_idx", "<i4"), ("n_loaded", "<i4"), ("n_failed", "<i4"), ("pad", "<i4")],
                 align=True)
SIM_MODEL = np.dtype([("last_used", "<i8"), ("type_idx", "<i4"), ("size_units", "<i4")], align=True)
SIM_EVENT = np.dtype([("type", "<i4"), ("model", "<i4"), ("caller", "<i4"), ("u", "<u4"), ("t", "<i8")], align=True)
SIM_DECISION = np.dtype([("model", "<i4"), ("self", "<i4"), ("target", "<i4"), ("n_candidates", "<i4"), ("status", "<i4"),
                         ("event", "<i4")], align=True)
SIM_EVICTION = np.dtype([("instance", "<i4"), ("model", "<i4"), ("last_used", "<i8"), ("weight", "<i4"), ("order", "<i4"),
                         ("reload", "<i4")], align=True)
assert INST.itemsize == 64 and DECISION.itemsize == 32 and RESULT.itemsize == 24 and MODEL.itemsize == 24
assert SIM_MODEL.itemsize == 16 and SIM_EVENT.itemsize == 24 and SIM_DECISION.itemsize == 24 and SIM_EVICTION.itemsize == 32
SCALE_IN = np.dtype([("instance", "<i4"), ("model", "<i4"), ("count", "<i8"), ("last_used", "<i8"), ("last_heavy", "<i8"), ("i1", "<i4"),
                     ("i2", "<i4"), ("weight", "<i4"), ("flags", "<i4")], align=True)
SCALE_PARAMS = np.dtype([("now", "<i8"), ("last_check_time", "<i8"), ("iteration", "<i4"), ("scale_up_rpm_threshold", "<i4"),
                         ("second_copy_min_age_iters", "<i4"), ("second_copy_max_age_iters", "<i4"), ("second_copy_lru_threshold_ms", "<i8"),
                         ("rate_check_interval_ms", "<i8"), ("assume_completed_ms", "<i8"), ("second_copy_remove_max_age_ms", "<i8"),
                         ("can_remove", "<i4"), ("pad", "<i4")], align=True)
SCALE_OUT = np.dtype([("action", "<i4"), ("copies_to_load", "<i4"), ("load_last_used", "<i8"), ("rpm", "<i4"), ("i1", "<i4"), ("i2", "<i4"),
                      ("set_heavy", "<i4"), ("remove", "<i4")], align=True)
assert SCALE_IN.itemsize == 48 and SCALE_PARAMS.itemsize == 72 and SCALE_OUT.itemsize == 40
SIM_REQUEST, SIM_REMOVE = 0, 1
(SIM_ACCEPTED, SIM_NOWHERE, SIM_CHURN, SIM_FALLTHRU, SIM_EARLY, SIM_GROW_EVICTED, SIM_EXISTS, SIM_SKIPPED, SIM_INVALID,
 SIM_EVICTED_LATER) = range(10)

NONE, SELF = -1, -2
ADDED, UPDATED, DELETED = 0, 1, 2


def build(force: bool = False) -> str:
    if force or not os.path.exists(SO) or any(
            os.path.getmtime(os.path.join(HERE, f)) > os.path.getmtime(SO) for f in ("mm_oracle.cpp", "mm_sim.inc", "mm_oracle.h")):
        subprocess.check_call(["make", "-C", HERE, "-s"])
    return SO


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(SO):
            build()
        L = C.CDLL(SO)
        P, I32, I64, U64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64
        STRS = C.POINTER(C.c_char_p)
        sig = {
            "orc_create": (P, [I64, I64, I32]), "orc_destroy": (None, [P]),
            "orc_instance_event": (C.c_int, [P, C.c_int, I32, P, C.c_char_p, C.c_char_p, C.c_char_p, STRS, I32, I64]),
            "orc_set_active": (C.c_int, [P, I32, I32]),
            "orc_bulk_add": (C.c_int, [P, I32, P, STRS, STRS, STRS, P, STRS]),
            "orc_types_set": (C.c_int, [P, I32, STRS, P, STRS, P, STRS]),
            "orc_tc_converge": (C.c_int, [P]),
            "orc_tc_defer_refresh": (C.c_int, [P, C.c_int]),
            "orc_set_replaced_replicasets": (C.c_int, [P, STRS, I32]),
            "orc_get_replaced_replicasets": (C.c_int, [P, C.c_char_p, I32]),
            "orc_type_sets": (C.c_int, [P, C.c_char_p, I32, P, C.POINTER(I32), P, C.POINTER(I32)]),
            "orc_cluster_order": (C.c_int, [P, P, I32]), "orc_compare": (C.c_int, [P, I32, I32]),
            "orc_cluster_stats": (C.c_int, [P, P]), "orc_partition_stats": (C.c_int, [P, P, P, I32]),
            "orc_instance_partition": (C.c_int, [P, I32]), "orc_type_stats": (C.c_int, [P, C.c_char_p, P]),
            "orc_get_next_batch": (I64, [P, I32, P, STRS, I32, P, I32, P, P, I64, U64, I32, P, P, P, P, P, I64]),
            "orc_get_next_batch_dense": (I64, [P, I32, P, STRS, I32, P, I32, P, P, I64, U64, I32, P]),
            "orc_lru_create": (P, [I64]), "orc_lru_destroy": (None, [P]),
            "orc_lru_apply": (I64, [P, P, I64, I64, P, I64]), "orc_lru_oldest_time": (I64, [P]),
            "orc_lru_weighted_size": (I64, [P]), "orc_lru_size": (I64, [P]), "orc_lru_dump": (I64, [P, P, P, P, I64]),
            "orc_unload_reserve_units": (I64, [I64, I32, I32]), "orc_min_space_units": (I64, [I64, I32, I32, I32]),
            "orc_churn_reject": (C.c_int, [I64, I64, I64, I64, I64, I64]),
            "orc_early_reject": (C.c_int, [I64, I64, I64, I64, I64]),
            "orc_reaper_select": (I64, [P, I32, P, STRS, I32, I32, I64, P, P, I64]),
            "orc_hash64": (U64, [U64, U64]),
            "orc_sim_create": (P, [P, I32, P, STRS, I32, P, P, P, I32, P, I64, I64]), "orc_sim_destroy": (None, [P]),
            "orc_sim_seed": (C.c_int, [P, I32, I32, P, P, P, P, I64]),
            "orc_sim_step": (I64, [P, P, I32, I64, I64, U64, P, I32, C.POINTER(I32), P, I32, C.POINTER(I32), P, C.POINTER(I32)]),
            "orc_sim_model_copies": (I64, [P, I32, P, I32, C.POINTER(I64)]),
            "orc_sim_lru_state": (I64, [P, I32, C.POINTER(I64), C.POINTER(I64), C.POINTER(I64)]),
            "orc_sim_coalesced": (I64, [P]),
            "orc_second_copy_trigger": (C.c_int, [C.POINTER(I32), C.POINTER(I32), I32, I32, I32, I64, I64, I64, I64, I64]),
            "orc_scaleup_copies": (I32, [I64, I64, I32, I32, I32, I32, I32, I32, I32, C.POINTER(I32)]),
            "orc_scaleup_exclude_set": (I32, [P, I32, I32, I32, P, I32]),
            "orc_loaded_since": (C.c_int, [P, P, I32, I64, I32]),
            "orc_rate_task_eval": (C.c_int, [P, I32, P, P, STRS, I32, P, P, P, P, P, P]),
            "orc_janitor_eval": (C.c_int, [P, I32, P, P, P, P, P, P, P, P]),
            "orc_prune_missing": (I32, [P, I32, P, P, I32, I64, I64, P, P]),
            "orc_scale_down": (C.c_int, [P, I32, P, P, I32, I64, I64, I64, I64, I64, I64, I32, I64, I64, I32]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _strs(items: Sequence[str]):
    arr = (C.c_char_p * max(1, len(items)))()
    for i, s in enumerate(items):
        arr[i] = s.encode("utf-8")
    return arr


class OracleFleet:
    """Event-driven restatement of ModelMesh's instance table + TypeConstraintManager + CacheMissForwardingLB."""

    def __init__(self, min_space_units: int, min_churn_age_ms: int, default_model_size_units: int):
        self.L = lib()
        self.h = C.c_void_p(self.L.orc_create(min_space_units, min_churn_age_ms, default_model_size_units))

    def close(self):
        if self.h:
            self.L.orc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def instance_event(self, etype: int, idx: int, row: Optional[np.ndarray], iid: str, loc=None, zone=None, labels=(),
                       now_ms: int = 0):
        labels = list(labels)
        r = None if row is None else np.ascontiguousarray(row, dtype=INST).reshape(1)
        rc = self.L.orc_instance_event(self.h, etype, idx, _ptr(r), iid.encode(), None if loc is None else loc.encode(),
                                       None if zone is None else zone.encode(), _strs(labels), len(labels), now_ms)
        assert rc == 0

    def bulk_add(self, rows: np.ndarray, ids, locs, zones, labels):
        rows = np.ascontiguousarray(rows, dtype=INST)
        n = len(rows)
        off = np.zeros(n + 1, dtype=np.int32)
        flat = []
        for i, l in enumerate(labels):
            flat += list(l)
            off[i + 1] = len(flat)

        def opt(items):
            arr = (C.c_char_p * max(1, n))()
            for i, s_ in enumerate(items):
                arr[i] = None if s_ is None else s_.encode("utf-8")
            return arr
        assert self.L.orc_bulk_add(self.h, n, _ptr(rows), _strs(ids), opt(locs), opt(zones), _ptr(off), _strs(flat)) == 0

    def set_active(self, idx: int, active: bool):
        assert self.L.orc_set_active(self.h, idx, int(active)) == 0

    def types_set(self, config: Optional[dict]):
        """config: {type: {"required": [...], "preferred": [...]}} or None (typeConstraints == null)."""
        if config is None:
            assert self.L.orc_types_set(self.h, -1, None, None, None, None, None) == 0
            return
        names = list(config.keys())
        req_off, pref_off, req, pref = [0], [0], [], []
        for t in names:
            req += list(config[t].get("required") or [])
            pref += list(config[t].get("preferred") or [])
            req_off.append(len(req))
            pref_off.append(len(pref))
        ro, po = np.asarray(req_off, dtype=np.int32), np.asarray(pref_off, dtype=np.int32)
        assert self.L.orc_types_set(self.h, len(names), _strs(names), _ptr(ro), _strs(req), _ptr(po), _strs(pref)) == 0

    def tc_defer_refresh(self, defer: bool):
        assert self.L.orc_tc_defer_refresh(self.h, int(defer)) == 0

    def tc_converge(self):
        assert self.L.orc_tc_converge(self.h) == 0

    def set_replaced_replicasets(self, prefixes: Sequence[str]):
        assert self.L.orc_set_replaced_replicasets(self.h, _strs(prefixes), len(prefixes)) == 0

    def get_replaced_replicasets(self):
        buf = C.create_string_buffer(4096)
        n = self.L.orc_get_replaced_replicasets(self.h, buf, 4096)
        return sorted(x for x in buf.value.decode().split(",") if x) if n else []

    def type_sets(self, type_name: str, n_idx: int):
        a = np.zeros(n_idx, dtype=np.uint8)
        p = np.zeros(n_idx, dtype=np.uint8)
        an, pn = C.c_int32(), C.c_int32()
        assert self.L.orc_type_sets(self.h, type_name.encode(), n_idx, _ptr(a), C.byref(an), _ptr(p), C.byref(pn)) == 0
        return (None if an.value else a.astype(bool)), (None if pn.value else p.astype(bool))

    def cluster_order(self, cap: int = 1 << 17) -> np.ndarray:
        buf = np.zeros(cap, dtype=np.int32)
        n = self.L.orc_cluster_order(self.h, _ptr(buf), cap)
        return buf[:n].copy()

    def compare(self, a: int, b: int) -> int:
        return int(self.L.orc_compare(self.h, a, b))

    def cluster_stats(self) -> np.ndarray:
        s = np.zeros(1, dtype=STATS)
        assert self.L.orc_cluster_stats(self.h, _ptr(s)) == 0
        return s[0]

    def partition_stats(self, cap: int = 256):
        s = np.zeros(cap, dtype=STATS)
        ids = np.zeros(cap, dtype=np.int32)
        n = self.L.orc_partition_stats(self.h, _ptr(s), _ptr(ids), cap)
        return s[:n].copy(), ids[:n].copy()

    def instance_partition(self, idx: int) -> int:
        return int(self.L.orc_instance_partition(self.h, idx))

    def type_stats(self, type_name: str) -> np.ndarray:
        s = np.zeros(1, dtype=STATS)
        assert self.L.orc_type_stats(self.h, type_name.encode(), _ptr(s)) == 0
        return s[0]

    def get_next_batch(self, dec: np.ndarray, type_names: Sequence[str], excl_off: np.ndarray, excl_idx: np.ndarray,
                       now_ms: int, seed: int, fresh: Optional[np.ndarray] = None, threads: int = 1,
                       want_candidates: bool = False, cand_cap: Optional[int] = None, dense: bool = False):
        dec = np.ascontiguousarray(dec, dtype=DECISION)
        n = len(dec)
        excl_off = np.ascontiguousarray(excl_off, dtype=np.int64)
        excl_idx = np.ascontiguousarray(excl_idx, dtype=np.int32)
        fresh_a = None if fresh is None else np.ascontiguousarray(fresh, dtype=INST)
        out = np.zeros(n, dtype=RESULT)
        if dense:  # CPU-baseline mode (ii): entries through a rank-ordered array
            rc = self.L.orc_get_next_batch_dense(self.h, n, _ptr(dec), _strs(type_names), len(type_names), _ptr(fresh_a),
                                                 0 if fresh_a is None else len(fresh_a), _ptr(excl_off), _ptr(excl_idx), now_ms, seed,
                                                 threads, _ptr(out))
            assert rc >= 0, rc
            return out
        if not want_candidates:
            rc = self.L.orc_get_next_batch(self.h, n, _ptr(dec), _strs(type_names), len(type_names), _ptr(fresh_a),
                                           0 if fresh_a is None else len(fresh_a), _ptr(excl_off), _ptr(excl_idx),
                                           now_ms, seed, threads, _ptr(out), None, None, None, None, 0)
            assert rc >= 0, rc
            return out
        cap = cand_cap or (1 << 22)
        while True:
            off = np.zeros(n + 1, dtype=np.int64)
            ci = np.zeros(cap, dtype=np.int32)
            cl = np.zeros(cap, dtype=np.int32)
            ck = np.zeros(cap, dtype=np.uint8)
            rc = self.L.orc_get_next_batch(self.h, n, _ptr(dec), _strs(type_names), len(type_names), _ptr(fresh_a),
                                           0 if fresh_a is None else len(fresh_a), _ptr(excl_off), _ptr(excl_idx),
                                           now_ms, seed, 1, _ptr(out), _ptr(off), _ptr(ci), _ptr(cl), _ptr(ck), cap)
            assert rc >= 0, rc
            if rc <= cap:
                return out, off, ci[:rc], cl[:rc], ck[:rc]
            cap = int(rc)

    def reaper_select(self, models: np.ndarray, type_names: Sequence[str], part_id: int, now_ms: int,
                      taken: Optional[np.ndarray] = None) -> np.ndarray:
        models = np.ascontiguousarray(models, dtype=MODEL)
        out = np.zeros(len(models), dtype=np.int32)
        n = self.L.orc_reaper_select(self.h, len(models), _ptr(models), _strs(type_names), len(type_names), part_id,
                                     now_ms, _ptr(taken), _ptr(out), len(out))
        assert n >= 0, n
        return out[:n].copy()


class OracleLru:
    def __init__(self, capacity: int):
        self.L = lib()
        self.h = C.c_void_p(self.L.orc_lru_create(capacity))

    def __del__(self):
        try:
            if self.h:
                self.L.orc_lru_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def apply(self, events: np.ndarray, now_ms: int) -> np.ndarray:
        events = np.ascontiguousarray(events, dtype=LRU_EVENT)
        cap = max(16, 4 * len(events)) + self.size()  # evictions <= resident entries + inserts
        out = np.zeros(cap, dtype=EVICTION)
        n = self.L.orc_lru_apply(self.h, _ptr(events), len(events), now_ms, _ptr(out), cap)
        assert 0 <= n <= cap
        return out[:n].copy()

    def oldest_time(self) -> int:
        return int(self.L.orc_lru_oldest_time(self.h))

    def weighted_size(self) -> int:
        return int(self.L.orc_lru_weighted_size(self.h))

    def size(self) -> int:
        return int(self.L.orc_lru_size(self.h))

    def dump(self):
        n = self.size()
        k = np.zeros(n, dtype=np.int32)
        t = np.zeros(n, dtype=np.int64)
        w = np.zeros(n, dtype=np.int64)
        self.L.orc_lru_dump(self.h, _ptr(k), _ptr(t), _ptr(w), n)
        return k, t, w


class OracleSim:
    """The closed loop (oracle/mm_sim.inc): one call of step() = one republish window of the whole fleet."""

    def __init__(self, fleet: OracleFleet, models: np.ndarray, type_names: Sequence[str], edge_off: np.ndarray,
                 edge_inst: np.ndarray, n_loaded: np.ndarray, capacity: np.ndarray, load_timeout_ms: int,
                 last_published_ms: int):
        self.L = lib()
        self.fleet = fleet  # keep alive
        models = np.ascontiguousarray(models, dtype=SIM_MODEL)
        self.n_models, self.n_instances = len(models), len(capacity)
        edge_off = np.ascontiguousarray(edge_off, dtype=np.int64)
        edge_inst = np.ascontiguousarray(edge_inst, dtype=np.int32)
        n_loaded = np.ascontiguousarray(n_loaded, dtype=np.int32)
        capacity = np.ascontiguousarray(capacity, dtype=np.int64)
        self.h = C.c_void_p(self.L.orc_sim_create(fleet.h, len(models), _ptr(models), _strs(type_names), len(type_names),
                                                   _ptr(edge_off), _ptr(edge_inst), _ptr(n_loaded), len(capacity),
                                                   _ptr(capacity), load_timeout_ms, last_published_ms))
        assert self.h

    def __del__(self):
        try:
            if self.h:
                self.L.orc_sim_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def seed(self, instance: int, model, last_used, weight, load_ts, now_ms: int):
        m = np.ascontiguousarray(model, dtype=np.int32)
        lu = np.ascontiguousarray(last_used, dtype=np.int64)
        w = np.ascontiguousarray(weight, dtype=np.int32)
        lt = np.ascontiguousarray(load_ts, dtype=np.int64)
        rc = self.L.orc_sim_seed(self.h, instance, len(m), _ptr(m), _ptr(lu), _ptr(w), _ptr(lt), now_ms)
        assert rc == 0, rc

    def step(self, events: np.ndarray, now0: int, now1: int, seed: int):
        ev = np.ascontiguousarray(events, dtype=SIM_EVENT)
        cap_d = len(ev) + 65536
        cap_e = 4 * len(ev) + 65536
        dec = np.zeros(cap_d, dtype=SIM_DECISION)
        evi = np.zeros(cap_e, dtype=SIM_EVICTION)
        rows = np.zeros(self.n_instances, dtype=INST)
        nd, ne, npub = C.c_int32(), C.c_int32(), C.c_int32()
        carry = self.L.orc_sim_step(self.h, _ptr(ev), len(ev), now0, now1, seed, _ptr(dec), cap_d, C.byref(nd), _ptr(evi), cap_e,
                                    C.byref(ne), _ptr(rows), C.byref(npub))
        assert carry >= 0 and nd.value <= cap_d and ne.value <= cap_e
        return dec[:nd.value].copy(), evi[:ne.value].copy(), rows, int(npub.value), int(carry)

    def model_copies(self, model: int):
        out = np.zeros(64, dtype=np.int32)
        lu = C.c_int64()
        n = self.L.orc_sim_model_copies(self.h, model, _ptr(out), 64, C.byref(lu))
        return out[:n].copy(), int(lu.value)

    def lru_state(self, instance: int):
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        assert self.L.orc_sim_lru_state(self.h, instance, C.byref(a), C.byref(b), C.byref(c)) == 0
        return int(a.value), int(b.value), int(c.value)

    def coalesced(self) -> int:
        return int(self.L.orc_sim_coalesced(self.h))
