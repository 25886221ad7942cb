"""ctypes binding of the libmmplace C ABI (include/mmplace.h).

The shipped library is ``modelmesh_b200/csrc/libmmplace.so`` (built by ``__graft_entry__.build()`` /
``python -m modelmesh_b200.build``).  There is no CPU implementation behind this package: ``load_product()`` raises if
the CUDA library has not been built, and ``mmp_fleet_create`` fails with MMP_E_CUDA when no device is usable.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PRODUCT_SO = os.path.join(HERE, "csrc", "libmmplace.so")

# numpy mirrors of the C structs (include/mmplace.h); itemsize is asserted against the header's layout in tests
INSTANCE_ROW = np.dtype(
    [("lru_time", "<i8"), ("capacity", "<i8"), ("used", "<i8"), ("start_time", "<i8"), ("vers", "<i8"),
     ("count", "<i4"), ("l_threads", "<i4"), ("l_in_prog", "<i4"), ("rpm", "<i4"), ("shutting_down", "<i4"),
     ("active", "<i4")], align=True)
MODEL_ROW = np.dtype(
    [("last_used", "<i8"), ("size_units", "<i4"), ("rpm", "<i4"), ("type_id", "<u2"), ("copy_count", "u1"),
     ("fail_count", "u1"), ("reserved", "<u4")], align=True)
DECISION_IN = np.dtype(
    [("model", "<i4"), ("self", "<i4"), ("last_used", "<i8"), ("flags", "<u4"), ("fresh", "<i4"),
     ("extra_off", "<i4"), ("extra_n", "<i4")], align=True)
DECISION_OUT = np.dtype([("target", "<i4"), ("n_candidates", "<i4")], align=True)
DECISION_TRACE = np.dtype(
    [("best", "<i4"), ("n_remaining", "<i4"), ("pick_index", "<i4"), ("flags", "<i4"), ("cut_rank", "<i4"),
     ("best_rank", "<i4"), ("reserved", "<i4", (2,))], align=True)
CLUSTER_STATS = np.dtype(
    [("total_capacity", "<i8"), ("total_free", "<i8"), ("global_lru", "<i8"), ("instance_count", "<i4"),
     ("model_copy_count", "<i4")], align=True)
LRU_EVENT = np.dtype([("op", "<i4"), ("instance", "<i4"), ("model", "<i4"), ("weight", "<i4"), ("last_used", "<i8")],
                     align=True)
EVICTION = np.dtype([("instance", "<i4"), ("model", "<i4"), ("last_used", "<i8"), ("weight", "<i4"), ("event", "<i4")],
                    align=True)
assert INSTANCE_ROW.itemsize == 64 and MODEL_ROW.itemsize == 24 and DECISION_IN.itemsize == 32
assert DECISION_OUT.itemsize == 8 and DECISION_TRACE.itemsize == 32 and CLUSTER_STATS.itemsize == 32
CHURN_EVENT = np.dtype([("type", "<i4"), ("model", "<i4"), ("caller", "<i4"), ("u", "<u4"), ("t", "<i8")], align=True)
CHURN_DECISION = np.dtype([("model", "<i4"), ("self", "<i4"), ("target", "<i4"), ("n_candidates", "<i4"), ("status", "<i4"),
                           ("event", "<i4")], align=True)
CHURN_EVICTION = np.dtype([("instance", "<i4"), ("model", "<i4"), ("last_used", "<i8"), ("weight", "<i4"), ("order", "<i4"),
                           ("reload", "<i4")], align=True)
LRU_ENTRY = np.dtype([("model", "<i4"), ("weight", "<i4"), ("last_used", "<i8"), ("load_ts", "<i8")], align=True)
assert LRU_EVENT.itemsize == 24 and EVICTION.itemsize == 24 and LRU_ENTRY.itemsize == 24
assert CHURN_EVENT.itemsize == 24 and CHURN_DECISION.itemsize == 24 and CHURN_EVICTION.itemsize == 32
SCALE_IN = np.dtype([("instance", "<i4"), ("model", "<i4"), ("count", "<i8"), ("last_used", "<i8"), ("last_heavy", "<i8"), ("i1", "<i4"),
                     ("i2", "<i4"), ("weight", "<i4"), ("flags", "<i4")], align=True)
SCALE_PARAMS = np.dtype([("now", "<i8"), ("last_check_time", "<i8"), ("iteration", "<i4"), ("scale_up_rpm_threshold", "<i4"),
                         ("second_copy_min_age_iters", "<i4"), ("second_copy_max_age_iters", "<i4"), ("second_copy_lru_threshold_ms", "<i8"),
                         ("rate_check_interval_ms", "<i8"), ("assume_completed_ms", "<i8"), ("second_copy_remove_max_age_ms", "<i8"),
                         ("can_remove", "<i4"), ("reserved", "<i4")], align=True)
SCALE_OUT = np.dtype([("action", "<i4"), ("copies_to_load", "<i4"), ("load_last_used", "<i8"), ("rpm", "<i4"), ("i1", "<i4"), ("i2", "<i4"),
                      ("set_heavy", "<i4"), ("remove", "<i4")], align=True)
assert SCALE_IN.itemsize == 48 and SCALE_PARAMS.itemsize == 72 and SCALE_OUT.itemsize == 40
REAPER_LOAD = np.dtype([("model", "<i4"), ("target", "<i4"), ("n_candidates", "<i4"), ("reserved", "<i4"), ("last_used", "<i8")],
                       align=True)
assert REAPER_LOAD.itemsize == 24
JANITOR_FAILED = 1
JE_UNREGISTER, JE_DROP_FAILURE, JE_REMOVE_LOCAL, JE_SCALE_DOWN, JE_UNDECIDED = 1, 2, 4, 8, 16
JANITOR_ENTRY = np.dtype([("model", "<i4"), ("weight", "<i4"), ("last_used", "<i8"), ("load_ts", "<i8"), ("last_heavy", "<i8"),
                          ("count", "<i8"), ("flags", "<u4"), ("reserved", "<u4")], align=True)
JANITOR_PARAMS = np.dtype([("scale", SCALE_PARAMS), ("load_failure_expiry_ms", "<i8"), ("adjusted_capacity", "<i8"), ("flags", "<u4"),
                           ("reserved", "<u4")], align=True)
JANITOR_EDIT = np.dtype([("model", "<i4"), ("what", "<u4"), ("last_used", "<i8"), ("last_unload_time", "<i8")], align=True)
assert JANITOR_ENTRY.itemsize == 48 and JANITOR_PARAMS.itemsize == 96 and JANITOR_EDIT.itemsize == 24
JANITOR_NOT_DONE, JANITOR_NOT_LIVE, JANITOR_UNLOAD_RECENT = 2, 4, 8
JANITOR_TASK_ENTRY = np.dtype([("e", JANITOR_ENTRY), ("load_complete_ts", "<i8")], align=True)
JANITOR_TASK_PARAMS = np.dtype([("janitor", JANITOR_PARAMS), ("min_stale_age_ms", "<i8"), ("janitor_freq_secs", "<i8"),
                                ("load_timeout_ms", "<i8")], align=True)
JANITOR_CACHE_ACTION = np.dtype([("model", "<i4"), ("what", "<u4"), ("last_used", "<i8"), ("replaced_ts", "<i8")], align=True)
assert JANITOR_TASK_ENTRY.itemsize == 56 and JANITOR_TASK_PARAMS.itemsize == 120 and JANITOR_CACHE_ACTION.itemsize == 24
JC_NOT_DONE, JC_NOT_CACHED, JC_OUT_OF_ORDER, JC_STOP, JC_REPAIR = 1, 2, 4, 8, 16
JC_NOT_REACHED, JC_STALE_UPDATE, JC_REMOVE, JC_REREGISTER, JC_UNDECIDED = 32, 64, 128, 256, 512
RATE_PARAMS = np.dtype([("scale", SCALE_PARAMS), ("load_failure_expiry_ms", "<i8")], align=True)
RATE_LOAD = np.dtype([("entry", "<i4"), ("model", "<i4"), ("chain_pos", "<i4"), ("self", "<i4"), ("target", "<i4"), ("n_candidates", "<i4"),
                      ("last_used", "<i8"), ("flags", "<u4"), ("remaining", "<u4")], align=True)
assert RATE_PARAMS.itemsize == 80 and RATE_LOAD.itemsize == 40
RL_SECOND_COPY, RL_CHAIN_CUT = 1, 2
RATE_RAN, RATE_TOO_SOON, RATE_FEW_INSTANCES, RATE_NO_ENTRIES = 0, 1, 2, 3
RATE_CHAIN_MAX = 17   # decisions one chain places: decision j carries the j targets before it as extras (MAX_EXTRA)
SHUTDOWN_ENTRY = np.dtype([("model", "<i4"), ("flags", "<u4"), ("lru_t", "<i8"), ("last_used", "<i8")], align=True)
SHUTDOWN_PARAMS = np.dtype([("now", "<i8"), ("cutoff_age_ms", "<i8"), ("load_failure_expiry_ms", "<i8")], align=True)
SHUTDOWN_ACTION = np.dtype([("model", "<i4"), ("what", "<u4"), ("target", "<i4"), ("n_candidates", "<i4"), ("last_used", "<i8")],
                           align=True)
assert SHUTDOWN_ENTRY.itemsize == 24 and SHUTDOWN_PARAMS.itemsize == 24 and SHUTDOWN_ACTION.itemsize == 24
SD_ENTRY_GONE, SD_ENTRY_FAILED, SD_ENTRY_ABORTED = 1, 2, 4
SD_NOT_REGISTERED, SD_STALE, SD_REMOVE_LOCAL, SD_DEREGISTER_NOW, SD_PLACED, SD_REFUSED, SD_WAIT, SD_UNDECIDED = 1, 2, 4, 8, 16, 32, 64, 128
EVICT_ENTRY = np.dtype([("model", "<i4"), ("flags", "<u4"), ("last_used", "<i8"), ("load_ts", "<i8"), ("load_complete_ts", "<i8")],
                       align=True)
EVICT_PARAMS = np.dtype([("now", "<i8"), ("load_timeout_ms", "<i8"), ("load_failure_expiry_ms", "<i8")], align=True)
EVICT_ACTION = np.dtype([("model", "<i4"), ("what", "<u4"), ("target", "<i4"), ("n_candidates", "<i4"), ("last_used", "<i8"),
                         ("last_unload_time", "<i8")], align=True)
assert EVICT_ENTRY.itemsize == 32 and EVICT_PARAMS.itemsize == 24 and EVICT_ACTION.itemsize == 32
EV_ENTRY_FAILED = 1
EV_UNREGISTER, EV_DROP_FAILURE, EV_RELOAD, EV_CLUSTER_FULL, EV_LOADED_ELSEWHERE, EV_REFUSED, EV_PLACED, EV_UNDECIDED = 1, 2, 4, 8, 16, 32, 64, 128
LRU_LOAD = 5
CHURN_REQUEST, CHURN_REMOVE, CHURN_REAPER = 0, 1, 2


class ChurnConfig(C.Structure):
    _fields_ = [("load_timeout_ms", C.c_int64), ("last_published_ms", C.c_int64), ("slots_per_instance", C.c_int32),
                ("reserved", C.c_int32)]


class ChurnReport(C.Structure):
    _fields_ = [("n_published", C.c_int32), ("n_carry", C.c_int32), ("n_coalesced", C.c_int32), ("n_lru_events", C.c_int32),
                ("ms_classify", C.c_float), ("ms_place", C.c_float), ("ms_route", C.c_float), ("ms_apply", C.c_float),
                ("ms_registry", C.c_float), ("ms_commit", C.c_float), ("ms_total", C.c_float), ("ms_reaper", C.c_float)]

class ReaperReport(C.Structure):
    _fields_ = [("n_pruned", C.c_int32), ("n_repaired", C.c_int32), ("n_loads", C.c_int32), ("stopped_partition", C.c_int32)]


class JanitorReport(C.Structure):
    _fields_ = [("n_referencing", C.c_int32), ("n_edits", C.c_int32), ("n_candidates", C.c_int32), ("n_removed", C.c_int32),
                ("weight_removed", C.c_int64)]


class JanitorTaskReport(C.Structure):
    _fields_ = [("n_not_done", C.c_int32), ("n_not_cached", C.c_int32), ("n_out_of_order", C.c_int32), ("n_stop", C.c_int32),
                ("n_repair", C.c_int32), ("n_not_reached", C.c_int32), ("n_stale_update", C.c_int32), ("n_remove", C.c_int32),
                ("n_reregister", C.c_int32), ("n_undecided", C.c_int32), ("stopped_at", C.c_int32), ("registry_ran", C.c_int32),
                ("cache_changed", C.c_int32), ("reserved", C.c_int32), ("registry", JanitorReport)]


assert C.sizeof(JanitorTaskReport) == 80


class RateReport(C.Structure):
    _fields_ = [("gate", C.c_int32), ("n_second", C.c_int32), ("n_scale_up", C.c_int32), ("n_loads", C.c_int32), ("n_heavy", C.c_int32),
                ("n_chains_cut", C.c_int32), ("n_refused_failures", C.c_int32), ("reserved", C.c_int32)]


class ShutdownReport(C.Structure):
    _fields_ = [("found_other", C.c_int32), ("n_registered", C.c_int32), ("will_be_skipped", C.c_int32), ("n_placed", C.c_int32),
                ("n_none", C.c_int32), ("n_refused", C.c_int32), ("n_wait", C.c_int32), ("reserved", C.c_int32)]


class EvictReport(C.Structure):
    _fields_ = [("n_unregister", C.c_int32), ("n_drop_failure", C.c_int32), ("n_reload", C.c_int32), ("n_cluster_full", C.c_int32),
                ("n_loaded_elsewhere", C.c_int32), ("n_refused", C.c_int32), ("n_placed", C.c_int32), ("n_none", C.c_int32)]


DF_FAVOUR_SELF = 1
DF_MODEL_LAST_USED = 2
DF_OWN_ID = 4
DF_REQUEST_MODEL = 8  # model = type id, the model's loaded ∪ failed instances in extra[] (MMP_DF_REQUEST_MODEL)
MAX_EXTRA = 16
TARGET_NONE = -1
TARGET_SELF = -2
TARGET_INVALID = -3
TF_RS_RETRY, TF_SIMPLE, TF_BEST_FULL, TF_FAVOUR_EXIT = 1, 2, 4, 8
TF_KEEP_BEST, TF_KEEP_OTHERS, TF_KEEP_SELF, TF_PREF_B = 16, 32, 64, 128

E_ARG, E_CUDA, E_NCCL, E_EPOCH, E_NOMEM, E_STATE = -1, -2, -3, -4, -5, -6


class MmpConfig(C.Structure):
    _fields_ = [("min_space_units", C.c_int64), ("min_churn_age_ms", C.c_int64),
                ("default_model_size_units", C.c_int32), ("max_instances", C.c_int32), ("max_models", C.c_int32),
                ("device", C.c_int32), ("shard_rank", C.c_int32), ("shard_count", C.c_int32), ("flags", C.c_uint32),
                ("reserved", C.c_uint32)]


# every symbol include/mmplace.h declares: (name, restype, argtypes)
_P = C.c_void_p
_I32, _I64, _U64 = C.c_int32, C.c_int64, C.c_uint64
_STRS = C.POINTER(C.c_char_p)
SYMBOLS = [
    ("mmp_abi_version", _I32, []),
    ("mmp_fleet_create", _I32, [C.POINTER(MmpConfig), C.POINTER(_P)]),
    ("mmp_fleet_destroy", None, [_P]),
    ("mmp_last_error", C.c_char_p, [_P]),
    ("mmp_instance_upsert", _I32, [_P, _I32, _P, C.c_char_p, C.c_char_p, C.c_char_p, _STRS, _I32]),
    ("mmp_instance_update", _I32, [_P, _I32, _P]),
    ("mmp_instance_remove", _I32, [_P, _I32]),
    ("mmp_instance_upsert_json", _I32, [_P, _I32, C.c_char_p, C.c_char_p, _I32]),
    ("mmp_model_upsert_json", _I32, [_P, _I32, C.c_char_p, _I32]),
    ("mmp_types_set_json", _I32, [_P, C.c_char_p]),
    ("mmp_type_id", _I32, [_P, C.c_char_p]),
    ("mmp_replicasets_set", _I32, [_P, _STRS, _I32]),
    ("mmp_model_upsert", _I32, [_P, _I32, _P, _P, _I32]),
    ("mmp_models_bulk", _I32, [_P, _I32, _I32, _P, _P, _P]),
    ("mmp_fleet_commit", _I32, [_P]),
    ("mmp_place_batch", _I32, [_P, _P, _I32, _P, _I32, _P, _I32, _P, _I64, _U64]),
    ("mmp_place_batch_trace", _I32, [_P, _P, _I32, _P, _I32, _P, _I32, _P, _P, _P, _I64, _U64]),
    ("mmp_place_batch_excluding", _I32, [_P, _P, _I32, _P, _I32, _P, _I32, _P, _I32, _P, _P, _P, _I64, _U64]),
    ("mmp_place_one", _I32, [_P, _P, _P, _P, _P, _I64, _U64]),
    ("mmp_place_sweep", _I32, [_P, _I32, _I32, _P, _I32, _P, _P, _I64, _U64]),
    ("mmp_place_batch_device", _I32, [_P, _P, _I32, _P, _I64, _U64, C.POINTER(C.c_float)]),
    ("mmp_slot_summaries", _I32, [_P, _I64, _P, _P, _I32]),
    ("mmp_device_alloc", _I32, [_P, _I64, C.POINTER(_P)]),
    ("mmp_device_free", _I32, [_P, _P]),
    ("mmp_device_upload", _I32, [_P, _P, _P, _I64]),
    ("mmp_device_download", _I32, [_P, _P, _P, _I64]),
    ("mmp_host_alloc", _I32, [_P, _I64, C.POINTER(_P)]),
    ("mmp_host_free", _I32, [_P, _P]),
    ("mmp_flush_l2", _I32, [_P]),
    ("mmp_row_words", _I32, [_P]),
    ("mmp_live_instances", _I32, [_P]),
    ("mmp_cluster_order", _I32, [_P, _P, _I32]),
    ("mmp_type_sets", _I32, [_P, _I32, _I32, _P, C.POINTER(_I32), _P, C.POINTER(_I32)]),
    ("mmp_kernel_launches", _I64, [_P]),
    ("mmp_stats", _I32, [_P, _P, _P, _I32]),
    ("mmp_instance_partition", _I32, [_P, _I32]),
    ("mmp_reaper_select", _I32, [_P, _I32, _I64, _P, _P, _I32]),
    ("mmp_reaper_run", _I32, [_P, _I32, _I64, _I64, _P, _U64, _P, _P, _I32, _P, _I32, _P, _I32, C.c_void_p]),
    ("mmp_janitor_run", _I32, [_P, _I32, _P, _I32, _P, _P, _I32, C.c_void_p]),
    ("mmp_janitor_task", _I32, [_P, _I32, _P, _I32, _P, _P, _P, _I32, C.c_void_p]),
    ("mmp_rate_run", _I32, [_P, _I32, _P, _I32, _P, _P, _U64, _P, _P, _I32, C.c_void_p]),
    ("mmp_shutdown_run", _I32, [_P, _I32, _P, _I32, _P, _P, _U64, _P, C.c_void_p]),
    ("mmp_evict_run", _I32, [_P, _I32, _P, _I32, _P, _P, _U64, _P, C.c_void_p]),
    ("mmp_lru_init", _I32, [_P, _I32, _P, _I32]),
    ("mmp_lru_apply", _I32, [_P, _P, _I32, _I64, _P, _I32]),
    ("mmp_lru_state", _I32, [_P, _I32, _P, _P, _P]),
    ("mmp_lru_apply_status", _I32, [_P, _P, _I32, _I64, _P, _I32, _P]),
    ("mmp_lru_read", _I32, [_P, _P, _I32, _I64, _P, _P, _I64]),
    ("mmp_lru_lookup", _I32, [_P, _I32, _P, _P, _P, _P, _P]),
    ("mmp_churn_init", _I32, [_P, C.c_void_p]),
    ("mmp_churn_seed", _I32, [_P, _I32, _P, _P, _P, _P, _P, _I64]),
    ("mmp_churn_step", _I32, [_P, _P, _I32, _I64, _I64, _U64, _P, _I32, C.POINTER(_I32), _P, _I32, C.POINTER(_I32), _P, C.c_void_p]),
    ("mmp_churn_model", _I32, [_P, _I32, _P, _P]),
    ("mmp_churn_model_ids", _I32, [_P, _I32, _P, _P, _I32]),
    ("mmp_commit_info", _I32, [_P, C.POINTER(_I32), C.POINTER(C.c_double)]),
    ("mmp_server_stats", _I32, [_P, _P]),
    ("mmp_model_times", _I32, [_P, _I32, _P, _I32, _I64]),
    ("mmp_scale_eval", _I32, [_P, _P, _I32, _P, _P]),
    ("mmp_registry_prune", _I32, [_P, _I32, _I64, _I64, _P, _P, _P, _I32]),
    ("mmp_registry_prune_ids", _I32, [_P, _I32, _I64, _I64, _P, _P, _P, _I32]),
    ("mmp_tune", _I32, [_P, C.c_char_p, _I64]),
    ("mmp_last_timing", _I32, [_P, C.c_char_p, C.POINTER(C.c_double)]),
    ("mmp_batcher_create", _I32, [_P, _I32, _I32, _U64, C.POINTER(_P)]),
    ("mmp_batcher_destroy", None, [_P]),
    ("mmp_place_submit", _I32, [_P, _P, _P, _P, _I64, _P, C.POINTER(C.c_uint32)]),
    ("mmp_batcher_stats", _I32, [_P, C.POINTER(_I64), C.POINTER(_I64)]),
    ("mmp_shard_unique_id", _I32, [_P]),
    ("mmp_shard_connect", _I32, [_P, _P]),
    ("mmp_shard_words", _I32, [_P, C.POINTER(_I32), C.POINTER(_I32)]),
    ("mmp_shard_open_decisions", _I64, [_P]),
    ("mmp_shard_ipc_export", _I32, [_P, _I32, _P]),
    ("mmp_shard_ipc_import", _I32, [_P, _P]),
    ("mmp_shard_peer_stats", _I32, [_P, _P]),
    ("mmp_fleet_set_id_base", _I32, [_P, _U64]),
]


def bind(lib: C.CDLL, require_all: bool = True) -> C.CDLL:
    missing = []
    for name, res, args in SYMBOLS:
        try:
            fn = getattr(lib, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    if missing and require_all:
        raise ImportError(f"libmmplace is missing symbols declared in include/mmplace.h: {missing}")
    lib._mmp_missing = missing
    return lib


def load(path: str, require_all: bool = True) -> C.CDLL:
    if not os.path.exists(path):
        raise ImportError(
            f"{path} not found: the CUDA library has not been built. Run `python -c 'import __graft_entry__ as g; "
            f"g.build()'` (needs nvcc). There is no CPU fallback.")
    return bind(C.CDLL(path), require_all)  # RTLD_LOCAL: never interpose with another copy of the ABI


_product = None


SHARD_IPC_BYTES = 512  # MMP_SHARD_IPC_BYTES


def load_product() -> C.CDLL:
    global _product
    if _product is None:
        # MMP_LIB: an alternative build of the same CUDA library (A/B runs of kernel variants on one GPU box)
        _product = load(os.environ.get("MMP_LIB", PRODUCT_SO))
    return _product
