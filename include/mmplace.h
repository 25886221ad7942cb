/*
 * mmplace.h — C ABI of libmmplace: an H100-native (sm_90a CUDA) placement / LRU-eviction solver that drops in
 * behind ModelMesh's decision API.  Plain pointers and sizes only; no CUDA/torch types.  This is the boundary a
 * JNI shim binds (see INTEGRATION.md for the Java side).  Reference = kserve/modelmesh @ ea13cdc5;
 * MM = src/main/java/com/ibm/watson/modelmesh/ModelMesh.java, IR = InstanceRecord.java, MR = ModelRecord.java,
 * TCM = TypeConstraintManager.java, UT = UpgradeTracker.java, CLHM = clhm/ConcurrentLinkedHashMap.java.
 *
 * Every function returns >= 0 on success or a negative MMP_E_* code; mmp_last_error() gives the message.
 * The library never falls back to a CPU path: if no CUDA device is usable, mmp_fleet_create fails with MMP_E_CUDA.
 *
 * Threading: ingest calls (mmp_instance_*, mmp_model*, mmp_types_*, mmp_replicasets_set, mmp_fleet_commit) are
 * single-writer (the reference serialises them on TypeConstraintManager.executor(), TCM:145-147, MM:1423-1427).
 * mmp_place_* / mmp_stats / mmp_reaper_select may be called from any number of threads concurrently with each
 * other and with ingest; they always see the last committed snapshot epoch (SURVEY.md §8a N6).
 */
#ifndef MMPLACE_H
#define MMPLACE_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define MMP_ABI_VERSION 2

enum {
  MMP_OK = 0,
  MMP_E_ARG = -1,    /* bad argument / out-of-range index / value outside the supported domain */
  MMP_E_CUDA = -2,   /* CUDA runtime failure (including "no device") */
  MMP_E_NCCL = -3,   /* collective failure in the instance-sharded path */
  MMP_E_EPOCH = -4,  /* no committed snapshot yet */
  MMP_E_NOMEM = -5,
  MMP_E_STATE = -6
};

/* per-decision result codes in mmp_decision_out.target */
enum {
  MMP_TARGET_NONE = -1,   /* getNext returned null        (MM:4796,4801,4872,4941) */
  MMP_TARGET_SELF = -2,   /* getNext returned ABORT_REQUEST (MM:4894,4932,4990)    */
  MMP_TARGET_INVALID = -3 /* malformed decision, nothing was decided: model / self index out of range, self not live and no
                             fresh row given, or an extra[] slice outside the table passed with the call (extra_off < 0,
                             extra_n outside [0, MMP_MAX_EXTRA], extra_off + extra_n > n_extra); with MMP_DF_REQUEST_MODEL
                             also a type id outside [0, 65535), the flag combined with MMP_DF_MODEL_LAST_USED, or an
                             instance-sharded fleet.  The reference has no counterpart (a Java caller cannot form such a
                             call); the batch itself still succeeds. */
};
#define MMP_MAX_EXTRA 16  /* per-decision additional excludes (tried-this-request ∪ explicit, MM:4706-4715) */

typedef struct mmp_fleet mmp_fleet;

/* Replaces the per-JVM constants ModelMesh derives in initialize() (MM:697, MM:767-771). */
typedef struct {
  int64_t min_space_units;           /* isFull threshold, MM:4640-4642 / MM:767-769 */
  int64_t min_churn_age_ms;          /* MM:697 */
  int32_t default_model_size_units;  /* MM:712 (runtime's default model size / 8 KiB) */
  int32_t max_instances;             /* capacity of the instance index space (<= 65536) */
  int32_t max_models;                /* capacity of the model index space */
  int32_t device;                    /* CUDA device ordinal */
  int32_t shard_rank;                /* instance-shard of this process (0 when not sharded) */
  int32_t shard_count;               /* number of instance shards (1 when not sharded) */
  uint32_t flags;                    /* reserved, 0 */
  uint32_t reserved;
} mmp_config;

/* Numeric part of InstanceRecord (IR:37-73).  Strings travel beside it in mmp_instance_upsert. */
typedef struct {
  int64_t lru_time;      /* IR:37  "lruTime", Long.MAX_VALUE when the cache is empty */
  int64_t capacity;      /* IR:41  "cap"  units of 8 KiB */
  int64_t used;          /* IR:43  "used" */
  int64_t start_time;    /* IR:60  "startTime" */
  int64_t vers;          /* IR:62  "vers" */
  int32_t count;         /* IR:39  "count" */
  int32_t l_threads;     /* IR:45  "lThreads" */
  int32_t l_in_prog;     /* IR:47  "lInProg" */
  int32_t rpm;           /* IR:51  "rpm"; must be <= 500,000,000 */
  int32_t shutting_down; /* IR:56  "shutdown": treated as a deletion, MM:1462-1464 */
  int32_t active;        /* 1 if the instance is in litelinks' service-instance list (siMap, MM:4765,4778) */
} mmp_instance_row;

/* Per-model registry state needed on the path (MR:61-114): 24 bytes. */
typedef struct {
  int64_t last_used;     /* MR:105 "lu" */
  int32_t size_units;    /* CacheEntry weight / KNOWN_SIZE (MM:5160-5178) */
  int32_t rpm;           /* request rate, informational */
  uint16_t type_id;      /* from mmp_type_id(); 0 = a type with no configured constraints */
  uint8_t copy_count;    /* MR:69  instanceIds.size() (saturating at 255) */
  uint8_t fail_count;    /* MR:73  loadFailedInstanceIds.size() */
  uint32_t reserved;
} mmp_model_row;

/* One call of CacheMissForwardingLB.getNext (MM:4776-5004): 32 bytes.
 * The model's exclusion set (loaded ∪ failed, MM:4735-4743) and type come from the model table of the last committed
 * snapshot -- or, with MMP_DF_REQUEST_MODEL, from the decision itself. */
#define MMP_DF_FAVOUR_SELF 1u        /* CacheMissExcludeSet.favourSelf (MM:4721) */
#define MMP_DF_MODEL_LAST_USED 2u    /* take last_used from the model row instead of this struct */
#define MMP_DF_OWN_ID 4u             /* bits 8..31 of flags carry the decision's own id for the hash-indexed pick (N4, MM:4981)
                                        instead of its position in the batch: the result of a decision then does not depend on
                                        which batch it travelled in (mmp_place_submit coalesces callers this way) */
#define MMP_DF_REQUEST_MODEL 8u      /* the model record this request read (MM:3537, refreshed after a failed load MM:4088-4097)
                                        instead of the committed one: `model` holds the model's TYPE ID (mmp_type_id; an id the
                                        snapshot does not know resolves like type 0, as a model row holding it would), and its
                                        loaded ∪ failed instance indices (MR:69,73) travel in the extra[] slice together with the
                                        request's own excludes -- at most MMP_MAX_EXTRA in all.  No registry state of the snapshot
                                        is read, so a model registered or changed since the last commit is placed on its current
                                        record.  Not with MMP_DF_MODEL_LAST_USED; unsharded fleets only (else MMP_TARGET_INVALID) */
typedef struct {
  int32_t model;        /* model index, or the type id with MMP_DF_REQUEST_MODEL */
  int32_t self;         /* instance index of the calling pod ("instanceId", MM:4780,4808) */
  int64_t last_used;    /* CacheMissExcludeSet.lastUsedTime (MM:4730, 4949) */
  uint32_t flags;       /* MMP_DF_* */
  int32_t fresh;        /* index into the fresh[] rows of the call (getFreshInstanceRecord MM:5369), or -1:
                           self's published row with rpm = 0 (the reference never sets rpm on the fresh record) */
  int32_t extra_off;    /* offset into extra[] of this decision's additional excluded instance indices
                           (tried-this-request ∪ explicit, MM:4706-4715) */
  int32_t extra_n;      /* how many, 0..MMP_MAX_EXTRA; the slice must lie inside extra[0, n_extra) or the decision is
                           answered MMP_TARGET_INVALID (checked on the device; never read out of bounds) */
} mmp_decision_in;

typedef struct {
  int32_t target;        /* instance index, MMP_TARGET_NONE or MMP_TARGET_SELF */
  int32_t n_candidates;  /* candidates.size() at MM:4939 (0 if getNext returned before that) */
} mmp_decision_out;

/* Optional per-decision trace for parity checking (everything before and after the random draw). */
#define MMP_TF_RS_RETRY 1       /* replicaset filter dropped and retried (MM:4798-4802) */
#define MMP_TF_SIMPLE 2         /* reached the simple-case walk (MM:4889) */
#define MMP_TF_BEST_FULL 4      /* bestIsFull (MM:4811) */
#define MMP_TF_FAVOUR_EXIT 8    /* returned through a favourSelf short-circuit */
#define MMP_TF_KEEP_BEST 16     /* best survived the rpm filter */
#define MMP_TF_KEEP_OTHERS 32   /* non-self candidates survived the rpm filter (all share one recorded rpm, N2) */
#define MMP_TF_KEEP_SELF 64     /* the self candidate survived the rpm filter */
#define MMP_TF_PREF_B 128       /* non-simple case (b) with preferred candidates (MM:4866-4880) */
typedef struct {
  int32_t best;          /* bestIid after preferred handling (instance index), -1 if none */
  int32_t n_remaining;   /* remainingCount (MM:4956) */
  int32_t pick_index;    /* index of the chosen non-null candidate (MM:4981) */
  int32_t flags;         /* MMP_TF_* */
  int32_t cut_rank;      /* rank (position in PLACEMENT_ORDER) of the first violator, INT32_MAX if none */
  int32_t best_rank;
  int32_t reserved[2];
} mmp_decision_trace;

typedef struct {  /* ModelMesh.ClusterStats MM:1570-1591 */
  int64_t total_capacity, total_free, global_lru;
  int32_t instance_count, model_copy_count;
} mmp_cluster_stats;

/* ---- lifecycle ---- */
int32_t mmp_abi_version(void);
int32_t mmp_fleet_create(const mmp_config *cfg, mmp_fleet **out);
void mmp_fleet_destroy(mmp_fleet *);
const char *mmp_last_error(mmp_fleet *); /* thread-local message of the last failing call (fleet may be NULL) */

/* ---- plug point 2: fleet-state ingest.  Replaces handleInstanceTableChange (MM:1455-1568) feeding
 * clusterState, and ModelMesh.event(type,key,ModelRecord) (MM:2807-2854). ---- */
/* id/loc/zone/labels are UTF-8; ordered as UTF-16 code units like String.compareTo (MM:4697-4700). loc/zone may be NULL. */
int32_t mmp_instance_upsert(mmp_fleet *, int32_t idx, const mmp_instance_row *row, const char *id, const char *loc,
                            const char *zone, const char *const *labels, int32_t n_labels);
/* update only the numeric columns of an instance already present (the common KV update event) */
int32_t mmp_instance_update(mmp_fleet *, int32_t idx, const mmp_instance_row *row);
int32_t mmp_instance_remove(mmp_fleet *, int32_t idx);
/* The same from the records as the KV store holds them (jackson JSON): InstanceRecord (IR:37-69: lruTime count cap used
 * lThreads lInProg rpm shutdown startTime vers loc zone labels) and ModelRecord (MR:61-114: type, instanceIds and failedIn
 * maps keyed by instance id, lu).  Unknown properties are ignored, absent ones keep the jackson-constructor defaults.
 * `active` = the instance is in litelinks' service-instance list (not part of the record).  Instance ids in a model
 * record are kept BY ID and resolved against the instance table at every mmp_fleet_commit (the reference tests membership
 * by id at decision time, MM:4735-4743), so model and instance records may arrive in any order and an instance may
 * re-register under another index.  A record without "type" gets ModelRecord's DEFAULT_TYPE "NLCLASSIFIER" (MR:117-130).
 * size_units = CacheEntry weight / KNOWN_SIZE (not part of the record). */
int32_t mmp_instance_upsert_json(mmp_fleet *, int32_t idx, const char *id, const char *record_json, int32_t active);
int32_t mmp_model_upsert_json(mmp_fleet *, int32_t model, const char *record_json, int32_t size_units);
/* MM_TYPE_CONSTRAINTS json (TCM:79-98, 193-206; config/examples/type-constraints-example):
 * {"type": {"required": ["l1",..], "preferred": ["l2",..]}, "_default": {...}}.  NULL/"" = typeConstraints == null. */
int32_t mmp_types_set_json(mmp_fleet *, const char *json);
/* type id for a model-type name: >= 1 for configured types, 0 for any other name (falls to "_default" if configured). */
int32_t mmp_type_id(mmp_fleet *, const char *type_name);
/* UpgradeTracker.getLikelyReplacedReplicaSets() keys (UT:78): 6-char replicaset prefixes to avoid (MM:4769-4770). */
int32_t mmp_replicasets_set(mmp_fleet *, const char *const *prefixes, int32_t n);
/* instance_ids = loaded ∪ failed instance indices of the model (MR:69,73): the CacheMissExcludeSet row (MM:4735-4743) */
int32_t mmp_model_upsert(mmp_fleet *, int32_t model, const mmp_model_row *row, const int32_t *instance_ids, int32_t n_ids);
/* bulk form: models [first, first+n); edge_off has n+1 entries indexing edge_inst */
int32_t mmp_models_bulk(mmp_fleet *, int32_t first, int32_t n, const mmp_model_row *rows, const int64_t *edge_off,
                        const int32_t *edge_inst);
/* Publish everything ingested since the last commit as a new snapshot epoch: recomputes PLACEMENT_ORDER ranks
 * (MM:4646-4703), type/preferred masks (TCM:680-747), stats columns and the rank-space exclusion bitmap in HBM.
 * Returns the new epoch number (>= 1). */
int32_t mmp_fleet_commit(mmp_fleet *);

/* ---- plug point 1: placement.  Replaces CacheMissForwardingLB.getNext (MM:4776-5004). ---- */
/* Host buffers in, host buffers out (copies included).  fresh[]/extra[] may be NULL when unused. */
int32_t mmp_place_batch(mmp_fleet *, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                        const int32_t *extra, int32_t n_extra, mmp_decision_out *out, int64_t now_ms, uint64_t seed);
/* Same with the optional trace (trace may be NULL) and candidate masks: cand_mask (may be NULL) receives, per decision,
 * TWO planes of mmp_row_words() 32-bit words each, i.e. the caller provides n * 2 * mmp_row_words() * 4 bytes:
 *   plane 0 (words [0, RW)):    bit r set iff the instance at PLACEMENT_ORDER rank r is a candidate other than best
 *   plane 1 (words [RW, 2 RW)): bit r set iff that candidate survived the rpm filter (MM:4957-4980)
 * (non-simple case (b), MMP_TF_PREF_B: both planes include best's own bit, see tests/helpers.py). */
int32_t mmp_place_batch_trace(mmp_fleet *, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh,
                              int32_t n_fresh, const int32_t *extra, int32_t n_extra, mmp_decision_out *out,
                              mmp_decision_trace *trace, uint32_t *cand_mask, int64_t now_ms, uint64_t seed);
/* Registry sweep -- the reference's natural batched caller: the leader's reaper walks the registry and calls
 * ensureLoadedInternal per model (MM:6616-6735), i.e. getNext for model first_model + i on behalf of instance self[i]
 * (self_stride = 1) or of one instance for the whole sweep (self_stride = 0: self[0]), lastUsedTime from the model record,
 * no extra excludes; favour_bits (may be NULL): bit i = CacheMissExcludeSet.favourSelf.  Same results as mmp_place_batch
 * on the equivalent 32-byte records, with 4 bytes (+1 bit) instead of 32 going to the device per decision. */
int32_t mmp_place_sweep(mmp_fleet *, int32_t first_model, int32_t n, const int32_t *self, int32_t self_stride,
                        const uint32_t *favour_bits, mmp_decision_out *out, int64_t now_ms, uint64_t seed);
/* Micro-batcher for plug point 1 (SURVEY.md §8b): getNext is called on arbitrary request threads (litelinks pool / gRPC
 * pool, MM:918-925, MM:1107-1110).  mmp_place_submit blocks the calling thread while ONE submit thread drains the queue into
 * a single mmp_place_batch against the current epoch: every `max_wait_us` or as soon as `max_batch` decisions wait.  Each
 * decision is numbered by the batcher (MMP_DF_OWN_ID; *decision_id receives the id), so its result equals
 * mmp_place_batch on that one record with seed = the batcher's seed -- whichever batch carried it. */
typedef struct mmp_batcher mmp_batcher;
int32_t mmp_batcher_create(mmp_fleet *, int32_t max_batch, int32_t max_wait_us, uint64_t seed, mmp_batcher **out);
void mmp_batcher_destroy(mmp_batcher *);
int32_t mmp_place_submit(mmp_batcher *, const mmp_decision_in *in, const mmp_instance_row *fresh, const int32_t *extra, int64_t now_ms,
                         mmp_decision_out *out, uint32_t *decision_id);
int32_t mmp_batcher_stats(mmp_batcher *, int64_t *batches, int64_t *decisions);
/* Single decision (latency path, B = 1). */
int32_t mmp_place_one(mmp_fleet *, const mmp_decision_in *in, const mmp_instance_row *fresh, const int32_t *extra,
                      mmp_decision_out *out, int64_t now_ms, uint64_t seed);
/* Device-resident variant used to time the kernel alone: d_in/d_out are device pointers obtained from
 * mmp_device_alloc; returns after the kernel has been enqueued AND completed; *kernel_ms (may be NULL) receives the
 * CUDA-event duration of the scoring kernel on its launch stream. */
int32_t mmp_place_batch_device(mmp_fleet *, const void *d_in, int32_t n, void *d_out, int64_t now_ms, uint64_t seed,
                               float *kernel_ms);
int32_t mmp_device_alloc(mmp_fleet *, int64_t bytes, void **out);
int32_t mmp_device_free(mmp_fleet *, void *p);
int32_t mmp_device_upload(mmp_fleet *, void *dst, const void *src, int64_t bytes);
int32_t mmp_device_download(mmp_fleet *, void *dst, const void *src, int64_t bytes);
/* pinned (page-locked) host memory for decision/result buffers, so that the copies in mmp_place_batch are true DMA;
 * a JNI shim wraps these in direct ByteBuffers (INTEGRATION.md) */
int32_t mmp_host_alloc(mmp_fleet *, int64_t bytes, void **out);
int32_t mmp_host_free(mmp_fleet *, void *p);
int32_t mmp_flush_l2(mmp_fleet *); /* writes a buffer larger than L2 (bench hygiene) */

/* ---- instance-sharded multi-GPU (SURVEY.md §8e): one process per GPU, mmp_config.shard_rank / shard_count.
 * Every process ingests the whole fleet; shard k keeps ranks [lo, hi) of every exclusion-bitmap row in its GPU's HBM
 * (contiguous ranges of PLACEMENT_ORDER ranks in 16-byte granules) and the small per-instance tables in full.
 * mmp_place_batch / mmp_place_batch_device on such a fleet must be called by all shards with the same batch; each shard
 * resolves every decision over its own range, ONE ncclAllReduce(min) over 64-bit min-loc keys picks the answer of the
 * shard that holds the first entry under PLACEMENT_ORDER (MM:4806), and decisions whose shortlist walk (MM:4901-4937)
 * left that shard's range are finished from all-gathered row blocks.  Every shard returns the full results.
 * Replaces nothing in the reference (one JVM decides alone); it is the scale-out of plug point 1. ---- */
int32_t mmp_shard_unique_id(void *id128);                       /* shard 0: ncclGetUniqueId; the host passes the 128 bytes to its peers */
int32_t mmp_shard_connect(mmp_fleet *, const void *id128);      /* all shards: ncclCommInitRank(shard_count, id, shard_rank) */
int32_t mmp_shard_words(mmp_fleet *, int32_t *word_lo, int32_t *word_hi); /* this shard's row words [lo, hi); returns the stored row stride */
int64_t mmp_shard_open_decisions(mmp_fleet *);                  /* decisions that needed the row-gather pass so far */
/* Peer access between the instance shards (one node, NVLink): once every shard has imported its peers' blobs, a batch is
 * DEALT across the shards -- each decides 1/shard_count of it, reading row words beyond the replicated front from the owning
 * shard's memory, and stores its results into every shard's result buffer.  No NCCL call and no host synchronisation on
 * that path (mmp_shard_connect is then optional).  Each shard: export (after its first commit or before), exchange the
 * blobs by any means, import all shard_count blobs ordered by rank.  Works across processes (CUDA IPC) and between fleets
 * of one process (peer access).  Same contract as the collective path: every shard commits the same epochs and is given
 * the same batches in the same order; every shard ends with the whole batch's results.  Batches of up to max_batch. */
#define MMP_SHARD_IPC_BYTES 512
int32_t mmp_shard_ipc_export(mmp_fleet *, int32_t max_batch, void *blob /* MMP_SHARD_IPC_BYTES */);
int32_t mmp_shard_ipc_import(mmp_fleet *, const void *blobs /* shard_count x MMP_SHARD_IPC_BYTES, by shard rank */);
/* out4: [0] batches taken by the peer path, [1] row words read from peers' memory, [2] result bytes stored to peers, [3] 1 = path active */
int32_t mmp_shard_peer_stats(mmp_fleet *, int64_t *out4);
/* Registry (model) sharding needs no exchange: each process places the decisions of its own models against the whole
 * instance table.  The only cross-shard convention is the numbering of decisions for the hash-indexed pick (N4, MM:4981):
 * decision i of a batch hashes as id_base + i, so a shard that is handed the slice [lo, hi) of a larger batch sets
 * id_base = lo and returns exactly what the unsharded run returns for that slice. */
int32_t mmp_fleet_set_id_base(mmp_fleet *, uint64_t id_base);

/* ---- snapshot introspection ---- */
int32_t mmp_row_words(mmp_fleet *);                                   /* 32-bit words per exclusion-bitmap row */
int32_t mmp_live_instances(mmp_fleet *);                              /* number of ranked instances in the snapshot */
int32_t mmp_cluster_order(mmp_fleet *, int32_t *out_idx, int32_t cap); /* instance idx by ascending PLACEMENT_ORDER rank */
/* candidate/preferred membership of a type id as computed at commit (TCM:242-251): 0/1 per instance idx;
 * *preferred_null = 1 when getPreferredInstances would return null */
int32_t mmp_type_sets(mmp_fleet *, int32_t type_id, int32_t n_idx, uint8_t *allowed, int32_t *allowed_null,
                      uint8_t *preferred, int32_t *preferred_null);
int64_t mmp_kernel_launches(mmp_fleet *);                             /* count of library kernels launched so far */

/* ---- plug point 4: batch scans ---- */
/* ClusterStats (MM:1570-1591, ISST:63-92) reduced on the device from the snapshot: out[0] = whole cluster, then one
 * per prohibited-type-set partition (TCM:557-579) in TCM.getPartitionStats order (TCM:264-292). part_ids gets the
 * partition id of each entry (-1 for the cluster). Returns the number of entries. */
int32_t mmp_stats(mmp_fleet *, mmp_cluster_stats *out, int32_t *part_ids, int32_t cap);
int32_t mmp_instance_partition(mmp_fleet *, int32_t idx);
/* Reaper candidate scan + proactive-load selection (MM:6574-6577, 6616-6735) for one partition (-1: no type
 * constraints).  taken[] (max_models bytes, in/out, may be NULL) mirrors allCandidates.set(i, null).
 * Writes the selected model indices most-recently-used first; returns how many. */
int32_t mmp_reaper_select(mmp_fleet *, int32_t partition, int64_t now_ms, uint8_t *taken, int32_t *out_models, int32_t cap);

/* ---- plug point 3: per-instance time-ordered weighted LRU (CLHM:821-858, 590-652, 329-352; LD:243-288) ---- */
enum { MMP_LRU_INSERT = 0, MMP_LRU_TOUCH = 1, MMP_LRU_RESIZE = 2, MMP_LRU_REMOVE = 3, MMP_LRU_SET_CAPACITY = 4,
       /* loadLocal's admission as ONE checked event (SURVEY.md §8a row a11): churn guard (MM:3872-3884: instance full and its
        * oldest entry younger than min_churn_age_ms -> rejected), putIfAbsent of a 1-unit placeholder at last_used
        * (INSERTION_WEIGHT MM:5011, 5061), "the new entry was immediately evicted" (MM:5145-5148), early reject (MM:5185-5190:
        * weight > capacity, or last_used > 0 && weight > free && last_used < oldestTime), then inflate to `weight` and
        * "check whether we were evicted when growing" (MM:2094-2106).  Outcome per event through mmp_lru_apply_status. */
       MMP_LRU_LOAD = 5 };
/* outcome of an MMP_LRU_LOAD event (-1 for other events) */
enum { MMP_LOAD_ACCEPTED = 0, MMP_LOAD_CHURN_REJECT = 2, MMP_LOAD_FELL_THROUGH = 3, MMP_LOAD_EARLY_REJECT = 4, MMP_LOAD_EVICTED_GROWING = 5,
       MMP_LOAD_ENTRY_EXISTS = 6 };
typedef struct {
  int32_t op;         /* MMP_LRU_* */
  int32_t instance;   /* which instance's cache */
  int32_t model;      /* key */
  int32_t weight;     /* INSERT/RESIZE: entry weight; SET_CAPACITY: unused */
  int64_t last_used;  /* INSERT/TOUCH: 0 = now;  SET_CAPACITY: the new capacity */
} mmp_lru_event;
typedef struct {
  int32_t instance, model;
  int64_t last_used;
  int32_t weight;
  int32_t event;      /* index of the event that triggered the eviction */
} mmp_eviction;
/* (re)initialise the LRU store: one cache per instance index with the given capacities (units) */
int32_t mmp_lru_init(mmp_fleet *, int32_t n_instances, const int64_t *capacity, int32_t slots_per_instance);
/* applies events in order per instance (instances are independent); evictions are returned grouped by event order
 * within each instance, oldest first (CLHM:329-352).  Returns the number of evictions (<= cap written). */
int32_t mmp_lru_apply(mmp_fleet *, const mmp_lru_event *ev, int32_t n, int64_t now_ms, mmp_eviction *out, int32_t cap);
/* the same, also returning the outcome of every event (status[i] = MMP_LOAD_* for MMP_LRU_LOAD events, -1 otherwise) */
int32_t mmp_lru_apply_status(mmp_fleet *, const mmp_lru_event *ev, int32_t n, int64_t now_ms, mmp_eviction *out, int32_t cap,
                             int32_t *status);
/* per-instance oldestTime() (CLHM:1125-1133, -1 if empty), weightedSize() and size().  oldestTime() is the field CLHM
 * caches: after an MMP_LRU_SET_CAPACITY it keeps the head from before that event's evictions until the next insert,
 * read of a present key, resize with a new weight or removal of a present key (quirk N14); MMP_LRU_LOAD's churn guard
 * reads the same value. */
int32_t mmp_lru_state(mmp_fleet *, int32_t n_instances, int64_t *oldest, int64_t *weighted, int32_t *count);

/* ---- the closed loop on the device (SURVEY.md §8a rows a11 admission, a12 rebalance; §8f-1 ingest / ordering maintenance,
 * §8f-4 fleet simulator; BASELINE.json configs[3] "churn").  One call = one republish window (2 s, INSTANCE_REC_PUBLISH_MIN_
 * PERIOD_MS MM:232) of the WHOLE fleet, evaluated against the instance and model records as committed at its start (N6):
 *   REQUEST of a model with registered copies -> runtimeCache.get on copy (u mod copies) in registration order;
 *   REQUEST of a model with none: the first one in the window is a cache miss -> getNext (self = caller, lastUsed = t) ->
 *     loadLocal on the target (MMP_LRU_LOAD's admission rules) -> evictions -> onEviction (MM:2875-2931: deregistration;
 *     a copy loaded more than 2 x load_timeout_ms ago whose type set is < 95 % full is queued for ensureLoadedElsewhere and
 *     placed first in the next window, MM:2915-2931); later misses of the same model in the window are coalesced;
 *   REMOVE -> runtimeCache.remove on every registered copy;
 *   then the registry changes, publishInstanceRecord with its significance thresholds (MM:5390-5470) per instance, and a
 *   commit (re-rank under PLACEMENT_ORDER, tables, bitmap) -- all on the device.  The host only reads the reports.
 * Requires an unsharded fleet whose models have at most 4 registered copies + failed loads.  Replaces nothing in the
 * reference 1:1 (each pod runs its own loop there); it is the batched, fleet-wide form of it for simulation / what-if runs. ---- */
enum { MMP_CHURN_REQUEST = 0, MMP_CHURN_REMOVE = 1 };
typedef struct { int32_t type; int32_t model; int32_t caller; uint32_t u; int64_t t; } mmp_churn_event;
typedef struct {
  int32_t model, self, target, n_candidates;
  int32_t status;  /* MMP_LOAD_* of the load, 1 = nowhere to load (getNext null), 7 = queued reload skipped (the model has a
                      copy again), 8 = malformed, 9 = accepted but evicted again later in the window */
  int32_t event;   /* index of the REQUEST that caused it, or -1 - k for the k-th queued ensureLoadedElsewhere */
} mmp_churn_decision;
typedef struct { int32_t instance, model; int64_t last_used; int32_t weight, order, reload; } mmp_churn_eviction;
typedef struct { int64_t load_timeout_ms; int64_t last_published_ms; int32_t slots_per_instance; int32_t reserved; } mmp_churn_config;
typedef struct {
  int32_t n_published, n_carry, n_coalesced, n_lru_events;
  float ms_classify, ms_place, ms_route, ms_apply, ms_registry, ms_commit, ms_total;  /* CUDA-event times of the phases */
  float reserved;
} mmp_churn_report;
/* one cache per instance index (capacity = its published capacity), empty; needs a committed snapshot */
int32_t mmp_churn_init(mmp_fleet *, const mmp_churn_config *cfg);
/* resident copies at the start of a trace: putIfAbsent(model, weight, last_used) on `instance`, registered at load_ts.
 * (The registry side -- mmp_model_upsert with the same instances as loaded copies -- is the caller's.) */
int32_t mmp_churn_seed(mmp_fleet *, int32_t n, const int32_t *instance, const int32_t *model, const int64_t *last_used,
                       const int32_t *weight, const int64_t *load_ts, int64_t now_ms);
/* events in trace order with now0 <= t < now1.  Reports: the window's decisions in order (queued reloads first), its
 * evictions grouped by instance in listener order, every instance's published row after the window (rows_out: max_instances
 * rows, may be NULL).  Ends with a committed snapshot: placement calls after it see the new epoch. */
int32_t mmp_churn_step(mmp_fleet *, const mmp_churn_event *ev, int32_t n, int64_t now0, int64_t now1, uint64_t seed,
                       mmp_churn_decision *dec_out, int32_t dec_cap, int32_t *n_dec, mmp_churn_eviction *evict_out, int32_t evict_cap,
                       int32_t *n_evict, mmp_instance_row *rows_out, mmp_churn_report *report);
/* registry state of one model as the device holds it: row + the 4 inline instance indices (first copy_count = loaded) */
int32_t mmp_churn_model(mmp_fleet *, int32_t model, mmp_model_row *row, int32_t *instances4);
/* ---- registry-side batch scans (SURVEY.md §8a row a14, §8f-2) ---- */
/* MR.instanceIds / failedIn VALUES (load-start / failure times of the model's inline edges, same order as the ids given to
 * mmp_model_upsert) and MR.lastUnloadTime ("lul").  mmp_model_upsert_json takes them from the record.  0 = unknown. */
int32_t mmp_model_times(mmp_fleet *, int32_t model, const int64_t *edge_ts, int32_t n, int64_t last_unload_time);
/* One cache entry of one pod, as its rate-tracking / janitor tasks see it (CacheEntry counters are pod-local): */
typedef struct {
  int32_t instance, model;
  int64_t count;        /* ce.getAndResetIntervalCount(): invocations since the last run (MM:5689) */
  int64_t last_used;    /* the entry's lastUsed in the pod's cache */
  int64_t last_heavy;   /* ce.getLastHeavyTime() */
  int32_t i1, i2;       /* ce.earlierUseIteration / lastUsedIteration (MM:1647-1648) */
  int32_t weight, flags; /* MMP_SCALE_NO_LOCAL_STATS */
} mmp_scale_in;
/* The pod's TypeConstraintManager.localInstanceSetStats is null: it is only assigned when the pod's own ADDED event created its
 * instance set (TCM:557-583), so a pod that joined an existing set sees EMPTY_STATS (TCM:236-239) and never scales down.  The
 * adapter passes `typeConstraints != null && typeConstraints.getLocalInstanceSetStats().totalCapacity == 0` here. */
#define MMP_SCALE_NO_LOCAL_STATS 1
typedef struct {
  int64_t now, last_check_time;                     /* timeDelta = now - lastCheckTime (MM:5641-5642) */
  int32_t iteration, scale_up_rpm_threshold;        /* iterationCounter, scaleUpRpmThreshold */
  int32_t second_copy_min_age_iters, second_copy_max_age_iters;  /* MM:5621-5622 */
  int64_t second_copy_lru_threshold_ms;             /* MM:5628 */
  int64_t rate_check_interval_ms;                   /* RATE_CHECK_INTERVAL_MS MM:238 */
  int64_t assume_completed_ms;                      /* loadingTimeStats(type).assumeCompletedAfterMillis() (MM:5765-5766) */
  int64_t second_copy_remove_max_age_ms;            /* SECOND_COPY_REMOVE_MAX_AGE_MS MM:257 */
  int32_t can_remove, reserved;                     /* the janitor's canRemove (MM:6197) */
} mmp_scale_params;
typedef struct {
  int32_t action;          /* 0 nothing, 1 add a second copy (regular-usage trigger MM:5726-5758), 2 scale up by copies_to_load
                              (MM:5760-5795), -1 the model has more registered instances than the device list holds: host path */
  int32_t copies_to_load;
  int64_t load_last_used;  /* lastUsed for the triggered loads: lastCheckTime (second copy) or now + 20 s (scale-up, MM:5675) */
  int32_t rpm, i1, i2;     /* measured rate; the updated usage iterations */
  int32_t set_heavy;       /* rpm above 3/4 of the threshold: ce.setLastHeavyTime(now) (MM:5712) */
  int32_t remove;          /* removeModelCopies (MM:6197-6335): this pod should drop its copy */
} mmp_scale_out;
/* rateTrackingTask's loop body (MM:5684-5806, exclude set MM:5835-5856, loadedSince MM:5858-5870) and the janitor's
 * removeModelCopies (MM:6197-6310, who-drops-the-copy by PLACEMENT_ORDER MM:6314-6335) for a batch of cache entries,
 * against the committed snapshot (instance table, type-set stats) and the registry (copies, failures, load times). */
int32_t mmp_scale_eval(mmp_fleet *, const mmp_scale_in *in, int32_t n, const mmp_scale_params *params, mmp_scale_out *out);
/* The reaper's prune pass (pruneModelRegistry MM:6524-6609, pruneMissingInstances MM:6752-6784) over the whole registry in one
 * sweep: registrations on instances that are not in the instance table, older than assume_gone_ms and missing for longer than
 * assume_gone_ms (ASSUME_INSTANCE_GONE_AFTER_MS, MM:270).  missing_since (max_instances entries, in/out) is the reaper's
 * `missings` map by instance index, 0 = absent.  Writes the models with entries to prune and, per model, the bit mask of the
 * pruned inline edges; returns how many (the registry itself is updated by the caller through mmp_model_upsert, as the
 * reference does through a conditional KV write). */
int32_t mmp_registry_prune(mmp_fleet *, int32_t self, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, int32_t *out_models,
                           uint8_t *out_masks, int32_t cap);

/* tuning / measurement knobs, same meaning as the MMP_* environment variables read at mmp_fleet_create:
 *   "one_mode"        how a batch of <= 32 decisions is launched: 0 the streaming kernel (k_place_lanes), 1 the latency kernel
 *                     k_place_small as a stream launch, 2 k_place_small as a replayed CUDA graph, 3 (default) a request to the
 *                     resident server kernel k_place_server (no launch per call: the host posts the request into mapped memory
 *                     and spins on the answer; one caller at a time, concurrent callers take the graph path)
 *   "server_life_us"  longest residence of one k_place_server launch (default 2000): bounds how long a device-wide wait
 *                     (cudaFree inside a commit) can be held up; "server_idle_us" (default 300): it leaves earlier when idle
 *   "direct"          1 (default): batches are resolved by k_place_direct (rows read straight from memory); 0: by the streaming
 *                     kernel k_place_lanes (whole rows through TMA landing stages) -- MMP_KERNEL=direct | lanes | tile
 *   "sort_slots"      k_place_direct resolves a batch of >= 8192 decisions in type-slot order: 0 never, 1 always, 2 (default) when
 *                     the committed snapshot's candidate sets are sparse (long walks: lanes of a warp then finish together)
 *   "small_max"       untraced batches of up to this many decisions run on k_place_small (one wave of 32-thread blocks, rows
 *                     read straight from memory) instead of the streaming kernel
 *   "lane_budget"     walk steps a lane may spend before its decision is redone by the whole warp
 *   "lane_warps"      warps per block of k_place_lanes (0 = default 12)
 *   "commit_host_only" 1: every commit takes the structural (host) path */
int32_t mmp_tune(mmp_fleet *, const char *key, int64_t value);
/* CUDA-event duration (ms) of the device part of the last mmp_stats ("stats"), mmp_reaper_select ("reaper": registry sweep +
 * sort + select), mmp_lru_apply ("lru_apply": the event kernel) on this fleet; "commit": host-clock ms of the last commit; "prune": mmp_registry_prune;
 * "dealt_kernel" / "dealt_wait": k_place_dealt and the arrival wait of the last peer-access step of an instance-sharded fleet */
int32_t mmp_last_timing(mmp_fleet *, const char *key, double *ms);
/* which path the last mmp_fleet_commit took: 1 = structural (host: string ranks, type-constraint sets, sort), 2 = device
 * (numeric instance updates / model-record deltas only: scattered into the device-resident tables, re-ranked and rebuilt
 * there); and its duration on the host clock */
int32_t mmp_commit_info(mmp_fleet *, int32_t *path, double *ms);

#ifdef __cplusplus
}
#endif
#endif
