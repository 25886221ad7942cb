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
/* Same with a CALL-WIDE exclude set of any size: every decision of the call behaves as if exclude[0, n_exclude) (instance
 * indices) were added to its CacheMissExcludeSet -- the rate-tracking scale-up's getExcludeSet() ∪ copies (MM:5771-5806,
 * 5835-5856), the janitor's every-copy-plus-self (MM:6915-6927), chained ensureLoadedElsewhere targets (MM:4575-4584) --
 * on top of its own extras (still <= MMP_MAX_EXTRA) and MMP_DF_* flags.  Its members leave the filtered iterator like
 * instances the type does not allow (MM:4760-4771).  trace / cand_mask may be NULL and mean what they mean for
 * mmp_place_batch_trace.  Duplicate ids are allowed; ids of instances that are not live are ignored.  An id outside
 * [0, max_instances), or exclude == NULL with n_exclude > 0, fails the call with MMP_E_ARG before anything is written.
 * n_exclude == 0 is exactly mmp_place_batch / _trace.  A call with a set that would take the instance-sharded path (an
 * instance-sharded fleet, or an untraced call on one that connected a communicator) fails with MMP_E_STATE.
 * Latency: the call derives its own copy of the per-type-slot tables on the device (two small launches), so a batch of
 * <= 32 decisions skips the resident server and the captured graph (one_mode 2 / 3, which hold the epoch's tables) and is
 * launched as k_place_small (one_mode 0: the batch kernel).  The micro-batcher never sees such calls. */
int32_t mmp_place_batch_excluding(mmp_fleet *, const mmp_decision_in *in, int32_t n, const mmp_instance_row *fresh, int32_t n_fresh,
                                  const int32_t *extra, int32_t n_extra, const int32_t *exclude, int32_t n_exclude,
                                  mmp_decision_out *out, mmp_decision_trace *trace, uint32_t *cand_mask, int64_t now_ms, uint64_t seed);
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
#define MMP_SERVER_SLOTS 8  /* concurrent callers the resident server (one_mode 3) answers without a launch: one slot and one
                               warp of k_place_server each; a call that finds every slot taken takes the graph path */
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
/* One run of the leader's reaper task (MM:6436-6494) against the committed epoch and the registry as of the last commit, in
 * one call: the prune of pruneModelRegistry (MM:6536-6590, 6752-6784), repairLastUsedTimeIfNeeded (MM:6837-6850), the
 * candidates of MM:6574-6577 on the pruned and repaired records, the selection of mmp_reaper_select over every partition and
 * the placement of every selected model, in the reference's order:
 *   prune     every registration, loaded and failed, exactly as mmp_registry_prune_ids (self = leader: the leader's own
 *             registrations are never pruned; missing_since stamped the same way).  Pruned pairs in (model, registration
 *             position) order: pruned_models[k] / pruned_instances[k].
 *   repair    every model whose last_used is INT64_MAX (mmp_model_upsert and mmp_model_upsert_json accept the value) is taken as
 *             now_ms - 3 x 3 600 000 (LASTUSED_AGE_ON_ADD_MS x 3) from here on: its sort position and its load's lastUsed.
 *             Repaired models in model order.
 *   select    the gate and globalLru of MM:6456-6463 from the epoch's stats; the candidates of a pruned record count its
 *             remaining registrations (a pruned registration at position < copy_count was a loaded copy, any other a failed
 *             load).  Then the closed loop's REAPER run at t = now_ms: the whole cluster without type constraints, otherwise
 *             every partition in mmp_stats order with one shared taken set; N12 and the emission rule as mmp_reaper_select.  A
 *             size estimate of 0 (the reference's ArithmeticException, MM:6651) ends the run at that partition: not an error,
 *             the report names it and everything before it is real.
 *   place     each selected model, in emission order, is getNext(model, self = leader, lastUsed = its (repaired) lastUsed)
 *             with no flags and no extra excludes, all against the one epoch (N6); decision k draws with id k (+ id_base):
 *             loads[k] equals mmp_place_batch of those records with the same seed.  A leader that is not live in the epoch
 *             gets MMP_TARGET_INVALID, as mmp_place_batch answers such a decision.
 * missing_since (max_instances entries, in/out) comes back as the reaper's `missings` map after its cleanup (MM:6601-6607):
 * entries with now_ms - v > assume_gone_ms, or whose instance is in the instance table, are cleared (0).  This is the one
 * difference from mmp_registry_prune_ids, which leaves the cleanup to its caller.
 * The caller writes the pruned and repaired records back (KV conditional writes) and calls ensureLoadedInternal(model,
 * last_used, ...) for each load whose target is not MMP_TARGET_NONE.  The outputs hold the first cap of each list; the report
 * gives the totals.  Returns the number of loads.  Errors (nothing written): MMP_E_ARG for a leader outside
 * [0, max_instances), a negative cap or assume_gone_ms, missing_since or report NULL, or a NULL output with a positive cap;
 * MMP_E_EPOCH without a commit; MMP_E_STATE on an instance-sharded fleet or one that connected a communicator (placement there
 * is a collective call every shard makes: keep mmp_registry_prune_ids + mmp_reaper_select + mmp_place_batch).  Sets the
 * "reaper_run" timing. */
typedef struct {
  int32_t model, target, n_candidates, reserved;  /* target: instance index, MMP_TARGET_NONE, MMP_TARGET_SELF or MMP_TARGET_INVALID */
  int64_t last_used;  /* the lastUsed ensureLoadedInternal is called with (MM:6712, 6727): the repaired value where repaired */
} mmp_reaper_load;    /* 24 B */
typedef struct {
  int32_t n_pruned, n_repaired, n_loads;  /* totals; the outputs hold the first cap of each */
  int32_t stopped_partition;  /* mmp_stats index of the partition whose size estimate was 0 (0: the whole cluster), -1 when
                                 the run completed */
} mmp_reaper_report;
int32_t mmp_reaper_run(mmp_fleet *, int32_t leader, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, uint64_t seed,
                       int32_t *pruned_models, int32_t *pruned_instances, int32_t pruned_cap, int32_t *repaired_models,
                       int32_t repaired_cap, mmp_reaper_load *loads, int32_t loads_cap, mmp_reaper_report *report);

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
/* The read side of the same caches (of the standalone store or of the closed loop's).  A read sees every event of every
 * mmp_lru_apply(_status) / mmp_churn_seed / mmp_churn_step call that has returned and none of a call still in progress. */
typedef struct {
  int32_t model, weight;
  int64_t last_used;
  int64_t load_ts;    /* registration time of a closed-loop copy (MR.instanceIds value); -1 in the standalone store and when
                         the copy is not registered */
} mmp_lru_entry;      /* 24 B */
/* descendingMapWithCutoff(used_since) of each listed cache (CLHM:1226-1260): from the most recently used entry down, up to
 * the first with 0 < last_used < used_since; used_since <= 0 is descendingLruMap() (CLHM:1087-1116), the whole deque.
 * instances: n cache indices, repeats allowed (listed again), NULL = 0 .. n-1.  offsets[0 .. n]: cache i's walk is entries
 * offsets[i] .. offsets[i+1] of the concatenation, whatever cap is; out receives its first cap entries (MRU first within
 * each cache).  Nothing is written on an error.  Sets the "lru_read" timing. */
int32_t mmp_lru_read(mmp_fleet *, const int32_t *instances, int32_t n, int64_t used_since, int64_t *offsets, mmp_lru_entry *out,
                     int64_t cap);
/* getLastUsedTime (CLHM:742-746: -1 when absent or last_used <= 0) and getWeight (CLHM:768-771: -1 when absent) of n
 * (instance, model) pairs, with the copy's load_ts as mmp_lru_entry has it (-1 when absent).  Nothing is written on an error. */
int32_t mmp_lru_lookup(mmp_fleet *, int32_t n, const int32_t *instance, const int32_t *model, int64_t *last_used, int32_t *weight,
                       int64_t *load_ts);

/* ---- the closed loop on the device (SURVEY.md §8a rows a11 admission, a12 rebalance; §8f-1 ingest / ordering maintenance,
 * §8f-4 fleet simulator; BASELINE.json configs[3] "churn").  One call = one republish window (2 s, INSTANCE_REC_PUBLISH_MIN_
 * PERIOD_MS MM:232) of the WHOLE fleet, evaluated against the instance and model records as committed at its start (N6):
 *   REQUEST of a model with registered copies -> runtimeCache.get on copy (u mod copies) in registration order;
 *   REQUEST of a model with none: the first one in the window is a cache miss -> getNext (self = caller, lastUsed = t) ->
 *     loadLocal on the target (MMP_LRU_LOAD's admission rules) -> evictions -> onEviction (MM:2875-2931: deregistration;
 *     a copy loaded more than 2 x load_timeout_ms ago whose type set is < 95 % full is queued for ensureLoadedElsewhere and
 *     placed first in the next window, MM:2915-2931); later misses of the same model in the window are coalesced;
 *   REMOVE -> runtimeCache.remove on every registered copy;
 *   REAPER (caller = the leader instance, t = the reaper's clock; model and u ignored) -> one run of the reaper's proactive
 *     loads (MM:6456-6494): the gate and globalLru of MM:6456-6463, the candidates of MM:6574-6577 (no loaded copy, fewer
 *     than 2 failed loads, used after globalLru unless the cluster has free space), then triggerProactiveLoadsForInstanceSubset
 *     (MM:6616-6747) for the whole cluster, or with type constraints for each partition in mmp_stats order with one `taken`
 *     set: size estimate, spaceToFill, the free-space and total counts and the lastUsed cutoff (age() at t), the bounded
 *     most-recently-used selection (N12: of equal lastUsed the first model in index order) and the emission rule of
 *     MM:6711-6719.  Every emitted model is a decision getNext(model, self = caller, lastUsed = the model's lastUsed) with no
 *     extra excludes, loaded on its target at last_used = the model's lastUsed on the clock t (ensureLoadedInternal MM:6727);
 *     its decisions stand at the REAPER's trace position, in emission order, and coalesce with the window's other decisions
 *     as misses do (a model already decided in the window is not decided again; a later miss of a model the reaper decided
 *     is coalesced).  A size estimate of 0 (the reference's ArithmeticException, MM:6651) ends the run at that partition.
 *     An out-of-range caller makes the run's decisions malformed (status 8), as for a REQUEST.
 *     Epoch-batching choices (the oracle makes the same): every partition reads the one snapshot of the window's start (the
 *     reference sleeps 2 x INSTANCE_REC_PUBLISH_MIN_PERIOD_MS between partitions, MM:6481-6484: put the runs in separate
 *     windows for that); the prune half of pruneModelRegistry is a no-op (no instance leaves the table in the loop);
 *     repairLastUsedTimeIfNeeded, vmodels and leaseless-record cleanup are not modelled; the caller picks the leader;
 *     DISABLE_PROACTIVE_LOADING is a trace without REAPER events.  A window with REAPER events reads the selections' count
 *     back once (one host synchronisation) to size its decision buffers; a window without them runs as before;
 *   then the registry changes, publishInstanceRecord with its significance thresholds (MM:5390-5470) per instance, and a
 *   commit (re-rank under PLACEMENT_ORDER, tables, bitmap) -- all on the device.  The host only reads the reports.
 * Requires an unsharded fleet; a model may hold any number of registrations (loaded copies, then failed loads), as long as
 * its copy_count tells its loaded copies apart (not saturated at 255 over more than 255 registrations).  Replaces nothing in the
 * reference 1:1 (each pod runs its own loop there); it is the batched, fleet-wide form of it for simulation / what-if runs. ---- */
enum { MMP_CHURN_REQUEST = 0, MMP_CHURN_REMOVE = 1, MMP_CHURN_REAPER = 2 };
typedef struct { int32_t type; int32_t model; int32_t caller; uint32_t u; int64_t t; } mmp_churn_event;
typedef struct {
  int32_t model, self, target, n_candidates;
  int32_t status;  /* MMP_LOAD_* of the load, 1 = nowhere to load (getNext null), 7 = queued reload skipped (the model has a
                      copy again), 8 = malformed, 9 = accepted but evicted again later in the window */
  int32_t event;   /* index of the REQUEST or REAPER event that caused it, or -1 - k for the k-th queued ensureLoadedElsewhere */
} mmp_churn_decision;
typedef struct { int32_t instance, model; int64_t last_used; int32_t weight, order, reload; } mmp_churn_eviction;
typedef struct { int64_t load_timeout_ms; int64_t last_published_ms; int32_t slots_per_instance; int32_t reserved; } mmp_churn_config;
typedef struct {
  int32_t n_published, n_carry, n_coalesced, n_lru_events;
  float ms_classify, ms_place, ms_route, ms_apply, ms_registry, ms_commit, ms_total;  /* CUDA-event times of the phases */
  float ms_reaper; /* the reaper pass of the window's REAPER events, its read-back included (0 without them); not in ms_classify */
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
/* the same, with every registration: ids[0 .. min(n, cap)) = the model's instance indices in registration order (the first
 * copy_count loaded, then the failed loads); returns n, the model's registration count (row may be NULL) */
int32_t mmp_churn_model_ids(mmp_fleet *, int32_t model, mmp_model_row *row, int32_t *ids, int32_t cap);
/* ---- registry-side batch scans (SURVEY.md §8a row a14, §8f-2) ---- */
/* MR.instanceIds / failedIn VALUES (load-start / failure times) and MR.lastUnloadTime ("lul").  edge_ts[i] is the time of the
 * i-th id of the model's last mmp_model_upsert (loaded first, then failed), for every registration; times past the model's
 * registration count are ignored, and a registration without one reads 0 (unknown).  A time stays with its position until the
 * next call.  mmp_model_upsert_json takes them from the record. */
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
                              (MM:5760-5795), -1 the entry's model or instance index is out of range, or its copy_count is saturated
                              (255) while it holds more than 255 registrations: where the loaded copies end is unknown */
  int32_t copies_to_load;
  int64_t load_last_used;  /* lastUsed for the triggered loads: lastCheckTime (second copy) or now + 20 s (scale-up, MM:5675) */
  int32_t rpm, i1, i2;     /* measured rate; the updated usage iterations */
  int32_t set_heavy;       /* rpm above 3/4 of the threshold: ce.setLastHeavyTime(now) (MM:5712) */
  int32_t remove;          /* removeModelCopies (MM:6197-6335): this pod should drop its copy */
} mmp_scale_out;
/* rateTrackingTask's loop body (MM:5684-5806, exclude set MM:5835-5856, loadedSince MM:5858-5870) and the janitor's
 * removeModelCopies (MM:6197-6310, who-drops-the-copy by PLACEMENT_ORDER MM:6314-6335) for a batch of cache entries,
 * against the committed snapshot (instance table, type-set stats) and the registry (copies, failures, load times): every
 * registration of the model, the first copy_count of them loaded, the rest failed loads. */
int32_t mmp_scale_eval(mmp_fleet *, const mmp_scale_in *in, int32_t n, const mmp_scale_params *params, mmp_scale_out *out);
/* The reaper's prune pass (pruneModelRegistry MM:6524-6609, pruneMissingInstances MM:6752-6784) over the whole registry in one
 * sweep: registrations on instances that are not in the instance table, older than assume_gone_ms and missing for longer than
 * assume_gone_ms (ASSUME_INSTANCE_GONE_AFTER_MS, MM:270).  missing_since (max_instances entries, in/out) is the reaper's
 * `missings` map by instance index, 0 = absent.  The four-registration view: it reads (and stamps missing_since for) the
 * first four registrations of each model only.  Writes the models with entries to prune and, per model, the bit mask of the
 * pruned inline edges; returns how many (the registry itself is updated by the caller through mmp_model_upsert, as the
 * reference does through a conditional KV write).  When that exceeds cap, the outputs hold the first cap of those models in
 * model order.  mmp_registry_prune_ids reads every registration. */
int32_t mmp_registry_prune(mmp_fleet *, int32_t self, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since, int32_t *out_models,
                           uint8_t *out_masks, int32_t cap);
/* The same pass over every registration of every model, stamping missing_since for each.  Reports each pruned registration
 * as a (model, instance) pair, in (model, registration position) order, and returns how many there are; when that exceeds
 * cap the outputs hold the first cap pairs of that order.  A second call with the same now_ms and the updated missing_since
 * returns the same pairs.  assume_gone_ms >= 0.  Sets the "prune" timing. */
int32_t mmp_registry_prune_ids(mmp_fleet *, int32_t self, int64_t now_ms, int64_t assume_gone_ms, int64_t *missing_since,
                               int32_t *out_models, int32_t *out_instances, int32_t cap);
/* The registry loop of one pod's janitor task (MM:6013-6145) against the committed epoch and the registry as of the last
 * commit, in one call.  entries[] is the pod's runtimeCache.descendingMap() (MM:5892) as the loop reads it, at most one entry per
 * model, in any order.  For every model with a registration of `self` (every registration, the overflow ones included):
 *   loaded     self is among the first copy_count registrations; failedTime = the time of self's first failed registration
 *   remLoaded  loaded && (no entry || the entry is MMP_JANITOR_FAILED)
 *   remFailed  there is a failure record, and: an entry that is not failed; or now - failedTime > expiry (Java long
 *              arithmetic), expiry = load_failure_expiry_ms / 2 when lu > 0 && now - lu < 180 000, load_failure_expiry_ms
 *              otherwise, lu = the entry's last_used (-1 without one)
 *   candidate  loaded && !remLoaded && the entry's last_used > 0, keyed by that last_used.  VALUE_COMP compares the value only, so
 *              of candidates with equal last_used only the first in model order stays (quirk N15; N12's stand-in for registry
 *              order)
 * then, over the candidates by ascending last_used, the budget walk of MM:6117-6140: canRemove = removed == 0 || weight <= budget
 * (budget from adjusted_capacity / 20, less each removed weight: it may go negative), and removeModelCopies is mmp_scale_eval's
 * scale-down with that canRemove, and the registration time of self's copy equal to the entry's load_ts
 * (removeLocalModelCopyAsync MM:6347-6349).
 * One edit per model that has anything to do, in model order, what[] the OR of the MMP_JE_* bits; last_used / last_unload_time
 * are the record's after the edit (updateLastUsed of the entry's last_used where it is > 0, MR:239-246; updateLastUnloadTime:
 * 0 when at most 2 loaded copies remain, else now).  The edits hold the first cap; the report gives the totals (n_referencing:
 * the reference's j, the models that reference self; n_candidates after the VALUE_COMP ties are dropped).
 * Not modelled (stays in the pod): the first loop over the local cache (MM:5892-6008), shuttingDown, the KV conditional writes
 * and their retry on conflict, and the async removal's isLoadedElsewhere and ce.remove() (MM:6353-6373).
 * Returns the number of edits.  Errors (nothing written): MMP_E_ARG for self outside [0, max_instances), an entry's model out
 * of range or two entries of one model, n < 0, p or report NULL, edits NULL with cap > 0, or a p->scale mmp_scale_eval refuses;
 * MMP_E_EPOCH without a commit; MMP_E_STATE when the committed registry holds no registration times (neither mmp_model_times
 * nor a JSON record supplied any: every failure would read as expired).  Sets the "janitor_run" timing. */
#define MMP_JANITOR_FAILED 1u              /* ce.isFailed() */
typedef struct {
  int32_t model, weight;                   /* model index; ce.getWeight() */
  int64_t last_used;                       /* runtimeCache.getLastUsedTime(model): -1 when absent or <= 0 (CLHM:742-746) */
  int64_t load_ts;                         /* ce.loadTimestamp (removeLocalModelCopyAsync compares it, MM:6347-6349) */
  int64_t last_heavy;                      /* ce.getLastHeavyTime() */
  int64_t count;                           /* the interval count ce.getRpm(timeSinceLastCheck) divides (MM:6292) */
  uint32_t flags, reserved;                /* MMP_JANITOR_FAILED */
} mmp_janitor_entry;                       /* 48 B */
typedef struct {
  mmp_scale_params scale;                  /* now, last_check_time, scale_up_rpm_threshold, rate_check_interval_ms,
                                              second_copy_remove_max_age_ms as mmp_scale_eval reads them; can_remove ignored */
  int64_t load_failure_expiry_ms;          /* LOAD_FAILURE_EXPIRY_MS (MM:219); the in-use expiry is half of it (MM:221) */
  int64_t adjusted_capacity;               /* getAdjustedCacheCapacity() (MM:5363): the budget is a twentieth of it (MM:6117) */
  uint32_t flags, reserved;                /* MMP_SCALE_NO_LOCAL_STATS for this pod (quirk N13) */
} mmp_janitor_params;
#define MMP_JE_UNREGISTER   1u  /* remLoaded: remove self from instanceIds, updateLastUnloadTime (MM:6059-6062) */
#define MMP_JE_DROP_FAILURE 2u  /* remFailed: removeLoadFailure(self) (MM:6063-6065) */
#define MMP_JE_REMOVE_LOCAL 4u  /* the pod's failed cache entry goes too (MM:6089-6091) */
#define MMP_JE_SCALE_DOWN   8u  /* removeModelCopies returned true under the budget: the async removal of MM:6353-6373 starts */
#define MMP_JE_UNDECIDED   16u  /* copy_count saturated at 255 over > 255 registrations: nothing decided (as mmp_scale_eval's -1) */
typedef struct {
  int32_t model; uint32_t what;
  int64_t last_used;         /* the record's lastUsed after the updateLastUsed calls of the edit (MR:239-246) */
  int64_t last_unload_time;  /* after updateLastUnloadTime where the edit unregisters self, else the record's value */
} mmp_janitor_edit;          /* 24 B */
typedef struct { int32_t n_referencing, n_edits, n_candidates, n_removed; int64_t weight_removed; } mmp_janitor_report;
int32_t mmp_janitor_run(mmp_fleet *, int32_t self, const mmp_janitor_entry *entries, int32_t n, const mmp_janitor_params *p,
                        mmp_janitor_edit *edits, int32_t cap, mmp_janitor_report *report);
/* One run of one pod's whole janitor task (janitorTask MM:5876-6145) against the committed epoch and the registry as of the
 * last commit, in one call: the cache pass over the pod's cache (MM:5892-6008), then mmp_janitor_run's registry pass on the
 * records the cache pass left.  entries[] is runtimeCache.descendingMap() (MM:5892) after removeUnloadBufferEntry, IN THAT
 * ORDER (most recently used first), at most one entry per model.  In Java long arithmetic, now = p->janitor.scale.now,
 * window = janitor_freq_secs * 2000 + load_timeout_ms (MM:5933-5934); a "record" is the committed one (no record: the model
 * index is at or past the committed model count, a model never upserted).  Per entry, in order:
 *   skips       MMP_JANITOR_NOT_DONE: MMP_JC_NOT_DONE.  last_used <= 0: MMP_JC_NOT_CACHED.  Nothing else (MM:5905-5912).
 *   order       the entries past the skips "qualify": one whose last_used > the previous qualifying one's (Long.MAX_VALUE
 *               before the first) gets MMP_JC_OUT_OF_ORDER, the log line of MM:5913-5917.
 *   stop        the first qualifying entry with last_used == Long.MAX_VALUE (quirk N16): MMP_JC_STOP, the pod force-sets its
 *               cache entry's lastUsed to out[r].last_used = now - 3 x 3 600 000 (LASTUSED_AGE_ON_ADD_MS); MMP_JC_REPAIR where
 *               the record's lastUsed is Long.MAX_VALUE (repairLastUsedTimeIfNeeded MM:6837-6850: the record gets the same
 *               value).  The task ends there (`return`, MM:5929): every later entry is MMP_JC_NOT_REACHED alone, no registry
 *               pass runs (report.registry_ran = 0, its report zero, no edits).
 *   recent      now - last_used < window: the stale update where there is a record (MM:5933-5939).
 *   stale       updateLastUsedTimeInRegistryIfStale (MM:6165-6183): last_used - rec.lastUsed >= min_stale_age_ms writes the
 *               record's lastUsed, raised to last_used as updateLastUsed does (MR:239-246): MMP_JC_STALE_UPDATE.
 *   check       otherwise (MM:5941-5997), over every registration of the model (the overflow ones included):
 *                 undecided   a copy_count saturated at 255 over more than 255 registrations (as MMP_JE_UNDECIDED):
 *                             MMP_JC_UNDECIDED, nothing written; the pod runs the loop body for that entry itself
 *                 matched     the pod's first failed registration's time == load_complete_ts (an MMP_JANITOR_FAILED
 *                             entry), else its first loaded registration's time == load_ts: the stale update
 *                 remove      no record, MMP_JANITOR_NOT_LIVE or MMP_JANITOR_UNLOAD_RECENT: MMP_JC_REMOVE, ce.remove()
 *                 re-register otherwise MMP_JC_REREGISTER: instanceIds.put(self, load_ts), removeLoadFailure(self),
 *                             updateLastUsed(last_used) (MM:5980-5982); out[r].replaced_ts is the pod's loaded registration
 *                             time it replaced (not for a failed entry, as regLoadTimestamp), -1 where there was none.
 * out[r] is entries[r]'s action in entry order: the OR of its MMP_JC_* bits and last_used, the record's lastUsed after the
 * cache pass (its own where nothing was written, 0 without a record), or for MMP_JC_STOP the forced cache value.
 * The registry pass is mmp_janitor_run's on the same entries, with two differences: a record the cache pass wrote is read as
 * written (a re-registered model has the pod among its loaded copies at load_ts, one more loaded copy where the pod was not
 * loaded, and no failure record of the pod; a raised lastUsed), and an entry the cache pass removed reads last_used = -1
 * (getLastUsedTime of a key no longer in the cache, MM:6045, 6068, 6094) while its MMP_JANITOR_FAILED stays as given.
 * Edits come back in model order, as mmp_janitor_run's.
 * Epoch batching: one now for both loops (the reference reads the clock at MM:5899 and MM:6018); registry.get and getStrong
 * both read the committed record; every conditional write, forceSetLastUsedTime and ce.remove() of the cache pass succeeds,
 * and the registry pass sees them.  Not modelled (stays in the pod): shuttingDown, verifyKvStoreConnection, the unload-buffer
 * step, the KV writes and their retry, publishInstanceRecordAsync (report.cache_changed) and the log lines (INTEGRATION.md §8).
 * Returns the number of edits.  Errors (nothing written): MMP_E_ARG for self outside [0, max_instances), an entry's model out of
 * range or two entries of one model, n < 0 or n > 2^24, p or report NULL, out NULL with n > 0, edits NULL with cap > 0, or a
 * p->janitor mmp_janitor_run refuses; MMP_E_EPOCH without a commit; MMP_E_STATE when the committed registry holds no
 * registration times.  Sets the "janitor_task" timing. */
#define MMP_JANITOR_NOT_DONE 2u            /* !ce.isDone(): still loading (MM:5905) */
#define MMP_JANITOR_NOT_LIVE 4u            /* ce.state < CacheEntry.LOADING || ce.state > CacheEntry.ACTIVE (MM:5968) */
#define MMP_JANITOR_UNLOAD_RECENT 8u       /* ce.unloadAttemptedRecently() (MM:5969) */
typedef struct {
  mmp_janitor_entry e;                     /* as mmp_janitor_run reads it; flags MMP_JANITOR_FAILED | the bits above */
  int64_t load_complete_ts;                /* ce.loadCompleteTimestamp (a failed entry's registration time, MM:5952) */
} mmp_janitor_task_entry;                  /* 56 B */
typedef struct {
  mmp_janitor_params janitor;              /* as mmp_janitor_run reads them */
  int64_t min_stale_age_ms;                /* minStaleAge (MM:6162): the pod draws it once, 6 h + a random hour */
  int64_t janitor_freq_secs;               /* LOCAL_JANITOR_FREQ_SECS (MM:235) */
  int64_t load_timeout_ms;                 /* loadTimeoutMs */
} mmp_janitor_task_params;                 /* 120 B */
#define MMP_JC_NOT_DONE      1u   /* skipped: still loading */
#define MMP_JC_NOT_CACHED    2u   /* skipped: last_used <= 0 */
#define MMP_JC_OUT_OF_ORDER  4u   /* last_used above the previous qualifying entry's: log it */
#define MMP_JC_STOP          8u   /* Long.MAX_VALUE last_used: forceSetLastUsedTime(out.last_used); the task ends here */
#define MMP_JC_REPAIR       16u   /* with MMP_JC_STOP: the record's lastUsed was Long.MAX_VALUE, set it to out.last_used */
#define MMP_JC_NOT_REACHED  32u   /* after the stop: alone, nothing done */
#define MMP_JC_STALE_UPDATE 64u   /* conditionalSet of the record with lastUsed = out.last_used */
#define MMP_JC_REMOVE      128u   /* ce.remove() */
#define MMP_JC_REREGISTER  256u   /* put self at load_ts, removeLoadFailure(self), lastUsed = out.last_used; conditionalSetAndGet */
#define MMP_JC_UNDECIDED   512u   /* copy_count saturated at 255 over > 255 registrations: nothing decided */
typedef struct {
  int32_t model; uint32_t what;            /* model; the OR of MMP_JC_* */
  int64_t last_used;                       /* the record's lastUsed after the cache pass, or the forced cache value (MMP_JC_STOP) */
  int64_t replaced_ts;                     /* MMP_JC_REREGISTER: the registration time it replaced, -1 for none; else -1 */
} mmp_janitor_cache_action;                /* 24 B */
typedef struct {
  int32_t n_not_done, n_not_cached, n_out_of_order, n_stop, n_repair;  /* entries with each MMP_JC_* bit, in bit order */
  int32_t n_not_reached, n_stale_update, n_remove, n_reregister, n_undecided;
  int32_t stopped_at;                      /* the MMP_JC_STOP entry, -1 for none */
  int32_t registry_ran;                    /* 1: the registry pass ran (no stop) */
  int32_t cache_changed;                   /* some ce.remove(): the pod calls publishInstanceRecordAsync (MM:6002-6004) */
  int32_t reserved;
  mmp_janitor_report registry;             /* the registry pass's, zero where it did not run */
} mmp_janitor_task_report;                 /* 80 B */
int32_t mmp_janitor_task(mmp_fleet *, int32_t self, const mmp_janitor_task_entry *entries, int32_t n,
                         const mmp_janitor_task_params *p, mmp_janitor_cache_action *out, mmp_janitor_edit *edits, int32_t cap,
                         mmp_janitor_task_report *report);
/* One run of one pod's rate-tracking task (rateTrackingTask MM:5619-5858) against the committed epoch and the registry as of
 * the last commit, in one call: the loop body of every cache entry and the loads it triggers, placed.  entries[] is the
 * pod's runtimeCache as the loop reads it, every entry's instance == self, at most one entry per model, in any order.
 *   gates     report.gate (MM:5646-5670):
 *               MMP_RATE_TOO_SOON        timeDelta * 5 < rate_check_interval_ms * 3 (Java long arithmetic): nothing is
 *                                        evaluated, and the pod does NOT advance lastCheckTime or iterationCounter (the
 *                                        return comes before the task's finally block)
 *               MMP_RATE_FEW_INSTANCES   clusterStats.instanceCount < 2: nothing is evaluated (no interval count is reset);
 *                                        the pod advances its clock and iteration
 *               MMP_RATE_NO_ENTRIES      n == 0: as MMP_RATE_FEW_INSTANCES
 *               MMP_RATE_RAN             the loop ran
 *             Under a gate out[r] is action 0 with rpm 0 and the entry's own i1 / i2.
 *   out[r]    exactly mmp_scale_eval's result for entries[r] with can_remove = 0: rpm, set_heavy, i1 / i2, action,
 *             copies_to_load and load_last_used.
 *   refusal   checkLoadFailureCount (MM:3771, 4607-4627): a model with 3 or more failure records (registrations past its
 *             loaded copies) whose time is > now - load_failure_expiry_ms / 2 gets no decision (report.n_refused_failures).
 *             checkLoadLocationCount cannot fire on these paths: the explicit excludes hold every copy.
 *   second    action 1: one decision getNext(model, self, lastUsed = lastCheckTime) with extras {self}, no heavy set,
 *   copy      favourSelf set (self is in toExclude, so UNBALANCED is not set: MM:6940-6943, 3526, 3782).
 *   scale-up  action 2: a chain of copies_to_load decisions (triggerChainedLoadIfNecessary MM:4560-4585, ensureLoadedInternal
 *             MM:6930-6952), lastUsed = now + 20 000 (MM:5675), every one excluding the call-wide heavy set of getExcludeSet
 *             (MM:5835-5856): the instances of the epoch other than self whose published rpm is > max(4 thr, ourRpm - 2 thr),
 *             ourRpm self's published rpm (0 when self is not in the epoch), as mmp_scale_eval reads it.
 *               decision 0      self = the pod; favourSelf only when the pod is a loaded registration of the model
 *               decision j > 0  self = target j-1 (the pod where target j-1 was MMP_TARGET_SELF), extras = targets 0..j-1
 *                               (the pod for a MMP_TARGET_SELF), favourSelf set
 *             A target of MMP_TARGET_NONE or MMP_TARGET_INVALID ends the chain (no chained trigger fires).  Decision j needs j
 *             extras: a chain longer than MMP_RATE_CHAIN_MAX is cut after its MMP_RATE_CHAIN_MAX-th decision, which carries
 *             MMP_RL_CHAIN_CUT and the copies not yet placed in `remaining`; the pod continues it with
 *             mmp_place_batch_excluding (INTEGRATION.md §9).
 *   fresh     every decision whose self is the pod reads fresh_self when given (getFreshInstanceRecord MM:5369), any other
 *             self its published row.
 *   draws     decision j of the chain of entries[r] (a second copy: j = 0) draws with id off[r] + j (MMP_DF_OWN_ID: id_base
 *             plays no part), off the exclusive prefix sum in entry order of each entry's decisions: 1 for a second copy,
 *             min(copies_to_load, MMP_RATE_CHAIN_MAX) for a scale-up, 0 when refused.  A call whose ids pass 2^24 is refused.
 * Epoch batching: every decision reads the one committed epoch; a chained decision's self is its target's published row,
 * not the record the target publishes mid-load; the chain assumes every target accepts its load (in the reference a
 * rejection ends the chain: the pod drops the rest of that chain, INTEGRATION.md §9).  The latency-based mode
 * (limitModelConcurrency, MaxConcCacheEntry) is not modelled.
 * Loads come back in (entry, chain_pos) order, the first loads_cap of them; the report gives the totals.  Returns the number
 * of loads.  Errors (nothing written): MMP_E_ARG for self outside [0, max_instances), an entry whose instance is not self,
 * an entry's model out of range or two entries of one model, n < 0, p or report NULL, out NULL with n > 0, loads NULL with
 * loads_cap > 0, a p->scale mmp_scale_eval refuses, a bad fresh_self, or ids past 2^24; MMP_E_EPOCH without a commit;
 * MMP_E_STATE when the committed registry holds no registration times, on an instance-sharded fleet or one that connected a
 * communicator.  Sets the "rate_run" timing. */
#define MMP_RATE_CHAIN_MAX (MMP_MAX_EXTRA + 1)
#define MMP_RATE_RAN 0
#define MMP_RATE_TOO_SOON 1
#define MMP_RATE_FEW_INSTANCES 2
#define MMP_RATE_NO_ENTRIES 3
typedef struct {
  mmp_scale_params scale;          /* as mmp_scale_eval reads them; can_remove ignored (no scale-down here) */
  int64_t load_failure_expiry_ms;  /* LOAD_FAILURE_EXPIRY_MS (MM:219); checkLoadFailureCount counts failures younger than half
                                      of it (IN_USE_LOAD_FAILURE_EXPIRY_MS, MM:221, 4607-4627) */
} mmp_rate_params;                 /* 80 B */
#define MMP_RL_SECOND_COPY 1u      /* a second copy (action 1), else a decision of a scale-up chain */
#define MMP_RL_CHAIN_CUT 2u        /* the chain was cut after this load: `remaining` copies are still to place */
typedef struct {
  int32_t entry, model;            /* index into entries[]; model */
  int32_t chain_pos;               /* 0 for a second copy; 0 .. MMP_RATE_CHAIN_MAX - 1 along a scale-up chain */
  int32_t self;                    /* the decision's self: the pod, or the previous load's target */
  int32_t target, n_candidates;    /* as mmp_decision_out; MMP_TARGET_INVALID also for a pod not live without fresh_self */
  int64_t last_used;               /* lastCheckTime (second copy, MM:5755) or now + 20 000 (scale-up, MM:5675) */
  uint32_t flags, remaining;       /* MMP_RL_*; remaining: copies of the chain not yet placed when it was cut */
} mmp_rate_load;                   /* 40 B */
typedef struct {
  int32_t gate;                    /* MMP_RATE_* */
  int32_t n_second, n_scale_up;    /* entries with action 1 / 2 */
  int32_t n_loads;                 /* decisions placed, every one of them in loads[] up to loads_cap */
  int32_t n_heavy;                 /* size of the heavy-instance exclude set */
  int32_t n_chains_cut, n_refused_failures, reserved;
} mmp_rate_report;
int32_t mmp_rate_run(mmp_fleet *, int32_t self, const mmp_scale_in *entries, int32_t n, const mmp_rate_params *p,
                     const mmp_instance_row *fresh_self, uint64_t seed, mmp_scale_out *out, mmp_rate_load *loads,
                     int32_t loads_cap, mmp_rate_report *report);
/* One pod's pre-shutdown migration (preShutdown MM:6959-7147, the distribution loop MM:6990-7047) against the committed epoch
 * and the registry as of the last commit, in one call: for every cache entry the pod holds and is registered for, a new copy
 * elsewhere (triggerNewModelCopyElsewhere MM:6913-6928), placed.  entries[] is runtimeCache.descendingLruMap() (MM:6990), most
 * recently used first, at most one entry per model.  In Java long arithmetic, cutoff = now - cutoff_age_ms (MM:7000):
 *   foundOther  some ranked instance of the epoch other than self (MM:6968-6976).  Without one nothing is evaluated or placed
 *               (every out[r] has what 0): report.found_other = 0 and the pod deregisters every entry (MM:7133-7143).
 *   registered  self is among the model's LOADED registrations in the committed registry, every registration looked at
 *               (MM:7007-7010).  Otherwise (registered only as a failed load, or no record) MMP_SD_NOT_REGISTERED and nothing
 *               else.  The registered entries are the reference's waitFor (report.n_registered).
 *   undecided   a model whose copy_count is saturated at 255 over more than 255 registrations (where its loaded copies end is
 *               unknown, as for mmp_scale_eval's -1 and MMP_JE_UNDECIDED): MMP_SD_UNDECIDED alone, no decision, counted in no
 *               report field; the pod runs the reference's loop body for that entry itself.
 *   stale       a registered entry with lru_t < cutoff: MMP_SD_STALE, counted in report.will_be_skipped (MM:7011-7014).
 *   task body   (MM:7016-7040), registered entries:
 *                 MMP_SD_ENTRY_GONE or _FAILED: nothing more (MM:7017-7020)
 *                 lruTime = lru_t != 0 ? lru_t : last_used (MM:7021), into out[r].last_used
 *                 lruTime >= 0: MMP_SD_REMOVE_LOCAL (ce.remove(), MM:7022-7024)
 *                 MMP_SD_ENTRY_ABORTED: MMP_SD_DEREGISTER_NOW (deregisterModelAsync now, MM:7027-7030)
 *                 lruTime > 0: checkLoadFailureCount (MM:3771, 4607-4627): 3 or more failure records (registrations past the
 *                   loaded copies) whose time is > now - load_failure_expiry_ms / 2 refuse the load: MMP_SD_REFUSED, no decision.
 *                   Otherwise MMP_SD_PLACED: one decision getNext(model, self, lastUsed = lruTime) excluding loaded u failed
 *                   (the committed row) and {self}, favourSelf set (self is in toExclude, so UNBALANCED is not set:
 *                   MM:6940-6943; with self excluded the flag cannot change the answer).  checkLoadLocationCount cannot fire:
 *                   every copy is excluded.
 *                 target an instance (>= 0) and lruTime >= cutoff: MMP_SD_WAIT, the `return ent` of MM:7037-7038 -- the pod
 *                   waits for this load.  MMP_TARGET_NONE is "Nowhere available to load": logged, not waited for.
 *   fresh       every decision reads fresh_self when given, else the pod's published row; a pod that is not ranked and has no
 *               fresh_self is answered MMP_TARGET_INVALID (as by mmp_rate_run).  The answers do not depend on whether the pod's
 *               own shutting-down record has been committed: self is excluded, and an unranked instance is in no candidate set.
 *   draws       entries[r]'s decision draws with id r (MMP_DF_OWN_ID: id_base plays no part), so an answer does not depend on
 *               which other entries were placed, and equals mmp_place_batch's on the same 32-byte record with the same seed.
 * Epoch batching: every decision reads the one committed epoch (the reference's tasks run concurrently on taskPool against a
 * clusterState that has not seen their loads yet); one fresh_self for every decision (the reference's fresh record drifts
 * as the tasks' ce.remove() calls empty the cache); the registry as of the last commit (the pod's KV writes catch the
 * difference).  Not modelled (stays in the pod): abortLoadings, publishInstanceRecord, removeUnloadBufferEntry, the wait
 * phase (MM:7048-7122) and every deregisterModelAsync write (INTEGRATION.md §10).
 * out[r] is entries[r]'s action, in entry order; without a decision target is MMP_TARGET_INVALID and n_candidates 0, and
 * last_used is 0 where the task body did not compute lruTime.  Returns n.  Errors (nothing written): MMP_E_ARG for self
 * outside [0, max_instances), an entry's model out of range or two entries of one model, n < 0 or n > 2^24, p or report
 * NULL, entries or out NULL with n > 0, or a bad fresh_self; MMP_E_EPOCH without a commit; MMP_E_STATE when the committed
 * registry holds no registration times, on an instance-sharded fleet or one that connected a communicator.  Sets the
 * "shutdown_run" timing. */
#define MMP_SD_ENTRY_GONE 1u       /* runtimeCache.getQuietly(model) returned null */
#define MMP_SD_ENTRY_FAILED 2u     /* ce.isFailed() */
#define MMP_SD_ENTRY_ABORTED 4u    /* ce.isAborted() after abortLoadings() */
typedef struct {
  int32_t model; uint32_t flags;   /* model index; MMP_SD_ENTRY_* */
  int64_t lru_t;                   /* the descendingLruMap value */
  int64_t last_used;               /* runtimeCache.getLastUsedTime(model): -1 when absent or <= 0 (CLHM:742-746) */
} mmp_shutdown_entry;              /* 24 B */
typedef struct {
  int64_t now;
  int64_t cutoff_age_ms;           /* CUTOFF_AGE_MS (MM:276): 3 600 000 */
  int64_t load_failure_expiry_ms;  /* LOAD_FAILURE_EXPIRY_MS (MM:219); checkLoadFailureCount counts failures younger than half */
} mmp_shutdown_params;             /* 24 B */
#define MMP_SD_NOT_REGISTERED 1u   /* self is not a loaded registration of the model: skipped (MM:7008-7010) */
#define MMP_SD_STALE 2u            /* lru_t < cutoff: counted in willBeSkipped (MM:7012-7014) */
#define MMP_SD_REMOVE_LOCAL 4u     /* lruTime >= 0: ce.remove() (MM:7022-7024) */
#define MMP_SD_DEREGISTER_NOW 8u   /* aborted: deregisterModelAsync(model, lruTime, loadTimestamp, ...) now (MM:7027-7030) */
#define MMP_SD_PLACED 16u          /* a decision was made: target / n_candidates are its answer */
#define MMP_SD_REFUSED 32u         /* lruTime > 0, but checkLoadFailureCount refused the load: no decision */
#define MMP_SD_WAIT 64u            /* target is an instance and lruTime >= cutoff: the pod waits for the load (MM:7037-7038) */
#define MMP_SD_UNDECIDED 128u      /* copy_count saturated at 255 over > 255 registrations: alone, nothing decided or counted */
typedef struct {
  int32_t model; uint32_t what;    /* model; the OR of MMP_SD_* */
  int32_t target, n_candidates;    /* as mmp_decision_out with MMP_SD_PLACED, else MMP_TARGET_INVALID and 0 */
  int64_t last_used;               /* the lruTime used, 0 where it was not computed */
} mmp_shutdown_action;             /* 24 B */
typedef struct {
  int32_t found_other;             /* 1: some ranked instance other than self; 0: nothing was evaluated */
  int32_t n_registered;            /* entries registered for self: the reference's waitFor.size() */
  int32_t will_be_skipped;         /* registered entries with lru_t < cutoff */
  int32_t n_placed, n_none, n_refused, n_wait;  /* entries with MMP_SD_PLACED, of them target MMP_TARGET_NONE; MMP_SD_REFUSED;
                                                   MMP_SD_WAIT */
  int32_t reserved;
} mmp_shutdown_report;             /* 32 B */
int32_t mmp_shutdown_run(mmp_fleet *, int32_t self, const mmp_shutdown_entry *entries, int32_t n, const mmp_shutdown_params *p,
                         const mmp_instance_row *fresh_self, uint64_t seed, mmp_shutdown_action *out, mmp_shutdown_report *report);
/* One pod's eviction listener (onEviction MM:2867-2933) for a burst of evictions, against the committed epoch and the registry
 * as of the last commit, in one call: every evicted copy deregistered (deregisterModel MM:2936-2962), and a copy elsewhere
 * placed for each one the rebalance rule reloads (ensureLoadedElsewhere MM:6905).  entries[] are the evictions the pod's cache
 * reported, in listener order, at most one entry per model.  Per entry, in Java long arithmetic, over every registration of the
 * model (the overflow ones included), loaded = the first copy_count registrations, the rest failed loads:
 *   undecided   a model whose copy_count is saturated at 255 over more than 255 registrations (where its loaded copies end is
 *               unknown, as for mmp_scale_eval's -1 and MMP_JE_UNDECIDED): MMP_EV_UNDECIDED alone, no decision, the record's
 *               own last_used / last_unload_time, counted in no report field; the pod runs the reference's listener task for
 *               that entry itself.
 *   deregister  MMP_EV_UNREGISTER: the pod's loaded registration has time load_ts (instanceIds.remove(self, loadTime)).
 *               MMP_EV_DROP_FAILURE: the pod's failed registration has time load_complete_ts (removeLoadFailure, MR:173-179).
 *               Neither: no write.  Otherwise out[r].last_used is the record's lastUsed after updateLastUsed(last_used) (0 reads
 *               as now, MR:239-246) and last_unload_time after updateLastUnloadTime where the pod is unregistered (0 when at
 *               most 2 loaded copies remain, else now, MR:260-262); both are mmp_janitor_run's record arithmetic.  Without a
 *               write, and for last_unload_time without MMP_EV_UNREGISTER, they are the record's own values.
 *   reload      MMP_EV_RELOAD (attemptReload, MM:2886-2896): the entry is not MMP_EV_ENTRY_FAILED, the pod has a registration,
 *               and now - t > 2 * load_timeout_ms, t the time of its loaded registration, else of its failed one (the record
 *               before the edit).
 *   gate        a reload whose model's type set is full (MM:2918-2920): typeSetStats of the model's committed type in the
 *               epoch, totalCapacity > 0 && instanceCount > 1 && 20 * totalFree / totalCapacity >= 1, fails:
 *               MMP_EV_CLUSTER_FULL, nothing more.
 *   elsewhere   ensureLoadedElsewhere on the record after the edit (MM:6905-6907, ensureLoadedInternal with {self} excluded):
 *                 MMP_EV_LOADED_ELSEWHERE  a loaded registration other than the pod on an instance the epoch ranks: the
 *                                          reference forwards to it and returns LOADED without a load (MM:3540-3760), so
 *                                          checkLoadLocationCount cannot fire either
 *                 MMP_EV_REFUSED           checkLoadFailureCount (MM:3771, 4607-4627): 3 or more failure records whose time is
 *                                          > now - load_failure_expiry_ms / 2; a failure record the edit dropped does not count
 *                 MMP_EV_PLACED            one decision getNext(model, self, lastUsed = last_used) excluding the committed
 *                                          registrations and {self}, favourSelf set (self is in toExclude, so UNBALANCED is
 *                                          not set: MM:6940-6943)
 *   fresh       every decision reads fresh_self when given, else the pod's published row; a pod that is not ranked and has no
 *               fresh_self is answered MMP_TARGET_INVALID (as by mmp_shutdown_run).
 *   draws       entries[r]'s decision draws with id r (MMP_DF_OWN_ID), so an answer equals mmp_place_batch's on the same 32-byte
 *               record with the same seed and does not depend on the other entries.
 * Epoch batching: every reload reads the one committed epoch and one fresh_self (the reference's tasks run concurrently on
 * taskPool against a clusterState that has not seen their loads yet); the registry is read as of the last commit, and the
 * pod's KV writes catch the difference; "live" is "ranked by the epoch".  Not modelled (stays in the pod): ce.doRemove, the
 * unload-buffer accounting, the conditional write and its retry, and issuing the load (INTEGRATION.md §11).
 * out[r] is entries[r]'s action, in entry order; without a decision target is MMP_TARGET_INVALID and n_candidates 0.  Returns
 * n.  Errors (nothing written): MMP_E_ARG for self outside [0, max_instances), an entry's model out of range or two entries
 * of one model, n < 0 or n > 2^24, p or report NULL, entries or out NULL with n > 0, or a bad fresh_self; MMP_E_EPOCH without
 * a commit; MMP_E_STATE when the committed registry holds no registration times, on an instance-sharded fleet or one that
 * connected a communicator.  Sets the "evict_run" timing. */
#define MMP_EV_ENTRY_FAILED 1u     /* ce.isFailed(): a cached load failure */
typedef struct {
  int32_t model; uint32_t flags;   /* model index; MMP_EV_ENTRY_* */
  int64_t last_used;               /* the listener's lastUsed */
  int64_t load_ts;                 /* ce.loadTimestamp */
  int64_t load_complete_ts;        /* ce.loadCompleteTimestamp */
} mmp_evict_entry;                 /* 32 B */
typedef struct {
  int64_t now;
  int64_t load_timeout_ms;         /* loadTimeoutMs: attemptReload needs the registration to be older than twice it */
  int64_t load_failure_expiry_ms;  /* LOAD_FAILURE_EXPIRY_MS (MM:219); checkLoadFailureCount counts failures younger than half */
} mmp_evict_params;                /* 24 B */
#define MMP_EV_UNREGISTER 1u       /* the pod's loaded registration (time load_ts) is removed, updateLastUnloadTime */
#define MMP_EV_DROP_FAILURE 2u     /* the pod's failed registration (time load_complete_ts) is removed */
#define MMP_EV_RELOAD 4u           /* attemptReload */
#define MMP_EV_CLUSTER_FULL 8u     /* a reload the rebalance gate stops: the model's type set is 95 % full or has one instance */
#define MMP_EV_LOADED_ELSEWHERE 16u /* a reload answered by a loaded copy on another ranked instance: no load */
#define MMP_EV_REFUSED 32u         /* a reload checkLoadFailureCount refused: no decision */
#define MMP_EV_PLACED 64u          /* a decision was made: target / n_candidates are its answer */
#define MMP_EV_UNDECIDED 128u      /* copy_count saturated at 255 over > 255 registrations: alone, nothing decided or counted */
typedef struct {
  int32_t model; uint32_t what;    /* model; the OR of MMP_EV_* */
  int32_t target, n_candidates;    /* as mmp_decision_out with MMP_EV_PLACED, else MMP_TARGET_INVALID and 0 */
  int64_t last_used;               /* the record's lastUsed after the edit (its own without a write) */
  int64_t last_unload_time;        /* the record's lastUnloadTime after the edit (its own without MMP_EV_UNREGISTER) */
} mmp_evict_action;                /* 32 B */
typedef struct {
  int32_t n_unregister, n_drop_failure, n_reload, n_cluster_full;  /* entries with each MMP_EV_* bit */
  int32_t n_loaded_elsewhere, n_refused, n_placed;
  int32_t n_none;                  /* of the MMP_EV_PLACED entries, those answered MMP_TARGET_NONE */
} mmp_evict_report;                /* 32 B */
int32_t mmp_evict_run(mmp_fleet *, int32_t self, const mmp_evict_entry *entries, int32_t n, const mmp_evict_params *p,
                      const mmp_instance_row *fresh_self, uint64_t seed, mmp_evict_action *out, mmp_evict_report *report);

/* tuning / measurement knobs, same meaning as the MMP_* environment variables read at mmp_fleet_create:
 *   "one_mode"        how a batch of <= 32 decisions is launched: 0 the batch kernel ("direct" below), 1 the latency kernel
 *                     k_place_small as a stream launch, 2 k_place_small as a replayed CUDA graph, 3 (default) a request to the
 *                     resident server kernel k_place_server (no launch per call: the host posts the request into mapped memory
 *                     and spins on the answer; up to MMP_SERVER_SLOTS concurrent callers each have a slot of their own,
 *                     a caller that finds every slot taken takes the graph path -- see mmp_server_stats)
 *   "server_life_us"  longest residence of one k_place_server launch (default 2000): bounds how long a device-wide wait
 *                     (cudaFree inside a commit) can be held up; "server_idle_us" (default 300): it leaves earlier when idle
 *   "direct"          1 (default): batches are resolved by k_place_direct (rows read straight from memory); 0: by the streaming
 *                     kernel k_place_lanes (whole rows through TMA landing stages) -- MMP_KERNEL=direct | lanes | tile
 *   "sort_slots"      k_place_direct resolves a batch of >= 8192 decisions in type-slot order: 0 never, 1 always, 2 (default) when
 *                     the committed snapshot's candidate sets are sparse (long walks: lanes of a warp then finish together)
 *   "lane_budget"     walk steps a lane may spend before its decision is redone by the whole warp
 *   "commit_host_only" 1: every commit takes the structural (host) path */
int32_t mmp_tune(mmp_fleet *, const char *key, int64_t value);
/* CUDA-event duration (ms) of the device part of the last mmp_stats ("stats"), mmp_reaper_select ("reaper": the candidate
 * sweep through the selection, k_rp_flag to k_rp_pick, without the stats and plan), mmp_lru_apply ("lru_apply": the event kernel), mmp_lru_read ("lru_read": count, scan and emit kernels) on
 * this fleet; "commit": host-clock ms of the last commit; "prune": mmp_registry_prune / mmp_registry_prune_ids;
 * "reaper_run": mmp_reaper_run from its prune sweep to its last placement kernel; "janitor_run": mmp_janitor_run from its stats
 * kernel to its budget walk; "janitor_task": mmp_janitor_task from its cache-pass plan kernel to its budget walk; "rate_run": mmp_rate_run from its stats kernel to its last placement round; "shutdown_run":
 * mmp_shutdown_run from its index kernel to its pack kernel; "evict_run": mmp_evict_run from its stats kernel to its pack kernel;
 * "dealt_kernel" / "dealt_wait": k_place_dealt and the arrival wait of the last peer-access step of an instance-sharded fleet */
int32_t mmp_last_timing(mmp_fleet *, const char *key, double *ms);
/* which path the last mmp_fleet_commit took: 1 = structural (host: string ranks, type-constraint sets, sort), 2 = device
 * (numeric instance updates / model-record deltas only: scattered into the device-resident tables, re-ranked and rebuilt
 * there); and its duration on the host clock */
int32_t mmp_commit_info(mmp_fleet *, int32_t *path, double *ms);
/* the resident server (one_mode 3) since mmp_fleet_create: out4[0] requests it answered, out4[1] calls that found all
 * MMP_SERVER_SLOTS slots taken and took the graph path, out4[2] launches of k_place_server, out4[3] the most slots busy at
 * once.  Its answers equal the graph path's by design: these counts are how a caller sees which path answered */
int32_t mmp_server_stats(mmp_fleet *, int64_t *out4);

#ifdef __cplusplus
}
#endif
#endif
