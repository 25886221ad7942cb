/* jni/mmplace_jni.c — the JNI shim between ModelMesh (Java) and libmmplace's C ABI (include/mmplace.h).
 *
 * One native per ABI entry point, class com.ibm.watson.modelmesh.gpu.MmPlace (java/com/ibm/watson/modelmesh/gpu/MmPlace.java).
 * Conventions: the fleet handle travels as a jlong; every struct array (instance rows, model rows, decisions, results, LRU
 * events, churn events, reports) is a DIRECT ByteBuffer in the C layout of mmplace.h (little-endian, natural alignment) --
 * for the batch paths a pinned one from allocPinned(), so the library's copies are true DMA and the JVM copies nothing;
 * small index lists are int[] accessed as critical arrays; strings are UTF-8 (GetStringUTFChars: modified UTF-8 equals
 * UTF-8 for the BMP ids, labels and JSON ModelMesh uses).  Nothing is retained across calls.
 *
 * Build: jni/Makefile (real JDK headers when JAVA_HOME is set, the compile-check stub jni/stub/jni.h otherwise).
 * Reference call sites these natives are used from: MM:1107-1110 (load balancer factory), MM:1455 (instance table listener),
 * MM:2807-2854 (registry listener), TCM:607 (type mappings), UT:78, MM:6616/6711 (reaper), see INTEGRATION.md. */
#include <jni.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "mmplace.h"

#define H(h) ((mmp_fleet *)(intptr_t)(h))
#define FN(name) JNIEXPORT JNICALL Java_com_ibm_watson_modelmesh_gpu_MmPlace_##name
#define BUF(b) ((b) ? (*env)->GetDirectBufferAddress(env, (b)) : NULL)

static const char *utf(JNIEnv *env, jstring s) { return s ? (*env)->GetStringUTFChars(env, s, NULL) : NULL; }
static void unutf(JNIEnv *env, jstring s, const char *c) { if (c) (*env)->ReleaseStringUTFChars(env, s, c); }

/* ---- lifecycle ---- */
jint FN(abiVersion)(JNIEnv *env, jclass c) { (void)env; (void)c; return mmp_abi_version(); }
jlong FN(create)(JNIEnv *env, jclass c, jlong minSpaceUnits, jlong minChurnAgeMs, jint defaultModelSizeUnits, jint maxInstances,
                 jint maxModels, jint device, jint shardRank, jint shardCount) {
  mmp_config cfg;
  mmp_fleet *f = NULL;
  (void)c;
  memset(&cfg, 0, sizeof(cfg));
  cfg.min_space_units = minSpaceUnits; cfg.min_churn_age_ms = minChurnAgeMs; cfg.default_model_size_units = defaultModelSizeUnits;
  cfg.max_instances = maxInstances; cfg.max_models = maxModels; cfg.device = device; cfg.shard_rank = shardRank; cfg.shard_count = shardCount;
  if (mmp_fleet_create(&cfg, &f) < 0) {
    (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/IllegalStateException"), mmp_last_error(NULL));
    return 0;
  }
  return (jlong)(intptr_t)f;
}
void FN(destroy)(JNIEnv *env, jclass c, jlong h) { (void)env; (void)c; mmp_fleet_destroy(H(h)); }
jstring FN(lastError)(JNIEnv *env, jclass c, jlong h) { (void)c; return (*env)->NewStringUTF(env, mmp_last_error(H(h))); }

/* ---- plug point 2: ingest ---- */
jint FN(instanceUpsert)(JNIEnv *env, jclass c, jlong h, jint idx, jobject row, jstring id, jstring loc, jstring zone, jobjectArray labels) {
  const char *cid = utf(env, id), *cloc = utf(env, loc), *czone = utf(env, zone);
  jsize n = labels ? (*env)->GetArrayLength(env, labels) : 0, i;
  const char *ls[64] = {0};
  jstring js[64];
  jint rc;
  (void)c;
  if (n > 64) n = 64;
  for (i = 0; i < n; i++) { js[i] = (jstring)(*env)->GetObjectArrayElement(env, labels, i); ls[i] = utf(env, js[i]); }
  rc = mmp_instance_upsert(H(h), idx, (const mmp_instance_row *)BUF(row), cid, cloc, czone, ls, n);
  for (i = 0; i < n; i++) { unutf(env, js[i], ls[i]); (*env)->DeleteLocalRef(env, js[i]); }
  unutf(env, zone, czone); unutf(env, loc, cloc); unutf(env, id, cid);
  return rc;
}
jint FN(instanceUpdate)(JNIEnv *env, jclass c, jlong h, jint idx, jobject row) { (void)c; return mmp_instance_update(H(h), idx, (const mmp_instance_row *)BUF(row)); }
jint FN(instanceRemove)(JNIEnv *env, jclass c, jlong h, jint idx) { (void)env; (void)c; return mmp_instance_remove(H(h), idx); }
jint FN(instanceUpsertJson)(JNIEnv *env, jclass c, jlong h, jint idx, jstring id, jstring json, jboolean active) {
  const char *cid = utf(env, id), *cj = utf(env, json);
  jint rc = mmp_instance_upsert_json(H(h), idx, cid, cj, active ? 1 : 0);
  (void)c;
  unutf(env, json, cj); unutf(env, id, cid);
  return rc;
}
jint FN(modelUpsertJson)(JNIEnv *env, jclass c, jlong h, jint model, jstring json, jint sizeUnits) {
  const char *cj = utf(env, json);
  jint rc = mmp_model_upsert_json(H(h), model, cj, sizeUnits);
  (void)c;
  unutf(env, json, cj);
  return rc;
}
jint FN(typesSetJson)(JNIEnv *env, jclass c, jlong h, jstring json) {
  const char *cj = utf(env, json);
  jint rc = mmp_types_set_json(H(h), cj);
  (void)c;
  unutf(env, json, cj);
  return rc;
}
jint FN(typeId)(JNIEnv *env, jclass c, jlong h, jstring name) {
  const char *cn = utf(env, name);
  jint rc = mmp_type_id(H(h), cn);
  (void)c;
  unutf(env, name, cn);
  return rc;
}
jint FN(replicasetsSet)(JNIEnv *env, jclass c, jlong h, jobjectArray prefixes) {
  jsize n = prefixes ? (*env)->GetArrayLength(env, prefixes) : 0, i;
  const char *ps[256] = {0};
  jstring js[256];
  jint rc;
  (void)c;
  if (n > 256) n = 256;
  for (i = 0; i < n; i++) { js[i] = (jstring)(*env)->GetObjectArrayElement(env, prefixes, i); ps[i] = utf(env, js[i]); }
  rc = mmp_replicasets_set(H(h), ps, n);
  for (i = 0; i < n; i++) { unutf(env, js[i], ps[i]); (*env)->DeleteLocalRef(env, js[i]); }
  return rc;
}
jint FN(modelUpsert)(JNIEnv *env, jclass c, jlong h, jint model, jobject row, jintArray ids) {
  jsize n = ids ? (*env)->GetArrayLength(env, ids) : 0;
  jint *p = n ? (jint *)(*env)->GetPrimitiveArrayCritical(env, ids, NULL) : NULL;
  jint rc = mmp_model_upsert(H(h), model, (const mmp_model_row *)BUF(row), (const int32_t *)p, n);
  (void)c;
  if (p) (*env)->ReleasePrimitiveArrayCritical(env, ids, p, JNI_ABORT);
  return rc;
}
/* rows: n x mmp_model_row, edgeOff: (n + 1) x int64, edgeInst: int32[] -- all direct buffers */
jint FN(modelsBulk)(JNIEnv *env, jclass c, jlong h, jint first, jint n, jobject rows, jobject edgeOff, jobject edgeInst) {
  (void)c;
  return mmp_models_bulk(H(h), first, n, (const mmp_model_row *)BUF(rows), (const int64_t *)BUF(edgeOff), (const int32_t *)BUF(edgeInst));
}
jint FN(commit)(JNIEnv *env, jclass c, jlong h) { (void)env; (void)c; return mmp_fleet_commit(H(h)); }
/* ts: int64[n] direct buffer of the edges' load-start / failure times, same order as modelUpsert's ids */
jint FN(modelTimes)(JNIEnv *env, jclass c, jlong h, jint model, jobject ts, jint n, jlong lastUnloadTime) {
  (void)c;
  return mmp_model_times(H(h), model, (const int64_t *)BUF(ts), n, lastUnloadTime);
}
/* in: n x mmp_scale_in (48 B), params: one mmp_scale_params (72 B), out: n x mmp_scale_out (40 B) -- direct buffers */
jint FN(scaleEval)(JNIEnv *env, jclass c, jlong h, jobject in, jint n, jobject params, jobject out) {
  (void)c;
  return mmp_scale_eval(H(h), (const mmp_scale_in *)BUF(in), n, (const mmp_scale_params *)BUF(params), (mmp_scale_out *)BUF(out));
}
/* missingSince: int64[max_instances] (in/out), outModels: int32[cap], outMasks: byte[cap] -- direct buffers */
jint FN(registryPrune)(JNIEnv *env, jclass c, jlong h, jint self, jlong nowMs, jlong assumeGoneMs, jobject missingSince, jobject outModels,
                       jobject outMasks, jint cap) {
  (void)c;
  return mmp_registry_prune(H(h), self, nowMs, assumeGoneMs, (int64_t *)BUF(missingSince), (int32_t *)BUF(outModels), (uint8_t *)BUF(outMasks), cap);
}
/* missingSince: int64[max_instances] (in/out), outModels / outInstances: int32[cap] -- direct buffers */
jint FN(registryPruneIds)(JNIEnv *env, jclass c, jlong h, jint self, jlong nowMs, jlong assumeGoneMs, jobject missingSince, jobject outModels,
                          jobject outInstances, jint cap) {
  (void)c;
  return mmp_registry_prune_ids(H(h), self, nowMs, assumeGoneMs, (int64_t *)BUF(missingSince), (int32_t *)BUF(outModels),
                                (int32_t *)BUF(outInstances), cap);
}
/* one run of the leader's reaper task.  missingSince: int64[max_instances] (in/out), prunedModels / prunedInstances:
 * int32[prunedCap], repairedModels: int32[repairedCap], loads: loadsCap x mmp_reaper_load (24 B), report: one
 * mmp_reaper_report (16 B) -- direct buffers */
jint FN(reaperRun)(JNIEnv *env, jclass c, jlong h, jint leader, jlong nowMs, jlong assumeGoneMs, jobject missingSince, jlong seed,
                   jobject prunedModels, jobject prunedInstances, jint prunedCap, jobject repairedModels, jint repairedCap, jobject loads,
                   jint loadsCap, jobject report) {
  (void)c;
  return mmp_reaper_run(H(h), leader, nowMs, assumeGoneMs, (int64_t *)BUF(missingSince), (uint64_t)seed, (int32_t *)BUF(prunedModels),
                        (int32_t *)BUF(prunedInstances), prunedCap, (int32_t *)BUF(repairedModels), repairedCap,
                        (mmp_reaper_load *)BUF(loads), loadsCap, (mmp_reaper_report *)BUF(report));
}
/* the registry loop of one pod's janitor task.  entries: n x mmp_janitor_entry (48 B), params: one mmp_janitor_params (96 B),
 * edits: cap x mmp_janitor_edit (24 B), report: one mmp_janitor_report (24 B) -- direct buffers */
jint FN(janitorRun)(JNIEnv *env, jclass c, jlong h, jint self, jobject entries, jint n, jobject params, jobject edits, jint cap,
                    jobject report) {
  (void)c;
  return mmp_janitor_run(H(h), self, (const mmp_janitor_entry *)BUF(entries), n, (const mmp_janitor_params *)BUF(params),
                         (mmp_janitor_edit *)BUF(edits), cap, (mmp_janitor_report *)BUF(report));
}
/* one run of one pod's whole janitor task.  entries: n x mmp_janitor_task_entry (56 B) most recently used first, params: one
 * mmp_janitor_task_params (120 B), out: n x mmp_janitor_cache_action (24 B), edits: cap x mmp_janitor_edit (24 B), report: one
 * mmp_janitor_task_report (80 B) -- direct buffers */
jint FN(janitorTask)(JNIEnv *env, jclass c, jlong h, jint self, jobject entries, jint n, jobject params, jobject out, jobject edits,
                     jint cap, jobject report) {
  (void)c;
  return mmp_janitor_task(H(h), self, (const mmp_janitor_task_entry *)BUF(entries), n, (const mmp_janitor_task_params *)BUF(params),
                          (mmp_janitor_cache_action *)BUF(out), (mmp_janitor_edit *)BUF(edits), cap, (mmp_janitor_task_report *)BUF(report));
}
/* one run of one pod's rate-tracking task.  entries: n x mmp_scale_in (48 B), params: one mmp_rate_params (80 B), freshSelf:
 * one mmp_instance_row (64 B) or null, out: n x mmp_scale_out (40 B), loads: loadsCap x mmp_rate_load (40 B), report: one
 * mmp_rate_report (32 B) -- direct buffers */
jint FN(rateRun)(JNIEnv *env, jclass c, jlong h, jint self, jobject entries, jint n, jobject params, jobject freshSelf, jlong seed,
                 jobject out, jobject loads, jint loadsCap, jobject report) {
  (void)c;
  return mmp_rate_run(H(h), self, (const mmp_scale_in *)BUF(entries), n, (const mmp_rate_params *)BUF(params),
                      (const mmp_instance_row *)BUF(freshSelf), (uint64_t)seed, (mmp_scale_out *)BUF(out), (mmp_rate_load *)BUF(loads),
                      loadsCap, (mmp_rate_report *)BUF(report));
}
/* one pod's pre-shutdown migration.  entries: n x mmp_shutdown_entry (24 B), params: one mmp_shutdown_params (24 B), freshSelf:
 * one mmp_instance_row (64 B) or null, out: n x mmp_shutdown_action (24 B), report: one mmp_shutdown_report (32 B) -- direct
 * buffers */
jint FN(shutdownRun)(JNIEnv *env, jclass c, jlong h, jint self, jobject entries, jint n, jobject params, jobject freshSelf, jlong seed,
                     jobject out, jobject report) {
  (void)c;
  return mmp_shutdown_run(H(h), self, (const mmp_shutdown_entry *)BUF(entries), n, (const mmp_shutdown_params *)BUF(params),
                          (const mmp_instance_row *)BUF(freshSelf), (uint64_t)seed, (mmp_shutdown_action *)BUF(out),
                          (mmp_shutdown_report *)BUF(report));
}
/* one pod's eviction listener over a burst of evictions.  entries: n x mmp_evict_entry (32 B), params: one mmp_evict_params
 * (24 B), freshSelf: one mmp_instance_row (64 B) or null, out: n x mmp_evict_action (32 B), report: one mmp_evict_report
 * (32 B) -- direct buffers */
jint FN(evictRun)(JNIEnv *env, jclass c, jlong h, jint self, jobject entries, jint n, jobject params, jobject freshSelf, jlong seed,
                  jobject out, jobject report) {
  (void)c;
  return mmp_evict_run(H(h), self, (const mmp_evict_entry *)BUF(entries), n, (const mmp_evict_params *)BUF(params),
                       (const mmp_instance_row *)BUF(freshSelf), (uint64_t)seed, (mmp_evict_action *)BUF(out),
                       (mmp_evict_report *)BUF(report));
}
jint FN(tune)(JNIEnv *env, jclass c, jlong h, jstring key, jlong value) {
  const char *ck = utf(env, key);
  jint rc = mmp_tune(H(h), ck, value);
  (void)c;
  unutf(env, key, ck);
  return rc;
}
jdouble FN(lastTiming)(JNIEnv *env, jclass c, jlong h, jstring key) {
  const char *ck = utf(env, key);
  double ms = -1.0;
  (void)c;
  if (mmp_last_timing(H(h), ck, &ms) < 0) ms = -1.0;
  unutf(env, key, ck);
  return ms;
}
/* out[0] = path (1 structural, 2 device), returns the duration in ms */
jdouble FN(commitInfo)(JNIEnv *env, jclass c, jlong h, jintArray pathOut) {
  int32_t path = 0;
  double ms = 0;
  (void)c;
  mmp_commit_info(H(h), &path, &ms);
  if (pathOut) { jint p = path; (*env)->SetIntArrayRegion(env, pathOut, 0, 1, &p); }
  return ms;
}

/* out[0..3] = the resident server's requests answered, graph-path fallbacks, launches, most slots busy at once */
jint FN(serverStats)(JNIEnv *env, jclass c, jlong h, jlongArray out) {
  int64_t v[4] = {0, 0, 0, 0};
  jint rc = mmp_server_stats(H(h), v);
  (void)c;
  if (rc >= 0 && out) {
    jlong j[4] = {v[0], v[1], v[2], v[3]};
    (*env)->SetLongArrayRegion(env, out, 0, 4, j);
  }
  return rc;
}

/* ---- plug point 1: placement ---- */
jint FN(placeBatch)(JNIEnv *env, jclass c, jlong h, jobject in, jint n, jobject fresh, jint nFresh, jobject extra, jint nExtra, jobject out,
                    jlong nowMs, jlong seed) {
  (void)c;
  return mmp_place_batch(H(h), (const mmp_decision_in *)BUF(in), n, (const mmp_instance_row *)BUF(fresh), nFresh, (const int32_t *)BUF(extra),
                         nExtra, (mmp_decision_out *)BUF(out), nowMs, (uint64_t)seed);
}
jint FN(placeBatchTrace)(JNIEnv *env, jclass c, jlong h, jobject in, jint n, jobject fresh, jint nFresh, jobject extra, jint nExtra,
                         jobject out, jobject trace, jobject candMask, jlong nowMs, jlong seed) {
  (void)c;
  return mmp_place_batch_trace(H(h), (const mmp_decision_in *)BUF(in), n, (const mmp_instance_row *)BUF(fresh), nFresh,
                               (const int32_t *)BUF(extra), nExtra, (mmp_decision_out *)BUF(out), (mmp_decision_trace *)BUF(trace),
                               (uint32_t *)BUF(candMask), nowMs, (uint64_t)seed);
}
/* a call-wide exclude set (int[] of instance indices, or null) on top of every decision's own exclusions; trace / candMask may be null */
jint FN(placeBatchExcluding)(JNIEnv *env, jclass c, jlong h, jobject in, jint n, jobject fresh, jint nFresh, jobject extra, jint nExtra,
                             jintArray exclude, jobject out, jobject trace, jobject candMask, jlong nowMs, jlong seed) {
  jsize nx = exclude ? (*env)->GetArrayLength(env, exclude) : 0;
  jint *px = nx ? (jint *)(*env)->GetPrimitiveArrayCritical(env, exclude, NULL) : NULL;
  jint rc = mmp_place_batch_excluding(H(h), (const mmp_decision_in *)BUF(in), n, (const mmp_instance_row *)BUF(fresh), nFresh,
                                      (const int32_t *)BUF(extra), nExtra, (const int32_t *)px, nx, (mmp_decision_out *)BUF(out),
                                      (mmp_decision_trace *)BUF(trace), (uint32_t *)BUF(candMask), nowMs, (uint64_t)seed);
  (void)c;
  if (px) (*env)->ReleasePrimitiveArrayCritical(env, exclude, px, JNI_ABORT);
  return rc;
}
jint FN(placeSweep)(JNIEnv *env, jclass c, jlong h, jint first, jint n, jobject self, jint selfStride, jobject favour, jobject out,
                    jlong nowMs, jlong seed) {
  (void)c;
  return mmp_place_sweep(H(h), first, n, (const int32_t *)BUF(self), selfStride, (const uint32_t *)BUF(favour), (mmp_decision_out *)BUF(out),
                         nowMs, (uint64_t)seed);
}
/* one decision on the caller's thread: in = 32 bytes, fresh = one row or null, extra = int[] or null, out = 8 bytes */
jint FN(placeOne)(JNIEnv *env, jclass c, jlong h, jobject in, jobject fresh, jintArray extra, jobject out, jlong nowMs, jlong seed) {
  jsize ne = extra ? (*env)->GetArrayLength(env, extra) : 0;
  jint *pe = ne ? (jint *)(*env)->GetPrimitiveArrayCritical(env, extra, NULL) : NULL;
  jint rc = mmp_place_one(H(h), (const mmp_decision_in *)BUF(in), (const mmp_instance_row *)BUF(fresh), (const int32_t *)pe,
                          (mmp_decision_out *)BUF(out), nowMs, (uint64_t)seed);
  (void)c;
  if (pe) (*env)->ReleasePrimitiveArrayCritical(env, extra, pe, JNI_ABORT);
  return rc;
}
/* micro-batcher: many request threads, one mmp_place_batch per drain (idOut[0] = the decision's own id) */
jlong FN(batcherCreate)(JNIEnv *env, jclass c, jlong h, jint maxBatch, jint maxWaitUs, jlong seed) {
  mmp_batcher *b = NULL;
  (void)env; (void)c;
  return mmp_batcher_create(H(h), maxBatch, maxWaitUs, (uint64_t)seed, &b) < 0 ? 0 : (jlong)(intptr_t)b;
}
void FN(batcherDestroy)(JNIEnv *env, jclass c, jlong b) { (void)env; (void)c; mmp_batcher_destroy((mmp_batcher *)(intptr_t)b); }
jint FN(placeSubmit)(JNIEnv *env, jclass c, jlong b, jobject in, jobject fresh, jintArray extra, jlong nowMs, jobject out, jintArray idOut) {
  jsize ne = extra ? (*env)->GetArrayLength(env, extra) : 0;
  jint tmp[MMP_MAX_EXTRA], id;
  uint32_t did = 0;
  jint rc;
  (void)c;
  if (ne > MMP_MAX_EXTRA) ne = MMP_MAX_EXTRA;
  if (ne) { jint *pe = (jint *)(*env)->GetPrimitiveArrayCritical(env, extra, NULL); memcpy(tmp, pe, (size_t)ne * sizeof(jint)); (*env)->ReleasePrimitiveArrayCritical(env, extra, pe, JNI_ABORT); }
  rc = mmp_place_submit((mmp_batcher *)(intptr_t)b, (const mmp_decision_in *)BUF(in), (const mmp_instance_row *)BUF(fresh), ne ? (const int32_t *)tmp : NULL,
                        nowMs, (mmp_decision_out *)BUF(out), &did);
  id = (jint)did;
  if (idOut) (*env)->SetIntArrayRegion(env, idOut, 0, 1, &id);
  return rc;
}
jint FN(batcherStats)(JNIEnv *env, jclass c, jlong b, jlongArray out) {
  int64_t v[2] = {0, 0};
  jlong w[2];
  jint rc = mmp_batcher_stats((mmp_batcher *)(intptr_t)b, &v[0], &v[1]);
  (void)c;
  w[0] = v[0]; w[1] = v[1];
  if (out) (*env)->SetLongArrayRegion(env, out, 0, 2, w);
  return rc;
}
jdouble FN(placeBatchDevice)(JNIEnv *env, jclass c, jlong h, jlong dIn, jint n, jlong dOut, jlong nowMs, jlong seed) {
  float ms = -1.0f;
  (void)env; (void)c;
  if (mmp_place_batch_device(H(h), (const void *)(intptr_t)dIn, n, (void *)(intptr_t)dOut, nowMs, (uint64_t)seed, &ms) < 0) return -1.0;
  return ms;
}
jlong FN(deviceAlloc)(JNIEnv *env, jclass c, jlong h, jlong bytes) { void *p = NULL; (void)env; (void)c; return mmp_device_alloc(H(h), bytes, &p) < 0 ? 0 : (jlong)(intptr_t)p; }
jint FN(deviceFree)(JNIEnv *env, jclass c, jlong h, jlong p) { (void)env; (void)c; return mmp_device_free(H(h), (void *)(intptr_t)p); }
jint FN(deviceUpload)(JNIEnv *env, jclass c, jlong h, jlong dst, jobject src, jlong bytes) { (void)c; return mmp_device_upload(H(h), (void *)(intptr_t)dst, BUF(src), bytes); }
jint FN(deviceDownload)(JNIEnv *env, jclass c, jlong h, jobject dst, jlong src, jlong bytes) { (void)c; return mmp_device_download(H(h), BUF(dst), (const void *)(intptr_t)src, bytes); }
/* pinned host memory as a direct ByteBuffer (free with freePinned) */
jobject FN(allocPinned)(JNIEnv *env, jclass c, jlong h, jlong bytes) {
  void *p = NULL;
  (void)c;
  if (mmp_host_alloc(H(h), bytes, &p) < 0) return NULL;
  return (*env)->NewDirectByteBuffer(env, p, bytes);
}
jint FN(freePinned)(JNIEnv *env, jclass c, jlong h, jobject buf) { (void)c; return mmp_host_free(H(h), BUF(buf)); }
jint FN(flushL2)(JNIEnv *env, jclass c, jlong h) { (void)env; (void)c; return mmp_flush_l2(H(h)); }

/* ---- instance-sharded fleets ---- */
jint FN(shardUniqueId)(JNIEnv *env, jclass c, jbyteArray out) {
  unsigned char id[128];
  jint rc = mmp_shard_unique_id(id);
  (void)c;
  if (rc == 0) (*env)->SetByteArrayRegion(env, out, 0, 128, (const jbyte *)id);
  return rc;
}
jint FN(shardConnect)(JNIEnv *env, jclass c, jlong h, jbyteArray id) {
  jbyte buf[128];
  (void)c;
  (*env)->GetByteArrayRegion(env, id, 0, 128, buf);
  return mmp_shard_connect(H(h), buf);
}
/* out = {word_lo, word_hi}; returns the stored row stride in words */
jint FN(shardWords)(JNIEnv *env, jclass c, jlong h, jintArray out) {
  int32_t lo = 0, hi = 0;
  jint v[2], rc = mmp_shard_words(H(h), &lo, &hi);
  (void)c;
  v[0] = lo; v[1] = hi;
  if (out) (*env)->SetIntArrayRegion(env, out, 0, 2, v);
  return rc;
}
jlong FN(shardOpenDecisions)(JNIEnv *env, jclass c, jlong h) { (void)env; (void)c; return mmp_shard_open_decisions(H(h)); }
/* peer access between the shards: blob = byte[MMP_SHARD_IPC_BYTES]; blobs = byte[shardCount * MMP_SHARD_IPC_BYTES] by rank */
jint FN(shardIpcExport)(JNIEnv *env, jclass c, jlong h, jint maxBatch, jbyteArray blob) {
  unsigned char buf[MMP_SHARD_IPC_BYTES];
  jint rc = mmp_shard_ipc_export(H(h), maxBatch, buf);
  (void)c;
  if (rc == 0) (*env)->SetByteArrayRegion(env, blob, 0, MMP_SHARD_IPC_BYTES, (const jbyte *)buf);
  return rc;
}
jint FN(shardIpcImport)(JNIEnv *env, jclass c, jlong h, jbyteArray blobs) {
  const jsize len = (*env)->GetArrayLength(env, blobs);
  jbyte *p = (jbyte *)malloc(len > 0 ? (size_t)len : 1);  /* (opening IPC handles may block: no critical section here) */
  jint rc;
  (void)c;
  if (!p) return MMP_E_ARG;
  (*env)->GetByteArrayRegion(env, blobs, 0, len, p);
  rc = mmp_shard_ipc_import(H(h), p);
  free(p);
  return rc;
}
jint FN(shardPeerStats)(JNIEnv *env, jclass c, jlong h, jlongArray out4) {
  int64_t v[4] = {0, 0, 0, 0};
  jlong w[4];
  jint rc = mmp_shard_peer_stats(H(h), v);
  int i;
  (void)c;
  for (i = 0; i < 4; i++) w[i] = (jlong)v[i];
  if (rc == 0) (*env)->SetLongArrayRegion(env, out4, 0, 4, w);
  return rc;
}
jint FN(setIdBase)(JNIEnv *env, jclass c, jlong h, jlong base) { (void)env; (void)c; return mmp_fleet_set_id_base(H(h), (uint64_t)base); }

/* ---- introspection ---- */
jint FN(rowWords)(JNIEnv *env, jclass c, jlong h) { (void)env; (void)c; return mmp_row_words(H(h)); }
jint FN(liveInstances)(JNIEnv *env, jclass c, jlong h) { (void)env; (void)c; return mmp_live_instances(H(h)); }
jint FN(clusterOrder)(JNIEnv *env, jclass c, jlong h, jobject outIdx, jint cap) { (void)c; return mmp_cluster_order(H(h), (int32_t *)BUF(outIdx), cap); }
/* allowed / preferred: nIdx bytes each (direct); nulls = {allowedNull, preferredNull} */
jint FN(typeSets)(JNIEnv *env, jclass c, jlong h, jint typeId, jint nIdx, jobject allowed, jobject preferred, jintArray nulls) {
  int32_t an = 0, pn = 0;
  jint v[2], rc = mmp_type_sets(H(h), typeId, nIdx, (uint8_t *)BUF(allowed), &an, (uint8_t *)BUF(preferred), &pn);
  (void)c;
  v[0] = an; v[1] = pn;
  if (nulls) (*env)->SetIntArrayRegion(env, nulls, 0, 2, v);
  return rc;
}
jlong FN(kernelLaunches)(JNIEnv *env, jclass c, jlong h) { (void)env; (void)c; return mmp_kernel_launches(H(h)); }
jint FN(instancePartition)(JNIEnv *env, jclass c, jlong h, jint idx) { (void)env; (void)c; return mmp_instance_partition(H(h), idx); }

/* ---- plug point 4: batch scans ---- */
jint FN(stats)(JNIEnv *env, jclass c, jlong h, jobject out, jobject partIds, jint cap) {
  (void)c;
  return mmp_stats(H(h), (mmp_cluster_stats *)BUF(out), (int32_t *)BUF(partIds), cap);
}
jint FN(reaperSelect)(JNIEnv *env, jclass c, jlong h, jint partition, jlong nowMs, jobject taken, jobject outModels, jint cap) {
  (void)c;
  return mmp_reaper_select(H(h), partition, nowMs, (uint8_t *)BUF(taken), (int32_t *)BUF(outModels), cap);
}

/* ---- plug point 3: LRU ---- */
jint FN(lruInit)(JNIEnv *env, jclass c, jlong h, jint nInstances, jobject capacity, jint slotsPerInstance) {
  (void)c;
  return mmp_lru_init(H(h), nInstances, (const int64_t *)BUF(capacity), slotsPerInstance);
}
jint FN(lruApply)(JNIEnv *env, jclass c, jlong h, jobject events, jint n, jlong nowMs, jobject out, jint cap) {
  (void)c;
  return mmp_lru_apply(H(h), (const mmp_lru_event *)BUF(events), n, nowMs, (mmp_eviction *)BUF(out), cap);
}
jint FN(lruApplyStatus)(JNIEnv *env, jclass c, jlong h, jobject events, jint n, jlong nowMs, jobject out, jint cap, jobject status) {
  (void)c;
  return mmp_lru_apply_status(H(h), (const mmp_lru_event *)BUF(events), n, nowMs, (mmp_eviction *)BUF(out), cap, (int32_t *)BUF(status));
}
jint FN(lruState)(JNIEnv *env, jclass c, jlong h, jint nInstances, jobject oldest, jobject weighted, jobject count) {
  (void)c;
  return mmp_lru_state(H(h), nInstances, (int64_t *)BUF(oldest), (int64_t *)BUF(weighted), (int32_t *)BUF(count));
}
/* instances: int32[n] direct buffer or null (caches 0 .. n-1); offsets: int64[n + 1]; out: cap mmp_lru_entry records (24 B) */
jint FN(lruRead)(JNIEnv *env, jclass c, jlong h, jobject instances, jint n, jlong usedSince, jobject offsets, jobject out, jlong cap) {
  (void)c;
  return mmp_lru_read(H(h), (const int32_t *)BUF(instances), n, usedSince, (int64_t *)BUF(offsets), (mmp_lru_entry *)BUF(out), cap);
}
jint FN(lruLookup)(JNIEnv *env, jclass c, jlong h, jint n, jobject instance, jobject model, jobject lastUsed, jobject weight, jobject loadTs) {
  (void)c;
  return mmp_lru_lookup(H(h), n, (const int32_t *)BUF(instance), (const int32_t *)BUF(model), (int64_t *)BUF(lastUsed), (int32_t *)BUF(weight),
                        (int64_t *)BUF(loadTs));
}

/* ---- the closed loop ---- */
jint FN(churnInit)(JNIEnv *env, jclass c, jlong h, jlong loadTimeoutMs, jlong lastPublishedMs, jint slotsPerInstance) {
  mmp_churn_config cfg;
  (void)env; (void)c;
  memset(&cfg, 0, sizeof(cfg));
  cfg.load_timeout_ms = loadTimeoutMs; cfg.last_published_ms = lastPublishedMs; cfg.slots_per_instance = slotsPerInstance;
  return mmp_churn_init(H(h), &cfg);
}
jint FN(churnSeed)(JNIEnv *env, jclass c, jlong h, jint n, jobject instance, jobject model, jobject lastUsed, jobject weight, jobject loadTs,
                   jlong nowMs) {
  (void)c;
  return mmp_churn_seed(H(h), n, (const int32_t *)BUF(instance), (const int32_t *)BUF(model), (const int64_t *)BUF(lastUsed),
                        (const int32_t *)BUF(weight), (const int64_t *)BUF(loadTs), nowMs);
}
/* counts = {nDecisions, nEvictions}; report = one mmp_churn_report (direct, may be null) */
jint FN(churnStep)(JNIEnv *env, jclass c, jlong h, jobject events, jint n, jlong now0, jlong now1, jlong seed, jobject decOut, jint decCap,
                   jobject evictOut, jint evictCap, jobject rowsOut, jobject report, jintArray counts) {
  int32_t nd = 0, ne = 0;
  jint v[2], rc = mmp_churn_step(H(h), (const mmp_churn_event *)BUF(events), n, now0, now1, (uint64_t)seed, (mmp_churn_decision *)BUF(decOut),
                                decCap, &nd, (mmp_churn_eviction *)BUF(evictOut), evictCap, &ne, (mmp_instance_row *)BUF(rowsOut),
                                (mmp_churn_report *)BUF(report));
  (void)c;
  v[0] = nd; v[1] = ne;
  if (counts) (*env)->SetIntArrayRegion(env, counts, 0, 2, v);
  return rc;
}
jint FN(churnModel)(JNIEnv *env, jclass c, jlong h, jint model, jobject rowOut, jobject instances4) {
  (void)c;
  return mmp_churn_model(H(h), model, (mmp_model_row *)BUF(rowOut), (int32_t *)BUF(instances4));
}
/* ids: int32[cap] direct buffer; returns the model's registration count */
jint FN(churnModelIds)(JNIEnv *env, jclass c, jlong h, jint model, jobject rowOut, jobject ids, jint cap) {
  (void)c;
  return mmp_churn_model_ids(H(h), model, (mmp_model_row *)BUF(rowOut), (int32_t *)BUF(ids), cap);
}
