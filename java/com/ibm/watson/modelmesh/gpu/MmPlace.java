/*
 * MmPlace — the natives of jni/mmplace_jni.c, one per entry point of libmmplace's C ABI (include/mmplace.h).
 * Source only in this repository (no JDK in the build image); tests/test_jni_shim.py checks that every native declared
 * here has its JNI function in the shim and that the shim references every symbol the header declares.
 *
 * All struct arrays are DIRECT ByteBuffers in little-endian C layout (ByteOrder.LITTLE_ENDIAN); see the offsets in
 * GpuPlacement.  The handle is the mmp_fleet* as a long.
 */
package com.ibm.watson.modelmesh.gpu;

import java.nio.ByteBuffer;

final class MmPlace {
    static { System.loadLibrary("mmplace_jni"); }
    private MmPlace() {}

    static final int TARGET_NONE = -1, TARGET_SELF = -2, TARGET_INVALID = -3;     // mmp_decision_out.target
    static final int DF_FAVOUR_SELF = 1, DF_MODEL_LAST_USED = 2, DF_REQUEST_MODEL = 8;  // mmp_decision_in.flags
    static final int MAX_EXTRA = 16;                                               // MMP_MAX_EXTRA
    static final int INSTANCE_ROW_BYTES = 64, MODEL_ROW_BYTES = 24, DECISION_IN_BYTES = 32, DECISION_OUT_BYTES = 8;

    // lifecycle
    static native int abiVersion();
    static native long create(long minSpaceUnits, long minChurnAgeMs, int defaultModelSizeUnits, int maxInstances, int maxModels,
                              int device, int shardRank, int shardCount);
    static native void destroy(long h);
    static native String lastError(long h);
    // plug point 2: ingest (handleInstanceTableChange MM:1455, registry listener MM:2807-2854, TCM:607, UT:78)
    static native int instanceUpsert(long h, int idx, ByteBuffer row, String id, String loc, String zone, String[] labels);
    static native int instanceUpdate(long h, int idx, ByteBuffer row);
    static native int instanceRemove(long h, int idx);
    static native int instanceUpsertJson(long h, int idx, String id, String recordJson, boolean active);
    static native int modelUpsertJson(long h, int model, String recordJson, int sizeUnits);
    static native int typesSetJson(long h, String json);
    static native int typeId(long h, String typeName);
    static native int replicasetsSet(long h, String[] prefixes);
    static native int modelUpsert(long h, int model, ByteBuffer row, int[] loadedThenFailedInstanceIdx);
    static native int modelsBulk(long h, int first, int n, ByteBuffer rows, ByteBuffer edgeOff, ByteBuffer edgeInst);
    static native int commit(long h);
    static native double commitInfo(long h, int[] pathOut);
    // registry-side batch scans: rate-tracking / janitor arithmetic (MM:5640-5806, 6197-6335), reaper prune pass (MM:6524-6609)
    static native int modelTimes(long h, int model, ByteBuffer edgeTimes, int n, long lastUnloadTime);
    static native int scaleEval(long h, ByteBuffer in, int n, ByteBuffer params, ByteBuffer out);
    static native int registryPrune(long h, int self, long nowMs, long assumeGoneMs, ByteBuffer missingSince, ByteBuffer outModels,
                                    ByteBuffer outMasks, int cap);
    static native int registryPruneIds(long h, int self, long nowMs, long assumeGoneMs, ByteBuffer missingSince, ByteBuffer outModels,
                                       ByteBuffer outInstances, int cap);
    // the leader's reaper task in one call (MM:6436-6494): prune, repair, select over every partition, place (mmp_reaper_run)
    static native int reaperRun(long h, int leader, long nowMs, long assumeGoneMs, ByteBuffer missingSince, long seed,
                                ByteBuffer prunedModels, ByteBuffer prunedInstances, int prunedCap, ByteBuffer repairedModels,
                                int repairedCap, ByteBuffer loads, int loadsCap, ByteBuffer report);
    // the registry loop of one pod's janitor task (MM:6013-6145): stale registrations, expired failures, budgeted scale-down
    static native int janitorRun(long h, int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer edits, int cap,
                                 ByteBuffer report);
    // one run of one pod's whole janitor task (MM:5876-6145): the cache pass, then the registry loop on the records it left
    static native int janitorTask(long h, int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer out, ByteBuffer edits,
                                  int cap, ByteBuffer report);
    // one run of one pod's rate-tracking task (MM:5619-5858): second copies, scale-up chains under the heavy-instance set (mmp_rate_run)
    static native int rateRun(long h, int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer freshSelf, long seed,
                              ByteBuffer out, ByteBuffer loads, int loadsCap, ByteBuffer report);
    // one pod's pre-shutdown migration (MM:6990-7047): a new copy elsewhere for every registered cache entry (mmp_shutdown_run)
    static native int shutdownRun(long h, int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer freshSelf, long seed,
                                  ByteBuffer out, ByteBuffer report);
    // one pod's eviction listener (MM:2867-2933) over a burst of evictions: deregistration edits and reloads elsewhere (mmp_evict_run)
    static native int evictRun(long h, int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer freshSelf, long seed,
                               ByteBuffer out, ByteBuffer report);
    static native int tune(long h, String key, long value);
    static native double lastTiming(long h, String key);
    // the resident placement server (one_mode 3): out[0..3] = requests answered, graph-path fallbacks, launches, most slots busy
    static native int serverStats(long h, long[] out);
    // plug point 1: placement (CacheMissForwardingLB.getNext MM:4776-5004)
    static native int placeBatch(long h, ByteBuffer in, int n, ByteBuffer fresh, int nFresh, ByteBuffer extra, int nExtra, ByteBuffer out,
                                 long nowMs, long seed);
    static native int placeBatchTrace(long h, ByteBuffer in, int n, ByteBuffer fresh, int nFresh, ByteBuffer extra, int nExtra,
                                      ByteBuffer out, ByteBuffer trace, ByteBuffer candMask, long nowMs, long seed);
    static native int placeBatchExcluding(long h, ByteBuffer in, int n, ByteBuffer fresh, int nFresh, ByteBuffer extra, int nExtra,
                                          int[] exclude, ByteBuffer out, ByteBuffer trace, ByteBuffer candMask, long nowMs, long seed);
    static native int placeSweep(long h, int firstModel, int n, ByteBuffer self, int selfStride, ByteBuffer favourBits, ByteBuffer out,
                                 long nowMs, long seed);
    static native int placeOne(long h, ByteBuffer in, ByteBuffer fresh, int[] extra, ByteBuffer out, long nowMs, long seed);
    static native long batcherCreate(long h, int maxBatch, int maxWaitUs, long seed);
    static native void batcherDestroy(long batcher);
    static native int placeSubmit(long batcher, ByteBuffer in, ByteBuffer fresh, int[] extra, long nowMs, ByteBuffer out, int[] idOut);
    static native int batcherStats(long batcher, long[] batchesDecisionsOut);
    static native double placeBatchDevice(long h, long dIn, int n, long dOut, long nowMs, long seed);
    static native long deviceAlloc(long h, long bytes);
    static native int deviceFree(long h, long p);
    static native int deviceUpload(long h, long dst, ByteBuffer src, long bytes);
    static native int deviceDownload(long h, ByteBuffer dst, long src, long bytes);
    static native ByteBuffer allocPinned(long h, long bytes);
    static native int freePinned(long h, ByteBuffer buf);
    static native int flushL2(long h);
    // instance-sharded fleets
    static native int shardUniqueId(byte[] out128);
    static native int shardConnect(long h, byte[] id128);
    static native int shardWords(long h, int[] loHiOut);
    static native long shardOpenDecisions(long h);
    static final int SHARD_IPC_BYTES = 512;
    static native int shardIpcExport(long h, int maxBatch, byte[] blobOut);
    static native int shardIpcImport(long h, byte[] blobsByRank);
    static native int shardPeerStats(long h, long[] out4);
    static native int setIdBase(long h, long base);
    // introspection
    static native int rowWords(long h);
    static native int liveInstances(long h);
    static native int clusterOrder(long h, ByteBuffer outIdx, int cap);
    static native int typeSets(long h, int typeId, int nIdx, ByteBuffer allowed, ByteBuffer preferred, int[] nullsOut);
    static native long kernelLaunches(long h);
    static native int instancePartition(long h, int idx);
    // plug point 4: batch scans (ClusterStats MM:1570-1591, reaper MM:6616-6735)
    static native int stats(long h, ByteBuffer out, ByteBuffer partIds, int cap);
    static native int reaperSelect(long h, int partition, long nowMs, ByteBuffer taken, ByteBuffer outModels, int cap);
    // plug point 3: time-ordered weighted LRU (clhm/ConcurrentLinkedHashMap), fleet-wide batched form
    static native int lruInit(long h, int nInstances, ByteBuffer capacity, int slotsPerInstance);
    static native int lruApply(long h, ByteBuffer events, int n, long nowMs, ByteBuffer out, int cap);
    static native int lruApplyStatus(long h, ByteBuffer events, int n, long nowMs, ByteBuffer out, int cap, ByteBuffer status);
    static native int lruState(long h, int nInstances, ByteBuffer oldest, ByteBuffer weighted, ByteBuffer count);
    // read side: descendingMapWithCutoff / descendingLruMap (CLHM:1226-1260, 1087-1116), getLastUsedTime / getWeight (CLHM:742-771)
    static final int LRU_ENTRY_BYTES = 24;
    static native int lruRead(long h, ByteBuffer instances, int n, long usedSince, ByteBuffer offsets, ByteBuffer out, long cap);
    static native int lruLookup(long h, int n, ByteBuffer instance, ByteBuffer model, ByteBuffer lastUsed, ByteBuffer weight,
                                ByteBuffer loadTs);
    // the closed loop (simulation / what-if)
    static native int churnInit(long h, long loadTimeoutMs, long lastPublishedMs, int slotsPerInstance);
    static native int churnSeed(long h, int n, ByteBuffer instance, ByteBuffer model, ByteBuffer lastUsed, ByteBuffer weight,
                                ByteBuffer loadTs, long nowMs);
    static native int churnStep(long h, ByteBuffer events, int n, long now0, long now1, long seed, ByteBuffer decOut, int decCap,
                                ByteBuffer evictOut, int evictCap, ByteBuffer rowsOut, ByteBuffer report, int[] countsOut);
    static native int churnModel(long h, int model, ByteBuffer rowOut, ByteBuffer instances4);
    static native int churnModelIds(long h, int model, ByteBuffer rowOut, ByteBuffer ids, int cap);
}
