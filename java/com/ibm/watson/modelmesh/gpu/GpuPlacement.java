/*
 * GpuPlacement — host side of the libmmplace integration inside a ModelMesh pod: owns the fleet handle, the
 * string <-> dense-index dictionaries (instance ids, model ids), the record encoders and the debounced commit.
 * Source only (no JDK / litelinks / kv-utils jars in the build image); INTEGRATION.md walks through the three call sites.
 */
package com.ibm.watson.modelmesh.gpu;

import java.nio.ByteBuffer;
import java.nio.ByteOrder;
import java.util.ArrayDeque;
import java.util.HashMap;
import java.util.Map;
import java.util.concurrent.ConcurrentHashMap;
import java.util.concurrent.Executors;
import java.util.concurrent.ScheduledExecutorService;
import java.util.concurrent.TimeUnit;
import java.util.concurrent.atomic.AtomicBoolean;
import java.util.concurrent.atomic.AtomicLong;

import com.ibm.watson.modelmesh.InstanceRecord;
import com.ibm.watson.modelmesh.ModelRecord;

public final class GpuPlacement implements AutoCloseable {
    /** INSTANCE_REC_PUBLISH_MIN_PERIOD_MS (ModelMesh.java:232): records are never fresher than this, so neither are commits. */
    static final long COMMIT_DEBOUNCE_MS = 2_000L;

    final long h;
    private final int maxInstances, maxModels;
    private final Map<String, Integer> instanceIdx = new HashMap<>(), modelIdx = new ConcurrentHashMap<>();
    /** model-type name -> MmPlace.typeId (interned by the library, stable for the fleet's life) */
    private final Map<String, Integer> typeIdOf = new ConcurrentHashMap<>();
    private final ArrayDeque<Integer> freeInstanceIdx = new ArrayDeque<>();
    private final String[] instanceIdOf;
    private int nextModelIdx;
    private final AtomicBoolean commitScheduled = new AtomicBoolean();
    private final AtomicLong pickSeed = new AtomicLong(System.nanoTime());
    private final ScheduledExecutorService committer = Executors.newSingleThreadScheduledExecutor(r -> {
        Thread t = new Thread(r, "mmplace-commit"); t.setDaemon(true); return t; });
    /** per-thread pinned scratch: one decision in (32 B), one fresh row (64 B), one result (8 B) */
    private final ThreadLocal<ByteBuffer[]> scratch;

    public GpuPlacement(long minSpaceUnits, long minChurnAgeMs, int defaultModelSizeUnits, int maxInstances, int maxModels, int device) {
        this.h = MmPlace.create(minSpaceUnits, minChurnAgeMs, defaultModelSizeUnits, maxInstances, maxModels, device, 0, 1);
        this.maxInstances = maxInstances; this.maxModels = maxModels;
        this.instanceIdOf = new String[maxInstances];
        for (int i = maxInstances - 1; i >= 0; i--) freeInstanceIdx.push(i);
        this.scratch = ThreadLocal.withInitial(() -> new ByteBuffer[] { pinned(MmPlace.DECISION_IN_BYTES),
                pinned(MmPlace.INSTANCE_ROW_BYTES), pinned(MmPlace.DECISION_OUT_BYTES) });
    }

    private ByteBuffer pinned(int bytes) { return MmPlace.allocPinned(h, bytes).order(ByteOrder.LITTLE_ENDIAN); }

    /** mmp_instance_row (mmplace.h): lruTime, cap, used, startTime, vers : i64; count, lThreads, lInProg, rpm, shutdown, active : i32 */
    static ByteBuffer encode(InstanceRecord r, boolean active, ByteBuffer b) {
        b.clear();
        b.putLong(r.getLruTime()).putLong(r.getCapacity()).putLong(r.getUsed()).putLong(r.getStartTime()).putLong(r.getInstanceVersion());
        b.putInt(r.getCount()).putInt(r.getLoadingThreads()).putInt(r.getLoadingInProgress()).putInt(r.getReqsPerMinute());
        b.putInt(r.isShuttingDown() ? 1 : 0).putInt(active ? 1 : 0);
        return b;
    }

    // ---- plug point 2: called from handleInstanceTableChange (ModelMesh.java:1455) after the existing bookkeeping ----
    public synchronized void onInstanceEvent(boolean deleted, String key, InstanceRecord rec, boolean inServiceInstanceList) {
        Integer idx = instanceIdx.get(key);
        if (deleted || rec == null) {
            if (idx != null) { MmPlace.instanceRemove(h, idx); instanceIdx.remove(key); instanceIdOf[idx] = null; freeInstanceIdx.push(idx); }
        } else {
            if (idx == null) { idx = freeInstanceIdx.pop(); instanceIdx.put(key, idx); instanceIdOf[idx] = key; }
            ByteBuffer row = ByteBuffer.allocateDirect(MmPlace.INSTANCE_ROW_BYTES).order(ByteOrder.LITTLE_ENDIAN);
            check(MmPlace.instanceUpsert(h, idx, encode(rec, inServiceInstanceList, row), key, rec.getLocation(), rec.getZone(), rec.getLabels()));
        }
        scheduleCommit();
    }

    // ---- called from ModelMesh.event(type, key, ModelRecord) (ModelMesh.java:2807-2854); knownSizeUnits = CacheEntry weight or 0 ----
    public void onModelEvent(boolean deleted, String modelId, String recordJson, int knownSizeUnits) {
        int m = modelIdx.computeIfAbsent(modelId, k -> { synchronized (this) { return nextModelIdx++; } });
        // the record travels as the KV store holds it: instance ids inside it are resolved by the library at every commit
        check(MmPlace.modelUpsertJson(h, m, deleted ? "{}" : recordJson, knownSizeUnits));
        scheduleCommit();
    }
    /** typeMappingsUpdated (TypeConstraintManager.java:607): the raw MM_TYPE_CONSTRAINTS document, null when unset */
    public void onTypeConstraints(String json) { check(MmPlace.typesSetJson(h, json)); scheduleCommit(); }
    /** UpgradeTracker.getLikelyReplacedReplicaSets() keys (UpgradeTracker.java:78) */
    public void onLikelyReplacedReplicaSets(String[] prefixes) { check(MmPlace.replicasetsSet(h, prefixes)); scheduleCommit(); }

    private void scheduleCommit() {
        if (commitScheduled.compareAndSet(false, true))
            committer.schedule(() -> { commitScheduled.set(false); check(MmPlace.commit(h)); }, COMMIT_DEBOUNCE_MS, TimeUnit.MILLISECONDS);
    }

    // ---- plug point 1: one getNext on the request thread (GpuCacheMissLB) ----
    /** @return instance id, null (getNext returned null) or SELF for LoadBalancer.ABORT_REQUEST */
    public static final String SELF = new String("<self>");
    /**
     * The model travels as the record this request read (MMP_DF_REQUEST_MODEL): its type and its loaded ∪ failed instances,
     * as the reference builds the CacheMissExcludeSet from the record (MM:3537, 3782-3785), so a model registered or changed
     * since the last commit is placed on its current record.  Instance ids the dictionary does not know are dropped (they
     * name no live instance).  Up to MMP_MAX_EXTRA ids travel as the decision's extras; more (a scale-up's exclude set, the
     * janitor's every-copy-plus-self, a long chain of ensureLoadedElsewhere targets) travel all together as the call's
     * exclude set (mmp_place_batch_excluding, a batch of one with no extras), which excludes them the same way.
     */
    public String placeOne(String modelType, java.util.Set<String> loadedAndFailed, String selfId, long lastUsedTime, boolean favourSelf,
                           InstanceRecord fresh, java.util.Set<String> requestExcludes, long nowMs) {
        // (ModelRecord's DEFAULT_TYPE for a record without one, MR:117-130, as the library reads a JSON record)
        int type = typeIdOf.computeIfAbsent(modelType == null ? "NLCLASSIFIER" : modelType, t -> check(MmPlace.typeId(h, t)));
        Integer self;
        int[] extra = new int[MmPlace.MAX_EXTRA];
        int n = 0;
        synchronized (this) {
            self = instanceIdx.get(selfId);
            for (java.util.Set<String> set : java.util.Arrays.asList(loadedAndFailed, requestExcludes))
                for (String e : set) {
                    Integer i = instanceIdx.get(e);
                    if (i == null) continue;
                    if (n == extra.length) extra = java.util.Arrays.copyOf(extra, 2 * n);
                    extra[n++] = i;
                }
        }
        if (self == null) return null;
        final boolean asSet = n > MmPlace.MAX_EXTRA;
        ByteBuffer[] s = scratch.get();
        ByteBuffer in = s[0], fr = s[1], out = s[2];
        in.clear();
        in.putInt(type).putInt(self).putLong(lastUsedTime).putInt(MmPlace.DF_REQUEST_MODEL | (favourSelf ? MmPlace.DF_FAVOUR_SELF : 0))
          .putInt(fresh != null ? 0 : -1).putInt(0).putInt(asSet ? 0 : n);
        extra = java.util.Arrays.copyOf(extra, n);
        if (fresh != null) encode(fresh, true, fr);
        int rc = asSet
                ? MmPlace.placeBatchExcluding(h, in, 1, fresh != null ? fr : null, fresh != null ? 1 : 0, null, 0, extra, out, null, null, nowMs,
                                              pickSeed.incrementAndGet())
                : MmPlace.placeOne(h, in, fresh != null ? fr : null, extra.length > 0 ? extra : null, out, nowMs, pickSeed.incrementAndGet());
        if (rc < 0) throw new IllegalStateException(MmPlace.lastError(h));  // the caller falls back to the Java load balancer
        int target = out.getInt(0);
        if (target == MmPlace.TARGET_SELF) return SELF;
        if (target < 0) return null;
        synchronized (this) { return instanceIdOf[target]; }
    }

    // ---- plug point 4: the reaper's sweep (ModelMesh.java:6616-6735) ----
    public int reaperSelect(int partition, long nowMs, ByteBuffer taken, ByteBuffer outModels, int cap) {
        return check(MmPlace.reaperSelect(h, partition, nowMs, taken, outModels, cap));
    }
    // one run of the leader's reaper task (ModelMesh.java:6436-6494): returns the number of loads; report gets the totals
    public int reaperRun(int leader, long nowMs, long assumeGoneMs, ByteBuffer missingSince, ByteBuffer prunedModels,
                         ByteBuffer prunedInstances, int prunedCap, ByteBuffer repairedModels, int repairedCap, ByteBuffer loads,
                         int loadsCap, ByteBuffer report) {
        return check(MmPlace.reaperRun(h, leader, nowMs, assumeGoneMs, missingSince, pickSeed.incrementAndGet(), prunedModels,
                                       prunedInstances, prunedCap, repairedModels, repairedCap, loads, loadsCap, report));
    }

    // the registry loop of this pod's janitor task (ModelMesh.java:6013-6145): returns the number of edits; report gets the totals
    public int janitorRun(int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer edits, int cap, ByteBuffer report) {
        return check(MmPlace.janitorRun(h, self, entries, n, params, edits, cap, report));
    }

    // one run of this pod's whole janitor task (ModelMesh.java:5876-6145): the cache pass over entries (most recently used
    // first), an action per entry in out, then the registry loop on the records it left; returns the number of edits
    public int janitorTask(int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer out, ByteBuffer edits, int cap,
                           ByteBuffer report) {
        return check(MmPlace.janitorTask(h, self, entries, n, params, out, edits, cap, report));
    }

    // one run of this pod's rate-tracking task (ModelMesh.java:5619-5858): returns the number of loads; report gets the gate
    // and the totals.  freshSelf may be null
    public int rateRun(int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer freshSelf, ByteBuffer out, ByteBuffer loads,
                       int loadsCap, ByteBuffer report) {
        return check(MmPlace.rateRun(h, self, entries, n, params, freshSelf, pickSeed.incrementAndGet(), out, loads, loadsCap, report));
    }

    // this pod's pre-shutdown migration (ModelMesh.java:6990-7047): out gets one action per entry of descendingLruMap(), report
    // foundOther and the totals; returns n.  freshSelf may be null
    public int shutdownRun(int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer freshSelf, ByteBuffer out, ByteBuffer report) {
        return check(MmPlace.shutdownRun(h, self, entries, n, params, freshSelf, pickSeed.incrementAndGet(), out, report));
    }

    // this pod's eviction listener (ModelMesh.java:2867-2933) for the evictions its cache reported, in listener order: out gets
    // one action per entry (the deregistration edit, and the reload's answer), report the totals; returns n.  freshSelf may be null
    public int evictRun(int self, ByteBuffer entries, int n, ByteBuffer params, ByteBuffer freshSelf, ByteBuffer out, ByteBuffer report) {
        return check(MmPlace.evictRun(h, self, entries, n, params, freshSelf, pickSeed.incrementAndGet(), out, report));
    }

    // for the pod's metrics: {requests the resident placement server answered, calls that found all its slots taken and took
    // the graph path, its launches, the most slots busy at once}, since this placement was created
    public long[] serverStats() {
        long[] out = new long[4];
        check(MmPlace.serverStats(h, out));
        return out;
    }

    private int check(int rc) { if (rc < 0) throw new IllegalStateException(MmPlace.lastError(h)); return rc; }
    @Override public void close() { committer.shutdownNow(); MmPlace.destroy(h); }
}
