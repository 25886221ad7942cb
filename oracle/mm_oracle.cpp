/*
 * mm_oracle.cpp — CPU ORACLE: a line-by-line C++17 restatement of the ModelMesh placement /
 * LRU-eviction hot path.  TEST INFRASTRUCTURE ONLY (see mm_oracle.h).  It deliberately keeps the
 * reference's *shape* (an ordered set of boxed records walked with an iterator, string tie-breaks,
 * Set<String>-style membership tests, a linked-list LRU) so that it is an independent check on the
 * rank-space/bitmask formulation used by the CUDA product, and so that timing it is a fair
 * "reference-shaped CPU path" baseline.
 *
 * Reference = kserve/modelmesh @ ea13cdc5.  Abbreviations: MM = ModelMesh.java, IR = InstanceRecord.java,
 * TCM = TypeConstraintManager.java, ISST = InstanceSetStatsTracker.java, UT = UpgradeTracker.java,
 * CLHM = clhm/ConcurrentLinkedHashMap.java, LD = clhm/LinkedDeque.java.
 *
 *   PlacementOrder::compare        MM:4646-4703   (isFull MM:4640-4642, Utils.STRING_ARRAY_COMP Utils.java:25-36)
 *   Fleet::instanceEvent           MM:1455-1568   (ISST:63-92, ClusterStats MM:1570-1591)
 *   Tcm::*                         TCM:242-262, 337-506, 512-747
 *   UpgradeTracker::*              UT:78-80, 85-115, 120-187
 *   Fleet::getNext                 MM:4757-5005   (filter MM:4760-4771, CacheMissExcludeSet MM:4717-4749)
 *   Lru::*                         CLHM:329-352, 438-452, 590-652, 821-858, 860-871, 963-984, 1125-1133, 1357-1360;
 *                                  LD:243-288
 *   orc_unload_reserve_units       MM:749-755      orc_min_space_units  MM:767-769
 *   orc_churn_reject               MM:3872-3884    orc_early_reject     MM:5185-5190
 *   Fleet::reaperSelect            MM:6574-6577, 6616-6735 (ModelToLoad MM:6393-6409)
 *
 * Quirks reproduced literally (SURVEY.md §8a N1-N6 plus ones found while restating):
 *   N1  MM:4663,4665 compare the absolute timestamp getLruTime() with the duration minChurnAgeMs*2.
 *   N2  MM:4909 `curInst = us ? bestEntry.getValue() : getFreshInstanceRecord()` — for every non-self
 *       candidate the range tests (MM:4913, 4919-4922) and the recorded rpm (MM:4936) use the CALLER's
 *       fresh record; for the self candidate they use the first filtered entry's record.  Only `count`
 *       (MM:4925) comes from the candidate.
 *   N3  `us = !us && ...` toggling (MM:4840, 4870, 4908).
 *   N4  ThreadLocalRandom.nextInt (MM:4981) is replaced by ((orc_hash64(seed, decisionId) >> 32) * remainingCount) >> 32.
 *   N5  age(t) = t==0 ? 0 : now - t (MM:4162-4164); `now` is an explicit input.
 *   N6  a batch is evaluated against one snapshot of the instance table; only self is fresh.
 *   N7  getFreshInstanceRecord (MM:5369-5386) never sets reqsPerMinute, so the fresh record's rpm is 0;
 *       the caller supplies the fresh row, orc_get_next_batch(fresh_idx=-1) reproduces rpm=0.
 *   N8  non-simple case (b) returns null — not ABORT_REQUEST — when self is a preferred candidate and
 *       favourSelf is set (MM:4871-4873).
 *   N9  UpgradeTracker keys its map by the labels String[] *object* (UT:67, identity hash): only records
 *       sharing InstanceRecord.NO_LABELS (IR:35,87-88) ever land in the same PerTypeLabelStats.
 *   N10 handleInstanceTableChange recomputes the changed subset's LRU over *all* cluster instances
 *       (MM:1519-1541), and refreshPerTypeInstanceSets runs before the new record is in clusterState
 *       (MM:1489-1493), so inferred-preferred sets lag one event behind.
 *   N11 ModelTypeConstraints.fromInstanceSet (TCM:418-433) never puts an instance that satisfies the
 *       required labels into the preferred set (else-if), whereas updateInstance (TCM:455-468) treats the
 *       two independently; refreshPerTypeInstanceSets (TCM:706-707) replaces the preferred set of every
 *       type without required labels by the default inferred one.
 *       orc_tc_converge() re-runs the refresh with all instances present so snapshot parity does not depend on
 *       arrival order (see mm_oracle.h).
 *   N12 ModelToLoad.compareTo (MM:6405-6408) orders by lastUsed only, so the reaper's TreeSet drops a
 *       candidate whose lastUsed equals one already held.
 *   N14 setCapacity (CLHM:305-316) evicts without updateOldestTime, which only afterWrite (CLHM:444) and
 *       tryToDrainBuffers (CLHM:463) call: oldestTime() keeps the head from before the evictions until the
 *       next write or read of a present key, and loadLocal's churn guard (MM:3876) reads that value.
 * Shutting-down records are treated as deletions (MM:1462-1464) so never sit in clusterState.
 * Java integer semantics: int/long arithmetic wraps, >> is arithmetic, / truncates toward zero,
 * (int)double saturates.
 */
#include "mm_oracle.h"

#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cstring>
#include <list>
#include <map>
#include <memory>
#include <optional>
#include <set>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

namespace {

typedef std::u16string JStr;  // java.lang.String: sequence of UTF-16 code units

JStr utf8to16(const char *s) {
  JStr out;
  if (!s) return out;
  const unsigned char *p = (const unsigned char *)s;
  while (*p) {
    uint32_t cp;
    if (*p < 0x80) { cp = *p++; }
    else if ((*p >> 5) == 6 && p[1]) { cp = ((p[0] & 0x1F) << 6) | (p[1] & 0x3F); p += 2; }
    else if ((*p >> 4) == 14 && p[1] && p[2]) { cp = ((p[0] & 0x0F) << 12) | ((p[1] & 0x3F) << 6) | (p[2] & 0x3F); p += 3; }
    else if ((*p >> 3) == 30 && p[1] && p[2] && p[3]) {
      cp = ((p[0] & 0x07) << 18) | ((p[1] & 0x3F) << 12) | ((p[2] & 0x3F) << 6) | (p[3] & 0x3F); p += 4;
    } else { cp = 0xFFFD; p++; }
    if (cp >= 0x10000) { cp -= 0x10000; out.push_back((char16_t)(0xD800 + (cp >> 10))); out.push_back((char16_t)(0xDC00 + (cp & 0x3FF))); }
    else out.push_back((char16_t)cp);
  }
  return out;
}
std::string u16to8(const JStr &s) {  // only for diagnostics / replicaset names (BMP subset is enough)
  std::string o;
  for (char16_t c : s) {
    if (c < 0x80) o.push_back((char)c);
    else if (c < 0x800) { o.push_back((char)(0xC0 | (c >> 6))); o.push_back((char)(0x80 | (c & 0x3F))); }
    else { o.push_back((char)(0xE0 | (c >> 12))); o.push_back((char)(0x80 | ((c >> 6) & 0x3F))); o.push_back((char)(0x80 | (c & 0x3F))); }
  }
  return o;
}
// String.compareTo: lexicographic over UTF-16 code units, then length
inline int jcompare(const JStr &a, const JStr &b) {
  size_t n = std::min(a.size(), b.size());
  for (size_t i = 0; i < n; i++)
    if (a[i] != b[i]) return (int)a[i] - (int)b[i];
  return (int)a.size() - (int)b.size();
}
// Utils.STRING_ARRAY_COMP (Utils.java:25-36)
inline int stringArrayComp(const std::vector<JStr> &l1, const std::vector<JStr> &l2) {
  int diff = (int)l1.size() - (int)l2.size();
  if (diff != 0) return diff;
  for (size_t i = 0; i < l1.size(); i++)
    if ((diff = jcompare(l1[i], l2[i])) != 0) return diff;
  return 0;
}
struct StringArrayLess {
  bool operator()(const std::vector<JStr> &a, const std::vector<JStr> &b) const { return stringArrayComp(a, b) < 0; }
};

// Java wrapping arithmetic helpers
inline int64_t jsub(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
inline int64_t jadd(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
inline int32_t jaddi(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
inline int32_t jsubi(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
inline int32_t jmuli(int32_t a, int32_t b) { return (int32_t)((uint32_t)a * (uint32_t)b); }
inline int64_t jmul(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
inline int32_t jd2i(double d) {  // (int) double: NaN->0, saturating
  if (d != d) return 0;
  if (d >= 2147483647.0) return INT32_MAX;
  if (d <= -2147483648.0) return INT32_MIN;
  return (int32_t)d;
}
inline int64_t jdiv(int64_t a, int64_t b) {  // Java long division (b != 0), MIN/-1 wraps
  if (b == -1) return (int64_t)(0 - (uint64_t)a);
  return a / b;
}

struct Pts;  // ProhibitedTypeSet

// InstanceRecord (IR:33-256)
struct IR {
  int64_t lruTime = 0;
  int32_t count = 0;
  int64_t capacity = 0, used = 0;
  int32_t lThreads = 0, lInProg = 0, rpm = 0;
  bool shuttingDown = false;
  int64_t startTime = 0, vers = 0;
  bool hasLoc = false, hasZone = false;
  JStr loc, zone;
  std::vector<JStr> labels;  // sorted (IR:90-91)
  uint64_t labelsIdentity = 0;  // 0 == the shared NO_LABELS constant (IR:35,87-88); else unique per record (N9)
  const Pts *prohibitedTypes = nullptr;
  int64_t getRemaining() const { return std::max<int64_t>(0, jsub(capacity, used)); }  // IR:203-205
};
typedef std::shared_ptr<IR> IRp;

struct Entry {  // Map.Entry<String, InstanceRecord>
  JStr key;
  int32_t idx;
  IRp rec;
};

// NULLS_LAST (MM:4644): Ordering.natural().nullsLast()
inline int nullsLastCompare(bool has1, const JStr &s1, bool has2, const JStr &s2) {
  if (!has1 && !has2) return 0;
  if (!has1) return 1;
  if (!has2) return -1;
  int c = jcompare(s1, s2);
  return c < 0 ? -1 : (c > 0 ? 1 : 0);
}
inline int sgn(int64_t a, int64_t b) { return a < b ? -1 : (a > b ? 1 : 0); }  // Long.compare / Ints.compare

struct PlacementOrder {  // MM:4646-4703
  int64_t minSpaceUnits = 0, minChurnAgeMs = 0;
  bool isFull(int64_t availableUnits) const { return availableUnits < minSpaceUnits; }  // MM:4640-4642
  int compare(const Entry &e1, const Entry &e2) const {
    const IR *ir1 = e1.rec.get(), *ir2 = e2.rec.get();
    if (ir1 == ir2) return jcompare(e1.key, e2.key);
    bool sd1 = ir1->shuttingDown;
    if (sd1 ^ ir2->shuttingDown) return sd1 ? 1 : -1;
    int64_t vers1 = ir1->vers, vers2 = ir2->vers;
    int64_t rem1 = ir1->getRemaining(), rem2 = ir2->getRemaining();
    bool full1 = isFull(rem1), full2 = isFull(rem2);
    if (vers1 != vers2) {
      // prefer newer version *unless* it's saturated  (N1)
      if (vers1 > vers2) {
        if (!full1 || ir1->lruTime > jmul(minChurnAgeMs, 2)) return -1;
      } else if (!full2 || ir2->lruTime > jmul(minChurnAgeMs, 2)) return 1;
    }
    if (full1 ^ full2) return full1 ? 1 : -1;
    if (full1) {
      int oldestDiff = sgn(ir1->lruTime, ir2->lruTime);
      if (oldestDiff != 0) return oldestDiff;
    }
    int countDiff = jsubi(ir1->count, ir2->count);  // int subtraction (may wrap, as in Java)
    if (countDiff != 0) return countDiff;
    int remDiff = sgn(rem2, rem1);
    if (remDiff != 0) return remDiff;
    if (!full1) {
      int oldestDiff = sgn(ir1->lruTime, ir2->lruTime);
      if (oldestDiff != 0) return oldestDiff;
    }
    int lip1 = ir1->lInProg, lip2 = ir2->lInProg;
    int c;
    // ComparisonChain: first non-zero result wins; int compares are Ints.compare (no wrap on the compare itself)
    if ((c = sgn(jsubi(ir2->lThreads, lip2), jsubi(ir1->lThreads, lip1))) != 0) return c;
    if ((c = sgn(lip1, lip2)) != 0) return c;
    if ((c = sgn(ir2->capacity, ir1->capacity)) != 0) return c;
    if ((c = sgn(ir1->rpm, ir2->rpm)) != 0) return c;
    if ((c = jcompare(e1.key, e2.key)) != 0) return c < 0 ? -1 : 1;
    if ((c = nullsLastCompare(ir1->hasLoc, ir1->loc, ir2->hasLoc, ir2->loc)) != 0) return c;
    if ((c = nullsLastCompare(ir1->hasZone, ir1->zone, ir2->hasZone, ir2->zone)) != 0) return c;
    if ((c = stringArrayComp(ir1->labels, ir2->labels)) != 0) return c < 0 ? -1 : 1;
    return 0;
  }
};
struct EntryLess {
  const PlacementOrder *po;
  bool operator()(const Entry &a, const Entry &b) const { return po->compare(a, b) < 0; }
};
typedef std::set<Entry, EntryLess> ClusterState;  // ConcurrentSkipListSet<>(PLACEMENT_ORDER) MM:774

// ClusterStats MM:1570-1591
struct ClusterStats {
  int64_t totalCapacity = 0, totalFree = 0, globalLru = INT64_MAX;
  int32_t instanceCount = 0, modelCopyCount = 0;
};

// ProhibitedTypeSet TCM:295-333
struct Pts {
  std::vector<std::string> types;  // sorted
  int id = 0;
  bool contains(const std::string &t) const { return std::binary_search(types.begin(), types.end(), t); }
};

// InstanceSetStatsTracker ISST:31-93
struct Isst {
  const PlacementOrder *po;
  const Pts *prohibitedTypesSet;  // null for the cluster-wide tracker
  int64_t totalCapacity = 0, totalFree = 0, lru = INT64_MAX;
  int32_t count = 0, modelCount = 0;
  ClusterStats currentStats;  // EMPTY_STATS
  Isst(const Pts *p, const PlacementOrder *po_) : po(po_), prohibitedTypesSet(p) {}
  void resetLru() { lru = INT64_MAX; }
  void addLru(int64_t l) { if (l > 0 && l < lru) lru = l; }
  void add(const IR &ir) {
    count++;
    modelCount = jaddi(modelCount, ir.count);
    totalCapacity = jadd(totalCapacity, ir.capacity);
    int64_t available = ir.getRemaining();
    if (!po->isFull(available)) totalFree = jadd(totalFree, available);
  }
  bool remove(const IR &ir) {
    count--;
    modelCount = jsubi(modelCount, ir.count);
    totalCapacity = jsub(totalCapacity, ir.capacity);
    int64_t available = ir.getRemaining();
    if (!po->isFull(available)) totalFree = jsub(totalFree, available);
    return count <= 0;
  }
  ClusterStats update() {
    ClusterStats ns;
    ns.totalCapacity = totalCapacity; ns.totalFree = totalFree; ns.globalLru = lru;
    ns.instanceCount = count; ns.modelCopyCount = modelCount;
    if (prohibitedTypesSet != nullptr) currentStats = ns;
    return ns;
  }
};

// Set<String> of instance ids (ids <-> idx bijection): sorted vector for iteration/equality + dense byte map so that
// contains() is O(1) like the reference's HashSet/ImmutableSet.
struct IdSet {
  std::vector<int32_t> v;
  std::vector<uint8_t> m;
  size_t count(int32_t i) const { return (i >= 0 && (size_t)i < m.size() && m[i]) ? 1 : 0; }
  size_t size() const { return v.size(); }
  bool empty() const { return v.empty(); }
  void insert(int32_t i) {
    if (count(i)) return;
    if ((size_t)i >= m.size()) m.resize((size_t)i + 1, 0);
    m[i] = 1;
    v.insert(std::lower_bound(v.begin(), v.end(), i), i);
  }
  void erase(int32_t i) {
    if (!count(i)) return;
    m[i] = 0;
    v.erase(std::lower_bound(v.begin(), v.end(), i));
  }
  void clear() { v.clear(); m.clear(); }
  std::vector<int32_t>::const_iterator begin() const { return v.begin(); }
  std::vector<int32_t>::const_iterator end() const { return v.end(); }
};
typedef std::optional<IdSet> OptSet;  // ... or null

// ModelTypeConstraints TCM:337-506
struct Mtc {
  std::vector<JStr> requiredLabels, preferredLabels;  // sorted, disjoint
  OptSet allowedInstances;               // null iff no required labels
  OptSet preferredInstances;             // resolved (configured or inferred)
  OptSet configuredPreferredInstances;
  bool hasStats = false;                 // instanceSetStats != null
  std::vector<Isst *> instanceSetStats;
  bool allowedOnInstance(int32_t iid) const { return !allowedInstances || allowedInstances->count(iid); }
};
typedef std::shared_ptr<const Mtc> Mtcp;

// instanceMatches TCM:478-486 (instanceLabels sorted)
bool instanceMatches(const std::vector<JStr> &instanceLabels, const std::vector<JStr> &typeLabels, bool matchAll) {
  if (instanceLabels.empty() || typeLabels.empty()) return false;
  auto hasLabel = [&](const JStr &l) {
    // Arrays.binarySearch over the sorted instance labels
    size_t lo = 0, hi = instanceLabels.size();
    while (lo < hi) {
      size_t mid = (lo + hi) / 2;
      int c = jcompare(instanceLabels[mid], l);
      if (c < 0) lo = mid + 1; else if (c > 0) hi = mid; else return true;
    }
    return false;
  };
  if (matchAll) { for (auto &l : typeLabels) if (!hasLabel(l)) return false; return true; }
  for (auto &l : typeLabels) if (hasLabel(l)) return true;
  return false;
}

// updateInstanceSet TCM:489-505; returns true if changed and writes `out`
bool updateInstanceSet(int32_t iid, const std::vector<JStr> &instanceLabels, const std::vector<JStr> &typeLabels,
                       const OptSet &instanceSet, bool matchAll, OptSet &out) {
  bool curMatch = instanceSet && instanceSet->count(iid);
  if (instanceMatches(instanceLabels, typeLabels, matchAll)) {
    if (!curMatch) {
      IdSet s = instanceSet ? *instanceSet : IdSet();
      s.insert(iid);
      out = std::move(s);
      return true;
    }
  } else if (curMatch) {
    if (instanceSet->size() == 1) {
      if (matchAll) out = IdSet(); else out = std::nullopt;
      return true;
    }
    IdSet s = *instanceSet;
    s.erase(iid);
    out = std::move(s);
    return true;
  }
  return false;
}

// sortAndDeduplicate TCM:100-113
std::vector<JStr> sortAndDeduplicate(std::vector<JStr> arr, const std::vector<JStr> *exclude) {
  if (arr.empty()) return arr;
  std::sort(arr.begin(), arr.end(), [](const JStr &a, const JStr &b) { return jcompare(a, b) < 0; });
  std::vector<JStr> out;
  for (auto &l : arr) {
    bool dupe = !out.empty() && out.back() == l;
    bool excl = exclude && std::binary_search(exclude->begin(), exclude->end(), l,
                                              [](const JStr &a, const JStr &b) { return jcompare(a, b) < 0; });
    if (!dupe && !excl) out.push_back(l);
  }
  return out;
}

struct ConfigTypeConstraints {  // TCM:79-98
  std::vector<JStr> required, preferred;
  bool isEmpty() const { return required.empty() && preferred.empty(); }
};

// UpgradeTracker UT:45-202
struct UpgradeTracker {
  static constexpr int64_t TEN_MINS = 600000, FIFTEEN_MINS = 900000, TWENTY_MINS = 1200000;
  struct ReplicaSetStats { int size = 0; int64_t earliestStartTime = INT64_MAX, latestStartTime = 0, lastChangeTime = 0; };
  typedef std::map<JStr, ReplicaSetStats> PerTypeLabelStats;  // HashMap<String, ReplicaSetStats>; order-insensitive use
  std::unordered_map<uint64_t, PerTypeLabelStats> upgradeTracker;  // keyed by labels array identity (N9)
  std::map<JStr, int64_t> likelyReplacedReplicaSets;

  void instanceRemoved(const JStr &iid, const IR &ir, int64_t now) {  // UT:85-115
    if (iid.size() < 7) return;
    auto it = upgradeTracker.find(ir.labelsIdentity);
    if (it == upgradeTracker.end()) return;
    PerTypeLabelStats &ptls = it->second;
    JStr replicaSet = iid.substr(0, 6);
    auto rit = ptls.find(replicaSet);
    if (rit != ptls.end()) {
      ReplicaSetStats rss = rit->second;  // copy: Java keeps the object after ptls.remove
      rss.size--;
      if (rss.size > 0) { rss.lastChangeTime = now; rit->second = rss; }
      else ptls.erase(rit);
      if (likelyReplacedReplicaSets.count(replicaSet)) {
        if (rss.size <= 0) likelyReplacedReplicaSets.erase(replicaSet);
        else likelyReplacedReplicaSets[replicaSet] = jadd(rss.lastChangeTime, FIFTEEN_MINS);
      }
    }
  }
  void instanceAdded(const JStr &iid, const IR &ir, int64_t now) {  // UT:120-187
    if (iid.size() < 7) return;
    PerTypeLabelStats &ptls = upgradeTracker[ir.labelsIdentity];
    JStr replicaSetId = iid.substr(0, 6);
    ReplicaSetStats &rss = ptls[replicaSetId];
    rss.lastChangeTime = now;
    rss.size++;
    int64_t startTime = ir.startTime;
    if (startTime < rss.earliestStartTime) rss.earliestStartTime = startTime;
    if (startTime > rss.latestStartTime) rss.latestStartTime = startTime;

    std::set<JStr> old;
    if (ptls.size() > 1) {
      // Stream.max(cmp) keeps the first of equal maxima in HashMap encounter order, which is not reproducible;
      // ties are outside the parity domain (replicasets of one Deployment start at distinct times).
      const ReplicaSetStats *newest = nullptr;
      for (auto &e : ptls)
        if (!newest || e.second.earliestStartTime > newest->earliestStartTime) newest = &e.second;
      if (newest->latestStartTime > jsub(now, TWENTY_MINS)) {
        for (auto &e : ptls)
          if (e.second.latestStartTime < newest->earliestStartTime &&
              (newest->latestStartTime > jsub(now, TEN_MINS) || e.second.lastChangeTime > jsub(now, FIFTEEN_MINS)))
            old.insert(e.first);
      }
    }
    if (likelyReplacedReplicaSets.empty() && old.empty()) return;
    for (auto &ent : ptls) {
      const JStr &rs = ent.first;
      if (old.count(rs)) {
        if (!likelyReplacedReplicaSets.count(rs))
          likelyReplacedReplicaSets[rs] = jadd(ent.second.lastChangeTime, FIFTEEN_MINS);
      } else if (likelyReplacedReplicaSets.count(rs)) {
        likelyReplacedReplicaSets.erase(rs);
      }
    }
  }
  void doHousekeeping(int64_t now) {  // UT:192-201
    for (auto it = likelyReplacedReplicaSets.begin(); it != likelyReplacedReplicaSets.end();)
      if (now >= it->second) it = likelyReplacedReplicaSets.erase(it); else ++it;
  }
};

struct Fleet;

// TypeConstraintManager TCM:64-748 (only the state/sets used by placement, stats and the reaper)
struct Tcm {
  Fleet *fleet;
  int32_t localInstanceId = -1;
  std::map<std::vector<JStr>, Isst *, StringArrayLess> labelsToInstanceSetStats;  // TreeMap(STRING_ARRAY_COMP)
  std::map<std::vector<std::string>, Isst *> ptsToInstanceSetStats;               // HashMap<PTS, ISST>
  std::vector<std::unique_ptr<Isst>> isstOwner;
  std::vector<std::unique_ptr<Pts>> ptsOwner;
  Isst *localInstanceSetStats = nullptr;
  std::map<std::string, Mtcp> typeConstraintsMap;
  OptSet defaultPreferredInstances;
  bool deferRefresh = false;  // test-harness switch for bulk loads, see orc_tc_defer_refresh

  // (raw pointers: the map is not mutated while decisions run, and a Java reference read costs no refcount traffic)
  const Mtc *getTypeConstraints(const std::string &type) const {  // TCM:258-262
    auto it = typeConstraintsMap.find(type);
    if (it != typeConstraintsMap.end()) return it->second.get();
    it = typeConstraintsMap.find("_default");
    return it != typeConstraintsMap.end() ? it->second.get() : nullptr;
  }
  // TCM:242-245: null means all
  const OptSet *getCandidateInstances(const std::string &type) const {
    const Mtc *m = getTypeConstraints(type);
    static const OptSet NULLSET;
    return m ? &m->allowedInstances : &NULLSET;
  }
  // TCM:248-251
  const OptSet *getPreferredInstances(const std::string &type) const {
    const Mtc *m = getTypeConstraints(type);
    return m ? &m->preferredInstances : &defaultPreferredInstances;
  }
  Isst *getStatsForLabels(const std::vector<JStr> &labels) {  // TCM:508-510
    auto it = labelsToInstanceSetStats.find(labels);
    return it == labelsToInstanceSetStats.end() ? nullptr : it->second;
  }

  static Mtcp fromInstanceSet(const std::vector<JStr> &requiredLabels, const std::vector<JStr> &preferredLabels,
                              const ClusterState &instances, bool hasStats, const std::vector<Isst *> &stats);
  static Mtcp updateInstance(const Mtcp &mtc, int32_t iid, const std::vector<JStr> &labels);
  static bool instanceUpdated(int32_t iid, const std::vector<JStr> &labels, const std::map<std::string, Mtcp> &mtcMap,
                              std::map<std::string, Mtcp> &newMap);
  Isst *getInstanceSetStats(int32_t iid, const std::vector<JStr> &labels, const std::map<std::string, Mtcp> &tcMap);
  Isst *instanceAdded(int32_t iid, const std::vector<JStr> &labels, bool includedInStats);
  void instanceRemoved(int32_t iid, const std::vector<JStr> &labels);
  void typeMappingsUpdated(std::map<std::string, ConfigTypeConstraints> newConfig);
  void refreshPerTypeInstanceSets(std::map<std::string, Mtcp> &mtcMap);
  static OptSet inferPreferredInstances(const std::map<int32_t, int32_t> &instanceScores, const IdSet *include);
};

struct Fleet {
  PlacementOrder po;
  int32_t defaultModelSizeUnits = 0;
  ClusterState clusterState;
  std::vector<uint8_t> siActive;  // litelinks siMap (MM:4778): instance idx -> known service instance
  bool haveTc = false;            // typeConstraints != null
  Tcm tcm;
  UpgradeTracker upgradeTracker;
  Isst clusterStatsTracker;
  ClusterStats clusterStats;
  int changeCounter = 0;
  uint64_t nextLabelsIdentity = 1;
  std::vector<IRp> byIdx;  // test convenience: latest record by instance idx (null if absent)
  std::vector<uint8_t> inTable;  // instanceInfo.contains(id): the KV table holds a record (a shutting-down one included)
  std::vector<JStr> keyByIdx;

  Fleet(int64_t minSpace, int64_t minChurn, int32_t defSize) : clusterState(EntryLess{&po}), clusterStatsTracker(nullptr, &po) {
    po.minSpaceUnits = minSpace;
    po.minChurnAgeMs = minChurn;
    defaultModelSizeUnits = defSize;
    tcm.fleet = this;
  }
  bool isFull(int64_t r) const { return po.isFull(r); }
  void instanceEvent(int type, int32_t idx, const JStr &key, IRp record, int64_t now);
  void bulkAdd(const std::vector<Entry> &ents);
};

// ---------------------------------------------------------------------------------------------
// TypeConstraintManager
// ---------------------------------------------------------------------------------------------

Mtcp Tcm::fromInstanceSet(const std::vector<JStr> &requiredLabels, const std::vector<JStr> &preferredLabels,
                          const ClusterState &instances, bool hasStats, const std::vector<Isst *> &stats) {  // TCM:418-446
  bool haveReq = !requiredLabels.empty();
  IdSet required;
  OptSet preferred;
  for (const Entry &ent : instances) {
    const std::vector<JStr> &instanceLabels = ent.rec->labels;
    if (haveReq && instanceMatches(instanceLabels, requiredLabels, true)) {
      required.insert(ent.idx);
    } else if (instanceMatches(instanceLabels, preferredLabels, false)) {  // N11 else-if
      if (!preferred) preferred = IdSet();
      preferred->insert(ent.idx);
    }
  }
  auto m = std::make_shared<Mtc>();
  m->requiredLabels = requiredLabels;
  m->preferredLabels = preferredLabels;
  if (haveReq) m->allowedInstances = required;
  m->configuredPreferredInstances = preferred;
  m->preferredInstances = preferred;
  m->hasStats = hasStats;
  m->instanceSetStats = stats;
  return m;
}

Mtcp Tcm::updateInstance(const Mtcp &mtc, int32_t iid, const std::vector<JStr> &labels) {  // TCM:455-468
  OptSet newReq = mtc->allowedInstances;
  bool reqChanged = false, prefChanged = false;
  if (mtc->allowedInstances) {
    OptSet o;
    if (updateInstanceSet(iid, labels, mtc->requiredLabels, mtc->allowedInstances, true, o)) { newReq = o; reqChanged = true; }
  }
  OptSet newPref = mtc->configuredPreferredInstances;
  {
    OptSet o;
    if (updateInstanceSet(iid, labels, mtc->preferredLabels, mtc->configuredPreferredInstances, false, o)) { newPref = o; prefChanged = true; }
  }
  if (!reqChanged && !prefChanged) return mtc;
  auto m = std::make_shared<Mtc>();
  m->requiredLabels = mtc->requiredLabels;
  m->preferredLabels = mtc->preferredLabels;
  m->allowedInstances = newReq;
  m->configuredPreferredInstances = newPref;
  m->preferredInstances = newPref;  // resolved := configured until the next refresh
  m->hasStats = mtc->hasStats;
  m->instanceSetStats = mtc->instanceSetStats;
  return m;
}

// TCM:585-603; returns true when a new map was produced
bool Tcm::instanceUpdated(int32_t iid, const std::vector<JStr> &labels, const std::map<std::string, Mtcp> &mtcMap,
                          std::map<std::string, Mtcp> &newMap) {
  bool changed = false;
  for (auto &ent : mtcMap) {
    Mtcp newMtc = updateInstance(ent.second, iid, labels);
    if (newMtc != ent.second) {
      if (!changed) { newMap = mtcMap; changed = true; }
      newMap[ent.first] = newMtc;
    }
  }
  return changed;
}

// TCM:557-583
Isst *Tcm::getInstanceSetStats(int32_t iid, const std::vector<JStr> &labels, const std::map<std::string, Mtcp> &tcMap) {
  Isst *instanceSetStats = getStatsForLabels(labels);
  if (instanceSetStats == nullptr) {
    std::vector<std::string> newPts;
    for (auto &ent : tcMap)
      if (!ent.second->allowedOnInstance(iid)) newPts.push_back(ent.first);
    std::sort(newPts.begin(), newPts.end());  // java String order == byte order for the ASCII/BMP type names used
    auto pit = ptsToInstanceSetStats.find(newPts);
    if (pit != ptsToInstanceSetStats.end()) {
      instanceSetStats = pit->second;
    } else {
      ptsOwner.push_back(std::make_unique<Pts>());
      Pts *pts = ptsOwner.back().get();
      pts->types = newPts;
      pts->id = (int)ptsOwner.size();
      isstOwner.push_back(std::make_unique<Isst>(pts, &fleet->po));
      instanceSetStats = isstOwner.back().get();
      ptsToInstanceSetStats[newPts] = instanceSetStats;
      labelsToInstanceSetStats[labels] = instanceSetStats;
      if (iid == localInstanceId) localInstanceSetStats = instanceSetStats;
    }
  }
  return instanceSetStats;
}

// TCM:513-526
Isst *Tcm::instanceAdded(int32_t iid, const std::vector<JStr> &labels, bool /*includedInStats*/) {
  std::map<std::string, Mtcp> newMap;
  bool changed = instanceUpdated(iid, labels, typeConstraintsMap, newMap);
  Isst *instanceSetStats = getInstanceSetStats(iid, labels, changed ? newMap : typeConstraintsMap);
  if (changed) {
    if (!deferRefresh) refreshPerTypeInstanceSets(newMap);
    typeConstraintsMap = newMap;
  }
  return instanceSetStats;
}

// TCM:528-551
void Tcm::instanceRemoved(int32_t iid, const std::vector<JStr> &labels) {
  static const std::vector<JStr> NO_LABELS;
  std::map<std::string, Mtcp> newMap;
  bool changed = instanceUpdated(iid, NO_LABELS, typeConstraintsMap, newMap);
  Isst *instanceSetStats = getStatsForLabels(labels);
  if (instanceSetStats != nullptr) {
    if (instanceSetStats->count == 0) {
      labelsToInstanceSetStats.erase(labels);
      ptsToInstanceSetStats.erase(instanceSetStats->prohibitedTypesSet->types);
      if (changed) refreshPerTypeInstanceSets(newMap);
    }
  }
  if (changed) typeConstraintsMap = newMap;
}

// TCM:607-668
void Tcm::typeMappingsUpdated(std::map<std::string, ConfigTypeConstraints> newConfig) {
  const std::map<std::string, Mtcp> &mtcMap = typeConstraintsMap;
  std::map<std::string, Mtcp> newMap;
  bool haveNew = false;
  auto ensureNew = [&]() { if (!haveNew) { newMap = mtcMap; haveNew = true; } };
  for (auto &ent : mtcMap) {
    const std::string &typeName = ent.first;
    auto cit = newConfig.find(typeName);
    bool present = cit != newConfig.end();
    ConfigTypeConstraints tc;
    if (present) { tc = cit->second; newConfig.erase(cit); }
    if (!present || tc.isEmpty()) {
      ensureNew();
      newMap.erase(typeName);
    } else {
      const Mtcp &mtc = ent.second;
      if (!(mtc->requiredLabels == tc.required && mtc->preferredLabels == tc.preferred)) {
        ensureNew();
        newMap[typeName] = fromInstanceSet(tc.required, tc.preferred, fleet->clusterState, mtc->hasStats, mtc->instanceSetStats);
      }
    }
  }
  for (auto &ent : newConfig) {
    // (an empty config for a *new* type is logged as ignored but still inserted, TCM:641-649)
    ensureNew();
    newMap[ent.first] = fromInstanceSet(ent.second.required, ent.second.preferred, fleet->clusterState, false, {});
  }
  if (haveNew) {
    labelsToInstanceSetStats.clear();
    ptsToInstanceSetStats.clear();
    for (const Entry &ent : fleet->clusterState) {
      Isst *isst = getInstanceSetStats(ent.idx, ent.rec->labels, newMap);
      isst->add(*ent.rec);
      ent.rec->prohibitedTypes = isst->prohibitedTypesSet;
    }
    for (auto &e : ptsToInstanceSetStats) e.second->update();
    refreshPerTypeInstanceSets(newMap);
    typeConstraintsMap = newMap;
  }
}

// TCM:680-725
void Tcm::refreshPerTypeInstanceSets(std::map<std::string, Mtcp> &mtcMap) {
  std::map<int32_t, int32_t> instanceScores;
  for (const Entry &ent : fleet->clusterState)
    instanceScores[ent.idx] = (int32_t)(ent.rec->prohibitedTypes ? ent.rec->prohibitedTypes->types.size() : 0) * 4;
  for (auto &ent : mtcMap) {
    const OptSet &preferred = ent.second->configuredPreferredInstances;
    if (preferred)
      for (int32_t p : *preferred) {
        auto it = instanceScores.find(p);
        if (it != instanceScores.end()) it->second -= 1;
      }
  }
  OptSet defaultPreferred = inferPreferredInstances(instanceScores, nullptr);
  defaultPreferredInstances = defaultPreferred;

  for (auto &ent : mtcMap) {
    const Mtcp &mtc = ent.second;
    auto withStats = [&](bool hasStats, std::vector<Isst *> stats, const OptSet &newInferredPreferred) -> Mtcp {
      // updateInstanceSetStats TCM:389-408 (identity short-cuts do not change observable state)
      auto m = std::make_shared<Mtc>(*mtc);
      m->hasStats = hasStats;
      m->instanceSetStats = std::move(stats);
      m->preferredInstances = newInferredPreferred;
      return m;
    };
    if (!mtc->allowedInstances) {
      ent.second = withStats(false, {}, defaultPreferred);  // N11
    } else {
      std::vector<Isst *> statSet;
      for (auto &pts : ptsToInstanceSetStats)
        if (!std::binary_search(pts.first.begin(), pts.first.end(), ent.first)) statSet.push_back(pts.second);
      OptSet inferredPreferred = (mtc->configuredPreferredInstances || mtc->allowedInstances->empty())
                                     ? mtc->preferredInstances
                                     : inferPreferredInstances(instanceScores, &*mtc->allowedInstances);
      ent.second = withStats(true, statSet, inferredPreferred);
    }
  }
}

// TCM:727-747
OptSet Tcm::inferPreferredInstances(const std::map<int32_t, int32_t> &instanceScores, const IdSet *include) {
  IdSet instanceIds;
  int32_t min = INT32_MAX, max = 0;
  for (auto &ent : instanceScores) {
    if (include != nullptr && !include->count(ent.first)) continue;
    int32_t score = ent.second;
    if (score < min) min = score;
    if (score >= max) {
      if (score > max) { instanceIds.clear(); max = score; }
      instanceIds.insert(ent.first);
    }
  }
  if (min < max) return instanceIds;
  return std::nullopt;
}

// ---------------------------------------------------------------------------------------------
// handleInstanceTableChange MM:1455-1568
// ---------------------------------------------------------------------------------------------
void Fleet::instanceEvent(int type, int32_t idx, const JStr &key, IRp record, int64_t now) {
  enum { ENTRY_ADDED = 0, ENTRY_UPDATED = 1, ENTRY_DELETED = 2 };
  const bool stays_in_table = type != ENTRY_DELETED && record != nullptr;
  Isst *subsetStats = nullptr;
  if (record) {
    if (record->shuttingDown) type = ENTRY_DELETED;
    if (haveTc) subsetStats = tcm.getStatsForLabels(record->labels);
  }
  bool wasAddedToTc = false;
  bool haveKeep = false;
  Entry keep;
  if (type == ENTRY_ADDED || type == ENTRY_UPDATED) {
    if (!record) return;
    if (haveTc) {
      if (type == ENTRY_ADDED || subsetStats == nullptr) {
        subsetStats = tcm.instanceAdded(idx, record->labels, false);
        wasAddedToTc = true;
      }
      record->prohibitedTypes = subsetStats->prohibitedTypesSet;
    }
    keep = Entry{key, idx, record};
    haveKeep = true;
    bool added = clusterState.insert(keep).second;
    if (!added) return;  // identical record already present
    clusterStatsTracker.add(*record);
    if (subsetStats != nullptr) subsetStats->add(*record);
  }
  // fall-thru / ENTRY_DELETED
  clusterStatsTracker.resetLru();
  if (subsetStats != nullptr) subsetStats->resetLru();
  bool existingWasRemoved = false;
  for (auto it = clusterState.begin(); it != clusterState.end();) {
    const Entry &ent = *it;
    IRp ir = ent.rec;
    if (key == ent.key && (!haveKeep || po.compare(ent, keep) != 0)) {
      clusterStatsTracker.remove(*ir);
      if (haveTc) {
        if (subsetStats != nullptr) subsetStats->remove(*ir);
        if (type == ENTRY_DELETED) tcm.instanceRemoved(idx, ir->labels);
      }
      if (type == ENTRY_DELETED) upgradeTracker.instanceRemoved(key, *ir, now);
      existingWasRemoved = true;
      it = clusterState.erase(it);
    } else {
      clusterStatsTracker.addLru(ir->lruTime);
      if (subsetStats != nullptr) subsetStats->addLru(ir->lruTime);  // N10: over all instances
      ++it;
    }
  }
  if (haveTc) {
    if (type != ENTRY_DELETED && !wasAddedToTc && !existingWasRemoved) tcm.instanceAdded(idx, record->labels, true);
    if (subsetStats != nullptr) subsetStats->update();
  }
  // NOTE MM:1552: upgradeTracker.instanceAdded only when an existing record was replaced
  if (type != ENTRY_DELETED && existingWasRemoved) upgradeTracker.instanceAdded(key, *record, now);
  clusterStats = clusterStatsTracker.update();
  if ((changeCounter++ & 63) == 0) upgradeTracker.doHousekeeping(now);

  if ((size_t)idx >= byIdx.size()) { byIdx.resize(idx + 1); keyByIdx.resize(idx + 1); siActive.resize(idx + 1, 0); }
  if ((size_t)idx >= inTable.size()) inTable.resize(idx + 1, 0);
  inTable[idx] = stays_in_table ? 1 : 0;
  keyByIdx[idx] = key;
  if (type == ENTRY_DELETED) byIdx[idx] = nullptr; else byIdx[idx] = record;
}

// Test-harness shortcut: the state that ENTRY_ADDED events for `ents` (fresh keys, empty fleet, type config already
// set, refresh deferred) followed by a converged refresh produce, computed without the per-event O(N) rescans of
// MM:1522-1542 and the per-event immutable-set rebuilds of TCM:489-505.  tests/test_host_logic.py checks it against the
// event-driven path; it exists only so that 40k-65k instance fleets can be set up in seconds.
void Fleet::bulkAdd(const std::vector<Entry> &ents) {
  if (haveTc) {
    std::map<std::string, Mtcp> newMap;
    for (auto &te : tcm.typeConstraintsMap) {
      auto m = std::make_shared<Mtc>(*te.second);
      if (!m->requiredLabels.empty() && !m->allowedInstances) m->allowedInstances = IdSet();
      for (const Entry &e : ents) {
        if (e.rec->shuttingDown) continue;  // MM:1462-1464: never reaches TypeConstraintManager.instanceAdded
        if (m->allowedInstances && instanceMatches(e.rec->labels, m->requiredLabels, true)) m->allowedInstances->insert(e.idx);
        if (instanceMatches(e.rec->labels, m->preferredLabels, false)) {
          if (!m->configuredPreferredInstances) m->configuredPreferredInstances = IdSet();
          m->configuredPreferredInstances->insert(e.idx);
        }
      }
      m->preferredInstances = m->configuredPreferredInstances;
      newMap[te.first] = m;
    }
    tcm.typeConstraintsMap = newMap;
  }
  int32_t maxIdx = -1;
  for (const Entry &e : ents) maxIdx = std::max(maxIdx, e.idx);
  if ((size_t)(maxIdx + 1) > byIdx.size()) { byIdx.resize(maxIdx + 1); keyByIdx.resize(maxIdx + 1); siActive.resize(maxIdx + 1, 0); }
  for (const Entry &e : ents) {
    if (e.rec->shuttingDown) { keyByIdx[e.idx] = e.key; continue; }  // treated as a deletion of an absent key: no-op
    Isst *ss = nullptr;
    if (haveTc) {
      ss = tcm.getInstanceSetStats(e.idx, e.rec->labels, tcm.typeConstraintsMap);
      e.rec->prohibitedTypes = ss->prohibitedTypesSet;
      ss->add(*e.rec);
    }
    clusterState.insert(e);
    clusterStatsTracker.add(*e.rec);
    byIdx[e.idx] = e.rec; keyByIdx[e.idx] = e.key;
  }
  clusterStatsTracker.resetLru();
  for (auto &ps : tcm.ptsToInstanceSetStats) ps.second->resetLru();
  for (const Entry &e : clusterState) {
    clusterStatsTracker.addLru(e.rec->lruTime);
    for (auto &ps : tcm.ptsToInstanceSetStats) ps.second->addLru(e.rec->lruTime);  // N10
  }
  for (auto &ps : tcm.ptsToInstanceSetStats) ps.second->update();
  clusterStats = clusterStatsTracker.update();
  if (haveTc) {
    std::map<std::string, Mtcp> m = tcm.typeConstraintsMap;
    tcm.refreshPerTypeInstanceSets(m);
    tcm.typeConstraintsMap = m;
  }
}

// ---------------------------------------------------------------------------------------------
// CacheMissForwardingLB.getNext MM:4776-5004
// ---------------------------------------------------------------------------------------------
struct ExcludeSet {  // CacheMissExcludeSet MM:4717-4749, as the union of its four member sets
  const int32_t *ids; int64_t n;
  bool isExcluded(int32_t iid) const { for (int64_t i = 0; i < n; i++) if (ids[i] == iid) return true; return false; }
};

struct GetNextOut {
  int32_t target = ORC_NONE, nCandidates = 0, nRemaining = 0, pickIndex = 0, best = -1, flags = 0;
  std::vector<int32_t> candidates, instReqLoad;
  std::vector<uint8_t> keep;
};

// Iterators.filter(clusterState.iterator(), pred) or a replay list iterator
struct EntIter {
  ClusterState::const_iterator cur, end;
  const std::vector<const Entry *> *list = nullptr;
  size_t li = 0;
  const Fleet *f; const OptSet *constrainTo; const ExcludeSet *exclude; bool useReplicaSets;
  const Entry *peeked = nullptr;
  // CPU-baseline mode (ii) "dense" (BASELINE.md §4): the same filtered iteration over a rank-ordered ARRAY of the entries
  // (built once per batch) instead of the ordered set's tree walk
  const std::vector<const Entry *> *dense = nullptr;
  size_t di = 0;
  bool pred(const Entry &ent) const {  // MM:4763-4770
    int32_t iid = ent.idx;
    if ((*constrainTo && !(*constrainTo)->count(iid)) || exclude->isExcluded(iid) ||
        !((size_t)iid < f->siActive.size() && f->siActive[iid]))
      return false;
    if (!useReplicaSets || f->upgradeTracker.likelyReplacedReplicaSets.empty() || ent.key.size() < 7) return true;
    return !f->upgradeTracker.likelyReplacedReplicaSets.count(ent.key.substr(0, 6));
  }
  bool hasNext() {
    if (list) return li < list->size();
    if (peeked) return true;
    if (dense) {
      while (di < dense->size()) {
        const Entry *e = (*dense)[di++];
        if (pred(*e)) { peeked = e; return true; }
      }
      return false;
    }
    while (cur != end) {
      const Entry &e = *cur;
      ++cur;
      if (pred(e)) { peeked = &e; return true; }
    }
    return false;
  }
  const Entry *next() {
    if (list) return (*list)[li++];
    hasNext();
    const Entry *e = peeked;
    peeked = nullptr;
    return e;
  }
  void rewindTo(const std::vector<const Entry *> *l) { list = l; li = 0; }
};

static const int64_t TWELVE_MIN_MS = 12LL * 60000, ONE_DAY_MS = 86400000LL, FIVE_DAYS_MS = 5 * 86400000LL;

inline int64_t age(int64_t t, int64_t now) { return t == 0 ? 0 : jsub(now, t); }  // MM:4162-4164

void getNext(const Fleet &f, const std::string &modelType, int32_t self, const IR &fresh, bool favourSelf,
             int64_t lastUsedTime, const ExcludeSet &exclude, int64_t now, uint64_t rnd, GetNextOut &o,
             const std::vector<const Entry *> *dense = nullptr) {
  const bool excludeSelf = exclude.isExcluded(self);
  static const OptSet NULLSET;
  const OptSet *constrainTo = f.haveTc ? f.tcm.getCandidateInstances(modelType) : &NULLSET;
  const bool rsEmpty = f.upgradeTracker.likelyReplacedReplicaSets.empty();

  EntIter it{f.clusterState.begin(), f.clusterState.end(), nullptr, 0, &f, constrainTo, &exclude, true, nullptr, dense, 0};
  if (!it.hasNext()) {
    if (rsEmpty) return;  // null
    o.flags |= 1;
    it = EntIter{f.clusterState.begin(), f.clusterState.end(), nullptr, 0, &f, constrainTo, &exclude, false, nullptr, dense, 0};
    if (!it.hasNext()) return;
  }
  const Entry *bestEntry = it.next();
  int32_t bestIid = bestEntry->idx;
  bool us = !excludeSelf && self == bestIid;
  const IR *bestInst = us ? &fresh : bestEntry->rec.get();
  const bool bestIsFull = f.isFull(bestInst->getRemaining());
  if (bestIsFull) o.flags |= 4;

  std::vector<int32_t> &candidates = o.candidates, &instReqLoad = o.instReqLoad;
  candidates.clear(); instReqLoad.clear();

  const OptSet *prefer = f.haveTc ? f.tcm.getPreferredInstances(modelType) : &NULLSET;
  auto preferContains = [&](int32_t iid) { return (*prefer)->count(iid) != 0; };

  bool simpleCase = !*prefer || preferContains(bestIid);
  std::vector<const Entry *> clusterStateReplay;
  bool replayNull = false;  // clusterStateReplay = null
  if (!simpleCase) {
    if (!bestIsFull) {
      // Non-simple case (a)  MM:4828-4852
      bool found = false;
      while (it.hasNext()) {
        const Entry *ent = it.next();
        if (preferContains(ent->idx)) {
          found = true;
          bestIid = ent->idx;
          bestInst = ent->rec.get();
          us = !us && !excludeSelf && self == bestIid;
          break;
        }
        if (f.isFull(ent->rec->getRemaining())) break;
        clusterStateReplay.push_back(ent);
      }
      if (!found) { it.rewindTo(&clusterStateReplay); prefer = &NULLSET; }
      simpleCase = true;
    } else {
      // Non-simple case (b)  MM:4853-4887
      int64_t oldest = bestInst->lruTime;
      while (it.hasNext()) {
        const Entry *ent = it.next();
        int32_t iid = ent->idx;
        const IR *curInst = ent->rec.get();
        int64_t diff = jsub(curInst->lruTime, oldest);
        if (diff > 120000 && diff > jdiv(age(oldest, now), 4)) break;
        if (preferContains(iid)) {
          us = !us && !excludeSelf && self == iid;
          if (us && favourSelf) { o.flags |= 8; o.best = bestIid; return; }  // N8: returns null
          replayNull = true;
          candidates.push_back(iid);
          instReqLoad.push_back(curInst->rpm);
        } else if (!replayNull) {
          clusterStateReplay.push_back(ent);
        }
      }
      if (!replayNull) { it.rewindTo(&clusterStateReplay); prefer = &NULLSET; simpleCase = true; }
    }
  }
  o.best = bestIid;
  if (simpleCase) {
    o.flags |= 2;
    if (us && favourSelf) { o.flags |= 8; o.target = ORC_SELF; return; }
    candidates.push_back(bestIid);
    instReqLoad.push_back(bestInst->rpm);
    const int64_t oldest = bestInst->lruTime;
    while (it.hasNext()) {
      const Entry *ent = it.next();
      int32_t iid = ent->idx;
      if (*prefer && !preferContains(iid)) continue;
      us = !us && !excludeSelf && self == iid;
      const IR *curInst = us ? bestEntry->rec.get() : &fresh;  // N2
      if (bestIsFull) {
        int64_t diff = jsub(curInst->lruTime, oldest);
        if (diff > 45000 && diff > jdiv(age(oldest, now), 10)) break;
      } else {
        int64_t rem = curInst->getRemaining();
        if (f.isFull(rem) || rem < (bestInst->getRemaining() >> 2)) break;
        int32_t count = ent->rec->count, firstCount = bestInst->count;
        if (count >= 10 && count > jaddi(firstCount, firstCount >> 2)) break;
      }
      if (us && favourSelf) { o.flags |= 8; o.target = ORC_SELF; return; }
      candidates.push_back(iid);
      instReqLoad.push_back(curInst->rpm);
    }
  }

  const int ccount = (int)candidates.size();
  o.nCandidates = ccount;
  o.keep.assign(ccount, 1);
  if (ccount == 0) return;  // null
  const int64_t lastUsedAgo = age(lastUsedTime, now);
  int32_t chosen = -1;
  if (ccount == 1) {
    chosen = candidates[0];
    o.nRemaining = 1; o.pickIndex = 0;
  } else {
    int remainingCount = ccount;
    if (lastUsedAgo < FIVE_DAYS_MS) {
      int32_t minRpm = *std::min_element(instReqLoad.begin(), instReqLoad.end());
      int32_t minLoad = std::max(100, minRpm);
      int32_t minLoad_1_1 = jd2i(1.1 * minLoad), minLoad_1_5 = jd2i(1.5 * minLoad);
      for (int i = 0; i < ccount; i++) {
        int32_t rpm = instReqLoad[i];
        if (rpm >= 100 && ((lastUsedAgo < -1000 && rpm > minLoad_1_1) || (lastUsedAgo < 5000 && rpm > minLoad_1_5) ||
                           (lastUsedAgo < TWELVE_MIN_MS && rpm > jmuli(minLoad, 3)) ||
                           (lastUsedAgo < ONE_DAY_MS && rpm > jmuli(minLoad, 4)))) {
          o.keep[i] = 0;
          remainingCount--;
          if (remainingCount == 1) break;
        }
      }
    }
    int index = remainingCount == 1 ? 0 : (int)(((rnd >> 32) * (uint64_t)remainingCount) >> 32);  // N4
    for (int i = 0, j = 0; i < ccount; i++) {
      if (o.keep[i]) { chosen = candidates[i]; if (index == j++) break; }
      else chosen = -1;
    }
    o.nRemaining = remainingCount; o.pickIndex = index;
  }
  if (!favourSelf && self == chosen) { o.target = ORC_SELF; return; }
  o.target = chosen;
}

// ---------------------------------------------------------------------------------------------
// Time-ordered weighted LRU: CLHM + LinkedDeque, single-threaded (reads drain immediately, see
// drainOnReadIfNeeded CLHM:425-431: a lone reader always finds the buffer below threshold and IDLE)
// ---------------------------------------------------------------------------------------------
struct Lru {
  struct Node { int32_t key; int64_t weight; int64_t lastUsed; bool alive; };
  typedef std::list<Node>::iterator NodeIt;
  std::list<Node> deque;   // evictionDeque, head = oldest
  std::list<Node> limbo;   // nodes in `data` but not linked (never happens single-threaded; kept for symmetry)
  std::unordered_map<int32_t, NodeIt> data;
  int64_t capacity, weightedSize = 0, oldestTime = -1;
  std::vector<orc_eviction_t> pendingNotifications;
  explicit Lru(int64_t cap) : capacity(cap) {}

  // LD:258-288 insert: walk from the tail to the last element with lastUsed <= ts, link after it
  void insert(NodeIt src_list_it, std::list<Node> &src) {
    int64_t ts = src_list_it->lastUsed;
    auto pos = deque.end();
    while (pos != deque.begin()) {
      auto prev = std::prev(pos);
      if (prev->lastUsed <= ts) break;
      pos = prev;
    }
    deque.splice(pos, src, src_list_it);
  }
  void reposition(NodeIt e) {  // LD:243-255
    int64_t lu = e->lastUsed;
    bool prevOk = (e == deque.begin()) || (std::prev(e)->lastUsed <= lu);
    if (prevOk) {
      auto nx = std::next(e);
      if (nx == deque.end() || nx->lastUsed >= lu) return;
    }
    std::list<Node> tmp;
    tmp.splice(tmp.begin(), deque, e);
    insert(tmp.begin(), tmp);
  }
  void evict(int32_t evIndex) {  // CLHM:329-352
    while (weightedSize > capacity) {
      if (deque.empty()) return;
      Node n = deque.front();
      deque.pop_front();
      weightedSize -= std::llabs(n.weight);  // makeDead
      data.erase(n.key);
      pendingNotifications.push_back(orc_eviction_t{n.key, evIndex, n.lastUsed, n.weight});
    }
  }
  void updateOldestTime() { oldestTime = deque.empty() ? -1 : deque.front().lastUsed; }  // CLHM:1129-1133
  static void touch(Node &n, int64_t time, int64_t now) { n.lastUsed = time == 0 ? now : std::max(n.lastUsed, time); }  // CLHM:1357-1360
  void notify(std::vector<orc_eviction_t> &out) {
    for (auto &e : pendingNotifications) out.push_back(e);
    pendingNotifications.clear();
  }
  void afterRead(NodeIt n, int64_t lastUsed, int64_t now) {  // CLHM:383-388 + drainReadBuffer 477-505
    touch(*n, lastUsed > 0 ? lastUsed : 0, now);
    reposition(n);  // applyRead: node is linked
    updateOldestTime();
  }
  void apply(const orc_lru_event_t &ev, int32_t evIndex, int64_t now, std::vector<orc_eviction_t> &out) {
    auto it = data.find(ev.key);
    switch (ev.op) {
      case 0: {  // putIfAbsent(key, value, lastUsed)  CLHM:821-836
        if (it == data.end()) {
          std::list<Node> tmp;
          Node n{ev.key, ev.weight, 0, true};
          touch(n, ev.last_used, now);
          tmp.push_back(n);
          data[ev.key] = tmp.begin();
          // AddTask CLHM:601-610
          weightedSize += ev.weight;
          insert(tmp.begin(), tmp);
          evict(evIndex);
          updateOldestTime();
          notify(out);
        } else {
          afterRead(it->second, ev.last_used, now);
        }
        break;
      }
      case 1:  // get(key, lastUsed) CLHM:731-738
        if (it != data.end()) afterRead(it->second, ev.last_used, now);
        break;
      case 2: {  // replaceQuietly with a new weight: UpdateTask(node, diff, -1)  CLHM:963-984, 631-652
        if (it == data.end()) break;
        int64_t diff = ev.weight - it->second->weight;
        it->second->weight = ev.weight;
        if (diff != 0) {
          weightedSize += diff;
          evict(evIndex);
          updateOldestTime();
          if (diff > 0) notify(out);
        }
        break;
      }
      case 3: {  // remove(key) CLHM:860-871: RemovalTask, no notification
        if (it == data.end()) break;
        weightedSize -= std::llabs(it->second->weight);
        deque.erase(it->second);
        data.erase(it);
        updateOldestTime();
        break;
      }
      case 4:  // setCapacity CLHM:305-316
        capacity = ev.weight;
        evict(evIndex);
        notify(out);
        break;  // (oldestTime is not refreshed by setCapacity in the reference)
      case 5:  // forceSetLastUsedTime CLHM:756-768: no reposition
        if (it != data.end()) it->second->lastUsed = ev.last_used;
        break;
    }
  }
};

}  // namespace

// ---------------------------------------------------------------------------------------------
// C API
// ---------------------------------------------------------------------------------------------
struct orc_fleet { Fleet f; orc_fleet(int64_t a, int64_t b, int32_t c) : f(a, b, c) {} };
struct orc_lru { Lru l; explicit orc_lru(int64_t c) : l(c) {} };

static void fillStats(const ClusterStats &s, orc_stats_t *o) {
  o->total_capacity = s.totalCapacity; o->total_free = s.totalFree; o->global_lru = s.globalLru;
  o->instance_count = s.instanceCount; o->model_copy_count = s.modelCopyCount;
}

extern "C" {

uint64_t orc_hash64(uint64_t seed, uint64_t decision_id) {  // SplitMix64 finaliser of a Weyl sequence
  uint64_t z = seed + 0x9E3779B97F4A7C15ULL * (decision_id + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
  return z ^ (z >> 31);
}

orc_fleet *orc_create(int64_t min_space_units, int64_t min_churn_age_ms, int32_t default_model_size_units) {
  return new orc_fleet(min_space_units, min_churn_age_ms, default_model_size_units);
}
void orc_destroy(orc_fleet *h) { delete h; }

int orc_instance_event(orc_fleet *h, int type, int32_t idx, const orc_inst_t *rec, const char *id, const char *loc,
                       const char *zone, const char *const *labels, int32_t n_labels, int64_t now_ms) {
  if (!h || idx < 0 || !id) return -1;
  Fleet &f = h->f;
  IRp r;
  if (rec) {
    r = std::make_shared<IR>();
    r->lruTime = rec->lru_time; r->count = rec->count; r->capacity = rec->capacity; r->used = rec->used;
    r->lThreads = rec->l_threads; r->lInProg = rec->l_in_prog; r->rpm = rec->rpm; r->shuttingDown = rec->shutting_down != 0;
    r->startTime = rec->start_time; r->vers = rec->vers;
    if (loc) { r->hasLoc = true; r->loc = utf8to16(loc); }
    if (zone) { r->hasZone = true; r->zone = utf8to16(zone); }
    for (int i = 0; i < n_labels; i++) r->labels.push_back(utf8to16(labels[i]));
    std::sort(r->labels.begin(), r->labels.end(), [](const JStr &a, const JStr &b) { return jcompare(a, b) < 0; });  // IR:90-91
    r->labelsIdentity = r->labels.empty() ? 0 : f.nextLabelsIdentity++;
  }
  f.instanceEvent(type, idx, utf8to16(id), r, now_ms);
  if (rec && (size_t)idx < f.siActive.size()) f.siActive[idx] = rec->active ? 1 : 0;
  return 0;
}

int orc_bulk_add(orc_fleet *h, int32_t n, const orc_inst_t *recs, const char *const *ids, const char *const *locs,
                 const char *const *zones, const int32_t *label_off, const char *const *labels) {
  if (!h || n < 0 || !h->f.clusterState.empty()) return -1;
  Fleet &f = h->f;
  std::vector<Entry> ents;
  for (int32_t i = 0; i < n; i++) {
    auto r = std::make_shared<IR>();
    const orc_inst_t *rec = &recs[i];
    r->lruTime = rec->lru_time; r->count = rec->count; r->capacity = rec->capacity; r->used = rec->used;
    r->lThreads = rec->l_threads; r->lInProg = rec->l_in_prog; r->rpm = rec->rpm; r->shuttingDown = rec->shutting_down != 0;
    r->startTime = rec->start_time; r->vers = rec->vers;
    if (locs[i]) { r->hasLoc = true; r->loc = utf8to16(locs[i]); }
    if (zones[i]) { r->hasZone = true; r->zone = utf8to16(zones[i]); }
    for (int k = label_off[i]; k < label_off[i + 1]; k++) r->labels.push_back(utf8to16(labels[k]));
    std::sort(r->labels.begin(), r->labels.end(), [](const JStr &a, const JStr &b) { return jcompare(a, b) < 0; });
    r->labelsIdentity = r->labels.empty() ? 0 : f.nextLabelsIdentity++;
    ents.push_back(Entry{utf8to16(ids[i]), i, r});
  }
  f.bulkAdd(ents);
  for (int32_t i = 0; i < n; i++) f.siActive[i] = recs[i].active ? 1 : 0;
  return 0;
}

int orc_set_active(orc_fleet *h, int32_t idx, int32_t active) {
  if (!h || idx < 0 || (size_t)idx >= h->f.siActive.size()) return -1;
  h->f.siActive[idx] = active ? 1 : 0;
  return 0;
}

int orc_types_set(orc_fleet *h, int32_t n, const char *const *names, const int32_t *req_off, const char *const *req_labels,
                  const int32_t *pref_off, const char *const *pref_labels) {
  if (!h) return -1;
  Fleet &f = h->f;
  if (n < 0) { f.haveTc = false; return 0; }
  f.haveTc = true;
  std::map<std::string, ConfigTypeConstraints> cfg;
  for (int t = 0; t < n; t++) {
    std::vector<JStr> req, pref;
    for (int i = req_off[t]; i < req_off[t + 1]; i++) req.push_back(utf8to16(req_labels[i]));
    for (int i = pref_off[t]; i < pref_off[t + 1]; i++) pref.push_back(utf8to16(pref_labels[i]));
    ConfigTypeConstraints c;  // TCM:91-94
    c.required = sortAndDeduplicate(req, nullptr);
    c.preferred = sortAndDeduplicate(pref, &c.required);
    cfg[names[t]] = c;
  }
  f.tcm.typeMappingsUpdated(cfg);
  return 0;
}

int orc_tc_defer_refresh(orc_fleet *h, int defer) {
  if (!h) return -1;
  h->f.tcm.deferRefresh = defer != 0;
  return 0;
}

int orc_tc_converge(orc_fleet *h) {
  if (!h || !h->f.haveTc) return -1;
  std::map<std::string, Mtcp> m = h->f.tcm.typeConstraintsMap;
  h->f.tcm.refreshPerTypeInstanceSets(m);
  h->f.tcm.typeConstraintsMap = m;
  return 0;
}

int orc_set_replaced_replicasets(orc_fleet *h, const char *const *prefixes, int32_t n) {
  if (!h) return -1;
  h->f.upgradeTracker.likelyReplacedReplicaSets.clear();
  for (int i = 0; i < n; i++) h->f.upgradeTracker.likelyReplacedReplicaSets[utf8to16(prefixes[i])] = INT64_MAX;
  return 0;
}
int orc_get_replaced_replicasets(orc_fleet *h, char *buf, int32_t cap) {
  if (!h) return -1;
  std::string s;
  int n = 0;
  for (auto &e : h->f.upgradeTracker.likelyReplacedReplicaSets) { if (n++) s += ","; s += u16to8(e.first); }
  if (buf && cap > 0) { strncpy(buf, s.c_str(), cap - 1); buf[cap - 1] = 0; }
  return n;
}

int orc_type_sets(orc_fleet *h, const char *type, int32_t n_idx, uint8_t *allowed, int32_t *allowed_null,
                  uint8_t *preferred, int32_t *preferred_null) {
  if (!h) return -1;
  Fleet &f = h->f;
  static const OptSet NULLSET;
  const OptSet *a = f.haveTc ? f.tcm.getCandidateInstances(type) : &NULLSET;
  const OptSet *p = f.haveTc ? f.tcm.getPreferredInstances(type) : &NULLSET;
  *allowed_null = !*a; *preferred_null = !*p;
  for (int i = 0; i < n_idx; i++) {
    allowed[i] = *a ? ((*a)->count(i) ? 1 : 0) : 0;
    preferred[i] = *p ? ((*p)->count(i) ? 1 : 0) : 0;
  }
  return 0;
}

int orc_cluster_order(orc_fleet *h, int32_t *out_idx, int32_t cap) {
  if (!h) return -1;
  int n = 0;
  for (const Entry &e : h->f.clusterState) { if (n < cap) out_idx[n] = e.idx; n++; }
  return n;
}

int orc_compare(orc_fleet *h, int32_t idx1, int32_t idx2) {
  Fleet &f = h->f;
  Entry a{f.keyByIdx[idx1], idx1, f.byIdx[idx1]}, b{f.keyByIdx[idx2], idx2, f.byIdx[idx2]};
  return f.po.compare(a, b);
}

int orc_cluster_stats(orc_fleet *h, orc_stats_t *out) { if (!h) return -1; fillStats(h->f.clusterStats, out); return 0; }

int orc_partition_stats(orc_fleet *h, orc_stats_t *out, int32_t *part_ids, int32_t cap) {
  if (!h) return -1;
  Tcm &t = h->f.tcm;
  std::vector<Isst *> result;
  for (auto &e : t.ptsToInstanceSetStats) result.push_back(e.second);
  // PARTITION_STATS_COMP TCM:264-271 (stable sort like List.sort)
  std::stable_sort(result.begin(), result.end(), [](Isst *a, Isst *b) {
    const ClusterStats &c1 = a->currentStats, &c2 = b->currentStats;
    if (c1.totalFree != c2.totalFree) return c2.totalFree < c1.totalFree;
    if (c1.globalLru != c2.globalLru) return c1.globalLru < c2.globalLru;
    return c2.totalCapacity < c1.totalCapacity;
  });
  int n = 0;
  for (Isst *i : result) { if (n < cap) { fillStats(i->currentStats, &out[n]); part_ids[n] = i->prohibitedTypesSet->id; } n++; }
  return n;
}
int orc_instance_partition(orc_fleet *h, int32_t idx) {
  Fleet &f = h->f;
  if ((size_t)idx >= f.byIdx.size() || !f.byIdx[idx] || !f.byIdx[idx]->prohibitedTypes) return -1;
  return f.byIdx[idx]->prohibitedTypes->id;
}
int orc_type_stats(orc_fleet *h, const char *type, orc_stats_t *out) {  // MM:1432-1438 + TCM:223-226, 356-376
  Fleet &f = h->f;
  if (!f.haveTc) { fillStats(f.clusterStats, out); return 0; }
  auto it = f.tcm.typeConstraintsMap.find(type);
  if (it == f.tcm.typeConstraintsMap.end() || !it->second->hasStats) { fillStats(f.clusterStats, out); return 0; }
  const Mtc &m = *it->second;
  if (m.instanceSetStats.size() == 1) { fillStats(m.instanceSetStats[0]->currentStats, out); return 0; }
  ClusterStats s; s.globalLru = INT64_MAX;
  for (Isst *is : m.instanceSetStats) {
    const ClusterStats &sub = is->currentStats;
    s.totalCapacity = jadd(s.totalCapacity, sub.totalCapacity); s.totalFree = jadd(s.totalFree, sub.totalFree);
    s.instanceCount += sub.instanceCount; s.modelCopyCount += sub.modelCopyCount;
    if (sub.globalLru < s.globalLru) s.globalLru = sub.globalLru;
  }
  fillStats(s, out);
  return 0;
}

static int64_t get_next_batch_impl(orc_fleet *h, int32_t n, const orc_decision_t *dec, const char *const *type_names, int32_t n_types,
                           const orc_inst_t *fresh, int32_t n_fresh, const int64_t *excl_off, const int32_t *excl_idx,
                           int64_t now_ms, uint64_t seed, int32_t threads, orc_result_t *out, int64_t *cand_off,
                           int32_t *cand_idx, int32_t *cand_load, uint8_t *cand_keep, int64_t cand_cap, bool dense_mode) {
  if (!h || n < 0) return -1;
  const Fleet &f = h->f;
  std::vector<const Entry *> dense_order;
  if (dense_mode) for (const Entry &e : f.clusterState) dense_order.push_back(&e);
  const std::vector<const Entry *> *dense = dense_mode ? &dense_order : nullptr;
  std::vector<std::string> tnames;
  for (int i = 0; i < n_types; i++) tnames.push_back(type_names[i]);
  static const std::string NOTYPE = "\x01<no-config>";
  const bool wantCands = cand_off != nullptr;
  if (threads < 1) threads = 1;
  if (wantCands) threads = 1;  // candidate lists are written sequentially
  std::atomic<int> bad{0};
  int64_t candPos = 0;
  auto work = [&](int lo, int hi) {
    GetNextOut o;
    for (int i = lo; i < hi; i++) {
      const orc_decision_t &d = dec[i];
      if (d.self < 0 || (size_t)d.self >= f.byIdx.size()) { bad = 1; continue; }
      IR freshRec;
      if (d.fresh_idx >= 0 && d.fresh_idx < n_fresh) {
        const orc_inst_t &r = fresh[d.fresh_idx];
        freshRec.lruTime = r.lru_time; freshRec.count = r.count; freshRec.capacity = r.capacity; freshRec.used = r.used;
        freshRec.lThreads = r.l_threads; freshRec.lInProg = r.l_in_prog; freshRec.rpm = r.rpm;
        freshRec.shuttingDown = r.shutting_down != 0; freshRec.startTime = r.start_time; freshRec.vers = r.vers;
      } else {
        if (!f.byIdx[d.self]) { bad = 1; continue; }
        freshRec = *f.byIdx[d.self];
        freshRec.rpm = 0;  // N7
      }
      ExcludeSet ex{excl_idx + excl_off[i], excl_off[i + 1] - excl_off[i]};
      const std::string &type = (d.type_idx >= 0 && d.type_idx < n_types) ? tnames[d.type_idx] : NOTYPE;
      o = GetNextOut();
      getNext(f, type, d.self, freshRec, d.favour_self != 0, d.last_used, ex, now_ms, orc_hash64(seed, d.decision_id), o, dense);
      out[i].target = o.target; out[i].n_candidates = o.nCandidates; out[i].n_remaining = o.nRemaining;
      out[i].pick_index = o.pickIndex; out[i].best = o.best; out[i].flags = o.flags;
      if (wantCands) {
        cand_off[i] = candPos;
        for (size_t k = 0; k < o.candidates.size() && (int)k < o.nCandidates; k++) {
          if (candPos < cand_cap) { cand_idx[candPos] = o.candidates[k]; cand_load[candPos] = o.instReqLoad[k]; cand_keep[candPos] = o.keep[k]; }
          candPos++;
        }
      }
    }
  };
  if (threads == 1) {
    work(0, n);
  } else {
    std::vector<std::thread> th;
    int per = (n + threads - 1) / threads;
    for (int t = 0; t < threads; t++) {
      int lo = t * per, hi = std::min(n, lo + per);
      if (lo < hi) th.emplace_back(work, lo, hi);
    }
    for (auto &t : th) t.join();
  }
  if (wantCands) cand_off[n] = candPos;
  if (bad) return -2;
  return candPos;
}

int64_t orc_get_next_batch(orc_fleet *h, int32_t n, const orc_decision_t *dec, const char *const *type_names, int32_t n_types,
                           const orc_inst_t *fresh, int32_t n_fresh, const int64_t *excl_off, const int32_t *excl_idx,
                           int64_t now_ms, uint64_t seed, int32_t threads, orc_result_t *out, int64_t *cand_off,
                           int32_t *cand_idx, int32_t *cand_load, uint8_t *cand_keep, int64_t cand_cap) {
  return get_next_batch_impl(h, n, dec, type_names, n_types, fresh, n_fresh, excl_off, excl_idx, now_ms, seed, threads, out, cand_off, cand_idx,
                             cand_load, cand_keep, cand_cap, false);
}
/* CPU-baseline mode (ii) "dense" (BASELINE.md §4): same decisions, entries walked through a rank-ordered array */
int64_t orc_get_next_batch_dense(orc_fleet *h, int32_t n, const orc_decision_t *dec, const char *const *type_names, int32_t n_types,
                                 const orc_inst_t *fresh, int32_t n_fresh, const int64_t *excl_off, const int32_t *excl_idx,
                                 int64_t now_ms, uint64_t seed, int32_t threads, orc_result_t *out) {
  return get_next_batch_impl(h, n, dec, type_names, n_types, fresh, n_fresh, excl_off, excl_idx, now_ms, seed, threads, out, nullptr, nullptr,
                             nullptr, nullptr, 0, true);
}

orc_lru *orc_lru_create(int64_t capacity) { return new orc_lru(capacity); }
void orc_lru_destroy(orc_lru *l) { delete l; }
int64_t orc_lru_apply(orc_lru *l, const orc_lru_event_t *ev, int64_t n, int64_t now_ms, orc_eviction_t *out, int64_t cap) {
  std::vector<orc_eviction_t> evs;
  for (int64_t i = 0; i < n; i++) l->l.apply(ev[i], (int32_t)i, now_ms, evs);
  for (size_t i = 0; i < evs.size() && (int64_t)i < cap; i++) out[i] = evs[i];
  return (int64_t)evs.size();
}
int64_t orc_lru_oldest_time(orc_lru *l) { return l->l.oldestTime; }
int64_t orc_lru_weighted_size(orc_lru *l) { return l->l.weightedSize; }
int64_t orc_lru_size(orc_lru *l) { return (int64_t)l->l.data.size(); }
int64_t orc_lru_dump(orc_lru *l, int32_t *keys, int64_t *last_used, int64_t *weights, int64_t cap) {
  int64_t n = 0;
  for (auto &nd : l->l.deque) { if (n < cap) { keys[n] = nd.key; last_used[n] = nd.lastUsed; weights[n] = nd.weight; } n++; }
  return n;
}

int64_t orc_unload_reserve_units(int64_t cacheCapacity, int32_t loadingThreads, int32_t defaultModelSizeUnits) {  // MM:749-755
  int32_t lowerBound = (int32_t)(cacheCapacity / 100), upperBound = (int32_t)(cacheCapacity / 10);
  int32_t unitsToReserve = jmuli(loadingThreads, defaultModelSizeUnits) / (loadingThreads <= 2 ? 2 : 4);
  return std::max(std::min(unitsToReserve, upperBound), lowerBound);
}
int64_t orc_min_space_units(int64_t capUnits, int32_t loadingThreads, int32_t defaultModelSizeUnits, int32_t hasUnloadManager) {  // MM:767-769
  int32_t mn = jmuli(defaultModelSizeUnits, (hasUnloadManager || loadingThreads <= 1) ? 1 : 2);
  int32_t target = std::min(jmuli(defaultModelSizeUnits, loadingThreads), (int32_t)(capUnits / 20));
  return std::max(mn, target);
}
int orc_churn_reject(int64_t capacity, int64_t weightedSize, int64_t oldestTime, int64_t minSpaceUnits, int64_t minChurnAgeMs,
                     int64_t now) {  // MM:3872-3884
  if (minChurnAgeMs > 0) {
    int64_t remaining = jsub(capacity, weightedSize);
    if (remaining < minSpaceUnits) {
      int64_t lru = oldestTime;
      if (lru >= 0 && lru != INT64_MAX && age(lru, now) < minChurnAgeMs) return 1;
    }
  }
  return 0;
}
int orc_early_reject(int64_t absSize, int64_t capacity, int64_t weightedSize, int64_t oldestTime, int64_t lastUsedTime) {  // MM:5185-5190
  return (absSize > capacity || (lastUsedTime > 0 && absSize > jsub(capacity, weightedSize) && lastUsedTime < oldestTime)) ? 1 : 0;
}

int64_t orc_reaper_select(orc_fleet *h, int32_t n, const orc_model_t *models, const char *const *type_names, int32_t n_types,
                          int32_t part_id, int64_t now, uint8_t *taken, int32_t *out_models, int64_t cap) {
  if (!h) return -1;
  Fleet &f = h->f;
  // reaper run(): MM:6455-6462
  const ClusterStats &globalStats = f.clusterStats;
  if (!(globalStats.totalCapacity > 0)) return 0;
  int64_t globalLru = globalStats.totalFree > 0 ? 0 : globalStats.globalLru;
  // pruneModelRegistry candidate rule MM:6574-6577 (instance pruning itself is KV I/O, out of scope)
  std::vector<int32_t> allCandidates;
  for (int i = 0; i < n; i++)
    if (models[i].n_loaded == 0 && models[i].n_failed < 2 && (globalLru == 0 || models[i].last_used > globalLru))
      allCandidates.push_back(i);
  if (allCandidates.empty()) return 0;
  ClusterStats stats;
  const Pts *excludeTypes = nullptr;
  if (part_id < 0) stats = f.clusterStats;
  else {
    Isst *is = nullptr;
    for (auto &e : f.tcm.ptsToInstanceSetStats) if (e.second->prohibitedTypesSet->id == part_id) is = e.second;
    if (!is) return -3;
    stats = is->currentStats; excludeTypes = is->prohibitedTypesSet;
  }
  // triggerProactiveLoadsForInstanceSubset MM:6616-6735
  int32_t freeSpaceProactiveLoadCount = 0, totalProactiveLoadCount = 0;
  if (stats.totalCapacity > 0 && stats.totalFree > 0) {
    int32_t sizeEstimate;
    if (stats.modelCopyCount < 3) sizeEstimate = f.defaultModelSizeUnits;
    else {
      int32_t averageSize = (int32_t)jsub(stats.totalCapacity, stats.totalFree) / stats.modelCopyCount;  // (int)(long) then int division
      sizeEstimate = stats.modelCopyCount > 10 ? averageSize : jaddi(averageSize, f.defaultModelSizeUnits) / 2;
    }
    int64_t spaceToFill = 0;
    for (const Entry &ent : f.clusterState) {
      const IR &ir = *ent.rec;
      if (excludeTypes != nullptr && !(ir.prohibitedTypes && ir.prohibitedTypes->types == excludeTypes->types)) continue;
      int32_t maxLoads = jsubi(jmuli(ir.lThreads, 50), ir.lInProg);
      if (maxLoads <= 0) continue;
      int64_t reserve = ir.capacity / 8, avail = jsub(ir.getRemaining(), reserve);
      if (avail > 0) spaceToFill = jadd(spaceToFill, std::min<int64_t>(avail, (int64_t)jmuli(maxLoads, sizeEstimate)));
    }
    spaceToFill /= 2;
    if (sizeEstimate == 0) return -4;  // Java would throw ArithmeticException
    freeSpaceProactiveLoadCount = (int32_t)(spaceToFill / sizeEstimate);
    totalProactiveLoadCount = std::max(freeSpaceProactiveLoadCount, (int32_t)jdiv(stats.totalCapacity, jmul(20, sizeEstimate)));
  }
  int64_t proactiveLastUsedCutoff = stats.globalLru == INT64_MAX ? 0
      : jadd(stats.globalLru, std::max<int64_t>(age(stats.globalLru, now) / 3, 1200000));
  // bounded TreeSet<ModelToLoad> keyed by lastUsed descending (N12)
  struct Mtl { int64_t lastUsed; int32_t model; };
  std::map<int64_t, Mtl, std::greater<int64_t>> toLoad;
  for (int32_t m : allCandidates) {
    if (taken && taken[m]) continue;
    const orc_model_t &mr = models[m];
    if (excludeTypes != nullptr && mr.type_idx >= 0 && mr.type_idx < n_types && excludeTypes->contains(type_names[mr.type_idx])) continue;
    int64_t lastUsed = mr.last_used;
    if (totalProactiveLoadCount > 0 && (freeSpaceProactiveLoadCount > 0 || lastUsed > proactiveLastUsedCutoff)) {
      if ((int64_t)toLoad.size() < totalProactiveLoadCount || std::prev(toLoad.end())->second.lastUsed < lastUsed) {
        toLoad.emplace(lastUsed, Mtl{lastUsed, m});  // no-op if equal key present
        if ((int64_t)toLoad.size() > totalProactiveLoadCount) toLoad.erase(std::prev(toLoad.end()));
      }
    }
  }
  int64_t count = 0;
  for (auto &e : toLoad) {
    int64_t timestamp = e.second.lastUsed;
    if (freeSpaceProactiveLoadCount > 0) freeSpaceProactiveLoadCount--;
    else if (timestamp < proactiveLastUsedCutoff) break;
    if (taken) taken[e.second.model] = 1;
    if (count < cap) out_models[count] = e.second.model;
    count++;
  }
  return count;
}

}  // extern "C"

#include "mm_sim.inc"
