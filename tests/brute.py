"""Deliberately naive Python re-derivations from the Java text that tests elsewhere share (tests/test_oracle_properties.py says
what each one pins): the janitor's removeModelCopies per cache entry, the PLACEMENT_ORDER comparator, and the time-ordered
weighted LRU as a plain list."""
from modelmesh_b200.synth import LONG_MAX


def trunc_div(a, b):  # Java integer division truncates toward zero
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def free_space(r):
    return max(0, int(r["capacity"]) - int(r["used"]))


def brute_janitor_entry(e, p, have_tc, local_stats, loaded, lul, ids, shutting_down, pos):
    """removeModelCopies for the entry's pod; local_stats: instanceSetStats() of that pod (None: EMPTY_STATS, quirk N13)."""
    if not p["can_remove"] or e["last_used"] == 0 or len(loaded) < 2:
        return 0
    st = local_stats if local_stats is not None else dict(total_capacity=0, total_free=0, global_lru=LONG_MAX)
    if st["total_capacity"] == 0 or trunc_div(st["total_free"] * 100, st["total_capacity"]) > 5:
        return 0
    other = None
    for i, _ in sorted(loaded, key=lambda x: ids[x[0]]):                # TreeMap key order
        if i != e["instance"] and not shutting_down[i]:
            other = i
            break
    if other is None:
        return 0
    now = p["now"]
    if len(loaded) == 2:
        cache_age = now - st["global_lru"]
        down_age = trunc_div(cache_age, 10)
        if e["last_heavy"] == 0 or (now - e["last_heavy"]) < trunc_div(cache_age, 5):
            down_age = min(p["second_copy_remove_max_age_ms"], down_age)
        if (now - e["last_used"]) > down_age:
            if shutting_down[e["instance"]]:
                return 0
            return 0 if pos[other] > pos[e["instance"]] else 1         # PLACEMENT_ORDER.compare(other, this) > 0: the other pod flushes
        return 0
    if lul > 0 and now - lul < 8 * p["rate_check_interval_ms"]:
        return 0
    if any(ts > now - 1_800_000 for _, ts in loaded):
        return 0
    min_age = trunc_div(3 * st["global_lru"] + 10_400_000, 100)
    min_age = 600_000 if min_age < 600_000 else (18_000_000 if min_age > 18_000_000 else min_age)
    if now - e["last_heavy"] < min_age:
        return 0
    since = now - p["last_check_time"]
    if since < p["rate_check_interval_ms"] // 10:
        return 0
    if trunc_div(e["count"] * 60_000, since) > trunc_div(p["scale_up_rpm_threshold"] * 2, 3):
        return 0
    return 1


def brute_compare(r1, id1, loc1, zone1, lab1, r2, id2, loc2, zone2, lab2, min_space, min_churn_age):
    """PLACEMENT_ORDER.compare (MM:4646-4703) for two DIFFERENT records, from the Java text; returns the sign."""
    sgn = lambda a, b: (a > b) - (a < b)
    def nulls_last(a, b):
        if a is None or b is None:
            return 0 if a is b else (1 if a is None else -1)
        return sgn(a, b)
    sd1, sd2 = bool(r1["shutting_down"]), bool(r2["shutting_down"])
    if sd1 != sd2:
        return 1 if sd1 else -1
    v1, v2 = int(r1["vers"]), int(r2["vers"])
    rem1, rem2 = free_space(r1), free_space(r2)
    full1, full2 = rem1 < min_space, rem2 < min_space
    if v1 != v2:                                                         # N1: "prefer newer version unless it's saturated"
        if v1 > v2:
            if not full1 or int(r1["lru_time"]) > min_churn_age * 2:
                return -1
        elif not full2 or int(r2["lru_time"]) > min_churn_age * 2:
            return 1
    if full1 != full2:
        return 1 if full1 else -1
    if full1:
        d = sgn(int(r1["lru_time"]), int(r2["lru_time"]))
        if d:
            return d
    d = sgn(int(r1["count"]) - int(r2["count"]), 0)
    if d:
        return d
    d = sgn(rem2, rem1)
    if d:
        return d
    if not full1:
        d = sgn(int(r1["lru_time"]), int(r2["lru_time"]))
        if d:
            return d
    lip1, lip2 = int(r1["l_in_prog"]), int(r2["l_in_prog"])
    for d in (sgn(int(r2["l_threads"]) - lip2, int(r1["l_threads"]) - lip1), sgn(lip1, lip2), sgn(int(r2["capacity"]), int(r1["capacity"])),
              sgn(int(r1["rpm"]), int(r2["rpm"])), sgn(id1, id2), nulls_last(loc1, loc2), nulls_last(zone1, zone2)):
        if d:
            return d
    l1, l2 = list(lab1 or []), list(lab2 or [])
    if len(l1) != len(l2):
        return sgn(len(l1), len(l2))
    for a, b in zip(l1, l2):
        if a != b:
            return sgn(a, b)
    return 0


# ---------------------------------------------------------------------------------------------------------------
# a10: the time-ordered weighted LRU (clhm/ConcurrentLinkedHashMap + LinkedDeque, single-threaded reading: every read is
# drained at once) as a plain Python list, from the Java text: put / putIfAbsent (CLHM:821-858, AddTask 590-610), get
# (731-738 -> touch 1357-1360 -> LinkedDeque.reposition / insert LD:243-288), replaceQuietly (963-984, UpdateTask 631-652),
# remove (860-871), setCapacity (305-316: evict, notify, oldestTime NOT refreshed), forceSetLastUsedTime (756-768: no
# reposition), evict from the head while weightedSize > capacity with |weight| on makeDead (329-352), oldestTime (1129-1133).
# ---------------------------------------------------------------------------------------------------------------
class BruteLru:
    def __init__(self, capacity):
        self.cap, self.wsize, self.oldest = capacity, 0, -1
        self.deque = []          # [key, weight, lastUsed], oldest first
        self.pending = []

    def _find(self, key):
        for n in self.deque:
            if n[0] == key:
                return n
        return None

    def _insert(self, node):    # LD:258-288: after the last element whose lastUsed <= ts, scanning from the tail
        pos = len(self.deque)
        while pos > 0 and self.deque[pos - 1][2] > node[2]:
            pos -= 1
        self.deque.insert(pos, node)

    def _reposition(self, node):  # LD:243-255
        i = next(k for k, n in enumerate(self.deque) if n is node)
        lu = node[2]
        if i == 0 or self.deque[i - 1][2] <= lu:
            if i == len(self.deque) - 1 or self.deque[i + 1][2] >= lu:
                return
        del self.deque[i]
        self._insert(node)

    def _evict(self, ev_index):
        while self.wsize > self.cap and self.deque:
            k, w, lu = self.deque.pop(0)
            self.wsize -= abs(w)
            self.pending.append((k, ev_index, lu, w))

    def _oldest(self):
        self.oldest = self.deque[0][2] if self.deque else -1

    def _after_read(self, node, last_used, now):
        t = last_used if last_used > 0 else 0
        node[2] = now if t == 0 else max(node[2], t)
        self._reposition(node)
        self._oldest()

    def apply(self, op, key, weight, last_used, ev_index, now, out):
        node = self._find(key)
        if op == 0:
            if node is None:
                n = [key, weight, now if last_used == 0 else max(0, last_used)]
                self.wsize += weight
                self._insert(n)
                self._evict(ev_index)
                self._oldest()
                out.extend(self.pending); self.pending = []
            else:
                self._after_read(node, last_used, now)
        elif op == 1:
            if node is not None:
                self._after_read(node, last_used, now)
        elif op == 2:
            if node is not None:
                diff = weight - node[1]
                node[1] = weight
                if diff != 0:
                    self.wsize += diff
                    self._evict(ev_index)
                    self._oldest()
                    if diff > 0:
                        out.extend(self.pending); self.pending = []
        elif op == 3:
            if node is not None:
                self.wsize -= abs(node[1])
                self.deque.remove(node)
                self._oldest()
        elif op == 4:
            self.cap = weight
            self._evict(ev_index)
            out.extend(self.pending); self.pending = []
        elif op == 5:
            if node is not None:
                node[2] = last_used
