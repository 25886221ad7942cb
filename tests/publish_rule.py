"""publishInstanceRecord (MM:5390-5470) with loadingChange / loadChange (MM:5536-5550), restated from the Java text for the
closed loop's end-of-window republish: one pod, its published record and its cache.  The oracle (publishNeeded and phase E
of oracle/mm_sim.inc) and the device (k_churn_republish) are checked against this in tests/test_publish_rule_oracle.py and
tests/test_publish_edges_gpu.py.

Java semantics throughout: long subtraction and `* 100` wrap, `/` truncates toward zero, Math.abs(Long.MIN_VALUE) is
Long.MIN_VALUE, and isFull(r) = r < minSpaceUnits (MM:4640-4642) on getRemaining() = max(0, capacity - used) (IR:203-205).

Out of the loop's reach, and so not restated as inputs: the unload manager's reserve (MM:5409-5422: the loop runs without
one), a pod without a record (MM:5432-5438: every pod in the loop has one) and the conditional-set retry (MM:5491-5511: a
pod is the only writer of its own record)."""
from common import LONG_MAX, jdiv, jlong, jsub

INSTANCE_REC_PUBLISH_MIN_PERIOD_MS = 2_000   # MM:232
INSTANCE_REC_PUBLISH_FREQ_MS = 40_000        # MM:231
FIELDS = ("capacity", "used", "count", "lru_time", "l_in_prog")  # what a republish writes (with the loop's constants)


def _jint(x: int) -> int:
    return ((int(x) + (1 << 31)) % (1 << 32)) - (1 << 31)


def _jabs(x: int) -> int:
    """Math.abs(long): Long.MIN_VALUE stays negative"""
    return jlong(-x) if x < 0 else x


def _jabsi(x: int) -> int:
    return _jint(-x) if x < 0 else x


def loading_change(cur_in_prog: int, l_threads: int, load_in_prog: int) -> bool:  # MM:5536-5543
    if load_in_prog == cur_in_prog:
        return False
    if (load_in_prog == 0) ^ (cur_in_prog == 0):
        return True
    if (load_in_prog <= l_threads) ^ (cur_in_prog <= l_threads):
        return True
    return _jabsi(_jint(load_in_prog - cur_in_prog)) >= 3


def load_change(cur_rec_rpms: int, rpms: int) -> bool:  # MM:5546-5550
    diff = _jabsi(_jint(cur_rec_rpms - rpms))
    return diff >= 100 or (rpms != 0 if cur_rec_rpms == 0 else jdiv(_jint(100 * diff), cur_rec_rpms) > 10)


def publish(cur, old_last_published: int, now: int, force: bool, cache, min_space_units: int):
    """(publish?, the record afterwards) for one pod at the end of a window.

    cur: the published record (a mapping with the INSTANCE_ROW fields); old_last_published: the pod's lastPublished;
    now: the window's end; force: whether the window forced a publish; cache: (capacity, weightedSize, size, the oldest
    entry's lastUsed or None when the cache is empty); min_space_units: the fleet's minSpaceUnits."""
    cap, used, count, oldest = (int(x) if x is not None else None for x in cache)
    last_done = jsub(now, old_last_published)
    # don't even check if last publish was < 2 sec ago (MM:5397-5400; preShutdown is false in the loop)
    if last_done < INSTANCE_REC_PUBLISH_MIN_PERIOD_MS or (not force and last_done < INSTANCE_REC_PUBLISH_FREQ_MS - 1000):
        return False, cur
    old = last_done > INSTANCE_REC_PUBLISH_FREQ_MS * 4
    if oldest is None:  # runtimeCache.oldestTime() == -1
        oldest = LONG_MAX
    # The loop holds these constant, so the clauses that compare them cannot fire from it: loadingThreads is the pod's
    # published value (no pod changes its thread count), no load is in progress when a window ends (every load of the
    # window completed inside it), the request rate is the published one (the loop tracks no rate) and no pod shuts down.
    load_threads, load_in_prog, rpms, is_shutting_down = int(cur["l_threads"]), 0, int(cur["rpm"]), bool(cur["shutting_down"])
    c_cap, c_used, c_count, c_lru = int(cur["capacity"]), int(cur["used"]), int(cur["count"]), int(cur["lru_time"])
    c_in_prog = int(cur["l_in_prog"])

    def is_full(r):
        return r < min_space_units

    if not old:
        # if changes are within thresholds, don't update (MM:5441-5458)
        within = bool(cur["shutting_down"]) == is_shutting_down
        within = within and _jabs(jsub(c_cap, cap)) < jdiv(cap, 50)
        if within:
            diff = _jabs(jsub(c_lru, oldest))
            within = diff < 20_000
        within = within and (c_lru == LONG_MAX or diff < jdiv(jsub(now, c_lru), 16))
        if within:
            diff = _jabsi(_jint(c_count - count))
            within = diff < 10
        within = within and ((count == 0) if c_count == 0 else jdiv(jlong(diff * 100), c_count) < 15)
        within = within and ((used == 0) if c_used == 0 else jdiv(jlong(_jabs(jsub(c_used, used)) * 100), c_used) < 20)
        within = within and is_full(max(0, jsub(c_cap, c_used))) == is_full(max(0, jsub(cap, used)))
        within = within and int(cur["l_threads"]) == load_threads
        within = within and not loading_change(c_in_prog, int(cur["l_threads"]), load_in_prog)
        within = within and not load_change(int(cur["rpm"]), rpms)
        if within:
            return False, cur
    # if not updated for a while, update if *any* change (MM:5460-5468)
    elif (bool(cur["shutting_down"]) == is_shutting_down and c_cap == cap and c_count == count and c_lru == oldest and c_used == used
          and int(cur["l_threads"]) == load_threads and c_in_prog == load_in_prog and int(cur["rpm"]) == rpms):
        return False, cur
    new = cur.copy()
    new["capacity"], new["lru_time"], new["count"], new["used"] = cap, oldest, count, used
    new["l_threads"], new["l_in_prog"], new["rpm"], new["shutting_down"] = load_threads, load_in_prog, rpms, is_shutting_down
    return True, new
