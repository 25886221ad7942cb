"""Brute-force cross-checks OF THE ORACLE (not of the GPU against the oracle) for the parts of getNext that no reference test
pins (SURVEY.md §8c: "parity unpinned by reference tests"): an independent, deliberately naive Python re-derivation from
the Java text, structured differently from oracle/mm_oracle.cpp (lists and dicts, the filtered set materialised, the
shortlist as a sorted-prefix enumeration), must give the same ordered shortlist, rpm-filter survivors and pick.

  * shortlist == brute-force filter -> sort -> prefix (MM:4760-4771, 4806-4811, 4889-4937, N2/N3 literal)
  * the same with type constraints and preferences: constrainTo, non-simple (a) and (b) (MM:4788-4790, 4816-4887), N8
  * the reaper's proactive-load selection (MM:6455-6462, 6574-6577, 6616-6735, N12) as plain Python arithmetic and a sorted list
  * a14: the rate-tracking loop body and the janitor's removeModelCopies / removeSecondModelCopy (MM:5684-5870, 6197-6335, N13)
  * ClusterStats / partition stats as plain sums (N10 literal)
  * a6: the converged per-type instance sets of TypeConstraintManager as set comprehensions (TCM:92-95, 455-486, 680-747, N11)
  * invariants of the closed loop (registry == caches, capacities) after every window
  * a10: the time-ordered weighted LRU as a plain Python list (CLHM / LinkedDeque)
  * rpm filter == independent re-derivation (MM:4957-4980)
  * PLACEMENT_ORDER is a strict weak order on uniform-`vers` fleets and the cluster order is sorted under it (MM:4646-4703);
    the comparator itself re-derived and compared on sampled pairs, mixed versions (N1) included
"""
import numpy as np
import pytest

from brute import BruteLru, brute_compare, brute_janitor_entry, free_space, trunc_div
from common import vp
from helpers import oracle_from_synth, oracle_inputs
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import LONG_MAX, make_decisions, make_fleet
from oracle import binding as ob

M64 = (1 << 64) - 1


def _i64(x):  # Java long wrap
    x &= M64
    return x - (1 << 64) if x >> 63 else x


def _age(t, now):  # MM:4162-4164
    return 0 if t == 0 else _i64(now - t)


def _hash64(seed, did):  # N4 (same contract as the oracle and the kernel)
    z = (seed + 0x9E3779B97F4A7C15 * (did + 1)) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def _java_int(d):  # (int) double: truncation toward zero, saturating
    if d != d:
        return 0
    return max(-(1 << 31), min((1 << 31) - 1, int(d)))


def brute_get_next(order, rows, ids, active, replaced, min_space, self_idx, fresh, favour_self, last_used, excluded, now, rnd):
    """getNext for a type WITHOUT constraints or preferences (constrainTo == null, prefer == null), naive form."""
    def in_filter(i, use_rs):
        if i in excluded or not active[i]:
            return False
        if use_rs and replaced and len(ids[i]) >= 7 and ids[i][:6] in replaced:
            return False
        return True
    flt = [i for i in order if in_filter(i, True)]                      # MM:4760-4771 materialised
    if not flt and replaced:
        flt = [i for i in order if in_filter(i, False)]                 # MM:4798-4802
    if not flt:
        return dict(target=ob.NONE, cands=[], keep=[], n_remaining=0, pick=0)
    best = flt[0]
    exclude_self = self_idx in excluded
    us = best == self_idx and not exclude_self                          # MM:4808
    best_rec = fresh if us else rows[best]
    best_full = free_space(best_rec) < min_space
    if us and favour_self:
        return dict(target=ob.SELF, cands=[], keep=[], n_remaining=0, pick=0)
    cands, loads = [best], [int(best_rec["rpm"])]
    oldest = int(best_rec["lru_time"])
    first_entry_rec = rows[best]                                        # bestEntry.getValue(): the PUBLISHED record of the first entry
    for i in flt[1:]:
        us = (not us) and (not exclude_self) and i == self_idx          # N3
        cur = first_entry_rec if us else fresh                          # N2 (literal)
        if best_full:
            diff = _i64(int(cur["lru_time"]) - oldest)
            a10 = int(_age(oldest, now) / 10)                           # Java long division truncates toward zero
            if diff > 45_000 and diff > a10:
                break
        else:
            rem = free_space(cur)
            if rem < min_space or rem < (free_space(best_rec) >> 2):
                break
            cnt, first = int(rows[i]["count"]), int(best_rec["count"])
            if cnt >= 10 and cnt > first + (first >> 2):
                break
        if us and favour_self:
            return dict(target=ob.SELF, cands=cands, keep=[], n_remaining=0, pick=0, early=True)
        cands.append(i)
        loads.append(int(cur["rpm"]))
    keep = [True] * len(cands)
    remaining, index = len(cands), 0
    if len(cands) > 1:
        ago = _age(last_used, now)
        if ago < 5 * 86_400_000:
            mn = max(100, min(loads))
            m11, m15 = _java_int(1.1 * mn), _java_int(1.5 * mn)
            for k, rpm in enumerate(loads):
                if rpm >= 100 and ((ago < -1000 and rpm > m11) or (ago < 5000 and rpm > m15) or (ago < 720_000 and rpm > mn * 3)
                                   or (ago < 86_400_000 and rpm > mn * 4)):
                    keep[k] = False
                    remaining -= 1
                    if remaining == 1:
                        break
        index = 0 if remaining == 1 else (((rnd >> 32) * remaining) >> 32)
    chosen = [c for c, k in zip(cands, keep) if k][index]
    target = ob.SELF if (not favour_self and chosen == self_idx) else chosen
    return dict(target=target, cands=cands, keep=keep, n_remaining=remaining, pick=index)


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 1500, 400, 2), ("C2", 1500, 97, 9), ("C1", 300, 16, 1), ("MIX", 500, 160, 2),
                                               ("MIX", 500, 300, 6), ("MIX", 500, 97, 8), ("MIX", 500, 64, 13), ("MIX", 500, 33, 20),
                                               ("MIX", 500, 160, 23), ("MIX", 500, 300, 24), ("MIX", 500, 200, 25), ("MIX", 500, 120, 29),
                                               ("MIX", 500, 250, 35), ("MIX", 500, 97, 36), ("MIX", 500, 180, 43)])
def test_shortlist_is_the_sorted_prefix_parity_unpinned_by_reference_tests(oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    if fl.type_config is not None:
        pytest.skip("this seed draws type constraints; the brute force covers constrainTo == null, prefer == null")
    o = oracle_from_synth(fl)
    sd = make_decisions(fl, 1200, seed)
    od, off, idx = oracle_inputs(fl, sd)
    fresh = sd.fresh if len(sd.fresh) else None
    res, coff, cidx, cload, ckeep = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed * 7, fresh=fresh, want_candidates=True)
    order = [int(x) for x in o.cluster_order()]
    rows = fl.inst_rows
    active = [bool(a) and not bool(s) for a, s in zip(rows["active"], rows["shutting_down"])]
    replaced = set(fl.replaced_replicasets)
    full_seen = nonfull_seen = multi = 0
    for i in range(len(od)):
        d = sd.dec[i]
        self_idx = int(d["self"])
        if d["fresh"] >= 0:
            fr = sd.fresh[int(d["fresh"])]
        else:
            fr = rows[self_idx].copy()
            fr["rpm"] = 0                                               # N7
        b = brute_get_next(order, rows, fl.inst_ids, active, replaced, fl.min_space_units, self_idx, fr,
                           bool(d["flags"] & L.DF_FAVOUR_SELF), int(od["last_used"][i]), set(int(x) for x in idx[off[i]:off[i + 1]]),
                           fl.now_ms, _hash64(seed * 7, i))
        assert b["target"] == int(res["target"][i]), (i, b, res[i])
        if b.get("early") or not b["cands"]:
            continue
        want = [int(x) for x in cidx[coff[i]:coff[i + 1]]]
        assert b["cands"] == want, (i, b["cands"][:6], want[:6])
        assert b["keep"] == [bool(k) for k in ckeep[coff[i]:coff[i + 1]]], i
        assert b["n_remaining"] == int(res["n_remaining"][i]) and b["pick"] == int(res["pick_index"][i]), i
        multi += len(want) > 1
        if res["flags"][i] & 4:
            full_seen += 1
        else:
            nonfull_seen += 1
    assert full_seen + nonfull_seen > 100  # (MIX seeds draw all-full, mixed and all-free regimes: both walk tests are reached over the set)
    test_shortlist_is_the_sorted_prefix_parity_unpinned_by_reference_tests.seen = getattr(
        test_shortlist_is_the_sorted_prefix_parity_unpinned_by_reference_tests, "seen", np.zeros(3, dtype=np.int64)) + [full_seen, nonfull_seen, multi]


def test_brute_force_reached_both_walk_tests():
    seen = getattr(test_shortlist_is_the_sorted_prefix_parity_unpinned_by_reference_tests, "seen", None)
    if seen is None:
        pytest.skip("runs after the brute-force cases")
    assert seen[0] > 200 and seen[1] > 200 and seen[2] > 200, seen  # full-case walks, non-full walks, multi-candidate shortlists


@pytest.mark.parametrize("config,ni,seed", [("C2", 300, 2), ("C3", 500, 3), ("C5", 400, 5), ("MIX", 200, 8), ("MIX", 200, 14), ("MIX", 120, 21)])
def test_placement_order_is_a_strict_weak_order_on_uniform_vers_fleets(oracle_lib, config, ni, seed):
    """Antisymmetry, transitivity (sampled triples) and agreement with the sorted cluster state; vers is uniform in the
    synthetic fleets, so N1's non-transitive corner cannot occur."""
    fl = make_fleet(config, 50, ni, seed)
    assert len(set(int(v) for v in fl.inst_rows["vers"])) == 1
    o = oracle_from_synth(fl)
    order = [int(x) for x in o.cluster_order()]
    n = len(order)
    assert n == int(np.count_nonzero(fl.inst_rows["shutting_down"] == 0))
    rng = np.random.default_rng(seed)
    for a, b in zip(order[:-1], order[1:]):
        assert o.compare(a, b) < 0 and o.compare(b, a) > 0
    pos = {x: k for k, x in enumerate(order)}
    for _ in range(3000):
        a, b, c = (order[int(k)] for k in rng.integers(0, n, 3))
        ab, ba = o.compare(a, b), o.compare(b, a)
        assert (ab > 0) == (ba < 0) and (ab == 0) == (ba == 0) == (a == b)
        assert (ab < 0) == (pos[a] < pos[b])
        if ab < 0 and o.compare(b, c) < 0:
            assert o.compare(a, c) < 0


def test_rpm_filter_thresholds_independent_rederivation(oracle_lib):
    """MM:4957-4980 on hand-built shortlists: three instances with equal keys except rpm, decisions whose lastUsed walks
    through the five age bands.  The caller is never a candidate (inactive), so every non-best candidate records the
    caller's fresh rpm (N2) -- given explicitly through a fresh row."""
    now = 1_760_000_000_000
    o = ob.OracleFleet(1000, 600_000, 2560)
    o.types_set(None)
    rows = np.zeros(4, dtype=ob.INST)
    rows["capacity"], rows["used"], rows["lru_time"], rows["l_threads"], rows["active"] = 100_000, 10_000, now - 3_600_000, 8, 1
    rows["rpm"] = [150, 400, 700, 0]
    rows["active"][3] = 0
    for i in range(4):
        o.instance_event(ob.ADDED, i, rows[i], f"pod-{i}", now_ms=now)
    for fresh_rpm in (0, 120, 200, 460, 650):
        fresh = rows[3:4].copy()
        fresh["rpm"] = fresh_rpm
        for ago in (-5000, 1000, 60_000, 3_600_000, 2 * 86_400_000, 6 * 86_400_000):
            od = np.zeros(1, dtype=ob.DECISION)
            od["type_idx"], od["self"], od["fresh_idx"], od["last_used"] = -1, 3, 0, now - ago
            res, coff, cidx, cload, ckeep = o.get_next_batch(od, [], np.zeros(2, dtype=np.int64), np.zeros(0, dtype=np.int32), now, 5,
                                                            fresh=fresh, want_candidates=True)
            loads = [150, fresh_rpm, fresh_rpm]                        # best records its own rpm, the others the caller's (N2)
            assert [int(x) for x in cload[:3]] == loads
            mn = max(100, min(loads))
            def drop(rpm):
                if rpm < 100 or ago >= 5 * 86_400_000:
                    return False
                return ((ago < -1000 and rpm > int(1.1 * mn)) or (ago < 5000 and rpm > int(1.5 * mn)) or (ago < 720_000 and rpm > 3 * mn)
                        or (ago < 86_400_000 and rpm > 4 * mn))
            assert [bool(k) for k in ckeep[:3]] == [not drop(r) for r in loads], (fresh_rpm, ago)


# ---------------------------------------------------------------------------------------------------------------
# The same brute force for types WITH constraints: constrainTo (required labels), prefer (preferred labels), the two
# non-simple cases.  Written from the Java text (MM:4776-5004) as an iterator over a materialised list, the way the Java
# reads -- `it`, `clusterStateReplay`, `prefer = null` -- and not the way the oracle or the kernels are structured.
# The candidate / preferred sets themselves come from the oracle's TypeConstraintManager restatement (this test pins
# getNext's use of them, test_type_masks_* pin the sets).
# ---------------------------------------------------------------------------------------------------------------
def _select(cands, loads, last_used, now, rnd, self_idx, favour_self):
    keep = [True] * len(cands)
    remaining, index = len(cands), 0
    if len(cands) > 1:
        ago = _age(last_used, now)
        if ago < 5 * 86_400_000:
            mn = max(100, min(loads))
            m11, m15 = _java_int(1.1 * mn), _java_int(1.5 * mn)
            for k, rpm in enumerate(loads):
                if rpm >= 100 and ((ago < -1000 and rpm > m11) or (ago < 5000 and rpm > m15) or (ago < 720_000 and rpm > mn * 3)
                                   or (ago < 86_400_000 and rpm > mn * 4)):
                    keep[k] = False
                    remaining -= 1
                    if remaining == 1:
                        break
        index = 0 if remaining == 1 else (((rnd >> 32) * remaining) >> 32)
    chosen = [c for c, k in zip(cands, keep) if k][index]
    target = ob.SELF if (not favour_self and chosen == self_idx) else chosen
    return dict(target=target, cands=cands, keep=keep, n_remaining=remaining, pick=index)


def brute_get_next_tc(order, rows, ids, active, replaced, min_space, self_idx, fresh, favour_self, last_used, excluded, now, rnd,
                      constrain_to, prefer):
    def passes(i, use_rs):
        if constrain_to is not None and i not in constrain_to:
            return False
        if i in excluded or not active[i]:
            return False
        if use_rs and replaced and len(ids[i]) >= 7 and ids[i][:6] in replaced:
            return False
        return True
    flt = [i for i in order if passes(i, True)]
    if not flt and replaced:
        flt = [i for i in order if passes(i, False)]
    if not flt:
        return dict(target=ob.NONE, cands=[], keep=[], n_remaining=0, pick=0)
    exclude_self = self_idx in excluded
    it = iter(flt)
    best_entry = next(it)                                               # bestEntry: never reassigned
    best_iid = best_entry
    us = (not exclude_self) and best_iid == self_idx
    best_inst = fresh if us else rows[best_iid]
    best_is_full = free_space(best_inst) < min_space                     # final: keeps the FIRST entry's verdict
    cands, loads = [], []
    case = "simple"
    simple = prefer is None or best_iid in prefer
    if not simple:
        replay = []
        if not best_is_full:                                            # (a) MM:4828-4852
            found = False
            for ent in it:
                if ent in prefer:
                    found = True
                    best_iid = ent
                    best_inst = rows[ent]                               # ent.getValue(): the published record, even for self
                    us = (not us) and (not exclude_self) and ent == self_idx
                    break
                if free_space(rows[ent]) < min_space:
                    break
                replay.append(ent)
            case = "a_found" if found else "a_rewind"
            if not found:
                it = iter(replay)
                prefer = None
            simple = True
        else:                                                           # (b) MM:4853-4887
            oldest = int(best_inst["lru_time"])
            for ent in it:
                diff = _i64(int(rows[ent]["lru_time"]) - oldest)
                if diff > 120_000 and diff > int(_age(oldest, now) / 4):
                    break
                if ent in prefer:
                    us = (not us) and (not exclude_self) and ent == self_idx
                    if us and favour_self:
                        return dict(target=ob.NONE, cands=[], keep=[], n_remaining=0, pick=0, early=True)  # N8: null
                    replay = None
                    cands.append(ent)
                    loads.append(int(rows[ent]["rpm"]))
                elif replay is not None:
                    replay.append(ent)
            case = "b_pref" if replay is None else "b_rewind"
            if replay is not None:
                it = iter(replay)
                prefer = None
                simple = True
    if simple:
        if us and favour_self:
            return dict(target=ob.SELF, cands=[], keep=[], n_remaining=0, pick=0, early=True)
        cands.append(best_iid)
        loads.append(int(best_inst["rpm"]))
        oldest = int(best_inst["lru_time"])
        for ent in it:
            if prefer is not None and ent not in prefer:
                continue
            us = (not us) and (not exclude_self) and ent == self_idx
            cur = rows[best_entry] if us else fresh                     # N2 / N3, literal
            if best_is_full:
                diff = _i64(int(cur["lru_time"]) - oldest)
                if diff > 45_000 and diff > int(_age(oldest, now) / 10):
                    break
            else:
                rem = free_space(cur)
                if rem < min_space or rem < (free_space(best_inst) >> 2):
                    break
                cnt, first = int(rows[ent]["count"]), int(best_inst["count"])
                if cnt >= 10 and cnt > first + (first >> 2):
                    break
            if us and favour_self:
                return dict(target=ob.SELF, cands=cands, keep=[], n_remaining=0, pick=0, early=True)
            cands.append(ent)
            loads.append(int(cur["rpm"]))
    if not cands:
        return dict(target=ob.NONE, cands=[], keep=[], n_remaining=0, pick=0)
    out = _select(cands, loads, last_used, now, rnd, self_idx, favour_self)
    out["case"] = case
    return out


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 1500, 400, 3), ("C3", 1500, 97, 4), ("C5", 1500, 500, 5), ("C5", 1500, 300, 7),
                                               ("MIX", 500, 160, 5), ("MIX", 500, 300, 8), ("MIX", 500, 97, 14), ("MIX", 500, 200, 21),
                                               ("MIX", 500, 250, 41), ("MIX", 500, 120, 3), ("MIX", 500, 64, 10), ("MIX", 500, 180, 11)])
def test_constrained_types_and_preferences_parity_unpinned_by_reference_tests(oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    if fl.type_config is None:
        pytest.skip("this seed draws no type constraints (covered by the test above)")
    o = oracle_from_synth(fl)
    sd = make_decisions(fl, 1200, seed)
    od, off, idx = oracle_inputs(fl, sd)
    fresh = sd.fresh if len(sd.fresh) else None
    res, coff, cidx, cload, ckeep = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed * 7, fresh=fresh, want_candidates=True)
    order = [int(x) for x in o.cluster_order()]
    rows = fl.inst_rows
    active = [bool(a) and not bool(s) for a, s in zip(rows["active"], rows["shutting_down"])]
    replaced = set(fl.replaced_replicasets)
    sets = {}
    for t, name in enumerate(fl.type_names):
        a, p = o.type_sets(name, fl.n_instances)
        sets[t] = (None if a is None else set(int(x) for x in np.nonzero(a)[0]), None if p is None else set(int(x) for x in np.nonzero(p)[0]))
    seen = dict(simple=0, a_found=0, a_rewind=0, b_pref=0, b_rewind=0, constrained=0)
    for i in range(len(od)):
        d = sd.dec[i]
        self_idx = int(d["self"])
        if d["fresh"] >= 0:
            fr = sd.fresh[int(d["fresh"])]
        else:
            fr = rows[self_idx].copy()
            fr["rpm"] = 0                                               # N7
        cto, prf = sets[int(od["type_idx"][i])]
        b = brute_get_next_tc(order, rows, fl.inst_ids, active, replaced, fl.min_space_units, self_idx, fr,
                              bool(d["flags"] & L.DF_FAVOUR_SELF), int(od["last_used"][i]), set(int(x) for x in idx[off[i]:off[i + 1]]),
                              fl.now_ms, _hash64(seed * 7, i), cto, prf)
        assert b["target"] == int(res["target"][i]), (i, b, res[i])
        if b.get("early") or not b["cands"]:
            continue
        want = [int(x) for x in cidx[coff[i]:coff[i + 1]]]
        assert b["cands"] == want, (i, b["cands"][:6], want[:6])
        assert b["keep"] == [bool(k) for k in ckeep[coff[i]:coff[i + 1]]], i
        assert b["n_remaining"] == int(res["n_remaining"][i]) and b["pick"] == int(res["pick_index"][i]), i
        seen["constrained"] += cto is not None
        seen[b["case"]] = seen.get(b["case"], 0) + 1
    acc = getattr(test_constrained_types_and_preferences_parity_unpinned_by_reference_tests, "seen", {})
    for k, v in seen.items():
        acc[k] = acc.get(k, 0) + v
    test_constrained_types_and_preferences_parity_unpinned_by_reference_tests.seen = acc


def test_constrained_brute_force_reached_every_case():
    seen = getattr(test_constrained_types_and_preferences_parity_unpinned_by_reference_tests, "seen", None)
    if seen is None:
        pytest.skip("runs after the constrained brute-force cases")
    # every branch of MM:4822-4887 was exercised: (a) with and without a preferred entry, (b) with preferred candidates and rewound
    assert seen["constrained"] > 500 and seen["a_found"] > 100 and seen["a_rewind"] > 20 and seen["b_pref"] > 20 and seen["b_rewind"] > 20, seen


# ---------------------------------------------------------------------------------------------------------------
# The reaper's proactive-load selection (MM:6455-6462 candidate rule inputs, MM:6574-6577, MM:6616-6735), naive form:
# plain Python ints for the Java arithmetic, a sorted list for the TreeSet<ModelToLoad> (whose compareTo looks at lastUsed
# only: two candidates with the same lastUsed are ONE element -- N12), partitions visited in getPartitionStats() order with
# the selected models nulled out of the shared candidate list.
# ---------------------------------------------------------------------------------------------------------------
def brute_reaper(stats, global_stats, insts_of_subset, rows, models, type_prohibited, default_size, now, taken):
    """stats / global_stats: ClusterStats dicts; insts_of_subset: instance indices the subset's loop visits (cluster order);
    models: list of (last_used, type_idx, n_loaded, n_failed); type_prohibited(type_idx) -> bool for this subset."""
    if not global_stats["total_capacity"] > 0:
        return []
    global_lru = 0 if global_stats["total_free"] > 0 else global_stats["global_lru"]
    cands = [m for m, (lu, t, nl, nf) in enumerate(models) if nl == 0 and nf < 2 and (global_lru == 0 or lu > global_lru)]
    free_count = total_count = 0
    if stats["total_capacity"] > 0 and stats["total_free"] > 0:
        if stats["model_copy_count"] < 3:
            size_est = default_size
        else:
            used = stats["total_capacity"] - stats["total_free"]
            used32 = ((used + (1 << 31)) % (1 << 32)) - (1 << 31)       # (int) of a long
            avg = trunc_div(used32, stats["model_copy_count"])
            size_est = avg if stats["model_copy_count"] > 10 else trunc_div(avg + default_size, 2)
        space = 0
        for i in insts_of_subset:
            r = rows[i]
            max_loads = int(r["l_threads"]) * 50 - int(r["l_in_prog"])
            if max_loads <= 0:
                continue
            avail = free_space(r) - int(r["capacity"]) // 8
            if avail > 0:
                space += min(avail, max_loads * size_est)
        space = trunc_div(space, 2)
        free_count = trunc_div(space, size_est)
        total_count = max(free_count, trunc_div(stats["total_capacity"], 20 * size_est))
    cutoff = 0 if stats["global_lru"] == LONG_MAX else stats["global_lru"] + max(trunc_div(_age(stats["global_lru"], now), 3), 1_200_000)
    to_load = []                                                        # [(lastUsed, model)], lastUsed descending, unique lastUsed
    for m in cands:
        if taken[m]:
            continue
        lu, t, _, _ = models[m]
        if type_prohibited(t):
            continue
        if total_count > 0 and (free_count > 0 or lu > cutoff):
            if len(to_load) < total_count or to_load[-1][0] < lu:
                if all(x[0] != lu for x in to_load):                    # TreeSet.add: equal under compareTo -> not added
                    to_load.append((lu, m))
                    to_load.sort(key=lambda x: -x[0])
                if len(to_load) > total_count:
                    to_load.pop()
    out = []
    for lu, m in to_load:
        if free_count > 0:
            free_count -= 1
        elif lu < cutoff:
            break
        taken[m] = 1
        out.append(m)
    return out


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 3000, 300, 2), ("C3", 3000, 400, 3), ("C5", 3000, 400, 5), ("MIX", 1500, 160, 5),
                                               ("MIX", 1500, 300, 8), ("MIX", 1500, 97, 14), ("MIX", 1500, 200, 2), ("MIX", 1500, 120, 29)])
def test_reaper_selection_parity_unpinned_by_reference_tests(oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    if config == "C5":  # leave some room so that the free-space branch is taken too
        fl.inst_rows["used"][::3] = fl.inst_rows["capacity"][::3] // 2
    o = oracle_from_synth(fl)
    om = np.zeros(nm, dtype=ob.MODEL)
    om["last_used"], om["type_idx"], om["n_loaded"], om["n_failed"] = fl.model_last_used, fl.model_type, fl.n_loaded, fl.n_failed
    models = [(int(a), int(b), int(c), int(d)) for a, b, c, d in zip(om["last_used"], om["type_idx"], om["n_loaded"], om["n_failed"])]
    names = ("total_capacity", "total_free", "global_lru", "instance_count", "model_copy_count")
    as_dict = lambda s: {k: int(s[k]) for k in names}
    gstats = as_dict(o.cluster_stats())
    order = [int(x) for x in o.cluster_order()]
    rows = fl.inst_rows
    total = 0
    if fl.type_config is None:
        want = o.reaper_select(om, fl.type_names, -1, fl.now_ms)
        got = brute_reaper(gstats, gstats, order, rows, models, lambda t: False, fl.default_model_size_units, fl.now_ms, np.zeros(nm, np.uint8))
        assert got == [int(x) for x in want], (got[:5], want[:5])
        total = len(got)
    else:
        pstats, pids = o.partition_stats()
        part_of = {i: o.instance_partition(i) for i in order}
        cand_sets = [o.type_sets(name, fl.n_instances)[0] for name in fl.type_names]
        taken_o, taken_b = np.zeros(nm, np.uint8), np.zeros(nm, np.uint8)
        for st, pid in zip(pstats, pids):                               # getPartitionStats() order (MM:6476-6489)
            members = [i for i in order if part_of[i] == int(pid)]
            rep = members[0]
            # a type is prohibited for the subset iff its candidate set exists and excludes the subset's instances (TCM:557-575)
            prohibited = lambda t, rep=rep: 0 <= t < len(cand_sets) and cand_sets[t] is not None and not bool(cand_sets[t][rep])
            want = o.reaper_select(om, fl.type_names, int(pid), fl.now_ms, taken=taken_o)
            got = brute_reaper(as_dict(st), gstats, members, rows, models, prohibited, fl.default_model_size_units, fl.now_ms, taken_b)
            assert got == [int(x) for x in want], (int(pid), got[:5], [int(x) for x in want[:5]])
            assert np.array_equal(taken_o, taken_b)
            total += len(got)
    acc = getattr(test_reaper_selection_parity_unpinned_by_reference_tests, "total", 0) + total
    test_reaper_selection_parity_unpinned_by_reference_tests.total = acc


def test_reaper_brute_force_selected_something():
    total = getattr(test_reaper_selection_parity_unpinned_by_reference_tests, "total", None)
    if total is None:
        pytest.skip("runs after the reaper brute-force cases")
    assert total > 200, total


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 500, 300, 2), ("C3", 500, 400, 3), ("C5", 500, 400, 5), ("MIX", 300, 160, 5), ("MIX", 300, 97, 14)])
def test_cluster_and_partition_stats_are_plain_sums(oracle_lib, config, nm, ni, seed):
    """ClusterStats (MM:1570-1591) / InstanceSetStatsTracker (ISST:63-92) against sums over the instance table: capacity, free space of
    the non-full instances only (ISST:67-71), instance and model-copy counts, the oldest positive lruTime (ISST:57-61); per partition
    the same over its members, with the LRU as quirk N10 leaves it."""
    fl = make_fleet(config, nm, ni, seed)
    o = oracle_from_synth(fl, bulk=False)
    rows = fl.inst_rows
    live = [int(x) for x in o.cluster_order()]                          # the instances in the cluster state (shutting-down ones are not)
    def sums(members):
        cap = sum(int(rows["capacity"][i]) for i in members)
        free = sum(free_space(rows[i]) for i in members if free_space(rows[i]) >= fl.min_space_units)
        copies = sum(int(rows["count"][i]) for i in members)
        return cap, free, len(members), copies
    lrus = [int(rows["lru_time"][i]) for i in live if int(rows["lru_time"][i]) > 0]
    glru = min(lrus) if lrus else LONG_MAX
    g = o.cluster_stats()
    assert (int(g["total_capacity"]), int(g["total_free"]), int(g["instance_count"]), int(g["model_copy_count"])) == sums(live)
    assert int(g["global_lru"]) == glru
    if fl.type_config is not None:
        pstats, pids = o.partition_stats()
        part_of = {i: o.instance_partition(i) for i in live}
        assert sorted(set(part_of.values())) == sorted(int(p) for p in pids)
        for st, pid in zip(pstats, pids):
            members = [i for i in live if part_of[i] == int(pid)]
            assert (int(st["total_capacity"]), int(st["total_free"]), int(st["instance_count"]), int(st["model_copy_count"])) == sums(members)
            # N10, literal: an instance event recomputes ITS subset's LRU over all instances known at that moment (MM:1519-1541);
            # the fleet was fed as ADDED events in index order, so a subset's LRU dates from its highest-index member's event
            upto = max(members)
            seen_l = [int(rows["lru_time"][i]) for i in live if i <= upto and int(rows["lru_time"][i]) > 0]
            assert int(st["global_lru"]) == (min(seen_l) if seen_l else LONG_MAX)
        # PARTITION_STATS_COMP (TCM:264-271): free desc, lru asc, capacity desc
        keys = [(-int(s["total_free"]), int(s["global_lru"]), -int(s["total_capacity"])) for s in pstats]
        assert keys == sorted(keys)


# ---------------------------------------------------------------------------------------------------------------
# a14: the rate-tracking task's loop body (MM:5684-5806, getExcludeSet MM:5835-5856, loadedSince MM:5858-5870) and the janitor's
# removeModelCopies / removeSecondModelCopy (MM:6197-6335), per cache entry, as plain Python over dicts -- against
# orc_rate_task_eval / orc_janitor_eval.  Inputs the Java reads from elsewhere (typeSetStats, instanceSetStats, PLACEMENT_ORDER)
# are taken from the oracle's own restatements of those, which other tests pin; what is re-derived here is the arithmetic.
# ---------------------------------------------------------------------------------------------------------------
def brute_rate_entry(e, p, inst_count, have_tc, tstats, loaded, failed, rows, order, order_set):
    """e: cache-entry dict; loaded / failed: [(instance, load time)]; returns the entry's outcome as a dict."""
    o = dict(action=0, copies_to_load=0, load_last_used=0, rpm=0, i1=e["i1"], i2=e["i2"], set_heavy=0)
    if inst_count < 2:
        return o
    time_delta = p["now"] - p["last_check_time"]
    lower, upper = p["iteration"] - p["second_copy_max_age_iters"], p["iteration"] - p["second_copy_min_age_iters"]
    suitable = inst_count
    if have_tc:
        suitable = tstats["instance_count"]
        if suitable < 2:
            return o
    thr = p["scale_up_rpm_threshold"]
    heavy = trunc_div(thr * 3, 4)
    rpm = trunc_div(e["count"] * 60_000, time_delta)
    o["rpm"] = rpm
    if rpm > heavy:
        o["set_heavy"] = 1
    if not loaded:
        return o
    cand = suitable - (len(loaded) + len(failed))
    if cand <= 0:
        return o
    if len(loaded) == 1:
        i1, i2 = e["i1"], e["i2"]
        in1 = in2 = False
        if i2 >= lower and i1 <= upper:
            in1, in2 = i1 >= lower, i2 <= upper
        if in2 or not in1:
            o["i1"] = i2
        o["i2"] = p["iteration"]
        if in1 or in2:
            if tstats["total_capacity"] == 0:
                return o                                                # ArithmeticException, caught at MM:5797
            if trunc_div(10 * tstats["total_free"], tstats["total_capacity"]) >= 1 or \
                    (p["now"] - tstats["global_lru"]) > p["second_copy_lru_threshold_ms"]:
                o.update(action=1, copies_to_load=1, load_last_used=p["last_check_time"])
                return o
    if rpm < thr:
        return o
    cutoff = p["now"] - (time_delta + p["rate_check_interval_ms"] + 2 * p["assume_completed_ms"])
    if any(i != e["instance"] and ts > cutoff for i, ts in loaded):     # loadedSince(mr, cutoff, instanceId)
        return o
    # invokeCounter.getBusyness(): the pod's own request rate; the oracle and the product take the pod's PUBLISHED rpm for it
    # (0 for a pod that is not in the cluster state, e.g. shutting down)
    our_rpm = int(rows[e["instance"]]["rpm"]) if e["instance"] in order_set else 0
    max_rpm = max(thr * 4, our_rpm - 2 * thr)
    exclude = [i for i in order if i != e["instance"] and int(rows[i]["rpm"]) > max_rpm]
    if exclude:
        holders = {i for i, _ in loaded} | {i for i, _ in failed}
        cand -= sum(1 for i in exclude if i not in holders)
        cand -= len(exclude)                                            # (sic: subtracted again, MM:5767)
        if cand <= 0:
            return o
    copies = min(trunc_div(rpm, thr), cand)
    if copies > 2:
        copies = min(copies, suitable // 3)
    o.update(action=2, copies_to_load=copies, load_last_used=p["now"] + 20_000)
    return o


@pytest.mark.parametrize("config,nm,ni,seed", [("C2", 3000, 300, 2), ("C3", 3000, 400, 3), ("C5", 3000, 400, 5), ("MIX", 1500, 160, 14),
                                               ("MIX", 1500, 200, 8)])
def test_scale_arithmetic_parity_unpinned_by_reference_tests(oracle_lib, config, nm, ni, seed):
    import ctypes as C
    rng = np.random.default_rng(seed)
    fl = make_fleet(config, nm, ni, seed)
    keep = np.minimum(fl.edge_off[1:] - fl.edge_off[:-1], 4)
    off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum(keep, out=off[1:])
    inst = np.concatenate([fl.edge_inst[fl.edge_off[m]:fl.edge_off[m] + keep[m]] for m in range(nm)]).astype(np.int32)
    n_loaded = np.minimum(fl.n_loaded, keep).astype(np.int32)
    ts = np.where(rng.uniform(size=len(inst)) < 0.3, fl.now_ms - rng.integers(0, 120_000, size=len(inst)),
                  fl.now_ms - rng.integers(0, 4 * 3_600_000, size=len(inst))).astype(np.int64)
    lul = np.where(rng.uniform(size=nm) < 0.3, fl.now_ms - rng.integers(0, 200_000, size=nm), 0).astype(np.int64)
    o = oracle_from_synth(fl)
    n = 4000
    rec = np.zeros(n, dtype=ob.SCALE_IN)
    models = rng.integers(0, nm, size=n)
    rec["model"] = models
    for r in range(n):
        m = int(models[r]); k = int(n_loaded[m])
        rec["instance"][r] = int(inst[off[m] + rng.integers(0, k)]) if k and rng.uniform() < 0.9 else int(rng.integers(0, ni))
    rec["count"] = np.where(rng.uniform(size=n) < 0.5, rng.integers(0, 50, size=n), rng.integers(0, 20_000, size=n))
    rec["last_used"] = np.where(rng.uniform(size=n) < 0.05, 0, fl.now_ms - rng.integers(0, 40 * 3_600_000, size=n))
    rec["last_heavy"] = np.where(rng.uniform(size=n) < 0.4, 0, fl.now_ms - rng.integers(0, 30 * 3_600_000, size=n))
    rec["flags"] = (rng.uniform(size=n) < 0.15).astype(np.int32)
    it = 5000
    rec["i1"] = it - rng.integers(0, 400, size=n)
    rec["i2"] = np.minimum(it, rec["i1"] + rng.integers(0, 300, size=n))
    m64 = models.astype(np.int64)
    deg = (off[m64 + 1] - off[m64]).astype(np.int64)
    eoff = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(deg, out=eoff[1:])
    einst = np.concatenate([inst[off[m]:off[m + 1]] for m in m64]).astype(np.int32)
    ets = np.concatenate([ts[off[m]:off[m + 1]] for m in m64]).astype(np.int64)
    nl = n_loaded[m64].astype(np.int32)
    tidx = fl.model_type[m64].astype(np.int32)
    lulr = lul[m64].astype(np.int64)
    names = (C.c_char_p * len(fl.type_names))(*[t.encode() for t in fl.type_names])
    # what the brute force reads
    stat_names = ("total_capacity", "total_free", "global_lru", "instance_count", "model_copy_count")
    as_dict = lambda s: {k: int(s[k]) for k in stat_names}
    gst = as_dict(o.cluster_stats())
    have_tc = fl.type_config is not None
    tst = {t: as_dict(o.type_stats(name)) for t, name in enumerate(fl.type_names)}
    order = [int(x) for x in o.cluster_order()]
    order_set = set(order)
    pos = {i: k for k, i in enumerate(order)}
    rows = fl.inst_rows
    sd = [bool(x) for x in rows["shutting_down"]]
    for i in range(ni):
        pos.setdefault(i, 1 << 30)
    pst = {}
    if have_tc:
        ps, pids = o.partition_stats()
        pst = {int(pid): as_dict(s) for s, pid in zip(ps, pids)}
    seen = dict(second=0, scale=0, remove=0)
    for thr, can_remove, lru_thr in ((2000, 1, 6 * 3_600_000), (300, 1, 1000), (5, 0, 6 * 3_600_000)):
        p = np.zeros(1, dtype=ob.SCALE_PARAMS)
        p["now"], p["last_check_time"], p["iteration"], p["scale_up_rpm_threshold"] = fl.now_ms, fl.now_ms - 10_000, it, thr
        p["second_copy_min_age_iters"], p["second_copy_max_age_iters"], p["second_copy_lru_threshold_ms"] = 42, 240, lru_thr
        p["rate_check_interval_ms"], p["assume_completed_ms"], p["second_copy_remove_max_age_ms"], p["can_remove"] = 10_000, 30_000, 36_000_000, can_remove
        pd = {k: int(p[k][0]) for k in p.dtype.names if k != "pad"}
        up, down = np.zeros(n, dtype=ob.SCALE_OUT), np.zeros(n, dtype=ob.SCALE_OUT)
        assert oracle_lib.orc_rate_task_eval(o.h, n, vp(rec), vp(p), names, len(fl.type_names), vp(tidx), vp(eoff), vp(einst), vp(ets), vp(nl), vp(up)) == 0
        assert oracle_lib.orc_janitor_eval(o.h, n, vp(rec), vp(p), vp(eoff), vp(einst), vp(ets), vp(nl), vp(lulr), vp(down)) == 0
        for r in range(n):
            e = {k: int(rec[k][r]) for k in ("instance", "model", "count", "last_used", "last_heavy", "i1", "i2", "flags")}
            edges = [(int(einst[q]), int(ets[q])) for q in range(eoff[r], eoff[r + 1])]
            loaded, failed = edges[:int(nl[r])], edges[int(nl[r]):]
            ty = int(tidx[r])
            b = brute_rate_entry(e, pd, gst["instance_count"], have_tc, tst[ty] if have_tc else gst, loaded, failed, rows, order, order_set)
            for k in ("action", "copies_to_load", "load_last_used", "rpm", "i1", "i2", "set_heavy"):
                assert b[k] == int(up[k][r]), str((thr, r, k, b, [int(up[x][r]) for x in up.dtype.names], ty, len(loaded), len(failed), e))
            if have_tc:
                part = o.instance_partition(e["instance"])
                local = None if (e["flags"] & 1) or part not in pst else pst[part]
            else:
                local = gst
            rm = brute_janitor_entry(e, pd, have_tc, local, loaded, int(lulr[r]), fl.inst_ids, sd, pos)
            assert rm == int(down["remove"][r]), (thr, r, rm, down[r], e)
            seen["second"] += b["action"] == 1
            seen["scale"] += b["action"] == 2
            seen["remove"] += rm
    acc = getattr(test_scale_arithmetic_parity_unpinned_by_reference_tests, "seen", dict(second=0, scale=0, remove=0))
    for k in seen:
        acc[k] += seen[k]
    test_scale_arithmetic_parity_unpinned_by_reference_tests.seen = acc


def test_scale_brute_force_reached_every_outcome():
    seen = getattr(test_scale_arithmetic_parity_unpinned_by_reference_tests, "seen", None)
    if seen is None:
        pytest.skip("runs after the scale brute-force cases")
    assert seen["second"] > 50 and seen["scale"] > 50 and seen["remove"] > 20, seen


@pytest.mark.parametrize("with_types,fill,seed", [(False, 0.95, 4), (True, 0.90, 5), (False, 0.99, 6)])
def test_closed_loop_oracle_conserves_copies_and_capacity(oracle_lib, with_types, fill, seed):
    """Invariants of the closed loop (oracle/mm_sim.inc) after every publish window of a churn trace: the registry holds
    exactly the copies that are resident in the per-instance caches (every admitted load registers, every eviction and removal
    deregisters: MM:5203, 2875-2931), no cache is over its capacity (CLHM:329-352), every eviction names a model that was
    admitted or seeded, and an accepted decision never targets an instance the model already held at the window's start."""
    from modelmesh_b200.synth import make_churn
    w = make_churn(8000, 60, seed, fill=fill, with_types=with_types)
    fl = w.fleet
    o = oracle_from_synth(fl, bulk=False)
    models = np.zeros(fl.n_models, dtype=ob.SIM_MODEL)
    models["last_used"], models["type_idx"], models["size_units"] = fl.model_last_used, fl.model_type, fl.model_size
    sim = ob.OracleSim(o, models, fl.type_names, fl.edge_off, fl.edge_inst, fl.n_loaded, w.capacity, w.load_timeout_ms, fl.now_ms - 60_000)
    order = np.argsort(w.seed_instance, kind="stable")
    bounds = np.searchsorted(w.seed_instance[order], np.arange(fl.n_instances + 1))
    for i in range(fl.n_instances):
        sel = order[bounds[i]:bounds[i + 1]]
        if len(sel):
            sim.seed(i, w.seed_model[sel], w.seed_last_used[sel], w.seed_weight[sel], w.seed_load_ts[sel], fl.now_ms)
    accepted = evicted = 0
    for ep in range(6):
        before = {m: set(int(x) for x in sim.model_copies(m)[0]) for m in range(fl.n_models)} if ep == 0 else after
        ev = w.events(ep, 1200, seed)
        now0 = fl.now_ms + ep * w.window_ms
        dec, evi, rows, npub, carry = sim.step(ev, now0, now0 + w.window_ms, 400 + ep)
        after = {m: set(int(x) for x in sim.model_copies(m)[0]) for m in range(fl.n_models)}
        resident = sum(sim.lru_state(i)[2] for i in range(fl.n_instances))
        assert resident == sum(len(v) for v in after.values()), ep
        for i in range(fl.n_instances):
            assert sim.lru_state(i)[1] <= int(w.capacity[i]), (ep, i)
            assert 0 <= int(rows["used"][i]) <= int(rows["capacity"][i]) + int(w.capacity[i])
        ok = dec[dec["status"] == ob.SIM_ACCEPTED]
        for d in ok:
            t = int(d["self"]) if int(d["target"]) == ob.SELF else int(d["target"])
            assert 0 <= t < fl.n_instances and t not in before[int(d["model"])], (ep, d)
        for e in evi:
            assert 0 <= int(e["model"]) < fl.n_models and 0 <= int(e["instance"]) < fl.n_instances and int(e["weight"]) != 0
        accepted += len(ok); evicted += len(evi)
    assert accepted > 100 and evicted > 50, (accepted, evicted)


# ---------------------------------------------------------------------------------------------------------------
# a6: the converged per-type instance sets of TypeConstraintManager as set comprehensions -- membership as updateInstance
# computes it (TCM:455-486: required = ALL labels, preferred = ANY label, independently), then one refreshPerTypeInstanceSets
# (TCM:680-747): instance scores = 4 x prohibited types - configured preferences, the default preferred set = the top-scoring
# instances (none when all scores are equal), N11: a type WITHOUT required labels gets the default preferred set even when it
# configures preferred labels; a type with required labels and no configured preference gets the top-scoring allowed ones.
# ---------------------------------------------------------------------------------------------------------------
def brute_type_sets(type_config, type_names, labels, live):
    def matches(inst, tl, all_):
        if not labels[inst] or not tl:
            return False
        return all(l in labels[inst] for l in tl) if all_ else any(l in labels[inst] for l in tl)
    # ConfigTypeConstraints (TCM:92-95): both lists sorted and de-duplicated, preferred labels that are also required dropped
    cfg = {t: (sorted(set(c.get("required", []))), sorted(set(c.get("preferred", [])) - set(c.get("required", [])))) for t, c in (type_config or {}).items()}
    allowed = {t: (None if not req else {i for i in live if matches(i, req, True)}) for t, (req, _) in cfg.items()}
    conf_pref = {}
    for t, (_, prf) in cfg.items():
        s = {i for i in live if matches(i, prf, False)}
        conf_pref[t] = s if s else None
    scores = {i: 4 * sum(1 for t in cfg if allowed[t] is not None and i not in allowed[t]) - sum(1 for t in cfg if conf_pref[t] and i in conf_pref[t])
              for i in live}
    def infer(include):
        pool = [i for i in live if include is None or i in include]
        if not pool:
            return None
        mn, mx = min(scores[i] for i in pool), max(max(scores[i] for i in pool), 0)
        top = {i for i in pool if scores[i] >= mx} if any(scores[i] >= mx for i in pool) else set()
        return top if mn < mx and top else None
    default_pref = infer(None)
    out = {}
    for t in type_names:
        if t not in cfg:
            out[t] = (None, default_pref)
        elif allowed[t] is None:
            out[t] = (None, default_pref)                              # N11
        else:
            pref = conf_pref[t] if (conf_pref[t] is not None or not allowed[t]) else infer(allowed[t])
            out[t] = (allowed[t], pref)
    return out


@pytest.mark.parametrize("config,nm,ni,seed", [("C3", 200, 400, 3), ("C3", 200, 97, 4), ("C5", 200, 500, 5), ("C5", 200, 64, 7),
                                               ("MIX", 200, 160, 5), ("MIX", 200, 300, 8), ("MIX", 200, 97, 14), ("MIX", 200, 200, 21)])
def test_type_sets_parity_unpinned_by_reference_tests(oracle_lib, config, nm, ni, seed):
    fl = make_fleet(config, nm, ni, seed)
    if fl.type_config is None:
        pytest.skip("no type constraints drawn")
    o = oracle_from_synth(fl, bulk=False)
    live = [int(x) for x in o.cluster_order()]
    want = brute_type_sets(fl.type_config, fl.type_names, [set(l) for l in fl.inst_labels], live)
    checked = 0
    for name in fl.type_names:
        a, p = o.type_sets(name, fl.n_instances)
        wa, wp = want[name]
        got_a = None if a is None else {int(x) for x in np.nonzero(a)[0]} & set(live)
        got_p = None if p is None else {int(x) for x in np.nonzero(p)[0]} & set(live)
        assert got_a == wa, (name, sorted(got_a or [])[:8], sorted(wa or [])[:8])
        assert (got_p or None) == (wp or None), (name, sorted(got_p or [])[:8], sorted(wp or [])[:8])
        checked += 1
    assert checked == len(fl.type_names)


@pytest.mark.parametrize("mixed_vers", [False, True])
@pytest.mark.parametrize("config,ni,seed", [("C2", 300, 2), ("C3", 400, 3), ("C5", 400, 5), ("MIX", 200, 8), ("MIX", 160, 14), ("MIX", 120, 21)])
def test_placement_order_comparator_parity_unpinned_by_reference_tests(oracle_lib, config, ni, seed, mixed_vers):
    """The oracle's comparator against the Java text re-derived in Python on sampled pairs, with uniform and with mixed
    instance versions (N1's corner: newer-but-saturated instances), equal-key instances included (MIX draws them)."""
    fl = make_fleet(config, 50, ni, seed)
    rng = np.random.default_rng(seed)
    if mixed_vers:
        fl.inst_rows["vers"] = np.where(rng.uniform(size=ni) < 0.4, 8, 7)
    o = oracle_from_synth(fl)
    live = [int(x) for x in o.cluster_order()]
    rows = fl.inst_rows
    seen_tie = 0
    for _ in range(6000):
        a, b = (live[int(k)] for k in rng.integers(0, len(live), 2))
        if a == b:
            continue
        want = brute_compare(rows[a], fl.inst_ids[a], fl.inst_locs[a], fl.inst_zones[a], fl.inst_labels[a],
                             rows[b], fl.inst_ids[b], fl.inst_locs[b], fl.inst_zones[b], fl.inst_labels[b],
                             fl.min_space_units, fl.min_churn_age_ms)
        got = o.compare(a, b)
        assert (got > 0) - (got < 0) == want, (a, b, got, want, rows[a], rows[b])
        ra, rb = rows[a], rows[b]
        seen_tie += all(int(ra[k]) == int(rb[k]) for k in ("count", "capacity", "used", "lru_time", "rpm", "l_in_prog", "l_threads"))
    if not mixed_vers:  # a uniform-vers cluster state is sorted under the re-derived comparator too
        for a, b in zip(live[:-1], live[1:]):
            assert brute_compare(rows[a], fl.inst_ids[a], fl.inst_locs[a], fl.inst_zones[a], fl.inst_labels[a],
                                 rows[b], fl.inst_ids[b], fl.inst_locs[b], fl.inst_zones[b], fl.inst_labels[b],
                                 fl.min_space_units, fl.min_churn_age_ms) < 0


@pytest.mark.parametrize("seed", range(8))
def test_time_ordered_lru_matches_a_plain_list(oracle_lib, seed):
    rng = np.random.default_rng(100 + seed)
    cap = int(rng.integers(20_000, 60_000))
    o, b = ob.OracleLru(cap), BruteLru(cap)
    now = 1_000_000
    evictions = 0
    for batch in range(10):
        n = 400
        ev = np.zeros(n, dtype=ob.LRU_EVENT)
        r = rng.uniform(size=n)
        ev["op"] = np.where(r < 0.45, 0, np.where(r < 0.72, 1, np.where(r < 0.85, 2, np.where(r < 0.94, 3, np.where(r < 0.97, 4, 5)))))
        ev["key"] = rng.integers(0, 120, size=n)
        ev["weight"] = np.where(ev["op"] == 4, rng.integers(15_000, 60_000, size=n), rng.integers(1, 6000, size=n))
        ev["last_used"] = np.where(rng.uniform(size=n) < 0.3, 0, now - rng.integers(0, 500_000, size=n))
        want = o.apply(ev, now)
        got = []
        for i in range(n):
            b.apply(int(ev["op"][i]), int(ev["key"][i]), int(ev["weight"][i]), int(ev["last_used"][i]), i, now, got)
        assert [(int(e["key"]), int(e["event"]), int(e["last_used"]), int(e["weight"])) for e in want] == got, batch
        k, t, w = o.dump()
        assert [list(x) for x in zip(k.tolist(), w.tolist(), t.tolist())] == b.deque, batch
        assert o.weighted_size() == b.wsize and o.oldest_time() == b.oldest and o.size() == len(b.deque), batch
        evictions += len(got)
        now += int(rng.integers(1, 200_000))
    assert evictions > 20
