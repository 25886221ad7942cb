"""The hand-built cases of the four pod tasks -- mmp_janitor_run, mmp_rate_run, mmp_shutdown_run and mmp_evict_run -- as data,
so that the same fleets, entries and parameters run through the restatements without a GPU (tests/test_*_run_oracle.py,
tests/test_pod_task_edges_oracle.py) and on the device (tests/test_pod_task_edges_gpu.py).

A Case is one call: the task, the fleet (a SynthFleet whose registrations were set by hand), the time of every registration,
lastUnloadTime per model, the pod, the entries, the parameters, the seed and the pod's fresh row.
  * hand_cases() runs every hand-built test of the four tests/test_*_run_oracle.py files, which assert their known answers
    on the restatement, and records each restatement call they make as a Case with the answer it gave;
  * all_pairs() are the edges those files miss, each written as two cases, one on each side of its line, with the part of the
    answer that tells the sides apart (the CPU test checks that it does);
  * saturated_cases() are the calls on a model whose copy count is saturated (280 loaded copies + 20 failed loads)."""
import copy
import dataclasses
import hashlib
import inspect
from typing import Any, Optional

import numpy as np

import evict_run_oracle as ero
import janitor_run_oracle as jro
import rate_run_oracle as rro
import shutdown_run_oracle as sro
from common import HOUR, LONG_MAX
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import NOW_MS, make_fleet
from pod_tasks import HAND_TIMEOUT, IT, evict_params, janitor_params, rate_params, shutdown_params

LONG_MIN = -(1 << 63)
TASKS = ("janitor", "rate", "shutdown", "evict")


def _set_edges(fl, regs):
    inst, ts, off, nl, nf = [], [], [0], [], []
    for loaded, failed in regs:
        for i, t in loaded + failed:
            inst.append(i)
            ts.append(t)
        off.append(len(inst))
        nl.append(len(loaded))
        nf.append(len(failed))
    fl.edge_inst, fl.edge_off = np.array(inst, dtype=np.int32), np.array(off, dtype=np.int64)
    fl.n_loaded, fl.n_failed = np.array(nl, dtype=np.int32), np.array(nf, dtype=np.int32)
    fl.model_last_used[:] = fl.now_ms - HOUR
    return np.array(ts, dtype=np.int64)


def hand_fleet(regs, ni, seed=3, rpm=None, inactive=()):
    """(fleet, times, oracle): a C3 fleet half full with no type constraints whose models hold exactly regs[m] = (loaded
    [(instance, ts)], failed [(instance, ts)]); rpm: per instance published rpm; inactive: instances out of the
    service-instance map (they count, but no decision can pick them).  The rate, shutdown and eviction cases use it."""
    fl = make_fleet("C3", len(regs), ni, seed)
    fl.type_config = None
    fl.type_names = fl.type_names[:1]
    fl.model_type[:] = 0
    fl.inst_rows["rpm"] = 0 if rpm is None else rpm
    fl.inst_rows["used"] = fl.inst_rows["capacity"] // 2
    fl.inst_rows["shutting_down"] = 0
    fl.inst_rows["active"] = 1
    for i in inactive:
        fl.inst_rows["active"][i] = 0
    ts = _set_edges(fl, regs)
    return fl, ts, oracle_from_synth(fl)


def janitor_hand_fleet(regs, seed=3, ni=24):
    """(fleet, times): a C3 fleet 2 % from full whose models hold exactly regs[m] = (loaded [(instance, ts)], failed
    [(instance, ts)])"""
    fl = make_fleet("C3", len(regs), ni, seed)
    fl.inst_rows["used"] = fl.inst_rows["capacity"] - fl.inst_rows["capacity"] // 50
    return fl, _set_edges(fl, regs)


# ---------------------------------------------------------------------------------------------------------------- cases

@dataclasses.dataclass
class Case:
    task: str                      # one of TASKS
    fl: Any
    ts: np.ndarray                 # the time of every registration of fl.edge_inst
    lul: np.ndarray                # lastUnloadTime per model
    pod: int
    entries: np.ndarray
    params: np.ndarray
    seed: int = 0
    fresh: Optional[np.ndarray] = None
    name: str = ""
    want: Any = None               # the restatement's answer, once run

    def fleet_key(self) -> str:
        """the device fleet a case runs on: equal keys, equal fleets"""
        fl, h = self.fl, hashlib.sha1()
        for a in (fl.inst_rows, fl.edge_inst, fl.edge_off, fl.n_loaded, fl.model_last_used, fl.model_type, self.ts, self.lul):
            h.update(np.ascontiguousarray(a).tobytes())
        h.update(repr((fl.type_config, fl.type_names, fl.inst_ids, fl.replaced_replicasets, fl.n_models)).encode())
        return h.hexdigest()


def restate(c: Case, o=None):
    """the restatement's answer to c: janitor (edits, report); rate (out, loads, report); shutdown / evict (out, report)"""
    own = o is None
    o = oracle_from_synth(c.fl) if own else o
    try:
        if c.task == "janitor":
            return jro.janitor_run(o, c.fl, c.ts, c.lul, c.pod, c.entries, c.params)
        if c.task == "rate":
            return rro.rate_run(o, c.fl, c.ts, c.pod, c.entries, c.params, c.seed, fresh_self=c.fresh)
        if c.task == "shutdown":
            return sro.shutdown_run(o, c.fl, c.ts, c.pod, c.entries, c.params, c.seed, fresh_self=c.fresh)
        return ero.evict_run(o, c.fl, c.ts, c.lul, c.pod, c.entries, c.params, c.seed, fresh_self=c.fresh)
    finally:
        if own:
            o.close()


def solved(c: Case) -> Case:
    c.want = restate(c)
    return c


# the hand-built tests of the four files, each of which makes at least one restatement call through its module
# (jro.janitor_run, rro.rate_run, sro.shutdown_run, ero.evict_run); test_pod_task_edges_oracle.py checks that the list names
# every test of those files but the random one, so a test added there is added here too
HAND_BUILT = {
    "test_janitor_run_oracle": ("test_known_answers",),
    "test_rate_run_oracle": ("test_gates_at_their_edges", "test_heavy_instance_second_copy_takes_it_scale_up_does_not",
                             "test_chain_ended_by_none", "test_chain_cut_at_17", "test_self_answer_continues_from_the_pod",
                             "test_failure_count_gate_edges"),
    "test_shutdown_run_oracle": ("test_cutoff_edges_stale_and_wait", "test_lru_zero_falls_back_to_last_used",
                                 "test_registered_means_a_loaded_registration_anywhere_in_the_record",
                                 "test_failure_count_at_the_expiry_edge", "test_nowhere_left_is_none_and_no_wait",
                                 "test_gone_failed_and_aborted_entries", "test_an_answer_does_not_depend_on_the_other_entries",
                                 "test_only_instance_places_nothing"),
    "test_evict_run_oracle": ("test_reload_needs_an_age_past_twice_the_timeout", "test_failed_entry_is_deregistered_and_not_reloaded",
                              "test_load_ts_that_does_not_match_writes_nothing_but_still_reloads",
                              "test_pod_only_in_failed_in_reloads_from_the_failure_time", "test_no_registration_of_the_pod",
                              "test_rebalance_gate_at_its_edges", "test_a_live_copy_elsewhere_is_a_forward_and_a_gone_one_is_not",
                              "test_failure_count_after_the_edit", "test_update_last_used_and_last_unload_time",
                              "test_registrations_past_the_fourth"),
}
NOT_HAND_BUILT = {"test_remove_model_copies_matches_brute_force"}   # (orc_janitor_eval on a random fleet: no task call)


def hand_cases(oracle_lib):
    """every restatement call of the HAND_BUILT tests, as Cases (named module::test) with the answers the tests checked.
    (The seed search of test_self_answer_continues_from_the_pod makes a call per seed it tries: each is a case.)"""
    import importlib
    cases, current = [], [""]
    mods = {"janitor": (jro, "janitor_run"), "rate": (rro, "rate_run"), "shutdown": (sro, "shutdown_run"), "evict": (ero, "evict_run")}
    saved = {t: getattr(m, f) for t, (m, f) in mods.items()}

    def recorder(task):
        real = saved[task]
        names = list(inspect.signature(real).parameters)

        def rec(*a, **kw):
            args = dict(zip(names, a), **kw)
            res = real(*a, **kw)
            lul = args.get("lul")
            fl = copy.deepcopy(args["fl"])
            cases.append(Case(task, fl, np.array(args["ts"], dtype=np.int64).copy(),
                              np.zeros(fl.n_models, dtype=np.int64) if lul is None else np.array(lul, dtype=np.int64).copy(),
                              int(args.get("pod", args.get("self_idx"))), args["entries"].copy(), np.array(args["params"]).copy(),
                              int(args.get("seed", 0)), None if args.get("fresh_self") is None else np.array(args["fresh_self"]).copy(),
                              current[0], copy.deepcopy(res)))
            return res
        return rec

    try:
        for t, (m, f) in mods.items():
            setattr(m, f, recorder(t))
        for mod_name, tests in HAND_BUILT.items():
            mod = importlib.import_module(mod_name)
            for name in tests:
                current[0] = f"{mod_name}::{name}"
                before = len(cases)
                getattr(mod, name)(oracle_lib)
                assert len(cases) > before, f"{current[0]} made no restatement call through its module"
    finally:
        for t, (m, f) in mods.items():
            setattr(m, f, saved[t])
    return cases


# ------------------------------------------------------------------------------------------------------- the edge pairs

def evict_entries(*rows):
    """rows of (model, last_used, load_ts, load_complete_ts, flags)"""
    e = np.zeros(len(rows), dtype=L.EVICT_ENTRY)
    for r, (m, lu, lt, lct, f) in enumerate(rows):
        e[r] = (m, f, lu, lt, lct)
    return e


def shutdown_entries(*rows):
    """rows of (model, lru_t, last_used, flags)"""
    e = np.zeros(len(rows), dtype=L.SHUTDOWN_ENTRY)
    for r, (m, lru_t, lu, f) in enumerate(rows):
        e[r] = (m, f, lru_t, lu)
    return e


def rate_entry(pod, model, rpm=0, second=False, delta=10_000):
    """an entry measuring at least rpm over delta ms; second: its usage iterations trigger the second-copy check"""
    e = np.zeros(1, dtype=L.SCALE_IN)
    e["instance"], e["model"], e["count"] = pod, model, -(-rpm * delta // 60_000)
    e["last_used"] = 1
    e["i1"], e["i2"] = (IT - 100, IT - 100) if second else (IT - 1000, IT - 1000)
    return e


def janitor_entry(model, last_used, weight=10, load_ts=0, failed=False):
    e = np.zeros(1, dtype=L.JANITOR_ENTRY)
    e["model"], e["weight"], e["last_used"], e["load_ts"] = model, weight, last_used, load_ts
    e["flags"] = L.JANITOR_FAILED if failed else 0
    return e


def _hand(task, regs, ni, entries, params, seed=5, lul=None, edit=None, pod=0, fresh=None, rpm=None, name=""):
    """a Case on hand_fleet(regs, ni); edit(fl) changes the instance rows first"""
    fl, ts, o = hand_fleet(regs, ni, seed=3, rpm=rpm)
    o.close()
    if edit is not None:
        edit(fl)
    lul = np.zeros(len(regs), dtype=np.int64) if lul is None else np.asarray(lul, dtype=np.int64)
    return Case(task, fl, ts, lul, pod, entries, params, seed, fresh, name)


def _janitor(S, regs, entries, params):
    fl, ts = janitor_hand_fleet(regs)
    return Case("janitor", fl, ts, np.zeros(len(regs), dtype=np.int64), S, entries, params)


def _janitor_self():
    """the least desirable pod of the janitor's fleet (it drops the second copies) and three others"""
    fl0 = make_fleet("C3", 1, 24, 3)
    fl0.inst_rows["used"] = fl0.inst_rows["capacity"] - fl0.inst_rows["capacity"] // 50
    o0 = oracle_from_synth(fl0)
    order = [int(x) for x in o0.cluster_order()]
    o0.close()
    return order[-1], order[0]


def _shut(fl, *i):
    fl.inst_rows["shutting_down"][list(i)] = 1


def _what(res):
    return [int(w) for w in res[0]["what"]]


def evict_pairs():
    now, old = NOW_MS, NOW_MS - 2 * HAND_TIMEOUT - 1
    P = 0
    one = [([(P, old)], [])]
    row = evict_entries((0, now - 10, old, 0, 0))
    pairs = []

    def big_rows(cap, used):
        def edit(fl):
            fl.inst_rows["capacity"][:3], fl.inst_rows["used"][:3] = cap, used
        return edit
    # three instances of 2^56 free: 20 * totalFree stays a long and the gate is open ...
    clear = _hand("evict", one, 12, row, evict_params(), edit=big_rows(1 << 56, 0))
    # ... of 3 * 2^61 with 2 * 2^61 free: totalCapacity wraps to 2^61 + the rest, totalFree to -2^62 + the rest, and 20 *
    # totalFree to 20 x the rest: 20 * free / cap reads 0
    pairs.append(("evict/gate-free-wrap", _hand("evict", one, 12, row, evict_params(), edit=big_rows(3 << 61, 1 << 61)), clear,
                  _what))
    # ... of 5 * 2^60, full: totalCapacity wraps negative
    pairs.append(("evict/gate-cap-negative", _hand("evict", one, 12, row, evict_params(), edit=big_rows(5 << 60, 5 << 60)),
                  copy.deepcopy(clear), _what))
    # 2 x load_timeout_ms wraps: 2^62 -> Long.MIN_VALUE, every age is past it; 2^62 - 1 -> no age is
    pairs.append(("evict/timeout-wrap",
                  _hand("evict", one, 12, row, evict_params(timeout=1 << 62)),
                  _hand("evict", one, 12, row, evict_params(timeout=(1 << 62) - 1)), _what))
    # registration times Long.MIN_VALUE (now - t wraps negative) and Long.MAX_VALUE against an old one
    for t, tag in ((LONG_MIN, "min"), (LONG_MAX, "max")):
        pairs.append((f"evict/reg-time-{tag}",
                      _hand("evict", [([(P, t)], [])], 12, evict_entries((0, now - 10, t, 0, 0)), evict_params()),
                      _hand("evict", one, 12, row, evict_params()), _what))
    # an odd expiry (900 001: half is 450 000): a third failure at exactly now - 450 000 is not counted, one ms after it is
    since = now - 450_000
    fails = lambda t3: [([(P, old)], [(2, since + 1), (3, since + 1), (4, t3)])]
    pairs.append(("evict/odd-expiry",
                  _hand("evict", fails(since), 12, row, evict_params(expiry=900_001)),
                  _hand("evict", fails(since + 1), 12, row, evict_params(expiry=900_001)), _what))
    # the pod loaded and failed on one model: the reload age reads the loaded registration (young here) ...
    young = now - 1000
    pairs.append(("evict/loaded-and-failed",
                  _hand("evict", [([(P, young)], [(P, old)])], 12, evict_entries((0, now - 10, young, old, 0)), evict_params()),
                  _hand("evict", [([(P, old)], [(P, young)])], 12, evict_entries((0, now - 10, old, young, 0)), evict_params()),
                  _what))
    # entry last_used Long.MAX_VALUE (updateLastUsed takes it, the decision carries it) and negative (the record keeps its own)
    pairs.append(("evict/last-used",
                  _hand("evict", one, 12, evict_entries((0, LONG_MAX, old, 0, 0)), evict_params()),
                  _hand("evict", one, 12, evict_entries((0, -5, old, 0, 0)), evict_params()),
                  lambda res: [int(x) for x in res[0]["last_used"]]))
    # the gate on a type-constrained fleet: each type set's own stats.  Type "ta" requires label ta (instances 1-4) and
    # has 20 * free / cap == 1, type "tb" label tb (5-8) and 0; model 2's type "plain" has no constraints and reads the
    # whole cluster (the unlabelled instances 0 and 9-11 half full)
    typed = [([(P, old)], []) for _ in range(3)]
    pairs.append(("evict/type-gate",
                  _hand("evict", typed, 12, evict_entries((0, now - 10, old, 0, 0), (2, now - 10, old, 0, 0)), evict_params(),
                        edit=_type_sets),
                  _hand("evict", typed, 12, evict_entries((1, now - 10, old, 0, 0), (2, now - 10, old, 0, 0)), evict_params(),
                        edit=_type_sets), _what))
    return pairs


TYPE_CAP = 1_000_000


def _type_sets(fl):
    """types plain / ta / tb on models 2 / 0 / 1; ta (instances 1-4) exactly a twentieth free, tb (5-8) one unit less"""
    fl.type_names = ["plain", "ta", "tb"]
    fl.model_type[:] = [1, 2, 0]
    fl.type_config = {"ta": {"required": ["ta"]}, "tb": {"required": ["tb"]}}
    fl.inst_labels = [["ta"] if 1 <= i <= 4 else ["tb"] if 5 <= i <= 8 else [] for i in range(fl.n_instances)]
    fl.inst_rows["capacity"] = TYPE_CAP
    fl.inst_rows["used"] = TYPE_CAP // 2
    fl.inst_rows["used"][1:9] = TYPE_CAP
    fl.inst_rows["used"][1] = TYPE_CAP - 4 * TYPE_CAP // 20
    fl.inst_rows["used"][5] = TYPE_CAP - 4 * TYPE_CAP // 20 + 1


def shutdown_pairs():
    now, P = NOW_MS, 0
    held = [([(P, 0), (1, 0)], []) for _ in range(2)]
    rows = shutdown_entries((0, now - 1000, -1, 0), (1, 0, now - 5000, 0))
    pairs = []
    # now - cutoff_age_ms wraps: to Long.MAX_VALUE every lru_t is stale; one ms further it wraps to Long.MIN_VALUE, none is
    edge = -(LONG_MAX - now)
    pairs.append(("shutdown/cutoff-wrap",
                  _hand("shutdown", held, 12, rows, shutdown_params(cutoff_age=edge)),
                  _hand("shutdown", held, 12, rows, shutdown_params(cutoff_age=edge - 1)), _what))
    # lru_t = Long.MIN_VALUE: lruTime < 0, nothing removed or placed; lru_t = 1: placed
    pairs.append(("shutdown/lru-min",
                  _hand("shutdown", held, 12, shutdown_entries((0, LONG_MIN, -1, 0)), shutdown_params()),
                  _hand("shutdown", held, 12, shutdown_entries((0, 1, -1, 0)), shutdown_params()), _what))

    # found_other with one ranked instance: the pod (nothing evaluated), or another (the pod places from its fresh row)
    def only(ranked):
        return lambda fl: _shut(fl, 1 - ranked)
    two = [([(0, 0), (1, 0)], [])]
    fl_probe, _, o = hand_fleet(two, 2)
    o.close()
    fresh1 = fl_probe.inst_rows[1].copy()
    fresh1["shutting_down"] = 0
    pairs.append(("shutdown/found-other",
                  _hand("shutdown", two, 2, shutdown_entries((0, now - 1000, -1, 0)), shutdown_params(), edit=only(0), pod=0),
                  _hand("shutdown", two, 2, shutdown_entries((0, now - 1000, -1, 0)), shutdown_params(), edit=only(0), pod=1,
                        fresh=fresh1),
                  lambda res: (res[1]["found_other"], _what(res))))
    return pairs


def rate_pairs():
    now, P, thr = NOW_MS, 0, 1000
    one = [([(P, now - HOUR), (1, now - HOUR)], [])]
    up = rate_entry(P, 0, rpm=3000)
    pairs = []
    rpm_at = lambda x: np.array([0] * 5 + [x] + [0] * 6, dtype=np.int32)
    # getExcludeSet: a published rpm exactly at max(4 thr, ourRpm - 2 thr) is not heavy, one above it is
    pairs.append(("rate/exclude-bound",
                  _hand("rate", one, 12, up, rate_params(now, thr), rpm=rpm_at(4000), seed=3),
                  _hand("rate", one, 12, up, rate_params(now, thr), rpm=rpm_at(4001), seed=3),
                  lambda res: res[2]["n_heavy"]))
    # the pod's own rpm (10 000) raises the bound to 8 000 while it is ranked; unranked it reads 0 and the bound is 4 000
    r = rpm_at(5000)
    r[P] = 10_000
    fl_probe, _, o = hand_fleet(one, 12, rpm=r)
    o.close()
    fresh = fl_probe.inst_rows[P].copy()
    pairs.append(("rate/unranked-pod",
                  _hand("rate", one, 12, up, rate_params(now, thr), rpm=r, seed=3),
                  _hand("rate", one, 12, up, rate_params(now, thr), rpm=r, seed=3, edit=lambda fl: _shut(fl, P), fresh=fresh),
                  lambda res: res[2]["n_heavy"]))
    # chains of 16, 17 (the longest a call places) and 18 copies (cut after 17)
    chain = lambda k: _hand("rate", one, 60, rate_entry(P, 0, rpm=k * thr), rate_params(now, thr), seed=7)
    pairs.append(("rate/chain-16-17", chain(16), chain(17), lambda res: len(res[1])))
    pairs.append(("rate/chain-17-18", chain(17), chain(18), lambda res: res[2]["n_chains_cut"]))
    pairs.append(("rate/self-fresh-row", *_self_answer_pair(), lambda res: [int(ld[4]) for ld in res[1]]))
    return pairs


def _self_answer_pair():
    """a chain whose decision 0 is answered MMP_TARGET_SELF and goes on from the pod (decision 1 has self = the pod), without
    a fresh row; and the same call with a fresh row that shows the pod full, which changes the chain's targets.  (Decision 0
    is the only one a chain's SELF can answer: decision j >= 1 has self = target j - 1, which the chain excludes, and
    favourSelf returns SELF only for a self that is not excluded.)  The pod does not hold the model; the pod and the seed
    are the first for which both hold"""
    now, ni = NOW_MS, 12
    regs = [([(1, now - HOUR), (2, now - HOUR)], [])]
    fl, ts, o = hand_fleet(regs, ni)
    try:
        for pod in range(3, ni):
            full = fl.inst_rows[pod].copy()
            full["used"] = full["capacity"]
            ent = rate_entry(pod, 0, rpm=3000)
            for seed in range(200):
                _, loads, _ = rro.rate_run(o, fl, ts, pod, ent, rate_params(now, 1000), seed)
                if len(loads) < 2 or loads[0][4] != L.TARGET_SELF:
                    continue
                _, with_row, _ = rro.rate_run(o, fl, ts, pod, ent, rate_params(now, 1000), seed, fresh_self=full)
                if [ld[4] for ld in with_row] == [ld[4] for ld in loads]:
                    continue
                a = _hand("rate", regs, ni, ent, rate_params(now, 1000), seed=seed, pod=pod)
                b = _hand("rate", regs, ni, ent, rate_params(now, 1000), seed=seed, pod=pod, fresh=full)
                return a, b
    finally:
        o.close()
    raise AssertionError("no draw answers SELF")


def janitor_pairs():
    S, A = _janitor_self()
    now = NOW_MS
    old = now - 2 * HOUR
    regs = [([(A, old), (S, old + m)], []) for m in range(4)]
    first = janitor_entry(0, now - 40_000, weight=5, load_ts=old)
    second = lambda w: janitor_entry(1, now - 30_000, weight=w, load_ts=old + 1)
    removed = lambda res: [m for m, w, _, _ in res[0] if w & L.JE_SCALE_DOWN]
    pairs = []
    # the budget (adjusted_capacity / 20 = 100): after a first removal of 5, a weight of 95 fits and 96 does not
    pairs.append(("janitor/budget-equal",
                  _janitor(S, regs, np.concatenate([first, second(95)]), janitor_params(now, 2000)),
                  _janitor(S, regs, np.concatenate([first, second(96)]), janitor_params(now, 2000)), removed))
    # adjusted_capacity not a multiple of 20: 1 999 / 20 = 99, so 95 no longer fits after 5
    pairs.append(("janitor/capacity-odd",
                  _janitor(S, regs, np.concatenate([first, second(95)]), janitor_params(now, 1999)),
                  _janitor(S, regs, np.concatenate([first, second(95)]), janitor_params(now, 2000)), removed))
    # an equal-lastUsed run whose lowest-index model does not remove (its load_ts does not match): the TreeSet keeps it and
    # drops the removable one (N15); with distinct lastUsed values the removable one goes
    T = now - 50_000
    pairs.append(("janitor/n15-first-keeps",
                  _janitor(S, regs, np.concatenate([janitor_entry(2, T, load_ts=old + 1), janitor_entry(3, T, load_ts=old + 3)]),
                           janitor_params(now, 2000)),
                  _janitor(S, regs, np.concatenate([janitor_entry(2, T, load_ts=old + 1), janitor_entry(3, T + 1, load_ts=old + 3)]),
                           janitor_params(now, 2000)), removed))
    # a candidate key of Long.MAX_VALUE (used "in the future": not removed) against an old one
    pairs.append(("janitor/key-long-max",
                  _janitor(S, regs, janitor_entry(0, LONG_MAX, load_ts=old), janitor_params(now, 2000)),
                  _janitor(S, regs, janitor_entry(0, now - 40_000, load_ts=old), janitor_params(now, 2000)), removed))
    return pairs


def saturation_pairs():
    """the saturation line itself: 255 loaded copies and no failed load (copy_count 255 over 255 registrations: decided)
    against 255 + 1 (over 256: undecided), the pod the first copy, for each task"""
    now, P = NOW_MS, 0
    ni = 300
    t = now - HOUR
    regs = lambda nf: [([(i, t) for i in range(255)], [(255 + i, t) for i in range(nf)])]
    a, b = regs(0), regs(1)
    sd, ev, up = shutdown_entries((0, now - 1000, -1, 0)), evict_entries((0, now - 10, t, 0, 0)), rate_entry(P, 0, rpm=3000)
    return [("saturation/shutdown", _hand("shutdown", a, ni, sd, shutdown_params()), _hand("shutdown", b, ni, sd, shutdown_params()), _what),
            ("saturation/evict", _hand("evict", a, ni, ev, evict_params()), _hand("evict", b, ni, ev, evict_params()), _what),
            ("saturation/rate", _hand("rate", a, ni, up, rate_params(now, 1000), seed=3),
             _hand("rate", b, ni, up, rate_params(now, 1000), seed=3), lambda res: [int(x) for x in res[0]["action"]])]


def all_pairs():
    """(name, case a, case b, the part of the answer that tells them apart), every case solved by the restatement"""
    out = []
    for make in (evict_pairs, shutdown_pairs, rate_pairs, janitor_pairs, saturation_pairs):
        for name, a, b, sig in make():
            a.name, b.name = name + "/a", name + "/b"
            out.append((name, solved(a), solved(b), sig))
    return out


# --------------------------------------------------------------------------------------------------- saturated records

SAT_NI = 320


def saturated_fleet():
    """(fleet, times, lastUnloadTime, pod, models): three models of 280 loaded copies + 20 failed loads (copy_count 255 over
    300 registrations) with the pod at loaded position 10, at loaded position 270 and as the failed load at 290, the
    loaded copies at positions 260-262 loaded recently (within expiry / 2, so a count that read them as failures would
    refuse), everything else an hour old; and a fourth model, 3 loaded + 3 recent failures with the pod the first copy,
    that decides as usual beside them"""
    P = 0
    now = NOW_MS
    old, recent = now - HOUR, now - 1000
    rng = np.random.default_rng(7)
    regs = []
    for pos in (10, 270, 290):
        ids = [int(i) for i in rng.permutation(np.arange(1, SAT_NI))[:299]]
        ids.insert(pos, P)
        loaded = [(i, recent if 260 <= j <= 262 else old) for j, i in enumerate(ids[:280])]
        failed = [(i, old) for i in ids[280:]]
        regs.append((loaded, failed))
    regs.append(([(P, old), (1, old), (2, old)], [(3, recent), (4, recent), (5, old)]))
    fl, ts, o = hand_fleet(regs, SAT_NI)
    o.close()
    fl.inst_rows["rpm"] = 0
    lul = np.array([now - 7, now - 8, now - 9, 0], dtype=np.int64)
    return fl, ts, lul, P


def saturated_cases():
    """one call of each task over the three saturated models and the ordinary one, solved"""
    fl, ts, lul, P = saturated_fleet()
    now = NOW_MS
    t = lambda m: int(ts[int(fl.edge_off[m]) + [10, 270, 290, 0][m]])
    cases = [
        Case("shutdown", fl, ts, lul, P, shutdown_entries(*[(m, now - 1000, -1, 0) for m in range(4)]), shutdown_params(), 5),
        Case("evict", fl, ts, lul, P,
             evict_entries(*[(m, now - 10, t(m) if m != 2 else 0, t(m) if m == 2 else 0, 0) for m in range(4)]), evict_params(), 5),
        Case("rate", fl, ts, lul, P, np.concatenate([rate_entry(P, m, rpm=3000) for m in range(4)]), rate_params(now, 1000), 5),
        Case("janitor", fl, ts, lul, P,
             np.concatenate([janitor_entry(m, now - 40_000, load_ts=t(m)) for m in range(4)]), janitor_params(now, 2000)),
    ]
    for c in cases:
        c.name = "saturated/" + c.task
        solved(c)
    return cases
