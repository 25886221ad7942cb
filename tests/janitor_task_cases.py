"""The hand-built cases of the janitor's whole task, as data: each @case function returns a HandCase (a fleet whose models hold
exactly the registrations it lists, the pod, the entries in cache order and the task's parameters), so that
tests/test_janitor_task_oracle.py checks their known answers on the restatement and tests/test_janitor_task_gpu.py runs every
one of them on the device."""
import numpy as np

import janitor_task_oracle as jto
from common import EXPIRY, HOUR, LONG_MAX
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from pod_task_edges import _janitor_self, janitor_hand_fleet
from pod_tasks import MIN_STALE, WINDOW, janitor_task_params


def tentry(model, last_used, load_ts=0, load_complete_ts=0, failed=False, not_done=False, not_live=False, unload_recent=False,
           weight=10, last_heavy=0, count=0):
    t = np.zeros(1, dtype=L.JANITOR_TASK_ENTRY)
    e = t["e"]
    e["model"], e["weight"], e["last_used"], e["load_ts"], e["last_heavy"], e["count"] = model, weight, last_used, load_ts, last_heavy, count
    e["flags"] = ((L.JANITOR_FAILED if failed else 0) | (L.JANITOR_NOT_DONE if not_done else 0) | (L.JANITOR_NOT_LIVE if not_live else 0)
                  | (L.JANITOR_UNLOAD_RECENT if unload_recent else 0))
    t["e"] = e
    t["load_complete_ts"] = load_complete_ts
    return t


NOW = 1_760_000_000_000   # the hand fleets' now (synth's)
OLD = NOW - 2 * HOUR
S_, A_ = _janitor_self()     # the least desirable pod of the janitor's fleet (it drops the second copies) and another
OTHERS = [i for i in range(24) if i not in (S_, A_)]


class HandCase:
    """a fleet whose models hold exactly regs[m] (loaded [(instance, ts)], failed [(instance, ts)]), record lastUsed rec_lu
    {m: value}, the pod S_, the entries in cache order, the task's params; extra_models: model indices past the fleet's
    models, without a record"""

    def __init__(self, name, regs, entries, rec_lu=None, extra_models=0, ni=24, **kw):
        self.name, self.S, self.now, self.old = name, S_, NOW, OLD
        self.fl, self.ts = janitor_hand_fleet(regs, ni=ni)
        assert int(self.fl.now_ms) == NOW
        for m, v in (rec_lu or {}).items():
            self.fl.model_last_used[m] = v
        self.lul = np.zeros(self.fl.n_models, dtype=np.int64)
        self.max_models = self.fl.n_models + extra_models
        self.entries = np.concatenate(entries)
        self.params = janitor_task_params(NOW, **kw)

    def run(self):
        o = oracle_from_synth(self.fl)
        try:
            return jto.janitor_task(o, self.fl, self.ts, self.lul, self.S, self.entries, self.params)
        finally:
            o.close()


def _pairs(n):
    """n models, each loaded on A and on the pod, the pod's registration at OLD + m"""
    return [([(A_, OLD), (S_, OLD + m)], []) for m in range(n)]


CASES = {}


def case(fn):
    CASES[fn.__name__] = fn
    return fn


@case
def skips():
    # not done, last_used 0 and -1: skipped, nothing written; the out-of-order count runs across them
    return HandCase("skips", _pairs(5), [tentry(0, NOW - 2 * HOUR, load_ts=OLD), tentry(1, NOW - HOUR, not_done=True), tentry(2, 0),
                                         tentry(3, -1), tentry(4, NOW - HOUR, load_ts=OLD + 4)])


@case
def stop_first():
    return HandCase("stop_first", _pairs(4), [tentry(0, LONG_MAX), tentry(1, NOW - HOUR, load_ts=OLD + 1), tentry(2, NOW - 2 * HOUR),
                                              tentry(3, LONG_MAX)], rec_lu={0: LONG_MAX})


@case
def stop_middle():
    return HandCase("stop_middle", _pairs(4), [tentry(0, NOW - 10 * HOUR, load_ts=OLD + 1), tentry(1, NOW - 2 * HOUR, load_ts=OLD + 1),
                                               tentry(2, LONG_MAX), tentry(3, NOW - 9 * HOUR)])


@case
def stop_last():
    return HandCase("stop_last", _pairs(3), [tentry(0, NOW - HOUR, load_ts=OLD), tentry(1, NOW - 2 * HOUR, load_ts=OLD + 1),
                                             tentry(2, LONG_MAX)], rec_lu={2: LONG_MAX})


@case
def stop_no_record():
    return HandCase("stop_no_record", _pairs(2), [tentry(0, NOW - HOUR, load_ts=OLD), tentry(3, LONG_MAX)], extra_models=4)


@case
def stop_behind_undone():
    # an undone Long.MAX_VALUE entry is skipped; the stop is the next one that passes the skips
    return HandCase("stop_behind_undone", _pairs(3), [tentry(0, LONG_MAX, not_done=True), tentry(1, LONG_MAX), tentry(2, NOW - HOUR)],
                    rec_lu={0: LONG_MAX, 1: LONG_MAX})


@case
def window_edges():
    # now - last_used = window - 1.. (recent: the stale test only) and = window (past it: the registration check); lu - rec
    # at min_stale (written), one short (not), one past (written); a record lastUsed of Long.MAX_VALUE (lu - MAX wraps
    # negative: not written)
    lu = [NOW - WINDOW + 1, NOW - WINDOW, NOW - WINDOW + 2, NOW - WINDOW + 3, NOW - WINDOW + 4]
    rec = {0: lu[0] - MIN_STALE, 2: lu[2] - MIN_STALE + 1, 3: LONG_MAX, 4: lu[4] - MIN_STALE - 1}
    return HandCase("window_edges", _pairs(5), [tentry(0, lu[0]), tentry(1, lu[1], load_ts=OLD + 1 + 7), tentry(2, lu[2]), tentry(3, lu[3]),
                                                tentry(4, lu[4])], rec_lu=rec)


@case
def matched():
    # the pod's loaded registration the sixth of seven, matched (stale update); a failed entry matched on its failure
    # record's time (load_complete_ts); a loaded registration matched with the record fresh: nothing
    regs = [([(OTHERS[k], OLD + k) for k in range(5)] + [(S_, OLD + 5), (OTHERS[5], OLD + 6)], []),
            ([(A_, OLD)], [(S_, NOW - 3 * HOUR)]),
            ([(A_, OLD), (S_, OLD + 2)], [])]
    return HandCase("matched", regs, [tentry(0, NOW - HOUR, load_ts=OLD + 5),
                                      tentry(1, NOW - HOUR - 1, failed=True, load_complete_ts=NOW - 3 * HOUR, not_live=True),
                                      tentry(2, NOW - HOUR - 2, load_ts=OLD + 2)],
                    rec_lu={0: NOW - 30 * HOUR, 1: NOW - 30 * HOUR, 2: NOW - HOUR})


@case
def removals():
    # not live, unload attempted recently, no record, and a failed entry (not live) whose failure time does not match: each
    # removes; the registry loop then reads lastUsed -1 for them
    regs = [([(A_, OLD), (S_, OLD)], []), ([(A_, OLD), (S_, OLD + 1)], []), ([(A_, OLD)], [(S_, NOW - EXPIRY // 2 - 10)])]
    return HandCase("removals", regs, [tentry(0, NOW - HOUR, load_ts=OLD + 1, not_live=True),
                                       tentry(1, NOW - HOUR - 5, load_ts=OLD + 2, unload_recent=True), tentry(5, NOW - HOUR - 6, load_ts=1),
                                       tentry(2, NOW - HOUR - 7, failed=True, not_live=True, load_complete_ts=1)], extra_models=4)


@case
def reregister():
    # no prior registration (a model with none), a mismatched time, a fresh failure record the re-registration drops, the
    # pod as a third copy and as a second copy; every one becomes a scale-down candidate
    regs = [([], []),                                            # 0 no registration at all: the pod becomes the only copy
            ([(A_, OLD), (S_, OLD + 1)], []),                    # 1 mismatched time: replaced, still 2 copies
            ([(A_, OLD)], [(S_, NOW - 1000)]),                   # 2 a fresh failure record: dropped by the re-registration
            ([(A_, OLD), (OTHERS[0], OLD)], []),                 # 3 two others: the pod is the third copy
            ([(A_, OLD)], []),                                   # 4 one other: the pod is the second copy
            ([(A_, OLD), (OTHERS[0], OLD)], []),                 # 5, 6 a failed entry that is not flagged out of LOADING..ACTIVE:
            ([(A_, OLD), (OTHERS[0], OLD), (OTHERS[1], OLD)], [])]  # re-registered, then unregistered with 2 / 3 copies left
    return HandCase("reregister", regs, [tentry(m, NOW - (10 + m) * HOUR, load_ts=OLD + 100 + m) for m in range(5)]
                    + [tentry(m, NOW - (10 + m) * HOUR, load_ts=OLD + 100 + m, failed=True) for m in (5, 6)],
                    rec_lu={m: NOW - 40 * HOUR for m in range(7)})


@case
def saturated_copy_count():
    ids = [i for i in range(320) if i != S_]
    regs = [([(i, OLD) for i in ids[:279]] + [(S_, OLD)], [(i, OLD) for i in ids[279:299]]), ([(A_, OLD), (S_, OLD + 1)], [])]
    return HandCase("saturated_copy_count", regs, [tentry(0, NOW - 3 * HOUR, load_ts=1), tentry(1, NOW - 4 * HOUR, load_ts=OLD + 1)], ni=320)
