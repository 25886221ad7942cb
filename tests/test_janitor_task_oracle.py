"""The oracle restatement of the janitor's whole task (tests/janitor_task_oracle.py), checked without a GPU on hand-built
records with known answers: the skips, the out-of-order count across a skipped entry, the early stop (quirk N16) first, in
the middle, last, behind an undone entry, with a record at Long.MAX_VALUE and with no record, the recent-use window and
min_stale_age_ms at their boundaries, matched loaded and failed registrations (the pod's the sixth of seven), each removal
reason, re-registration and what it does to the registry loop, a removed entry, and the saturated copy count.  The hand
cases live in CASES, so that tests/test_janitor_task_gpu.py runs every one of them on the device."""
import numpy as np
import pytest

import janitor_task_oracle as jto
from helpers import oracle_from_synth
from modelmesh_b200 import _lib as L
from pod_task_edges import _janitor_self, janitor_hand_fleet
from test_janitor_run_oracle import EXPIRY, HOUR, LONG_MAX, params as run_params

FREQ_S, LOAD_TIMEOUT = 360, 30_000
WINDOW = FREQ_S * 2000 + LOAD_TIMEOUT     # 750 000 ms
MIN_STALE = 6 * HOUR + 123_456


def params(now, adjusted_capacity=1 << 40, flags=0, min_stale=MIN_STALE, freq=FREQ_S, timeout=LOAD_TIMEOUT):
    p = np.zeros(1, dtype=L.JANITOR_TASK_PARAMS)
    p["janitor"] = run_params(now, adjusted_capacity, flags)[0]
    p["janitor"]["scale"]["second_copy_remove_max_age_ms"] = 36 * HOUR
    p["min_stale_age_ms"], p["janitor_freq_secs"], p["load_timeout_ms"] = min_stale, freq, timeout
    return p


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
        self.params = params(NOW, **kw)

    def run(self):
        o = oracle_from_synth(self.fl)
        try:
            return jto.janitor_task(o, self.fl, self.ts, self.lul, self.S, self.entries, self.params)
        finally:
            o.close()


def _whats(out):
    return [w for _, w, _, _ in out]


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


# ------------------------------------------------------------------------------------------------------------- the answers


def test_skips_and_out_of_order(oracle_lib):
    c = skips()
    out, edits, rep = c.run()
    assert _whats(out)[1:4] == [L.JC_NOT_DONE, L.JC_NOT_CACHED, L.JC_NOT_CACHED]
    # entry 4 (now - 1 h) follows entry 0 (now - 2 h) across the skipped ones: out of order; entry 0 is first (MAX before it)
    assert _whats(out)[4] & L.JC_OUT_OF_ORDER and not _whats(out)[0] & L.JC_OUT_OF_ORDER
    assert rep["n_out_of_order"] == 1 and rep["n_not_done"] == 1 and rep["n_not_cached"] == 2
    assert rep["registry_ran"] == 1 and rep["stopped_at"] == -1 and rep["cache_changed"] == 0
    # the undone entry (model 1) and the uncached ones are candidates or not as the registry loop reads them
    assert rep["registry"]["n_referencing"] == 5


@pytest.mark.parametrize("name,stop,repair", [("stop_first", 0, True), ("stop_middle", 2, False), ("stop_last", 2, True),
                                              ("stop_no_record", 1, False), ("stop_behind_undone", 1, True)])
def test_the_stop(oracle_lib, name, stop, repair):
    c = CASES[name]()
    out, edits, rep = c.run()
    forced = c.now - 3 * HOUR
    assert rep["stopped_at"] == stop and rep["registry_ran"] == 0 and edits == [] and rep["n_stop"] == 1
    assert rep["registry"] == dict(n_referencing=0, n_edits=0, n_candidates=0, n_removed=0, weight_removed=0)
    m, w, lu, _ = out[stop]
    assert w & L.JC_STOP and lu == forced and bool(w & L.JC_REPAIR) == repair
    assert all(x[1] == L.JC_NOT_REACHED for x in out[stop + 1:]) and rep["n_not_reached"] == len(out) - stop - 1
    assert all(not x[1] & (L.JC_STOP | L.JC_NOT_REACHED) for x in out[:stop])


def test_stop_middle_keeps_the_earlier_writes(oracle_lib):
    out, _, rep = stop_middle().run()
    assert out[0][1] == L.JC_REREGISTER and out[1][1] & L.JC_OUT_OF_ORDER  # (now - 2 h after now - 10 h)
    assert rep["n_reregister"] == 1


def test_window_and_min_stale(oracle_lib):
    c = window_edges()
    out, edits, rep = c.run()
    w = [x & ~L.JC_OUT_OF_ORDER for x in _whats(out)]
    assert w[0] == L.JC_STALE_UPDATE and out[0][2] == c.now - WINDOW + 1
    assert w[2] == 0 and out[2][2] == int(c.fl.model_last_used[2])
    assert w[3] == 0 and out[3][2] == LONG_MAX
    assert w[4] == L.JC_STALE_UPDATE
    # entry 1 is past the window: its registration time does not match (+ 7), so it is re-registered
    assert w[1] & L.JC_REREGISTER and out[1][3] == OLD + 1


def test_matched_registrations(oracle_lib):
    c = matched()
    out, _, rep = c.run()
    assert out[0][1] == L.JC_STALE_UPDATE and out[0][2] == c.now - HOUR           # the sixth of seven, matched
    assert out[1][1] & L.JC_STALE_UPDATE and not out[1][1] & L.JC_REMOVE          # failed entry matched on load_complete_ts
    assert out[2][1] & ~L.JC_OUT_OF_ORDER == 0 and out[2][2] == c.now - HOUR      # matched, the record is fresh


def test_each_removal_reason(oracle_lib):
    c = removals()
    out, edits, rep = c.run()
    assert [w & L.JC_REMOVE for w in _whats(out)] == [L.JC_REMOVE] * 4 and rep["cache_changed"] == 1 and rep["n_remove"] == 4
    assert out[2][2] == 0  # no record
    got = {m: w for m, w, _, _ in edits}
    # model 0 and 1: present, not failed, lastUsed -1: no candidate, no edit; model 2: failed, lastUsed -1: the full expiry
    assert 0 not in got and 1 not in got and 2 not in got
    assert rep["registry"]["n_candidates"] == 0
    # the same entries without the cache pass's removals: 0 and 1 are candidates, 2's failure takes the in-use expiry
    c2 = removals()
    c2.entries["e"]["flags"] &= np.uint32(0xffffffff & ~(L.JANITOR_NOT_LIVE | L.JANITOR_UNLOAD_RECENT))
    c2.entries["e"]["last_used"][3] = c2.now - 1000  # (recent: skipped by the cache loop, so the registry loop reads it)
    _, edits2, rep2 = c2.run()
    assert rep2["registry"]["n_candidates"] >= 1 and {m: w for m, w, _, _ in edits2}.get(2) == L.JE_DROP_FAILURE | L.JE_REMOVE_LOCAL


def test_reregistration_and_the_registry_loop(oracle_lib):
    c = reregister()
    out, edits, rep = c.run()
    assert _whats(out) == [L.JC_REREGISTER] * 7
    assert [r for _, _, _, r in out] == [-1, OLD + 1, -1, -1, -1, -1, -1]
    assert [lu for _, _, lu, _ in out] == [NOW - (10 + m) * HOUR for m in range(7)]
    got = {m: (w, lu, lul) for m, w, lu, lul in edits}
    assert not any(w & L.JE_DROP_FAILURE for w, _, _ in got.values())   # the re-registration dropped model 2's failure
    # every non-failed one is a scale-down candidate now; the pod's second copies (models 1, 2 and 4) scale down, leaving 1
    assert rep["registry"]["n_candidates"] == 5 and rep["registry"]["n_referencing"] == 7
    for m in (1, 2, 4):
        assert got[m] == (L.JE_SCALE_DOWN, NOW - (10 + m) * HOUR, 0)
    # the failed entries' re-registered copies are unregistered: updateLastUnloadTime with 2 copies left, then with 3
    assert got[5] == (L.JE_UNREGISTER, NOW - 15 * HOUR, 0) and got[6] == (L.JE_UNREGISTER, NOW - 16 * HOUR, NOW)
    # on the committed records none of this happens: model 2's failure record goes, 5 and 6 have nothing to unregister
    o = oracle_from_synth(c.fl)
    edits0, rep0 = jto.jro.janitor_run(o, c.fl, c.ts, c.lul, c.S, np.array([t["e"] for t in c.entries], dtype=L.JANITOR_ENTRY),
                                       np.array([c.params[0]["janitor"]]))
    o.close()
    got0 = {m: w for m, w, _, _ in edits0}
    assert got0.get(2) == L.JE_DROP_FAILURE and 5 not in got0 and 6 not in got0 and rep0["n_candidates"] == 1


def test_saturated(oracle_lib):
    c = saturated_copy_count()
    out, edits, rep = c.run()
    assert out[0][1] == L.JC_UNDECIDED and rep["n_undecided"] == 1
    assert {m: w for m, w, _, _ in edits}.get(0) == L.JE_UNDECIDED


def test_every_bit_is_reached():
    seen = 0
    for name, make in CASES.items():
        out, _, _ = make().run()
        for _, w, _, _ in out:
            seen |= w
    assert seen == (1 << 10) - 1, bin(seen)
