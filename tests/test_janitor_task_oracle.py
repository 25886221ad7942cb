"""The oracle restatement of the janitor's whole task (tests/janitor_task_oracle.py), checked without a GPU on hand-built
records with known answers: the skips, the out-of-order count across a skipped entry, the early stop (quirk N16) first, in
the middle, last, behind an undone entry, with a record at Long.MAX_VALUE and with no record, the recent-use window and
min_stale_age_ms at their boundaries, matched loaded and failed registrations (the pod's the sixth of seven), each removal
reason, re-registration and what it does to the registry loop, a removed entry, and the saturated copy count.  The hand
cases live in tests/janitor_task_cases.py, so that tests/test_janitor_task_gpu.py runs every one of them on the device."""
import numpy as np
import pytest

import janitor_task_oracle as jto
from common import HOUR, LONG_MAX
from helpers import oracle_from_synth
from janitor_task_cases import CASES, NOW, OLD, matched, removals, reregister, saturated_copy_count, skips, stop_middle, window_edges
from modelmesh_b200 import _lib as L
from pod_tasks import WINDOW


def _whats(out):
    return [w for _, w, _, _ in out]


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
