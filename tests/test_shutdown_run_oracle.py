"""The restatement of one pod's pre-shutdown migration (tests/shutdown_run_oracle.py), checked without a GPU on small
hand-built fleets with known answers, one edge each: lru_t at the cutoff and one ms before it, lruTime at the cutoff for the
wait test, lru_t == 0 falling back to a last_used of -1, 0 and > 0, the pod registered only as a failed load, past its fourth
registration and on a model with more than 16 registrations, 2 and 3 recent failures at the expiry edge, a model with nowhere
left to go, gone, failed and aborted entries, and the only-instance branch."""
import numpy as np

import shutdown_run_oracle as sro
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import NOW_MS
from common import EXPIRY, HOUR
from pod_task_edges import hand_fleet
from pod_tasks import shutdown_params

POD = 0

def ents(*rows):
    """rows of (model, lru_t, last_used, flags)"""
    e = np.zeros(len(rows), dtype=L.SHUTDOWN_ENTRY)
    for r, (m, lru_t, lu, fl) in enumerate(rows):
        e[r] = (m, fl, lru_t, lu)
    return e


def run(regs, ni, rows, seed=5, **kw):
    fl, ts, o = hand_fleet(regs, ni, **kw)
    out, rep = sro.shutdown_run(o, fl, ts, POD, ents(*rows), shutdown_params(fl.now_ms), seed)
    o.close()
    return fl, out, rep


def held(n_models, others=(1,), t=None):
    """n_models models loaded on the pod and `others`"""
    return [([(POD, t or 0)] + [(i, t or 0) for i in others], []) for _ in range(n_models)]


PLACED_WAIT = L.SD_REMOVE_LOCAL | L.SD_PLACED | L.SD_WAIT


def test_cutoff_edges_stale_and_wait(oracle_lib):
    now = NOW_MS
    cut = now - HOUR
    fl, out, rep = run(held(4), 12, [(0, cut, -1, 0), (1, cut - 1, -1, 0), (2, 0, cut, 0), (3, 0, cut - 1, 0)])
    assert list(out["what"]) == [PLACED_WAIT, L.SD_STALE | L.SD_REMOVE_LOCAL | L.SD_PLACED,
                                 L.SD_STALE | PLACED_WAIT, L.SD_STALE | L.SD_REMOVE_LOCAL | L.SD_PLACED]
    assert list(out["last_used"]) == [cut, cut - 1, cut, cut - 1]
    assert all(t >= 2 for t in out["target"])
    assert rep == dict(found_other=1, n_registered=4, will_be_skipped=3, n_placed=4, n_none=0, n_refused=0, n_wait=2)


def test_lru_zero_falls_back_to_last_used(oracle_lib):
    now = NOW_MS
    fl, out, rep = run(held(3), 12, [(0, 0, -1, 0), (1, 0, 0, 0), (2, 0, now - 5000, 0)])
    assert list(out["what"]) == [L.SD_STALE, L.SD_STALE | L.SD_REMOVE_LOCAL, L.SD_STALE | PLACED_WAIT]
    assert list(out["last_used"]) == [-1, 0, now - 5000]
    assert list(out["target"][:2]) == [L.TARGET_INVALID] * 2 and out["target"][2] >= 2
    assert rep["n_placed"] == 1 and rep["will_be_skipped"] == 3


def test_registered_means_a_loaded_registration_anywhere_in_the_record(oracle_lib):
    """model 0: the pod only as a failed load; model 1: the pod as the sixth loaded copy; model 2: 20 registrations (17
    loaded, 3 failed) with the pod the 17th loaded; model 3: no record"""
    ni = 40
    now = NOW_MS
    t = now - HOUR
    regs = [([(1, t)], [(POD, t)]),
            ([(i, t) for i in (1, 2, 3, 4, 5, POD)], []),
            ([(i, t) for i in range(1, 17)] + [(POD, t)], [(i, t) for i in (17, 18, 19)]),
            ([], [])]
    fl, out, rep = run(regs, ni, [(m, now - 1000, -1, 0) for m in range(4)])
    assert list(out["what"]) == [L.SD_NOT_REGISTERED, PLACED_WAIT, PLACED_WAIT, L.SD_NOT_REGISTERED]
    assert out["target"][1] not in (1, 2, 3, 4, 5, POD) and out["target"][1] >= 0
    assert out["target"][2] >= 20
    assert list(out["last_used"]) == [0, now - 1000, now - 1000, 0]
    assert rep["n_registered"] == 2 and rep["n_placed"] == 2 and rep["n_wait"] == 2


def test_failure_count_at_the_expiry_edge(oracle_lib):
    now = NOW_MS
    edge = now - EXPIRY // 2
    regs = [([(POD, 0)], [(2, edge + 1), (3, edge + 1), (4, edge)]),       # two counted: placed
            ([(POD, 0)], [(2, edge + 1), (3, edge + 1), (4, edge + 1)])]   # three: refused
    fl, out, rep = run(regs, 20, [(0, now - 1, -1, 0), (1, now - 1, -1, 0)])
    assert list(out["what"]) == [PLACED_WAIT, L.SD_REMOVE_LOCAL | L.SD_REFUSED]
    assert out["target"][1] == L.TARGET_INVALID and out["n_candidates"][1] == 0
    assert rep["n_refused"] == 1 and rep["n_placed"] == 1


def test_nowhere_left_is_none_and_no_wait(oracle_lib):
    """six instances: the model is loaded on 0-3 and failed on 4 and 5"""
    now = NOW_MS
    fl, out, rep = run([([(i, 0) for i in range(4)], [(4, 0), (5, 0)])], 6, [(0, now - 1, -1, 0)])
    assert out["what"][0] == L.SD_REMOVE_LOCAL | L.SD_PLACED and out["target"][0] == L.TARGET_NONE
    assert rep["n_none"] == 1 and rep["n_wait"] == 0


def test_gone_failed_and_aborted_entries(oracle_lib):
    now = NOW_MS
    rows = [(0, now - 1, -1, L.SD_ENTRY_GONE), (1, now - 1, -1, L.SD_ENTRY_FAILED), (2, now - 1, -1, L.SD_ENTRY_ABORTED),
            (3, 0, -1, L.SD_ENTRY_ABORTED), (4, 1, -1, L.SD_ENTRY_GONE | L.SD_ENTRY_ABORTED)]
    fl, out, rep = run(held(5), 12, rows)
    assert list(out["what"]) == [0, 0, PLACED_WAIT | L.SD_DEREGISTER_NOW, L.SD_STALE | L.SD_DEREGISTER_NOW, L.SD_STALE]
    assert list(out["last_used"]) == [0, 0, now - 1, -1, 0]
    assert rep == dict(found_other=1, n_registered=5, will_be_skipped=2, n_placed=1, n_none=0, n_refused=0, n_wait=1)


def test_an_answer_does_not_depend_on_the_other_entries(oracle_lib):
    now = NOW_MS
    rows = [(m, now - 1000 * m - 1, -1, 0) for m in range(8)]
    _, out, _ = run(held(8, others=(1, 2)), 40, rows, seed=11)
    rows2 = [(m, lru, lu, L.SD_ENTRY_GONE if m % 2 else 0) for m, lru, lu, _ in rows]
    _, out2, _ = run(held(8, others=(1, 2)), 40, rows2, seed=11)
    assert list(out2["target"][::2]) == list(out["target"][::2]) and all(t >= 3 for t in out["target"])


def test_only_instance_places_nothing(oracle_lib):
    now = NOW_MS
    fl, out, rep = run(held(2, others=()), 1, [(0, now - 1, -1, 0), (1, now - 1, -1, L.SD_ENTRY_ABORTED)])
    assert list(out["what"]) == [0, 0] and list(out["target"]) == [L.TARGET_INVALID] * 2
    assert rep == dict(found_other=0, n_registered=0, will_be_skipped=0, n_placed=0, n_none=0, n_refused=0, n_wait=0)
