"""The edge cases of tests/pod_task_edges.py on the restatements, without a GPU:
  * every pair answers differently on its two sides, so a case that misses its line fails here rather than passing
    silently on the device (tests/test_pod_task_edges_gpu.py runs both sides there);
  * a model whose copy count is saturated (280 loaded copies + 20 failed loads, copy_count 255) is undecided in every task,
    wherever the pod sits in it, and the model beside it decides as usual;
  * the hand-built cases of the four tests/test_*_run_oracle.py files are recorded as data, and together with the pairs
    they reach every MMP_JE_* / MMP_SD_* / MMP_EV_* bit."""
import pytest

import pod_task_edges as pe
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import NOW_MS

JE_BITS = (L.JE_UNREGISTER, L.JE_DROP_FAILURE, L.JE_REMOVE_LOCAL, L.JE_SCALE_DOWN, L.JE_UNDECIDED)
SD_BITS = (L.SD_NOT_REGISTERED, L.SD_STALE, L.SD_REMOVE_LOCAL, L.SD_DEREGISTER_NOW, L.SD_PLACED, L.SD_REFUSED, L.SD_WAIT,
           L.SD_UNDECIDED)
EV_BITS = (L.EV_UNREGISTER, L.EV_DROP_FAILURE, L.EV_RELOAD, L.EV_CLUSTER_FULL, L.EV_LOADED_ELSEWHERE, L.EV_REFUSED, L.EV_PLACED,
           L.EV_UNDECIDED)


def whats(c):
    """the MMP_*_ bits a solved case's answer holds, OR-ed over its entries"""
    if c.task == "janitor":
        return [int(w) for _, w, _, _ in c.want[0]]
    if c.task in ("shutdown", "evict"):
        return [int(w) for w in c.want[0]["what"]]
    return []


def bits_missing(cases):
    seen = {t: 0 for t in ("janitor", "shutdown", "evict")}
    for c in cases:
        for w in whats(c):
            seen[c.task] |= w
    want = {"janitor": JE_BITS, "shutdown": SD_BITS, "evict": EV_BITS}
    return {t: [b for b in want[t] if not seen[t] & b] for t in seen if any(not seen[t] & b for b in want[t])}


@pytest.fixture(scope="module")
def pairs(oracle_lib):
    return pe.all_pairs()


def test_every_pair_answers_differently(pairs):
    names = [name for name, _, _, _ in pairs]
    assert len(set(names)) == len(names)
    for name, a, b, sig in pairs:
        assert sig(a.want) != sig(b.want), (name, sig(a.want))


def test_pairs_on_the_lines_they_name(pairs):
    """the side each pair's known answer is on"""
    got = {name: (sig(a.want), sig(b.want)) for name, a, b, sig in pairs}
    UR = L.EV_UNREGISTER | L.EV_RELOAD
    assert got["evict/gate-free-wrap"] == ([UR | L.EV_CLUSTER_FULL], [UR | L.EV_PLACED])
    assert got["evict/gate-cap-negative"] == ([UR | L.EV_CLUSTER_FULL], [UR | L.EV_PLACED])
    assert got["evict/timeout-wrap"] == ([UR | L.EV_PLACED], [L.EV_UNREGISTER])
    assert got["evict/reg-time-min"][0] == [L.EV_UNREGISTER] and got["evict/reg-time-max"][0] == [L.EV_UNREGISTER]
    assert got["evict/odd-expiry"] == ([UR | L.EV_PLACED], [UR | L.EV_REFUSED])
    assert got["evict/loaded-and-failed"][0] == [L.EV_UNREGISTER | L.EV_DROP_FAILURE]
    assert got["evict/last-used"] == ([pe.LONG_MAX], [NOW_MS - pe.HOUR])
    assert got["shutdown/lru-min"][0] == [L.SD_STALE]
    assert got["shutdown/found-other"][0] == (0, [0]) and got["shutdown/found-other"][1][0] == 1
    assert got["rate/exclude-bound"] == (0, 1) and got["rate/unranked-pod"] == (0, 1)
    a, b = next((a, b) for name, a, b, _ in pairs if name == "rate/self-fresh-row")
    assert got["rate/self-fresh-row"][0][0] == L.TARGET_SELF and a.want[1][1][3] == a.pod and b.fresh is not None
    assert got["evict/type-gate"] == ([UR | L.EV_PLACED] * 2, [UR | L.EV_CLUSTER_FULL, UR | L.EV_PLACED])
    assert got["rate/chain-16-17"] == (16, 17) and got["rate/chain-17-18"] == (0, 1)
    assert got["janitor/budget-equal"] == ([0, 1], [0]) and got["janitor/capacity-odd"] == ([0], [0, 1])
    assert got["janitor/n15-first-keeps"] == ([], [3]) and got["janitor/key-long-max"] == ([], [0])
    assert got["saturation/shutdown"][1] == [L.SD_UNDECIDED] and got["saturation/evict"][1] == [L.EV_UNDECIDED]
    assert got["saturation/rate"] == ([2], [-1])


def test_saturated_records_are_undecided(oracle_lib):
    now = NOW_MS
    by = {c.task: c for c in pe.saturated_cases()}
    out, rep = by["shutdown"].want
    assert list(out["what"][:3]) == [L.SD_UNDECIDED] * 3 and list(out["target"][:3]) == [L.TARGET_INVALID] * 3
    assert out["what"][3] == L.SD_REMOVE_LOCAL | L.SD_PLACED | L.SD_WAIT and out["target"][3] >= 6
    assert rep["n_registered"] == 1 and rep["n_placed"] == 1 and rep["n_refused"] == 0
    out, rep = by["evict"].want
    assert list(out["what"][:3]) == [L.EV_UNDECIDED] * 3
    assert list(out["last_used"][:3]) == [now - pe.HOUR] * 3 and list(out["last_unload_time"][:3]) == [now - 7, now - 8, now - 9]
    assert out["what"][3] == L.EV_UNREGISTER | L.EV_RELOAD | L.EV_LOADED_ELSEWHERE
    assert rep["n_unregister"] == 1 and rep["n_reload"] == 1 and rep["n_placed"] == 0
    out, loads, rep = by["rate"].want
    assert list(out["action"]) == [-1, -1, -1, 2] and list(out["rpm"][:3]) == [0] * 3
    assert {ld[0] for ld in loads} == {3} and rep["n_scale_up"] == 1
    edits, rep = by["janitor"].want
    assert [(m, w) for m, w, _, _ in edits if m < 3] == [(m, L.JE_UNDECIDED) for m in range(3)]
    assert rep["n_referencing"] == 4


def test_hand_built_cases_are_data(oracle_lib, pairs):
    import importlib
    for mod_name, tests in pe.HAND_BUILT.items():
        mod = importlib.import_module(mod_name)
        assert set(tests) == {n for n in dir(mod) if n.startswith("test_")} - pe.NOT_HAND_BUILT, mod_name
    cases = pe.hand_cases(oracle_lib)
    assert {c.task for c in cases} == set(pe.TASKS)
    assert {c.name for c in cases} == {f"{m}::{t}" for m, ts in pe.HAND_BUILT.items() for t in ts}
    sat = pe.saturated_cases()
    assert bits_missing(cases + [c for _, a, b, _ in pairs for c in (a, b)] + sat) == {}
