"""The widened fast-path rule of k_place_split on the device (DESIGN.md §5.2.1): keys over every live candidate edge of a
model, inline and overflow, and selves that are not candidates of their slot left out of the test.  Batches are placed
with the two-pass path forced on (split = 1) and off (split = 0): the two must be byte identical, and both equal the
oracle.  Besides the bench-like fleets and split_widen.front_cases, keys are checked after a device-path commit that moves
the hand-built models' exclusions across the candidate line, and after closed-loop windows that re-lay the overflow
table, so that a key left from the epoch before would show."""
import numpy as np
import pytest

from churn_harness import build, compare_window
from helpers import oracle_from_synth, solver_from_synth
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthDecisions, make_churn, make_churn_overflow, make_decisions, make_fleet
from replay import NUMERIC, Replay, assert_same_results, oracle_batch
from split_widen import GROUPS, front_cases
from upgrade import upgrade

pytestmark = pytest.mark.gpu


def _place(f, lib, sd, now, seed, split):
    f._ck(lib.mmp_tune(f.h, b"split", split))
    try:
        return f.place_batch(sd.dec, now, seed, fresh=sd.fresh if len(sd.fresh) else None,
                             extra=sd.extra if len(sd.extra) else None)
    finally:
        f._ck(lib.mmp_tune(f.h, b"split", 2))


def _on_off(f, lib, sd, now, seed, what):
    """The batch placed with the two passes and with one launch.  The two passes launch k_slot_summary, k_place_split and
    k_place_tail where one launch runs k_place_direct: a call that takes neither (a batch small enough for the mapped
    tiny-batch path ignores the knob) would launch as many kernels either way."""
    n0 = f.kernel_launches()
    on = _place(f, lib, sd, now, seed, 1)
    n1 = f.kernel_launches()
    off = _place(f, lib, sd, now, seed, 0)
    n2 = f.kernel_launches()
    assert n1 - n0 >= 3 and n1 - n0 > n2 - n1, (what, n1 - n0, n2 - n1)
    assert on.tobytes() == off.tobytes(), (what, int(np.sum(on != off)))
    return on


CASES = [("C2", 2000, 400, 2, None), ("C3", 3000, 1300, 33, None), ("C5", 1500, 500, 5, None), ("MIX", 800, 300, 14, None),
         ("MIX", 800, 700, 41, None), ("C3", 3000, 1300, 33, "half"), ("MIX", 800, 300, 14, "saturated")]


@pytest.mark.parametrize("config,nm,ni,seed,pattern", CASES)
def test_split_on_off_and_oracle(product_lib, oracle_lib, config, nm, ni, seed, pattern):
    fl = make_fleet(config, nm, ni, seed)
    if pattern is not None:
        fl = upgrade(fl, pattern, seed)
    o = oracle_from_synth(fl)
    s = solver_from_synth(fl, product_lib)
    fav = make_decisions(fl, 2000, seed + 3, sweep=True, plain=True)
    fav.dec["flags"] |= L.DF_FAVOUR_SELF
    for k, sd in enumerate((make_decisions(fl, 3000, seed, sweep=True, plain=True), fav, make_decisions(fl, 2000, seed + 1))):
        on = _on_off(s, product_lib, sd, fl.now_ms, seed + k, (config, pattern, k))
        assert_same_results(on, oracle_batch(fl, sd, o, seed + k), (config, pattern, k))
    s.close()


def _front_lists(rank, allowed):
    order = np.argsort(np.where(rank >= 0, rank, np.iinfo(np.int64).max))[:int(np.sum(rank >= 0))]
    return order[~allowed[order]], order[allowed[order]]


def test_hand_built_cases_and_a_device_path_commit(product_lib, oracle_lib):
    fl, sd, group, rank, allowed = front_cases()
    # repeated past the mapped tiny-batch path's size (16 KB of records and results), so that the batch reaches the
    # launch that takes the split knob; each copy is numbered apart, so its picks differ
    n_cases = len(sd.dec)
    reps = -(-1024 // n_cases)
    sd = SynthDecisions(np.tile(sd.dec, reps), sd.fresh, sd.extra)
    rp = Replay(fl, product_lib, 33)
    _on_off(rp.f, product_lib, sd, rp.now, 5, "load")
    assert_same_results(_place(rp.f, product_lib, sd, rp.now, 5, 1), oracle_batch(rp.view(), sd, rp.oracle(), 5), "load")
    # across the candidate line: the models without exclusions (A, B) take the first candidate, the overflow models whose
    # fifth id is the first candidate (E) take non-candidates at the front and candidates at the back instead
    non, cand = _front_lists(rank, allowed)
    edits = 0
    for i, d in enumerate(sd.dec[:n_cases]):
        g = GROUPS[group[i]]
        if g in "AB":
            rp.upsert_model(int(d["model"]), [int(cand[0])])
        elif g == "E":
            rp.upsert_model(int(d["model"]), [int(x) for x in non[:3]] + [int(x) for x in cand[::-1][:3]])
        else:
            continue
        edits += 1
    assert rp.commit(NUMERIC, edits) == 2
    for k in range(2):
        on = _on_off(rp.f, product_lib, sd, rp.now, 6 + k, ("device path", k))
        assert_same_results(on, oracle_batch(rp.view(), sd, rp.oracle(), 6 + k), ("device path", k))
        sd.dec["flags"] ^= np.uint32(L.DF_FAVOUR_SELF)
    rp.f.close()


def test_after_windows_that_re_lay_the_overflow_table(product_lib, oracle_lib):
    """Closed-loop windows on a fleet whose models hold more than four registrations (the window re-lays the overflow
    table and commits on the device): after each, a sweep over every model with the two-pass path on and off."""
    w = make_churn_overflow(make_churn(20_000, 200, 4, fill=0.9), 0.05, 4)
    fl = w.fleet
    o, sim, s = build(product_lib, w, slots=256)
    rng = np.random.default_rng(4)
    for ep in range(3):
        ev = w.events(ep, 2000, 4)
        now0 = fl.now_ms + ep * w.window_ms
        compare_window(ep, o, sim, s, ev, now0, now0 + w.window_ms, 400 + ep)
        dec = np.zeros(fl.n_models, dtype=L.DECISION_IN)
        dec["model"] = np.arange(fl.n_models)
        dec["self"] = rng.integers(0, fl.n_instances, size=fl.n_models)
        dec["flags"] = np.where(rng.uniform(size=fl.n_models) < 0.3, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(L.DF_MODEL_LAST_USED)
        dec["fresh"] = -1
        sd = SynthDecisions(dec, np.zeros(0, dtype=L.INSTANCE_ROW), np.zeros(0, dtype=np.int32))
        on = _on_off(s, product_lib, sd, now0 + w.window_ms, 40 + ep, ep)
        assert np.count_nonzero(on["target"] >= 0) > 0, ep
    s.close()
