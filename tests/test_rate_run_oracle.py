"""The oracle composition of one pod's rate-tracking task (tests/rate_run_oracle.py), checked without a GPU on small
hand-built fleets with known answers: both gates at their edges (timeDelta 5 999 / 6 000 ms for a 10 s interval, one
instance), a second copy whose only target is a heavy instance (it takes it; a scale-up of another model does not), chains
that grow their excludes, a chain ended by MMP_TARGET_NONE, a chain cut at 17, decision 0 answered SELF by a pod that does not
hold the model (the chain continues from the pod), and checkLoadFailureCount with failure times at now - expiry / 2 and one
ms after it."""
import numpy as np

import rate_run_oracle as rro
from common import EXPIRY, HOUR
from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import make_fleet
from pod_task_edges import hand_fleet
from pod_tasks import IT, rate_params

def entry(pod, model, rpm=0, second=False, delta=10_000):
    """an entry measuring rpm over delta ms; second: its usage iterations trigger the second-copy check"""
    e = np.zeros(1, dtype=L.SCALE_IN)
    e["instance"], e["model"], e["count"] = pod, model, -(-rpm * delta // 60_000)   # (measured: at least rpm)
    e["last_used"] = 1
    e["i1"], e["i2"] = (IT - 100, IT - 100) if second else (IT - 1000, IT - 1000)
    return e


def by_entry(loads):
    out = {}
    for ld in loads:
        out.setdefault(ld[0], []).append(ld)
    return out


def test_gates_at_their_edges(oracle_lib):
    fl, ts, o = hand_fleet([([(0, 0)], [])], 4)
    now = fl.now_ms
    ents = entry(0, 0, rpm=5000, delta=6000)
    out, loads, rep = rro.rate_run(o, fl, ts, 0, ents, rate_params(now, 1000, delta=5999), 1)
    assert rep["gate"] == L.RATE_TOO_SOON and loads == [] and out["action"][0] == 0 and out["i1"][0] == ents["i1"][0]
    out, loads, rep = rro.rate_run(o, fl, ts, 0, ents, rate_params(now, 1000, delta=6000), 1)
    assert rep["gate"] == L.RATE_RAN and out["action"][0] == 2 and rep["n_scale_up"] == 1 and len(loads) > 0
    out, loads, rep = rro.rate_run(o, fl, ts, 0, ents[:0], rate_params(now, 1000), 1)
    assert rep["gate"] == L.RATE_NO_ENTRIES and loads == []
    o.close()
    fl, ts, o = hand_fleet([([(0, 0)], [])], 1)
    out, loads, rep = rro.rate_run(o, fl, ts, 0, entry(0, 0, rpm=5000), rate_params(fl.now_ms, 1000), 1)
    assert rep["gate"] == L.RATE_FEW_INSTANCES and loads == [] and out["rpm"][0] == 0
    o.close()


def picks(o, fl, m, self_idx, now, excl, seed, n=32):
    """the targets of n draws of getNext(m, self_idx) excluding m's registrations and excl"""
    own = list(fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]]) + list(excl)
    od = np.zeros(n, dtype=rro.ob.DECISION)
    od["self"], od["fresh_idx"], od["last_used"], od["decision_id"] = self_idx, -1, now + 20_000, np.arange(n)
    r = o.get_next_batch(od, fl.type_names, np.arange(n + 1) * len(own), np.tile(np.array(own, dtype=np.int32), n), now, seed)
    return set(int(t) for t in r["target"])


def test_heavy_instance_second_copy_takes_it_scale_up_does_not(oracle_lib):
    """pod P = 0, X = 1..7.  Model 1: copies on P and 1, a scale-up of two.  H: an instance model 1's decision 0 picks
    without a heavy set, made heavy (rpm 5 000 > 4 x 1 000).  Model 0: a copy on P and old failures on every other X: its
    second copy can only go to H."""
    ni = 8
    now = make_fleet("C3", 1, ni, 3).now_ms
    old = now - EXPIRY
    reg1 = ([(0, old), (1, old)], [])
    fl, ts, o = hand_fleet([([(0, old)], []), reg1], ni)
    H = min(picks(o, fl, 1, 0, now, [], 11) - {0, -2})
    o.close()
    rpm = np.zeros(ni, dtype=np.int32)
    rpm[H] = 5000
    fl, ts, o = hand_fleet([([(0, old)], [(x, old) for x in range(1, ni) if x != H]), reg1], ni, rpm=rpm)
    assert H in picks(o, fl, 1, 0, now, [], 11)
    ents = np.concatenate([entry(0, 0, rpm=10, second=True), entry(0, 1, rpm=3000)])
    out, loads, rep = rro.rate_run(o, fl, ts, 0, ents, rate_params(now, 1000), 11)
    assert list(out["action"]) == [1, 2] and rep["n_heavy"] == 1 and rep["n_second"] == 1 and rep["n_scale_up"] == 1
    got = by_entry(loads)
    assert got[0] == [(0, 0, 0, 0, H, got[0][0][5], out["load_last_used"][0], L.RL_SECOND_COPY, 0)]
    assert out["load_last_used"][0] == now - 10_000 and out["load_last_used"][1] == now + 20_000
    chain = got[1]
    assert len(chain) == out["copies_to_load"][1] == 2
    assert all(ld[4] not in (H, L.TARGET_NONE) for ld in chain)
    # the chain grows its excludes: decision 1 is self = target 0 and lands elsewhere
    assert chain[1][3] == chain[0][4] and chain[1][4] != chain[0][4]
    o.close()


def test_chain_ended_by_none(oracle_lib):
    """12 instances, 8 out of the service-instance map: model 0 on P = 0 and 1 asks for 4 copies, 2 and 3 take two, the third
    decision finds nothing and the chain ends"""
    ni = 12
    now = make_fleet("C3", 1, ni, 3).now_ms
    fl, ts, o = hand_fleet([([(0, now - HOUR), (1, now - HOUR)], [])], ni, inactive=range(4, 12))
    out, loads, rep = rro.rate_run(o, fl, ts, 0, entry(0, 0, rpm=4000), rate_params(now, 1000), 5)
    assert out["action"][0] == 2 and out["copies_to_load"][0] == 4
    assert [ld[2] for ld in loads] == [0, 1, 2] and loads[2][4] == L.TARGET_NONE
    assert sorted(ld[4] for ld in loads[:2]) == [2, 3] and rep["n_loads"] == 3 and rep["n_chains_cut"] == 0
    o.close()


def test_chain_cut_at_17(oracle_lib):
    """60 instances, threshold 5: 20 copies wanted (suitable / 3), 17 placed, the last one carries CHAIN_CUT and 3"""
    ni = 60
    now = make_fleet("C3", 1, ni, 3).now_ms
    fl, ts, o = hand_fleet([([(0, now - HOUR), (1, now - HOUR)], [])], ni)
    out, loads, rep = rro.rate_run(o, fl, ts, 0, entry(0, 0, rpm=100_000), rate_params(now, 5), 7)
    assert out["copies_to_load"][0] == 20
    assert [ld[2] for ld in loads] == list(range(17)) and rep["n_chains_cut"] == 1
    assert loads[-1][7] == L.RL_CHAIN_CUT and loads[-1][8] == 3 and all(ld[7] == 0 for ld in loads[:-1])
    targets = [ld[4] for ld in loads]
    assert len(set(targets)) == 17 and not set(targets) & {0, 1}
    assert [ld[3] for ld in loads[1:]] == targets[:-1]
    o.close()


def test_self_answer_continues_from_the_pod(oracle_lib):
    """the pod does not hold the model and is among decision 0's best candidates: a draw that answers SELF, then decision 1
    runs from the pod with the pod among its excludes"""
    ni = 12
    now = make_fleet("C3", 1, ni, 3).now_ms
    fl, ts, o = hand_fleet([([(1, now - HOUR), (2, now - HOUR)], [])], ni)
    P = min(picks(o, fl, 0, 1, now, [], 3) - {1, 2, -1, -2})
    ents = entry(P, 0, rpm=3000)
    # (the pick among the best candidates is a hash of the seed and the id: the first seed whose draw is the pod)
    seed = next(k for k in range(500) if rro.rate_run(o, fl, ts, P, ents, rate_params(now, 1000), k)[1][0][4] == L.TARGET_SELF)
    out, loads, rep = rro.rate_run(o, fl, ts, P, ents, rate_params(now, 1000), seed)
    assert out["action"][0] == 2 and len(loads) >= 2
    assert loads[0][3] == P and loads[0][4] == L.TARGET_SELF
    assert loads[1][3] == P and loads[1][4] not in (P, L.TARGET_SELF, L.TARGET_NONE)
    o.close()


def test_failure_count_gate_edges(oracle_lib):
    now = make_fleet("C3", 1, 8, 3).now_ms
    edge = now - EXPIRY // 2
    regs = [([(0, now - HOUR)], [(2, edge + 1), (3, edge + 1), (4, edge)]),       # two counted: placed
            ([(0, now - HOUR)], [(2, edge + 1), (3, edge + 1), (4, edge + 1)]),   # three: refused
            ([(0, now - HOUR)], [(2, edge + 1), (3, edge + 1), (4, edge + 1)])]   # ... a scale-up too
    fl, ts, o = hand_fleet(regs, 20)
    ents = np.concatenate([entry(0, 0, second=True), entry(0, 1, second=True), entry(0, 2, rpm=3000)])
    out, loads, rep = rro.rate_run(o, fl, ts, 0, ents, rate_params(now, 1000), 9)
    assert list(out["action"]) == [1, 1, 2]
    assert [ld[0] for ld in loads] == [0] and rep["n_refused_failures"] == 2 and rep["n_second"] == 2 and rep["n_scale_up"] == 1
    o.close()
