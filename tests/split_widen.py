"""Hand-built decisions for the widened fast-path rule of k_place_split (DESIGN.md §5.2.1): models of one type that allows
few of the fleet's instances, whose exclusions and selves sit at the front of the placement order, candidates of the
type or not.  front_cases() returns the fleet with those models' edges rewritten, one decision per case and each
decision's group:

  A  self not a candidate, at the front, no exclusions                  (answerable from the summary)
  B  self a candidate (the slot's first candidate), no exclusions       (walked)
  C  one exclusion, not a candidate, at the front                        (answerable)
  D  overflow ids: three non-candidates at the front, candidates last   (answerable)
  E  overflow ids: four candidates last, the fifth the first candidate  (walked)
  F  an exclusion on an instance that is not live, a candidate last     (answerable)
  G  overflow ids: four candidates last, the fifth not live             (answerable)

Selves of C-G are live instances from the back of the order."""
import numpy as np

from modelmesh_b200 import _lib as L
from modelmesh_b200.synth import SynthDecisions, make_fleet

from helpers import oracle_from_synth

GROUPS = "ABCDEFG"


def _set_edges(fl, edges):
    nm = fl.n_models
    fl.edge_off = np.zeros(nm + 1, dtype=np.int64)
    np.cumsum([len(e) for e in edges], out=fl.edge_off[1:])
    fl.edge_inst = np.asarray([int(x) for e in edges for x in e], dtype=np.int32)
    fl.n_loaded = np.asarray([len(e) for e in edges], dtype=np.int32)
    fl.n_failed = np.zeros(nm, dtype=np.int32)


def front_cases(nm=3000, ni=1300, seed=33, per_group=12):
    """(fleet, decisions, group index per decision, rank by instance (-1: not live), allowed mask of the chosen type)"""
    fl = make_fleet("C3", nm, ni, seed)
    order0 = oracle_from_synth(fl).cluster_order()
    gone = int(order0[2])  # an instance at the front leaves: shutting down, it has no rank
    fl.inst_rows["shutting_down"][gone] = 1
    o = oracle_from_synth(fl)
    order = o.cluster_order()
    rank = np.full(fl.n_instances, -1, dtype=np.int64)
    rank[order] = np.arange(len(order))
    # the type with the most models among those that allow at most half of the instances
    best_t, allowed = None, None
    counts = np.bincount(fl.model_type, minlength=len(fl.type_names))
    for t in np.argsort(-counts):
        a, _ = o.type_sets(fl.type_names[int(t)], fl.n_instances)
        if a is not None and 0 < a[order].mean() <= 0.5:
            best_t, allowed = int(t), a
            break
    assert best_t is not None, "no restricted type"
    live_allowed = order[allowed[order]]
    non_front = order[~allowed[order]][:8]
    cand_last = live_allowed[::-1][:6]
    back = order[::-1][:8]
    models = np.nonzero(fl.model_type == best_t)[0]
    need = len(GROUPS) * per_group
    assert len(models) >= need, (len(models), need)
    edges = [list(fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]]) for m in range(fl.n_models)]
    rng = np.random.default_rng(seed)
    dec = np.zeros(need, dtype=L.DECISION_IN)
    group = np.zeros(need, dtype=np.int32)
    for g, name in enumerate(GROUPS):
        for j in range(per_group):
            k = g * per_group + j
            m = int(models[k])
            self_ = int(back[j % len(back)])
            if name == "A":
                e, self_ = [], int(non_front[j % len(non_front)])
            elif name == "B":
                e, self_ = [], int(live_allowed[0])
            elif name == "C":
                e = [int(non_front[j % len(non_front)])]
            elif name == "D":
                e = [int(x) for x in np.roll(non_front, j)[:3]] + [int(x) for x in cand_last[:3]]
            elif name == "E":
                e = [int(x) for x in cand_last[:4]] + [int(live_allowed[0])]
            elif name == "F":
                e = [gone, int(cand_last[j % len(cand_last)])]
            else:
                e = [int(x) for x in cand_last[:4]] + [gone]
            edges[m] = e
            dec[k]["model"], dec[k]["self"], group[k] = m, self_, g
    _set_edges(fl, edges)
    dec["fresh"] = -1
    dec["flags"] = np.where(rng.uniform(size=need) < 0.25, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(L.DF_MODEL_LAST_USED)
    sd = SynthDecisions(dec, np.zeros(0, dtype=L.INSTANCE_ROW), np.zeros(0, dtype=np.int32))
    return fl, sd, group, rank, allowed
