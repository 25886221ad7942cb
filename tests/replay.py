"""Replayed ingest streams: a seeded chain of instance, model, type-config and replicaset events, committed window by
window, applied to a fleet and to a plain Python model of the same fleet.

At every checkpoint the references are rebuilt from the Python model, never carried along: the oracle gets a bulk load
of every index that was ever present, a DELETED event for each index that is absent now, the current type config and
replicaset list, and one converged refresh; `scratch()` loads a fresh fleet with a single commit.  So whatever the
fleet under test did incrementally (dirty rows scattered on the device, overflow pairs re-uploaded, JSON records
re-resolved by id, registry rows past the old end) is compared with a state that was never incremental.

Windows come in two kinds: "numeric" windows carry numeric instance updates and model-record edits only (the device
path of a commit, path 2), "structural" windows also add, remove, re-register and relabel instances or change the type
config or the replicaset list (the host path, path 1)."""
from __future__ import annotations

import copy
import ctypes as C
import json
from typing import Dict, List, Optional

import numpy as np

from helpers import compare_decisions, oracle_inputs_fast
from modelmesh_b200 import _lib as L
from modelmesh_b200.fleet import Fleet
from modelmesh_b200.synth import LONG_MAX, SynthDecisions, SynthFleet, load_into_fleet
from oracle import binding as ob

# the oracle's name for type id 0, the type of a registry row that was never upserted: absent from every constraint
# config, so it resolves like any unconfigured name ("_default", else unconstrained)
GAP_TYPE = "~never-upserted"

NUMERIC, STRUCTURAL = "numeric", "structural"


class Replay:
    def __init__(self, fl: SynthFleet, lib, seed: int, headroom: int = 48, max_models: Optional[int] = None):
        self.fl, self.lib = fl, lib
        self.rng = np.random.default_rng(seed)
        n0, nm = fl.n_instances, fl.n_models
        self.ni_max = n0 + headroom
        self.nm_max = max_models or nm + 2 * nm // 3 + 64
        self.now = fl.now_ms
        # ---- instances (index -> last published state; `present` says whether the index is in the table now) ----
        self.rows = np.zeros(self.ni_max, dtype=L.INSTANCE_ROW)
        self.rows[:n0] = fl.inst_rows
        self.ids: List[Optional[str]] = list(fl.inst_ids) + [None] * headroom
        self.locs: List[Optional[str]] = list(fl.inst_locs) + [None] * headroom
        self.zones: List[Optional[str]] = list(fl.inst_zones) + [None] * headroom
        self.labels: List[List[str]] = [list(x) for x in fl.inst_labels] + [[] for _ in range(headroom)]
        self.present = np.zeros(self.ni_max, dtype=bool)
        self.present[:n0] = True
        self.n_ever = n0           # indices [0, n_ever) have been present at some point; new pods take the next one
        self.gone_ids: List[str] = []
        self.moved: List[int] = []   # indices that changed pod (re-used, re-registered from / to)
        self.n_new = 0
        # ---- configuration ----
        self.type_config0 = copy.deepcopy(fl.type_config)
        self.type_config = copy.deepcopy(fl.type_config)
        self.replicasets = list(fl.replaced_replicasets)
        self.rs_prefixes = sorted({i.split("-")[0] for i in fl.inst_ids if "-" in i})
        labs = {l for ls in fl.inst_labels for l in ls}
        for ent in (fl.type_config or {}).values():
            labs |= set(ent.get("required") or []) | set(ent.get("preferred") or [])
        self.label_names = sorted(labs) or ["lbl-a", "lbl-b", "lbl-c"]
        self.type_names = list(fl.type_names)
        self.o_names = self.type_names + [GAP_TYPE]   # oracle type list: a model's type is an index into it
        # ---- registry: the row as the library stores it, the edges (index-based) or the pod ids (JSON records) ----
        self.mrow = np.zeros(self.nm_max, dtype=L.MODEL_ROW)
        self.mtype = np.full(self.nm_max, len(self.type_names), dtype=np.int32)
        self.edges: List[List[int]] = [[] for _ in range(self.nm_max)]
        self.json_ids: Dict[int, List[str]] = {}
        self.n_used = nm
        self.f = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, self.ni_max, self.nm_max, lib=lib)
        self.tid = load_into_fleet(fl, self.f)
        self.mrow["last_used"][:nm] = fl.model_last_used
        self.mrow["size_units"][:nm] = fl.model_size
        self.mrow["rpm"][:nm] = fl.model_rpm
        self.mrow["type_id"][:nm] = np.asarray([self.tid[t] for t in fl.type_names], dtype=np.uint16)[fl.model_type]
        self.mrow["copy_count"][:nm] = np.minimum(255, fl.n_loaded)
        self.mrow["fail_count"][:nm] = np.minimum(255, fl.n_failed)
        self.mtype[:nm] = fl.model_type
        for m in range(nm):
            self.edges[m] = [int(x) for x in fl.edge_inst[fl.edge_off[m]:fl.edge_off[m + 1]]]
        self.has_path = "mmp_commit_info" not in getattr(lib, "_mmp_missing", [])
        self.windows: List[tuple] = []   # (kind, commit path, model edits, structural events) per committed window
        self.n_compared = 0
        self.touched: set = set()          # models edited since the last commit
        self.last_touched = np.zeros(0, dtype=np.int64)  # ... and in the window before the last commit
        self.front = self._front()

    def _front(self) -> np.ndarray:
        """Where placements go in the committed epoch: the targets of a probe batch, then the first ranks of the order.
        Edges drawn from here are the exclusions that change answers."""
        live = self._live()
        n = 512
        dec = np.zeros(n, dtype=L.DECISION_IN)
        dec["model"] = self.rng.integers(0, self.n_used, size=n)
        dec["self"] = live[self.rng.integers(0, len(live), size=n)]
        dec["flags"], dec["fresh"] = L.DF_MODEL_LAST_USED, -1
        t = self.f.place_batch(dec, self.now, 1)["target"]
        hot = [int(x) for x in np.unique(t[t >= 0])]
        return np.asarray(list(dict.fromkeys(hot + [int(x) for x in self.f.cluster_order()[:8]]))[:32], dtype=np.int64)

    # ------------------------------------------------------------------------------------------------------------
    # events: each one goes to the fleet under test and to the Python model
    # ------------------------------------------------------------------------------------------------------------
    def _live(self) -> np.ndarray:
        return np.nonzero(self.present & (self.rows["shutting_down"] == 0))[0]

    def _numeric_row(self, i: int) -> np.ndarray:
        rng, r = self.rng, self.rows[i].copy()
        cap = int(r["capacity"])
        if rng.uniform() < 0.15:
            cap = int(cap * rng.uniform(0.6, 1.4))
            r["capacity"] = cap
        ms = self.fl.min_space_units
        # about half of the updates leave the instance within two minSpaceUnits of full (the "full" side of the order)
        r["used"] = cap - int(rng.integers(0, min(cap, 2 * ms) + 1)) if rng.uniform() < 0.5 else int(rng.integers(0, cap + 1))
        r["count"] = int(rng.integers(0, 400))
        r["lru_time"] = LONG_MAX if rng.uniform() < 0.05 else int(self.now - rng.integers(0, 10_000_000))
        r["rpm"] = int(rng.integers(0, 5000))
        r["l_in_prog"] = int(rng.integers(0, 4))
        return r

    def _arrived(self, row) -> np.ndarray:
        """A pod that has just (re)registered, with numbers like the rest of the fleet's."""
        row = row.copy()
        row["shutting_down"], row["active"] = 0, 1
        ms = self.fl.min_space_units
        row["used"] = max(0, int(row["capacity"]) - int(self.rng.integers(0, 2 * ms + 1))) if self.rng.uniform() < 0.5 else int(self.rng.integers(0, int(row["capacity"]) + 1))
        return row

    def update_numeric(self, i: int):
        r = self._numeric_row(i)
        self.f.instance_update(i, r)
        self.rows[i] = r

    def _ids_for_model(self, k: int) -> List[int]:
        # any index ever used, removed ones included, and now and then one that never held a pod; half of them from the
        # instances placements go to in the last committed epoch, where an exclusion changes the answer
        hi = min(self.ni_max, self.n_ever + 4)
        ids = [int(x) for x in self.rng.choice(hi, size=min(k, hi), replace=False)]
        front = self.front[self.rng.permutation(len(self.front))]
        for j in range(len(ids)):
            if self.rng.uniform() < 0.5 and len(front):
                i, front = int(front[0]), front[1:]
                if i not in ids:
                    ids[j] = i
        return ids

    def _n_ids(self, allow_overflow: bool) -> int:
        if allow_overflow and self.rng.uniform() < 0.25:
            return int(self.rng.integers(5, 13))
        return int(self.rng.integers(0, 5))

    def upsert_model(self, m: int, ids: List[int], tname: Optional[str] = None, last_used: Optional[int] = None):
        rng = self.rng
        if tname is None:
            tname = self.o_names[self.mtype[m]] if self.mtype[m] < len(self.type_names) else self.type_names[int(rng.integers(0, len(self.type_names)))]
        row = np.zeros(1, dtype=L.MODEL_ROW)[0]
        row["last_used"] = last_used if last_used is not None else int(self.now - rng.integers(0, 10_000_000))
        row["size_units"] = int(rng.integers(200, 40_000))
        row["rpm"] = int(rng.integers(0, 2000))
        row["type_id"] = self.tid[tname]
        nl = int(rng.integers(0, len(ids) + 1))
        row["copy_count"], row["fail_count"] = nl, len(ids) - nl
        self.f.model_upsert(m, row, ids)
        self.touched.add(m)
        self.mrow[m] = row
        self.mtype[m] = self.type_names.index(tname)
        self.edges[m] = list(ids)
        self.json_ids.pop(m, None)
        self.n_used = max(self.n_used, m + 1)

    def upsert_model_json(self, m: int, loaded: List[str], failed: List[str], tname: str, last_used: int, size: int):
        """A model record as the registry stores it (MR JSON): instances named by pod id, resolved against the id table at
        every commit after it changed.  Times 0: the record carries no load times."""
        doc = {"type": tname, "instanceIds": {p: 0 for p in loaded}, "failedIn": {p: 0 for p in failed}, "lu": int(last_used)}
        self.f._ck(self.lib.mmp_model_upsert_json(self.f.h, m, json.dumps(doc).encode(), int(size)))
        self.touched.add(m)
        row = np.zeros(1, dtype=L.MODEL_ROW)[0]
        row["last_used"], row["size_units"], row["type_id"] = last_used, size, self.tid[tname]
        row["copy_count"], row["fail_count"] = min(255, len(loaded)), min(255, len(failed))
        self.mrow[m] = row
        self.mtype[m] = self.type_names.index(tname)
        self.edges[m] = []
        self.json_ids[m] = list(loaded) + list(failed)
        self.n_used = max(self.n_used, m + 1)

    def _upsert_instance(self, i: int, row, iid: str, loc, zone, labels):
        self.f.instance_upsert(i, row, iid, loc, zone, labels)
        self.rows[i], self.ids[i], self.locs[i], self.zones[i], self.labels[i] = row, iid, loc, zone, list(labels)
        self.present[i] = True
        self.n_ever = max(self.n_ever, i + 1)

    def _new_id(self) -> str:
        self.n_new += 1
        rs = self.rs_prefixes[self.n_new % len(self.rs_prefixes)] if self.rs_prefixes else "pod"
        return f"{rs}-n{self.n_new:04x}"

    def remove(self, i: int):
        self.f.instance_remove(i)
        self.present[i] = False
        self.gone_ids.append(self.ids[i])

    def reuse_index(self, i: int):
        """A new pod id at index i (present or not)."""
        if self.present[i]:
            self.gone_ids.append(self.ids[i])
        self._upsert_instance(i, self._arrived(self.rows[i]), self._new_id(), self.locs[i], self.zones[i], self.labels[i])
        self.moved.append(i)

    def add_new(self) -> int:
        """A pod at an index that never held one (the fleet was created with headroom)."""
        i = self.n_ever
        assert i < self.ni_max
        src = int(self.rng.choice(self._live()))
        self._upsert_instance(i, self._arrived(self.rows[src]), self._new_id(), self.locs[src], self.zones[src], self.labels[src])
        return i

    def reregister(self, i: int) -> int:
        """The pod at index i leaves and comes back under the same id at another index."""
        iid = self.ids[i]
        row, loc, zone, labels = self.rows[i].copy(), self.locs[i], self.zones[i], list(self.labels[i])
        self.remove(i)
        self.gone_ids.remove(iid)
        free = [j for j in range(self.n_ever) if not self.present[j] and j != i]
        j = int(self.rng.choice(free)) if free and self.rng.uniform() < 0.5 else self.n_ever
        self._upsert_instance(j, row, iid, loc, zone, labels)
        self.moved += [i, j]
        return j

    def toggle(self, i: int, field: str):
        row = self.rows[i].copy()
        row[field] = 1 - int(row[field])
        self.f.instance_update(i, row)
        self.rows[i] = row

    def relabel(self, i: int):
        rng = self.rng
        labels, zone = list(self.labels[i]), self.zones[i]
        if rng.uniform() < 0.6:
            k = int(rng.integers(0, 4))
            labels = sorted({self.label_names[int(x)] for x in rng.integers(0, len(self.label_names), size=k)})
        else:
            zone = None if zone is not None and rng.uniform() < 0.3 else f"zone-{int(rng.integers(0, 5))}"
        self._upsert_instance(i, self.rows[i].copy(), self.ids[i], self.locs[i], zone, labels)

    def set_types(self, cfg: Optional[dict]):
        self.f.types_set_json(None if cfg is None else json.dumps(cfg))
        self.type_config = copy.deepcopy(cfg)

    def other_type_config(self) -> Optional[dict]:
        """A different constraint document over the same type and label names."""
        rng = self.rng
        if self.type_config0 is None:
            base = {}
        else:
            base = copy.deepcopy(self.type_config0)
        out = {}
        for t, ent in base.items():
            u = rng.uniform()
            if u < 0.25:
                continue
            if u < 0.5 and (ent.get("required") or ent.get("preferred")):
                ent = {"required": list(ent.get("preferred") or []), "preferred": list(ent.get("required") or [])}
                ent = {k: v for k, v in ent.items() if v}
            out[t] = ent
        for t in self.type_names[:4]:
            if t not in out and rng.uniform() < 0.5:
                out[t] = {"required": [self.label_names[int(rng.integers(0, len(self.label_names)))]]}
        return out

    def set_replicasets(self, prefixes: List[str]):
        self.f.replicasets_set(prefixes)
        self.replicasets = list(prefixes)

    # ------------------------------------------------------------------------------------------------------------
    # windows
    # ------------------------------------------------------------------------------------------------------------
    def numeric_window(self, n_inst: int, n_models: int, n_growth: int = 0, overflow: bool = True, n_json: int = 0,
                       distinct_models: bool = False):
        """Numeric instance updates and model edits only.  overflow=False: no upsert names more than 4 instances, and up to
        24 models that hold more are cut back to at most 4, so models only leave the overflow map in this window."""
        rng = self.rng
        if not overflow:
            ovf = [m for m in range(self.n_used) if len(self.edges[m]) > 4]
            for m in (rng.choice(ovf, size=min(24, len(ovf)), replace=False) if ovf else []):
                m = int(m)
                self.upsert_model(m, self.edges[m][:int(rng.integers(0, 5))])
        live = np.nonzero(self.present)[0]
        for i in rng.choice(live, size=min(n_inst, len(live)), replace=False):
            self.update_numeric(int(i))
        if distinct_models:
            ms = rng.choice(max(self.n_used, n_models), size=n_models, replace=False)
        else:
            ms = rng.integers(0, self.n_used, size=n_models)
        for m in ms:
            m = int(m)
            tname = self.type_names[int(rng.integers(0, len(self.type_names)))] if rng.uniform() < 0.2 else None
            lu = 0 if rng.uniform() < 0.05 else None
            self.upsert_model(m, self._ids_for_model(self._n_ids(overflow)), tname, lu)
        for _ in range(n_json):
            self._json_event(rng.integers(0, self.n_used), overflow)
        for _ in range(n_growth):  # registry growth: the indices in between are never upserted
            m = self.n_used + int(rng.integers(1, 40))
            if m < self.nm_max:
                self.upsert_model(m, self._ids_for_model(self._n_ids(overflow)))
        return self.commit(NUMERIC, len(ms) + n_json + n_growth)

    def _json_event(self, m, overflow: bool = True):
        rng = self.rng
        live_ids = [self.ids[i] for i in np.nonzero(self.present)[0]]
        front_ids = [self.ids[i] for i in self.front if self.present[i]]
        pool = live_ids + front_ids * max(1, len(live_ids) // (2 * max(1, len(front_ids)))) + self.gone_ids[-20:] + ["ghost-pod-1", "ghost-pod-2"]
        k = int(rng.integers(0, 7 if overflow else 4))
        pods = list(dict.fromkeys(pool[int(x)] for x in rng.choice(len(pool), size=min(k, len(pool)), replace=False)))
        nl = int(rng.integers(0, len(pods) + 1))
        tname = self.type_names[int(rng.integers(0, len(self.type_names)))]
        self.upsert_model_json(int(m), pods[:nl], pods[nl:], tname, int(self.now - rng.integers(0, 9_000_000)),
                               int(rng.integers(200, 40_000)))

    def structural_window(self, events: List[str], n_inst: int = 30, n_models: int = 60, n_json: int = 8):
        rng = self.rng
        for ev in events:
            live = self._live()
            if ev == "remove":
                for i in rng.choice(live, size=min(6, len(live) // 4), replace=False):
                    self.remove(int(i))
            elif ev == "reuse":
                for i in rng.choice(self.n_ever, size=4, replace=False):
                    self.reuse_index(int(i))
            elif ev == "add":
                for _ in range(3):
                    if self.n_ever < self.ni_max:
                        self.add_new()
            elif ev == "reregister":  # pods named by JSON records come back at other indices
                named = {p for pods in self.json_ids.values() for p in pods}
                cand = [int(i) for i in self.front if self.present[i] and self.ids[i] in named] or \
                    [int(i) for i in live if self.ids[i] in named] or [int(i) for i in live]
                for i in rng.choice(cand, size=min(3, len(cand)), replace=False):
                    if self.n_ever < self.ni_max:
                        self.reregister(int(i))
            elif ev == "toggle":
                for i in rng.choice(np.nonzero(self.present)[0], size=4, replace=False):
                    self.toggle(int(i), "shutting_down" if rng.uniform() < 0.5 else "active")
            elif ev == "relabel":
                for i in rng.choice(live, size=5, replace=False):
                    self.relabel(int(i))
            elif ev == "types":
                self.set_types(self.other_type_config() if self.type_config == self.type_config0 else copy.deepcopy(self.type_config0))
            elif ev == "replicasets":
                k = int(rng.integers(0, len(self.rs_prefixes) + 1))
                self.set_replicasets(sorted(rng.choice(self.rs_prefixes, size=min(k, 3), replace=False).tolist()) if k else [])
            else:
                raise ValueError(ev)
        live = np.nonzero(self.present)[0]
        for i in rng.choice(live, size=min(n_inst, len(live)), replace=False):
            self.update_numeric(int(i))
        for m in rng.integers(0, self.n_used, size=n_models):
            self.upsert_model(int(m), self._ids_for_model(self._n_ids(True)))
        for m in rng.integers(0, self.n_used, size=n_json):
            self._json_event(m)
        return self.commit(STRUCTURAL, n_models + n_json, events)

    def all_dirty_threshold(self) -> int:
        """More distinct dirty models than this in one window and the commit uploads the whole registry instead."""
        return self.nm_max // 8 + 1024

    def commit(self, kind: str, n_model_edits: int, events=()):
        self.f.commit()
        self.last_touched = np.asarray(sorted(self.touched), dtype=np.int64)
        self.touched = set()
        self.front = self._front()
        path = self.f.commit_info()[0] if self.has_path else None
        if self.has_path:
            assert path == (2 if kind == NUMERIC else 1), (kind, path, len(self.windows))
        self.windows.append((kind, path, n_model_edits, tuple(events)))
        return path

    # ------------------------------------------------------------------------------------------------------------
    # references, rebuilt from the Python model
    # ------------------------------------------------------------------------------------------------------------
    def current_edges(self) -> List[List[int]]:
        """Each model's loaded ∪ failed instance indices now: JSON records resolved against the current id table."""
        idx_of = {self.ids[i]: int(i) for i in np.nonzero(self.present)[0]}
        out = [list(self.edges[m]) for m in range(self.n_used)]
        for m, pods in self.json_ids.items():
            seen, e = set(), []
            for p in pods:
                if p in seen:
                    continue
                seen.add(p)
                i = idx_of.get(p)
                if i is not None and i not in e:
                    e.append(i)
            out[m] = e
        return out

    def view(self) -> SynthFleet:
        """The current state as a SynthFleet (the shape helpers.compare_decisions and oracle_inputs read)."""
        nm, K = self.n_used, self.n_ever
        edges = self.current_edges()
        deg = np.asarray([len(e) for e in edges], dtype=np.int64)
        off = np.zeros(nm + 1, dtype=np.int64)
        np.cumsum(deg, out=off[1:])
        inst = np.asarray([x for e in edges for x in e], dtype=np.int32)
        fl = self.fl
        return SynthFleet("replay", self.now, fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units,
                          self.rows[:K].copy(), self.ids[:K], self.locs[:K], self.zones[:K], self.labels[:K],
                          copy.deepcopy(self.type_config), list(self.o_names), self.mtype[:nm].copy(),
                          self.mrow["last_used"][:nm].astype(np.int64), self.mrow["size_units"][:nm].astype(np.int32),
                          self.mrow["rpm"][:nm].astype(np.int32), off, inst, self.mrow["copy_count"][:nm].astype(np.int32),
                          self.mrow["fail_count"][:nm].astype(np.int32), list(self.replicasets))

    def oracle(self) -> ob.OracleFleet:
        fl, K = self.fl, self.n_ever
        o = ob.OracleFleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units)
        o.types_set(self.type_config)
        ids = [self.ids[i] if self.present[i] else f"~gone-{i}" for i in range(K)]
        o.bulk_add(self.rows[:K], ids, self.locs[:K], self.zones[:K], self.labels[:K])
        for i in range(K):
            if not self.present[i]:
                o.instance_event(ob.DELETED, i, None, ids[i], now_ms=self.now)
        if self.type_config is not None:
            o.tc_converge()
        o.set_replaced_replicasets(self.replicasets)
        return o

    def scratch(self, lib=None) -> Fleet:
        """A fresh fleet loaded from the Python model with a single commit (type names interned in the same order, so the
        model rows are byte-identical)."""
        fl = self.fl
        g = Fleet(fl.min_space_units, fl.min_churn_age_ms, fl.default_model_size_units, self.ni_max, self.nm_max, lib=lib or self.lib)
        g.types_set_json(fl.type_json())
        assert all(g.type_id(t) == self.tid[t] for t in self.type_names)
        g.types_set_json(None if self.type_config is None else json.dumps(self.type_config))
        g.replicasets_set(self.replicasets)
        for i in np.nonzero(self.present)[0]:
            i = int(i)
            g.instance_upsert(i, self.rows[i], self.ids[i], self.locs[i], self.zones[i], self.labels[i])
        v = self.view()
        g.models_bulk(0, self.mrow[:self.n_used], v.edge_off, v.edge_inst)
        g.commit()
        return g

    # ------------------------------------------------------------------------------------------------------------
    # decisions
    # ------------------------------------------------------------------------------------------------------------
    def decisions(self, n: int, seed: int, plain: bool = False, models=None) -> SynthDecisions:
        rng = np.random.default_rng(seed)
        live = self._live()
        dec = np.zeros(n, dtype=L.DECISION_IN)
        if models is None:  # 40 % for models edited in the last window, 15 % for JSON records
            models = rng.integers(0, self.n_used, size=n)
            u = rng.uniform(size=n)
            if len(self.last_touched):
                models = np.where(u < 0.4, self.last_touched[rng.integers(0, len(self.last_touched), size=n)], models)
            if self.json_ids:
                js = np.asarray(sorted(self.json_ids), dtype=np.int64)
                models = np.where((u >= 0.4) & (u < 0.55), js[rng.integers(0, len(js), size=n)], models)
        dec["model"] = models
        dec["self"] = live[rng.integers(0, len(live), size=n)]
        # a third of the decisions are made by a pod that holds the model (self excluded: no favour-self exit for it)
        edges = self.current_edges()
        is_live = self.present & (self.rows["shutting_down"] == 0)
        for k in np.nonzero(rng.uniform(size=n) < 0.33)[0]:
            e = [i for i in edges[int(dec["model"][k])] if is_live[i]]
            if e:
                dec["self"][k] = e[int(rng.integers(0, len(e)))]
        fav = rng.uniform(size=n) < 0.3
        if plain:
            dec["flags"] = np.where(fav, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(L.DF_MODEL_LAST_USED)
            dec["fresh"] = -1
            return SynthDecisions(dec, np.zeros(0, dtype=L.INSTANCE_ROW), np.zeros(0, dtype=np.int32))
        r = rng.uniform(size=n)
        dec["last_used"] = np.where(r < 0.7, self.now + 20_000, np.where(r < 0.8, 0, np.where(
            r < 0.9, self.now - rng.integers(0, 3_000_000, size=n), self.now - 7 * 86_400_000)))
        dec["flags"] = (np.where(fav, L.DF_FAVOUR_SELF, 0) | np.where(r < 0.6, L.DF_MODEL_LAST_USED, 0)).astype(np.uint32)
        n_fresh = min(len(live), 48)
        fresh_inst = rng.choice(live, size=n_fresh, replace=False)
        fresh = self.rows[fresh_inst].copy()
        fresh["used"] = np.clip(fresh["used"] + rng.integers(-200_000, 200_001, size=n_fresh), 0, fresh["capacity"])
        fresh["count"] = np.maximum(0, fresh["count"] + rng.integers(-3, 4, size=n_fresh)).astype(np.int32)
        fresh["rpm"] = np.where(rng.uniform(size=n_fresh) < 0.25, rng.integers(0, 5000, size=n_fresh), 0).astype(np.int32)
        slot_of = np.full(self.ni_max, -1, dtype=np.int64)
        slot_of[fresh_inst] = np.arange(n_fresh)
        s = slot_of[dec["self"]]
        dec["fresh"] = np.where((s >= 0) & (rng.uniform(size=n) < 0.7), s, -1).astype(np.int32)
        k = np.where(rng.uniform(size=n) < 0.12, rng.integers(1, 4, size=n), 0).astype(np.int32)
        off = np.zeros(n + 1, dtype=np.int64)
        np.cumsum(k, out=off[1:])
        extra = rng.integers(0, self.n_ever, size=int(off[-1])).astype(np.int32)
        owner = np.repeat(np.arange(n), k)
        extra = np.where(rng.uniform(size=len(extra)) < 0.15, dec["self"][owner], extra).astype(np.int32)
        dec["extra_off"], dec["extra_n"] = off[:-1].astype(np.int32), k
        return SynthDecisions(dec, fresh, extra)

    def holder_decisions(self, seed: int, cap: int = 600) -> SynthDecisions:
        """Decisions made by a pod that holds the model (self = one of its live edges), half of them favouring self: the
        exclusion of self decides whether the answer can be self.  Every JSON record first (their edges are pod ids
        resolved against the current id table), then a sample of the other models."""
        rng = np.random.default_rng(seed)
        edges = self.current_edges()
        is_live = self.present & (self.rows["shutting_down"] == 0)
        others = [int(m) for m in rng.permutation(self.n_used) if int(m) not in self.json_ids]
        pairs = []
        moved = [i for i in dict.fromkeys(self.moved[-8:]) if is_live[i]]
        for m in sorted(self.json_ids) + others:
            e = [i for i in edges[m] if is_live[i]]
            # a JSON record also meets the pods that came and went at re-used indices: excluded only if it names them now
            pairs += [(m, i) for i in e + ([i for i in moved if i not in e] if m in self.json_ids else [])]
            if len(pairs) >= cap:
                break
        pairs = pairs[:cap]
        n = len(pairs)
        dec = np.zeros(n, dtype=L.DECISION_IN)
        dec["model"] = [m for m, _ in pairs]
        dec["self"] = [i for _, i in pairs]
        dec["flags"] = np.where(rng.uniform(size=n) < 0.5, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(L.DF_MODEL_LAST_USED)
        dec["fresh"] = -1
        return SynthDecisions(dec, np.zeros(0, dtype=L.INSTANCE_ROW), np.zeros(0, dtype=np.int32))

    def sweep_decisions(self, self_idx: np.ndarray, fav: np.ndarray) -> SynthDecisions:
        """What mmp_place_sweep(0, n_models, self_idx, favour) decides, as explicit decision records."""
        n = self.n_used
        dec = np.zeros(n, dtype=L.DECISION_IN)
        dec["model"] = np.arange(n)
        dec["self"] = self_idx
        dec["flags"] = np.where(fav, L.DF_FAVOUR_SELF, 0).astype(np.uint32) | np.uint32(L.DF_MODEL_LAST_USED)
        dec["fresh"] = -1
        return SynthDecisions(dec, np.zeros(0, dtype=L.INSTANCE_ROW), np.zeros(0, dtype=np.int32))


def oracle_batch(v: SynthFleet, sd: SynthDecisions, o: ob.OracleFleet, seed: int) -> np.ndarray:
    od, off, idx = oracle_inputs_fast(v, sd)
    return o.get_next_batch(od, v.type_names, off, idx, v.now_ms, seed, fresh=sd.fresh if len(sd.fresh) else None)


def assert_same_results(got: np.ndarray, want: np.ndarray, what):
    bad = np.nonzero((got["target"] != want["target"]) | (got["n_candidates"] != want["n_candidates"]))[0]
    assert len(bad) == 0, (what, len(bad), bad[:5], got[bad[:5]], want[bad[:5]])


def check_against_oracle(rp: Replay, seed: int, n_traced: int, n_batch: int) -> int:
    """cluster order, traced decisions with candidate masks (helpers.compare_decisions, which also runs the untraced
    entry point), a larger untraced batch and a sweep over the whole registry, gap models included.  Returns the number
    of decisions compared."""
    v, o, f = rp.view(), rp.oracle(), rp.f
    assert np.array_equal(f.cluster_order(), o.cluster_order()), ("cluster order", len(rp.windows))
    sd = rp.decisions(n_traced, seed)
    compare_decisions(v, sd, o, f, seed=seed)
    sh = rp.holder_decisions(seed)
    compare_decisions(v, sh, o, f, seed=seed + 2)
    sd = rp.decisions(n_batch, seed + 1, plain=bool(seed & 1))
    kw = dict(fresh=sd.fresh if len(sd.fresh) else None, extra=sd.extra if len(sd.extra) else None)
    assert_same_results(f.place_batch(sd.dec, rp.now, seed, **kw), oracle_batch(v, sd, o, seed), ("batch", len(rp.windows)))
    rng = np.random.default_rng(seed)
    live = rp._live()
    self_idx = live[rng.integers(0, len(live), size=rp.n_used)].astype(np.int32)
    fav = rng.uniform(size=rp.n_used) < 0.3
    got = f.place_sweep(0, rp.n_used, self_idx, rp.now, seed, favour=fav)
    assert_same_results(got, oracle_batch(v, rp.sweep_decisions(self_idx, fav), o, seed), ("sweep", len(rp.windows)))
    o.close()
    n = 3 * (n_traced + len(sh.dec)) + n_batch + rp.n_used
    rp.n_compared += n
    return n


# The window schedule of every stream: numeric windows (device-path commits) alternate with structural ones (host path).
# Numeric windows grow the registry past its end, edit JSON records, let models leave the overflow map only ("shrink"),
# and one of them edits more distinct models than the dirty-list threshold.
SCHEDULE = [
    (NUMERIC, dict(n_inst=40, n_models=80, n_growth=3, n_json=4)),
    (STRUCTURAL, ["remove", "reuse", "add"]),
    (NUMERIC, dict(n_inst=40, n_models=80, overflow=False)),
    (STRUCTURAL, ["reregister", "toggle", "relabel"]),
    (NUMERIC, "all_dirty"),
    (STRUCTURAL, ["types", "replicasets", "remove"]),
    (NUMERIC, dict(n_inst=60, n_models=120, n_growth=4, n_json=4)),
    (STRUCTURAL, ["reregister", "add", "types", "toggle"]),
    (NUMERIC, dict(n_inst=20, n_models=60, overflow=False, n_json=3)),
    (STRUCTURAL, ["reuse", "relabel", "replicasets"]),
    (NUMERIC, dict(n_inst=30, n_models=50, n_growth=2)),
    (STRUCTURAL, ["remove", "reregister", "add"]),
]


def run_window(rp: Replay, w: int):
    kind, spec = SCHEDULE[w % len(SCHEDULE)]
    if kind == STRUCTURAL:
        return rp.structural_window(spec)
    if spec == "all_dirty":
        return rp.numeric_window(n_inst=30, n_models=rp.all_dirty_threshold() + 64, distinct_models=True)
    return rp.numeric_window(**spec)


def describe(rp: Replay) -> str:
    """One line per window: kind, commit path taken, model edits, structural events."""
    return "; ".join(f"w{k}:{kind[0]}/path{path}/{n}{'/' + ','.join(ev) if ev else ''}" for k, (kind, path, n, ev) in enumerate(rp.windows))


def check_sorted_batch(rp: Replay, seed: int, n: int = 8192 + 77) -> int:
    """A batch large enough for k_place_direct to resolve it in type-slot order (sort_slots = 1), against the oracle."""
    f, lib = rp.f, rp.lib
    sd = rp.decisions(n, seed)
    f._ck(lib.mmp_tune(f.h, b"sort_slots", 1))
    try:
        got = f.place_batch(sd.dec, rp.now, seed, fresh=sd.fresh, extra=sd.extra if len(sd.extra) else None)
    finally:
        f._ck(lib.mmp_tune(f.h, b"sort_slots", 2))
    o = rp.oracle()
    assert_same_results(got, oracle_batch(rp.view(), sd, o, seed), ("sorted batch", len(rp.windows)))
    o.close()
    rp.n_compared += n
    return n


def prune(fleet: Fleet, self_idx: int, now: int, missing: np.ndarray, cap: int):
    outm = np.zeros(cap, dtype=np.int32)
    outk = np.zeros(cap, dtype=np.uint8)
    miss = missing.copy()
    n = fleet._ck(fleet.lib.mmp_registry_prune(fleet.h, self_idx, now, 600_000, miss.ctypes.data_as(C.c_void_p),
                                               outm.ctypes.data_as(C.c_void_p), outk.ctypes.data_as(C.c_void_p), cap))
    return {int(outm[i]): int(outk[i]) for i in range(n)}, miss


def check_against_scratch(rp: Replay, seed: int, n_batch: int = 4000) -> int:
    """The fleet the stream built incrementally against a fresh fleet loaded from the Python model with one commit:
    byte-identical placements and registry sweeps (never-upserted rows included), the same partition stats, reaper
    selections per partition and registry-prune results."""
    f, g = rp.f, rp.scratch()
    w = len(rp.windows)
    assert np.array_equal(f.cluster_order(), g.cluster_order()), ("scratch order", w)
    sd = rp.decisions(n_batch, seed)
    kw = dict(fresh=sd.fresh, extra=sd.extra if len(sd.extra) else None)
    a, b = f.place_batch(sd.dec, rp.now, seed, **kw), g.place_batch(sd.dec, rp.now, seed, **kw)
    assert a.tobytes() == b.tobytes(), ("scratch batch", w, np.nonzero(a != b)[0][:5])
    rng = np.random.default_rng(seed)
    live = rp._live()
    self_idx = live[rng.integers(0, len(live), size=rp.n_used)].astype(np.int32)
    fav = rng.uniform(size=rp.n_used) < 0.3
    a, b = f.place_sweep(0, rp.n_used, self_idx, rp.now, seed, favour=fav), g.place_sweep(0, rp.n_used, self_idx, rp.now, seed, favour=fav)
    assert a.tobytes() == b.tobytes(), ("scratch sweep", w, np.nonzero(a != b)[0][:5])
    # partition ids are opaque per fleet and break ties of the stats order: compare as sets, map ids through the instances
    sa, ia = f.stats()
    sb, ib = g.stats()
    assert np.array_equal(np.sort(sa, order=list(sa.dtype.names)), np.sort(sb, order=list(sb.dtype.names))), ("stats", w)
    pmap = {-1: -1}
    for i in np.nonzero(rp.present)[0]:
        pa, pb = f.instance_partition(int(i)), g.instance_partition(int(i))
        assert (pa < 0) == (pb < 0), ("partition", w, i)
        if pa >= 0:
            assert pmap.setdefault(pa, pb) == pb, ("partition map", w, i)
    for pa in ia:
        pb = pmap.get(int(pa))
        if pb is None:
            continue
        assert np.array_equal(sa[ia == pa], sb[ib == pb]), ("partition stats", w, pa)
        ra, rb = f.reaper_select(int(pa), rp.now), g.reaper_select(pb, rp.now)
        assert np.array_equal(ra, rb), ("reaper", w, pa, ra[:5], rb[:5])
    # registry prune: every absent pod was first seen missing 11 minutes ago, so its copies are pruned in this pass
    missing = np.zeros(rp.ni_max, dtype=np.int64)
    missing[~rp.present] = rp.now - 660_000
    pa, ma = prune(f, int(live[0]), rp.now, missing, rp.n_used)
    pb, mb = prune(g, int(live[0]), rp.now, missing, rp.n_used)
    assert pa == pb and np.array_equal(ma, mb), ("prune", w, len(pa), len(pb))
    g.close()
    rp.n_compared += n_batch + rp.n_used
    return len(pa)
