"""Which path the decisions of the bench workloads take under the two-pass placement (DESIGN.md §5.2), estimated on the
CPU from the oracle: a plain decision is answered from its slot's summary when its model's excluded instances and self all
lie at or past the reach, here taken as one past the last rank its shortlist (best included) reaches -- the kernel's
reach also covers the non-simple probes, so this is an upper bound on the fast share.  Models with more than four ids
go to the one-warp pass.  Prints, per configuration, the share of decisions on each path and the share of warps of 32
consecutive decisions that would have no decision to walk.

    python tools/split_census.py [--configs C2,C3,C5] [--n 40000]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SIZES = {"C2": (100_000, 1_000, 2), "C3": (1_000_000, 10_000, 3), "C5": (1_000_000, 10_000, 5)}


def census(cfg, n):
    import helpers
    from modelmesh_b200.synth import SynthDecisions, make_decisions, make_fleet
    nm, ni, seed = SIZES[cfg]
    fl = make_fleet(cfg, nm, ni, seed)
    sd = make_decisions(fl, nm, seed, sweep=True, plain=True)
    o = helpers.oracle_from_synth(fl)
    order = o.cluster_order()
    rank = np.full(fl.n_instances, 1 << 30, dtype=np.int64)
    rank[order] = np.arange(len(order))
    n = min(n, len(sd.dec))
    sub = SynthDecisions(sd.dec[:n], sd.fresh, sd.extra)
    od, off, idx = helpers.oracle_inputs_fast(fl, sub)
    out, coff, ci, _, _ = o.get_next_batch(od, fl.type_names, off, idx, fl.now_ms, seed, want_candidates=True)
    best_r = np.where(out["best"] >= 0, rank[np.maximum(out["best"], 0)], -1)
    reach = np.empty(n, dtype=np.int64)
    for i in range(n):
        c = ci[coff[i]:coff[i + 1]]
        reach[i] = max(rank[c].max() if len(c) else -1, best_r[i]) + 1
    m = sub.dec["model"].astype(np.int64)
    deg = fl.edge_off[m + 1] - fl.edge_off[m]
    first_ex = np.full(n, 1 << 30, dtype=np.int64)
    for i in range(n):
        e = fl.edge_inst[fl.edge_off[m[i]]:fl.edge_off[m[i] + 1]]
        if len(e):
            first_ex[i] = rank[e].min()
    self_r = rank[sub.dec["self"]]
    ovf = deg > 4
    fast = ~ovf & (out["best"] >= 0) & (first_ex >= reach) & (self_r >= reach)
    walk = ~ovf & ~fast
    w = n // 32 * 32
    print(f"{cfg}: {n} decisions  fast {fast.mean():.4f}  walk {walk.mean():.4f}  overflow {ovf.mean():.4f}  "
          f"warps without a walk {np.mean(~walk[:w].reshape(-1, 32).any(1)):.4f}  "
          f"shortlist size p50/p99/max {np.percentile(out['n_candidates'], 50):.0f}/{np.percentile(out['n_candidates'], 99):.0f}/"
          f"{out['n_candidates'].max()}  reach p50/p99 {np.percentile(reach, 50):.0f}/{np.percentile(reach, 99):.0f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="C2,C3,C5")
    ap.add_argument("--n", type=int, default=40_000)
    args = ap.parse_args()
    for cfg in args.configs.split(","):
        census(cfg, args.n)


if __name__ == "__main__":
    main()
