"""Bin-packing on the C4 workload: grove_run_cycle with no set, with every gang packed at block level (its Required level) and with
every gang packed at rack level.

The three arms run alternately, each cycle on a fresh engine (a fresh handle per cycle keeps one arm's state from reaching the
next).  Per arm: ms per cycle (device events, grove_cycle_stats_t.ms_total), rounds, evaluations, gangs admitted, pods bound, the
device time of the pick kernels (k_binpack_* and the radix sort that ranks the domains, from torch.profiler in a separate run, one
cycle per arm), and how fragmented the cycle leaves the cluster: nodes with every GPU free and blocks no pod of the cycle landed in.
Prints one JSON line with the card, its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_binpack.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from grove_b200 import synth  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402

GPUS_PER_NODE = 8   # synth.kwok_nodes' default, the C4 node size


def _cycle(cfg, levels):
    g, c, s = cfg["tables"]
    with PlacementEngine(cfg["n_levels"]) as e:
        e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
        if levels is not None:
            e.set_binpack(levels)
        st = e.run_cycle()
        after, pl = e.nodes(), e.placements()
    block = cfg["nodes"]["dom"][:, 1].astype(np.int64)
    touched = np.unique(block[pl["node"]])
    st["free_nodes"] = int((after["free_gpu"] == GPUS_PER_NODE).sum())
    st["untouched_blocks"] = int(len(np.unique(block)) - len(touched))
    return st


def _pick_ms(cfg, levels):
    """device time of the pick kernels in one cycle, from the profiler's kernel records"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _cycle(cfg, levels)
    us = sum(ev.device_time_total for ev in prof.key_averages() if "binpack" in ev.key or "RadixSort" in ev.key)
    return us / 1e3


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    cfg = synth.config_c4()
    g = cfg["tables"][0]
    arms = {"none": None, "block": synth.binpack_levels(g), "rack": synth.binpack_levels(g, 2)}
    rows = {k: [] for k in arms}
    for i in range(a.warmup + a.steps):
        for k, levels in arms.items():
            st = _cycle(cfg, levels)
            if i >= a.warmup:
                rows[k].append(st)
    out = dict(workload="C4 bin-packing", nodes=int(len(cfg["nodes"])), gangs=int(len(g)), steps=a.steps, **card())
    for k, r in rows.items():
        out[k] = dict(ms_median=statistics.median(x["ms_total"] for x in r), ms_min=min(x["ms_total"] for x in r),
                      ms_max=max(x["ms_total"] for x in r), rounds=r[-1]["rounds"], evaluations=r[-1]["evaluations"],
                      gangs_admitted=r[-1]["gangs_admitted"], pods_bound=r[-1]["pods_bound"], free_nodes=r[-1]["free_nodes"],
                      untouched_blocks=r[-1]["untouched_blocks"],
                      pick_ms=_pick_ms(cfg, arms[k]) if arms[k] is not None else 0.0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
