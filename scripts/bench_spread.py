"""Topology spread on the C4 workload: time grove_run_cycle with spread groups against the same submission without them.

C4's base gangs go into groups of eight by (priority, template) -- the replicas of one PodCliqueSet -- spread over zones (level 0)
with max skew 1 (synth.c4_spread_groups), once HARD (DoNotSchedule) and once SOFT (ScheduleAnyway).  The three forms run
alternately from the same node table: no groups, HARD, SOFT.  Prints one JSON line: ms per cycle (device events,
grove_cycle_stats_t.ms_total, and the host clock around the blocking call), rounds, evaluations, admitted gangs, skewed SOFT members,
and the card with its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_spread.py [--steps 10] [--warmup 2] [--level 0] [--size 8]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--level", type=int, default=0)
    ap.add_argument("--size", type=int, default=8)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    kinds = {"none": None}
    for name, mode in (("hard", T.SPREAD_HARD), ("soft", T.SPREAD_SOFT)):
        kinds[name] = synth.c4_spread_groups(g, c, size=a.size, level=a.level, mode=mode)
    res = {k: [] for k in kinds}
    with PlacementEngine(cfg["n_levels"]) as e:
        for i in range(a.warmup + a.steps):
            for kind, spread in kinds.items():
                e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
                if spread is not None:
                    e.set_spread(*spread)
                t0 = time.perf_counter()
                st = e.run_cycle()
                wall = (time.perf_counter() - t0) * 1e3
                if i >= a.warmup:
                    skewed = int(((e.gang_status()["reserved0"] & T.STATUS_SPREAD_SKEWED) != 0).sum())
                    res[kind].append(dict(ms=st["ms_total"], wall_ms=wall, rounds=st["rounds"], evaluations=st["evaluations"],
                                          admitted=st["gangs_admitted"], skewed=skewed))
    groups, gang_group = kinds["hard"]
    out = dict(workload="C4 with spread groups", nodes=int(len(cfg["nodes"])), gangs=int(len(g)), level=a.level, group_size=a.size,
               groups=int(len(groups)), members=int((gang_group != T.NONE_U32).sum()), max_skew=1, steps=a.steps, **card())
    for kind, rows in res.items():
        out[kind] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows),
                         ms_max=max(r["ms"] for r in rows), wall_ms_median=statistics.median(r["wall_ms"] for r in rows),
                         rounds=rows[-1]["rounds"], evaluations=rows[-1]["evaluations"], gangs_admitted=rows[-1]["admitted"],
                         skewed=rows[-1]["skewed"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
