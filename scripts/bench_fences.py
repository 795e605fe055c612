"""Fences on the C4 workload: time grove_run_cycle with 0, 16 and 64 fencing gangs on the same submission.

The fencing gangs are the highest-ranked gangs that an ordinary cycle on the same node table rejects and that have a gang Required
level -- the ones a starvation guard would fence first.  The three forms run alternately from the same node table.  Prints one JSON
line: per form, ms per cycle (device events, grove_cycle_stats_t.ms_total, and the host clock around the blocking call), rounds,
evaluations, admitted gangs and fences held at the end, and the card with its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_fences.py [--steps 10] [--warmup 2]
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
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    res = {}
    with PlacementEngine(cfg["n_levels"]) as e:
        e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
        e.run_cycle()
        st = e.gang_status()
        order = sorted(range(len(g)), key=lambda i: (-int(g["priority"][i]), i))
        cand = [x for x in order if st["state"][x] == T.GANG_REJECTED and g["level"][x] != T.LEVEL_NONE]
        kinds = {k: np.array(cand[:k], dtype=np.uint32) for k in (0, 16, 64)}
        res = {k: [] for k in kinds}
        for i in range(a.warmup + a.steps):
            for k, fencing in kinds.items():
                e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
                e.set_fences(fencing)
                t0 = time.perf_counter()
                st = e.run_cycle()
                wall = (time.perf_counter() - t0) * 1e3
                if i >= a.warmup:
                    held = int(((e.gang_status()["reserved0"] & T.STATUS_FENCING) != 0).sum())
                    res[k].append(dict(ms=st["ms_total"], wall_ms=wall, rounds=st["rounds"], evaluations=st["evaluations"],
                                       admitted=st["gangs_admitted"], held=held))
    out = dict(workload="C4 with fences", nodes=int(len(cfg["nodes"])), gangs=int(len(g)), rejected_with_level=len(cand),
               steps=a.steps, **card())
    for k, rows in res.items():
        out[f"fences_{k}"] = dict(fencing=len(kinds[k]), ms_median=statistics.median(r["ms"] for r in rows),
                                  ms_min=min(r["ms"] for r in rows), ms_max=max(r["ms"] for r in rows),
                                  wall_ms_median=statistics.median(r["wall_ms"] for r in rows), rounds=rows[-1]["rounds"],
                                  evaluations=rows[-1]["evaluations"], gangs_admitted=rows[-1]["admitted"],
                                  fences_held=rows[-1]["held"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
