"""ComputeDomain exclusivity on the C4 workload: grove_run_cycle without a set, and with one CD per PCS replica (every base gang and
the gangs scaled from it, their GPU cliques enrolled; synth.c4_compute_domains) and half of the pre-used nodes held by CDs that
already run.

The two arms run alternately on the same tables, each cycle on a fresh engine (a fresh handle per cycle keeps one arm's state from
reaching the next).  Per arm: ms per cycle (device events, grove_cycle_stats_t.ms_total), rounds, evaluations, gangs admitted and
pods bound.  Prints one JSON line with the card, its power limit, its maximum SM clock and the SM clock read right after the timed
cycles.  Needs a GPU; writes nothing.

    python scripts/bench_imex.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402


def sm_clock():
    """the SM clock the card runs at now (nvidia-smi clocks.sm), read in the same run as the cycles"""
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as ex:  # the measurement stands without it; say so
        return f"unknown ({ex})"


def _cycle(cfg, cds):
    with PlacementEngine(cfg["n_levels"]) as e:
        e.load_nodes(cfg["nodes"]); e.submit_gangs(*cfg["tables"])
        if cds is not None:
            e.set_compute_domains(*cds)
        return e.run_cycle()


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    cfg = synth.config_c4()
    g, c, _ = cfg["tables"]
    cd, owner0 = synth.c4_compute_domains(cfg["nodes"], g, c)
    arms = {"none": None, "cd": (cd, owner0)}
    rows = {k: [] for k in arms}
    for i in range(a.warmup + a.steps):
        for k, cds in arms.items():
            st = _cycle(cfg, cds)
            if i >= a.warmup:
                rows[k].append(st)
    clock = sm_clock()
    out = dict(workload="C4 ComputeDomains", nodes=int(len(cfg["nodes"])), gangs=int(len(g)), steps=a.steps,
               enrolled_cliques=int((cd != T.CD_NONE).sum()), owned_nodes=int((owner0 != T.CD_NONE).sum()), **card(), sm_clock_after=clock)
    for k, r in rows.items():
        out[k] = dict(ms_median=statistics.median(x["ms_total"] for x in r), ms_min=min(x["ms_total"] for x in r),
                      ms_max=max(x["ms_total"] for x in r), rounds=r[-1]["rounds"], evaluations=r[-1]["evaluations"],
                      gangs_admitted=r[-1]["gangs_admitted"], pods_bound=r[-1]["pods_bound"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
