"""Consolidation on the C4 workload: grove_run_cycle_consolidate against grove_run_cycle on the same submission.

The cluster is C4 (pre-used up to 60 % instead of 90 %, so that a displaced gang can find room) after an ordinary cycle: the gangs it
admitted are RUNNING and every one of them is movable, restated as a gated
spec row of the new submission (a second C4-shaped submission on the same nodes).  The targets are the 16 highest-ranked gangs with
a gang Required level that the ordinary cycle rejects -- the ones a starvation guard would name first.  The two entries run
alternately, each on an engine of its own created for the call (a second grove_run_cycle of this workload on one handle does not
reproduce the first one's result, with or without consolidation: DESIGN.md section 9), so every call includes its buffer
allocations.  Prints one JSON line: per entry, ms per call (the summed grove_cycle_stats_t.ms_total of device events, and the host
clock around the blocking call); for the consolidation pass the tries, commits and moves, with tries counted by the restatement in
tests/consolidate_cases.py over the CPU oracle, whose outputs the engine's must equal; and the card with its power limit, its
maximum SM clock and the SM clock read right after the timed calls.  Needs a GPU; writes nothing.

    python scripts/bench_consolidate.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_rolling import card, holdings  # noqa: E402
from consolidate_cases import run_cycle_consolidate, top_rejected, with_specs  # noqa: E402
from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    first = synth.config_c4(max_used_pct=60)
    second = synth.config_c4(seed=synth.SEED_BASE + 4 + 7919)
    L = first["n_levels"]
    with PlacementEngine(L) as e:
        e.load_nodes(first["nodes"]); e.submit_gangs(*first["tables"])
        e.run_cycle()
        st1 = e.gang_status()
        running, held = holdings(e.placements(), st1, *first["tables"][:2])
        free = e.nodes()
    admitted = [int(g) for g in np.nonzero(st1["state"] == T.GANG_ADMITTED)[0]]
    tables, spec_of = with_specs(second["tables"], first["tables"], admitted)
    with PlacementEngine(L) as e:
        e.load_nodes(free); e.submit_gangs(*tables)
        e.run_cycle()
        targets = top_rejected(dict(status=e.gang_status()), tables[0], level_only=True)
    res = {"plain": [], "consolidate": []}
    outs = None
    for i in range(a.warmup + a.steps):
        for kind in res:
            with PlacementEngine(L) as e:
                e.load_nodes(free); e.submit_gangs(*tables)
                t0 = time.perf_counter()
                st = e.run_cycle() if kind == "plain" else e.run_cycle_consolidate(targets, spec_of, running, held)
                wall = (time.perf_counter() - t0) * 1e3
                if i >= a.warmup:
                    res[kind].append(dict(ms=st["ms_total"], wall_ms=wall))
                if kind == "consolidate" and outs is None:
                    outs = dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                                moves=e.moves())
    sm_now = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    from oracle import oracle_py
    oracle_py.build()
    trace = {}
    ref = run_cycle_consolidate(oracle_py, free, L, *tables, targets, spec_of, running, held, trace=trace)
    same = all(np.array_equal(outs[k], ref[k]) for k in ("status", "placements", "scope_status", "nodes_after", "moves"))
    out = dict(workload="C4 with the gangs of an earlier cycle running, all movable", nodes=int(len(free)), gangs=int(len(tables[0])),
               running=int(len(running)), targets=int(len(targets)), steps=a.steps, sm_clock_after_timing=sm_now, **card())
    for kind, rows in res.items():
        out[kind] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows),
                         ms_max=max(r["ms"] for r in rows), wall_ms_median=statistics.median(r["wall_ms"] for r in rows),
                         wall_ms_min=min(r["wall_ms"] for r in rows), wall_ms_max=max(r["wall_ms"] for r in rows))
    out["consolidate"].update(tries=trace["tries"], commits=int(((outs["status"]["reserved0"] & T.STATUS_CONSOLIDATED) != 0).sum()),
                              moves=int(len(outs["moves"])), identical_to_restatement=bool(same))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
