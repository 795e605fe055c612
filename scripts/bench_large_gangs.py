"""PodGangs of up to 2048 pods on the C4 cluster: time grove_run_cycle on a wide submission against the same cycle without them.

Alternately, from the same node table:
  wide      C4 plus --large PodGangs of 256-2048 pods (synth.config_c4_large) through grove_submit_gangs_wide: the cycle runs
            the wide instantiations of k_eval / k_shape_plaus;
  ordinary  the C4 part alone through grove_submit_gangs: the ordinary instantiations.
Prints one JSON line: median ms per cycle (host clock around the blocking call, which ends in a device synchronise, and the
engine's device-event total), rounds, evaluations, gangs admitted, and the card with its power limit and SM clock read in the
same run.  Then one more wide cycle with GROVE_DEBUG_ADMIT=1 (not timed: the host looks at the control words after every round)
gives the slowest evaluation of a large gang: clock64() cycles on the SM, among the six slowest evaluations the engine reports
per round, and us at the SM clock read in this run.  Needs a GPU; writes nothing.

    python scripts/bench_large_gangs.py [--steps 10] [--warmup 2] [--large 24]
"""
from __future__ import annotations

import argparse
import json
import os
import re
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_rolling import card  # noqa: E402
from grove_b200 import synth  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402


SLOW_RE = re.compile(r"\[g(\d+) rank\d+ st\d+ scopes\d+: (\d+) cyc, (\d+) plaus, (\d+) att\]")


def slowest_large_evaluation(cfg, first_large) -> dict:
    """one wide cycle with GROVE_DEBUG_ADMIT=1: the slowest evaluation of a gang of index >= first_large in the per-round
    reports the engine writes to stderr"""
    os.environ["GROVE_DEBUG_ADMIT"] = "1"
    try:
        e = PlacementEngine(cfg["n_levels"])
    finally:
        del os.environ["GROVE_DEBUG_ADMIT"]
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            e.load_nodes(cfg["nodes"]); e.submit_gangs_wide(*cfg["tables"]); e.run_cycle()
        finally:
            os.dup2(saved, 2); os.close(saved)
        f.seek(0)
        text = f.read()
    e.close()
    every = [(int(g), int(c), int(a)) for g, c, _, a in SLOW_RE.findall(text)]
    ordinary = [x for x in every if x[0] < first_large]
    large = [x for x in every if x[0] >= first_large]
    out = dict(slowest_ordinary_cyc=max((x[1] for x in ordinary), default=None))
    if not large:
        return dict(out, slowest_large_cyc=None, note="no large gang among any round's six slowest evaluations")
    g, c, a = max(large, key=lambda x: x[1])
    return dict(out, slowest_large_cyc=c, slowest_large_gang=g, slowest_large_attempts=a)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--large", type=int, default=24)
    args = ap.parse_args()
    cfg = synth.config_c4_large(n_large=args.large)
    runs = {"wide": [], "ordinary": []}
    with PlacementEngine(cfg["n_levels"]) as e:
        for step in range(args.warmup + args.steps):
            for kind in ("wide", "ordinary"):
                e.load_nodes(cfg["nodes"])
                if kind == "wide":
                    e.submit_gangs_wide(*cfg["tables"])
                else:
                    e.submit_gangs(*cfg["ordinary"])
                t0 = time.perf_counter()
                st = e.run_cycle()
                ms = (time.perf_counter() - t0) * 1e3
                if step >= args.warmup:
                    runs[kind].append((ms, float(st["ms_total"]), int(st["rounds"]), int(st["evaluations"]), int(st["gangs_admitted"])))
    line = dict(bench="large_gangs", config="C4", gangs=len(cfg["tables"][0]), large=args.large, steps=args.steps, **card())
    for kind, rs in runs.items():
        line[kind] = dict(ms_host=statistics.median(r[0] for r in rs), ms_device=statistics.median(r[1] for r in rs),
                          rounds=rs[-1][2], evaluations=rs[-1][3], admitted=rs[-1][4])
    dbg = slowest_large_evaluation(cfg, len(cfg["ordinary"][0]))
    mhz = line.get("sm_clock_max", "").split()[0] if line.get("sm_clock_max") else None
    if dbg.get("slowest_large_cyc") and mhz:
        dbg["slowest_large_us"] = dbg["slowest_large_cyc"] / float(mhz)
    line["debug_admit"] = dbg
    print(json.dumps(line))


if __name__ == "__main__":
    main()
