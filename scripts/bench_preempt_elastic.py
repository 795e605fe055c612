"""Elastic reclaim on the C4 cluster: time grove_run_cycle_preempt_elastic against grove_run_cycle_preempt.

One ordinary cycle admits C4's gangs with about --surplus-share of the worker PodGroups scaled out by 1-3 pods above MinReplicas
(synth.c4_surplus); they are RUNNING from then on, and their pods above MinReplicas are the surplus pods.  The next submission
is copies of about --pressure of the running gangs below the top priority class (bench_reuse_preempt.with_pressure), every
other one a priority above the top class and the rest in it: they outrank part of what runs.
Alternately, from the same node table, each call on a fresh handle (a handle's node table after a running-gang cycle is the
caller's to refresh, DESIGN.md section 9):
  elastic   grove_run_cycle_preempt_elastic: every class takes surplus pods first (pass 1), then evicts whole gangs (pass 2);
  preempt   grove_run_cycle_preempt on the same inputs: whole-gang eviction only.
Prints one JSON line: ms per call (device events summed over the cycles of the call, and the host clock around the blocking
call), priority classes, preemptors per pass (read off the status flags), whole victims, surplus pods taken, running gangs
disrupted, and the card with its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_preempt_elastic.py [--steps 10] [--warmup 2] [--pressure 0.2] [--surplus-share 0.5]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_reuse_preempt import with_pressure  # noqa: E402
from bench_rolling import card, holdings  # noqa: E402
from elastic_cases import surplus_of  # noqa: E402
from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pressure", type=float, default=0.2)
    ap.add_argument("--surplus-share", type=float, default=0.5)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    c = synth.c4_surplus(c, share=a.surplus_share)
    L = cfg["n_levels"]
    with PlacementEngine(L) as e:
        e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
        e.run_cycle()
        status, placements, now = e.gang_status(), e.placements(), e.nodes()
    running, held = holdings(placements, status, g, c)
    surplus = surplus_of(placements, status, g, c)
    empty = (np.zeros(0, T.gang_dt), np.zeros(0, T.clique_dt), np.zeros(0, T.scope_dt))
    tables, _ = with_pressure(g, c, s, status, empty, np.zeros(0, np.uint32), a.pressure, seed=2)
    tables[0]["priority"][0::2] += 1
    kinds = ("elastic", "preempt")
    res = {k: [] for k in kinds}
    for i in range(a.warmup + a.steps):
        for kind in kinds:
            with PlacementEngine(L) as e:
                e.load_nodes(now); e.submit_gangs(*tables)
                t0 = time.perf_counter()
                if kind == "elastic":
                    st = e.run_cycle_preempt_elastic(running, held, surplus)
                else:
                    st = e.run_cycle_preempt(running, held)
                wall = (time.perf_counter() - t0) * 1e3
                if i < a.warmup:
                    continue
                gs, vs = e.gang_status(), e.victims()
                sv = e.surplus_victims() if kind == "elastic" else np.zeros(0, T.surplus_victim_dt)
            pre = (gs["reserved0"] & T.STATUS_PREEMPTOR) != 0
            only = (gs["reserved0"] & T.STATUS_SURPLUS_ONLY) != 0
            hit = set(int(x) for x in vs["running"]) | set(int(x) for x in surplus["running"][sv["pod"]])
            res[kind].append(dict(ms=st["ms_total"], wall_ms=wall, rounds=st["rounds"], evaluations=st["evaluations"],
                                  admitted=st["gangs_admitted"], preemptors_pass1=int(only.sum()),
                                  preemptors_pass2=int((pre & ~only).sum()), whole_victims=int(len(vs)),
                                  surplus_pods_taken=int(len(sv)), gangs_disrupted=len(hit)))
    prio = tables[0]["priority"]
    out = dict(workload="C4 elastic reclaim", nodes=int(len(now)), running=int(len(running)), surplus_pods=int(len(surplus)),
               gangs=int(len(prio)), priority_classes=int(len(np.unique(prio))), steps=a.steps, **card())
    for kind, rows in res.items():
        last = rows[-1]
        out[kind] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows),
                         ms_max=max(r["ms"] for r in rows), wall_ms_median=statistics.median(r["wall_ms"] for r in rows),
                         wall_ms_min=min(r["wall_ms"] for r in rows),
                         **{k: v for k, v in last.items() if k not in ("ms", "wall_ms")})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
