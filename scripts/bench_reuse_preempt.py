"""Rolling update under preemption on the C4 cluster: time grove_run_cycle_reuse_preempt against grove_run_cycle_preempt.

One ordinary cycle admits C4's gangs (three priority classes; they are RUNNING from then on).  The next submission carries the
gangs that stayed pending plus new versions of about --share of the running gangs (scripts/bench_rolling.py), every other one
asking for twice the memory per pod, plus copies of about --pressure of the running gangs below the top priority class, in
the top class: they outrank part of what runs, and the reclaim pass evicts to place them.
Alternately, from the same node table:
  reuse_preempt  grove_run_cycle_reuse_preempt: the new versions reuse their predecessors' reservations, then the reclaim pass
                 with class views built on the device;
  preempt        grove_run_cycle_preempt on the same submission with no replacements: the same reclaim loop with no holds;
  reuse, cycle   their ordinary passes alone (grove_run_cycle_reuse, grove_run_cycle), so that what the reclaim pass adds can
                 be told apart: (entry - its ordinary pass) / classes is the reclaim cost per class.
Prints one JSON line: ms per cycle (device events summed over the cycles of the call, and the host clock around the blocking
call), classes run, rounds, evaluations, victims, and the card with its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_reuse_preempt.py [--steps 10] [--warmup 2] [--share 0.1] [--pressure 0.2]
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_rolling import card, holdings, rolling_submission  # noqa: E402
from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402


def classes_run(gangs, first_status, released, victims, running):
    """the priority classes the reclaim pass ran a cycle for: those of the gangs the ordinary pass rejected while some running
    gang of a lower priority was still standing"""
    gone = np.zeros(len(running), dtype=bool)
    gone[list(released)] = True
    prio = running["priority"].astype(np.int64)
    by_class = {}
    for v in victims:
        by_class.setdefault(int(gangs["priority"][v["preemptor"]]), []).append(int(v["running"]))
    n = 0
    for p in sorted({int(x) for x in gangs["priority"][first_status["state"] == T.GANG_REJECTED]}, reverse=True):
        if not (~gone & (prio < p)).any():
            break
        n += 1
        gone[by_class.get(p, [])] = True
    return n


def with_pressure(gangs, cliques, scopes, status, tables, replaces, share, seed):
    """the submission plus copies of about `share` of the running gangs below the top priority class, in the top class: the
    gangs that stayed pending do not fit even with every running gang evicted (their shapes do not fit C4), copies of running
    gangs do, by evicting.  -> (tables, replaces)"""
    top = int(gangs["priority"].max())
    low = np.nonzero((status["state"] == T.GANG_ADMITTED) & (gangs["priority"] < top))[0]
    rng = np.random.default_rng(seed)
    picks = np.sort(rng.choice(low, size=max(1, int(len(low) * share)), replace=False))
    g, q, sc = tables
    ng, nq, ns = [g], [q], [sc]
    nc, nsc = len(q), len(sc)
    for i in picks:
        co, so = int(gangs["clique_off"][i]), int(gangs["scope_off"][i])
        x = gangs[i: i + 1].copy()
        x["clique_off"] = nc; x["scope_off"] = nsc; x["base_gang"] = T.NONE_U32; x["priority"] = top
        ng.append(x); nq.append(cliques[co: co + int(gangs["n_cliques"][i])]); ns.append(scopes[so: so + int(gangs["n_scopes"][i])])
        nc += int(gangs["n_cliques"][i]); nsc += int(gangs["n_scopes"][i])
    rep = np.concatenate([replaces, np.full(len(picks), T.NONE_U32, dtype=np.uint32)])
    return (np.concatenate(ng), np.concatenate(nq), np.concatenate(ns)), rep


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--share", type=float, default=0.1)
    ap.add_argument("--pressure", type=float, default=0.2)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    L = cfg["n_levels"]
    with PlacementEngine(L) as e:
        e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
        e.run_cycle()
        status, placements, now = e.gang_status(), e.placements(), e.nodes()
        running, held = holdings(placements, status, g, c)
        tables, replaces = rolling_submission(g, c, s, status, a.share, seed=1)
        tables, replaces = with_pressure(g, c, s, status, tables, replaces, a.pressure, seed=2)
        rep = replaces != T.NONE_U32
        kinds = ("reuse_preempt", "preempt", "reuse", "cycle")
        res = {k: [] for k in kinds}
        first = {}
        for i in range(a.warmup + a.steps):
            for kind in kinds:
                e.load_nodes(now); e.submit_gangs(*tables)
                t0 = time.perf_counter()
                if kind == "reuse_preempt":
                    st = e.run_cycle_reuse_preempt(replaces, running, held)
                elif kind == "preempt":
                    st = e.run_cycle_preempt(running, held)
                elif kind == "reuse":
                    st = e.run_cycle_reuse(replaces, running, held)
                else:
                    st = e.run_cycle()
                wall = (time.perf_counter() - t0) * 1e3
                gs = e.gang_status()
                if kind in ("reuse", "cycle"):
                    first[kind] = gs
                if i >= a.warmup:
                    row = dict(ms=st["ms_total"], wall_ms=wall, rounds=st["rounds"], evaluations=st["evaluations"],
                               admitted=st["gangs_admitted"], new_versions_admitted=int((gs["state"][rep] == T.GANG_ADMITTED).sum()))
                    if kind in ("reuse_preempt", "preempt"):
                        vs = e.victims()
                        row["victims"] = int(len(vs))
                        row["_v"] = vs
                        row["preemptors"] = int(((gs["reserved0"] & T.STATUS_PREEMPTOR) != 0).sum())
                        row["released"] = [int(replaces[k]) for k in np.nonzero(rep & (gs["state"] == T.GANG_ADMITTED))[0]] if kind == "reuse_preempt" else []
                    res[kind].append(row)
    out = dict(workload="C4 rolling update under preemption", nodes=int(len(cfg["nodes"])), gangs=int(len(replaces)),
               new_versions=int(rep.sum()), running=int(len(running)), priority_classes=int(len(np.unique(tables[0]["priority"]))),
               steps=a.steps, **card())
    for kind, rows in res.items():
        out[kind] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows),
                         ms_max=max(r["ms"] for r in rows), wall_ms_median=statistics.median(r["wall_ms"] for r in rows),
                         wall_ms_min=min(r["wall_ms"] for r in rows), rounds=rows[-1]["rounds"], evaluations=rows[-1]["evaluations"],
                         gangs_admitted=rows[-1]["admitted"], new_versions_admitted=rows[-1]["new_versions_admitted"])
    for kind, base in (("reuse_preempt", "reuse"), ("preempt", "cycle")):
        last = res[kind][-1]
        ncls = classes_run(tables[0], first[base], last["released"] if kind == "reuse_preempt" else [], last["_v"], running)
        extra = out[kind]["wall_ms_median"] - out[base]["wall_ms_median"]
        out[kind].update(classes_run=ncls, victims=last["victims"], preemptors=last["preemptors"],
                         reclaim_wall_ms=extra, reclaim_wall_ms_per_class=extra / ncls if ncls else None)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
