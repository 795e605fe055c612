"""Reclaim within queue limits on the C4 workload: time grove_run_cycle_preempt_queues on the reduced-C4 queue layout with running
gangs (synth.c4_queues, synth.queue_running: the gangs a C4 queue cycle admitted run in their queues, and the submission is those
gangs again, about half of them at a higher priority), alternating with grove_run_cycle_preempt on the same submission and running
gangs without a queue set.

Each call runs on an engine of its own from the same node table.  Prints one JSON line: per form, ms per call (device events summed
over the cycles, grove_cycle_stats_t.ms_total, and the host clock around the blocking call), priority classes reconsidered,
preemptors, victims (for the queue form split into those holding on a node of their preemptor, which include every node-step
victim, and the others, which the queue step chose), and the card with its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_preempt_queues.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402


def layout():
    cfg = synth.config_c4()
    tables = cfg["tables"]
    qs, gq = synth.c4_queues(*tables[:2])
    with PlacementEngine(cfg["n_levels"]) as e:   # the first cycle: its admitted gangs become the running ones
        e.load_nodes(cfg["nodes"]); e.submit_gangs(*tables); e.set_queues(qs, gq); e.run_cycle()
        nodes, pl, st = e.nodes(), e.placements(), e.gang_status()
    t2, q2, gq2, running, holdings, rq = synth.queue_running(tables, qs, gq, pl, st)
    return cfg["n_levels"], nodes, t2, q2, gq2, running, holdings, rq


def split_victims(victims, placements, status, running, holdings):
    """-> (victims holding on a node of their preemptor, the others)"""
    on = off = 0
    for v in victims:
        g = int(v["preemptor"])
        mine = set(placements["node"][status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]].tolist())
        r = int(v["running"])
        held = holdings["node"][running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]].tolist()
        if mine.intersection(held):
            on += 1
        else:
            off += 1
    return on, off


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    L, nodes, (g, c, s), qs, gq, running, holdings, rq = layout()
    with PlacementEngine(L) as e:   # the classes the reclaim pass reconsiders: priorities of the queue cycle's rejects above a running one
        e.load_nodes(nodes); e.submit_gangs(g, c, s); e.set_queues(qs, gq); e.run_cycle()
        rej = {int(p) for p in g["priority"][e.gang_status()["state"] == T.GANG_REJECTED]}
    classes = len([p for p in rej if len(running) and p > int(running["priority"].min())])
    res = {"queues": [], "no_queue_set": []}
    for i in range(a.warmup + a.steps):
        for k in res:
            with PlacementEngine(L) as e:
                e.load_nodes(nodes); e.submit_gangs(g, c, s)
                if k == "queues":
                    e.set_queues(qs, gq)
                t0 = time.perf_counter()
                st = e.run_cycle_preempt_queues(running, holdings, rq) if k == "queues" else e.run_cycle_preempt(running, holdings)
                host_ms = (time.perf_counter() - t0) * 1e3
                if i < a.warmup:
                    continue
                gs, v = e.gang_status(), e.victims()
                row = dict(ms=st["ms_total"], host_ms=host_ms, preemptors=int(((gs["reserved0"] & T.STATUS_PREEMPTOR) != 0).sum()),
                           victims=int(len(v)), admitted=st["gangs_admitted"])
                if k == "queues":
                    row["victims_on_preemptor_nodes"], row["victims_elsewhere"] = split_victims(v, e.placements(), gs, running, holdings)
                    row["over_limit_left"] = int(((gs["reserved0"] & T.STATUS_OVER_LIMIT) != 0).sum())
                res[k].append(row)
    out = dict(workload="C4 with queue limits and running gangs", nodes=int(len(nodes)), gangs=int(len(g)), running=int(len(running)),
               members=int((gq != T.NONE_U32).sum()), classes=classes, steps=a.steps, **card())
    for k, rows in res.items():
        out[k] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows), ms_max=max(r["ms"] for r in rows),
                      host_ms_median=statistics.median(r["host_ms"] for r in rows),
                      **{x: rows[-1][x] for x in rows[-1] if x not in ("ms", "host_ms")})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
