"""Reclaim across queues on the C4 workload: time grove_run_cycle_reclaim_queues on the C4 queue layout with running gangs
(synth.c4_queues, synth.queue_running) and deserved quotas from synth.c4_queue_quotas (the first leaves above their quota, the last
below it), alternating with grove_run_cycle_preempt_queues and the plain queue cycle (grove_run_cycle) on the same inputs.  The
defaults (leaf limits at 0.6 of demand, quota spread 1.2) are a layout in which the class pass admits gangs and evicts.

Each call runs on an engine of its own from the same node table.  Prints one JSON line: per form, ms per call (device events summed
over the cycles, grove_cycle_stats_t.ms_total, and the host clock around the blocking call), the classes the pass considers (queues
of the queue cycle's rejected gangs), reclaimers or preemptors, victims (split into those holding on a node of their reclaimer, which
include every node-step victim, and the others, which the queue step chose), and the card with its power limit and SM clock.  Needs
a GPU; writes nothing.

    python scripts/bench_reclaim_queues.py [--steps 10] [--warmup 2] [--share 0.6] [--spread 1.2]
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
from scripts.bench_preempt_queues import split_victims  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402

FORMS = ("reclaim_queues", "preempt_queues", "queue_cycle")


def layout(share):
    """bench_preempt_queues.layout with leaf limits at `share` of their members' demand"""
    cfg = synth.config_c4()
    tables = cfg["tables"]
    qs, gq = synth.c4_queues(*tables[:2], share=share)
    with PlacementEngine(cfg["n_levels"]) as e:   # the first cycle: its admitted gangs become the running ones
        e.load_nodes(cfg["nodes"]); e.submit_gangs(*tables); e.set_queues(qs, gq); e.run_cycle()
        nodes, pl, st = e.nodes(), e.placements(), e.gang_status()
    t2, q2, gq2, running, holdings, rq = synth.queue_running(tables, qs, gq, pl, st)
    return cfg["n_levels"], nodes, t2, q2, gq2, running, holdings, rq


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--share", type=float, default=0.6, help="leaf limits as a share of their members' demand (synth.c4_queues)")
    ap.add_argument("--spread", type=float, default=1.2, help="synth.c4_queue_quotas spread")
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    L, nodes, (g, c, s), qs, gq, running, holdings, rq = layout(a.share)
    quotas = synth.c4_queue_quotas(qs, running, holdings, rq, spread=a.spread)
    with PlacementEngine(L) as e:   # the classes: the queues of the queue cycle's rejected gangs
        e.load_nodes(nodes); e.submit_gangs(g, c, s); e.set_queues(qs, gq); e.run_cycle()
        rej = e.gang_status()["state"] == T.GANG_REJECTED
    classes = len({int(q) for q in gq[rej] if q != T.NONE_U32})
    res = {k: [] for k in FORMS}
    for i in range(a.warmup + a.steps):
        for k in FORMS:
            with PlacementEngine(L) as e:
                e.load_nodes(nodes); e.submit_gangs(g, c, s); e.set_queues(qs, gq)
                t0 = time.perf_counter()
                if k == "reclaim_queues":
                    st = e.run_cycle_reclaim_queues(quotas, running, holdings, rq)
                elif k == "preempt_queues":
                    st = e.run_cycle_preempt_queues(running, holdings, rq)
                else:
                    st = e.run_cycle()
                host_ms = (time.perf_counter() - t0) * 1e3
                if i < a.warmup:
                    continue
                gs = e.gang_status()
                row = dict(ms=st["ms_total"], host_ms=host_ms, admitted=st["gangs_admitted"], kernel_launches=st["kernel_launches"])
                if k != "queue_cycle":
                    v = e.victims()
                    flag = T.STATUS_RECLAIMER if k == "reclaim_queues" else T.STATUS_PREEMPTOR
                    row["admitted_by_pass"] = int(((gs["reserved0"] & flag) != 0).sum())
                    row["victims"] = int(len(v))
                    row["victims_on_admitted_nodes"], row["victims_elsewhere"] = split_victims(v, e.placements(), gs, running, holdings)
                res[k].append(row)
    out = dict(workload="C4 with queue limits, deserved quotas and running gangs", nodes=int(len(nodes)), gangs=int(len(g)),
               running=int(len(running)), members=int((gq != T.NONE_U32).sum()), classes=classes, share=a.share, spread=a.spread,
               steps=a.steps, **card())
    for k, rows in res.items():
        out[k] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows), ms_max=max(r["ms"] for r in rows),
                      host_ms_median=statistics.median(r["host_ms"] for r in rows),
                      **{x: rows[-1][x] for x in rows[-1] if x not in ("ms", "host_ms")})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
