"""Reclaim, then preempt, on the C4 workload: time grove_run_cycle_reclaim_preempt_queues on the C4 queue layout with running gangs
(synth.c4_queues, synth.queue_running) and deserved quotas from synth.c4_queue_quotas, alternating with
grove_run_cycle_reclaim_queues, grove_run_cycle_preempt_queues and the plain queue cycle (grove_run_cycle) on the same inputs.  The
layout is bench_reclaim_queues's (leaf limits at 0.6 of demand, quota spread 1.2), in which both passes admit gangs and evict.

Each call runs on an engine of its own from the same node table.  Prints one JSON line: per form, ms per call (device events summed
over the cycles, grove_cycle_stats_t.ms_total, and the host clock around the blocking call), per pass the classes it considers
(reclaim: the queues of the queue cycle's rejected gangs; preempt: the priorities of the gangs still rejected when it starts), the
gangs it admits and the victims it chooses (told apart by the flag of the gang that evicts them), and the card with its power limit
and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_reclaim_preempt_queues.py [--steps 10] [--warmup 2] [--share 0.6] [--spread 1.2]
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
from scripts.bench_reclaim_queues import layout  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402

FORMS = ("reclaim_preempt_queues", "reclaim_queues", "preempt_queues", "queue_cycle")


def run(form, L, nodes, tables, qs, gq, quotas, running, holdings, rq):
    """one call of `form` on an engine of its own -> (stats, host ms, statuses, victims)"""
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq)
        t0 = time.perf_counter()
        if form == "reclaim_preempt_queues":
            st = e.run_cycle_reclaim_preempt_queues(quotas, running, holdings, rq)
        elif form == "reclaim_queues":
            st = e.run_cycle_reclaim_queues(quotas, running, holdings, rq)
        elif form == "preempt_queues":
            st = e.run_cycle_preempt_queues(running, holdings, rq)
        else:
            st = e.run_cycle()
        host_ms = (time.perf_counter() - t0) * 1e3
        return st, host_ms, e.gang_status(), (e.victims() if form != "queue_cycle" else None)


def per_pass(gs, victims):
    """gangs admitted and victims chosen by each pass, told apart by the evicting gang's flag"""
    out = {}
    for name, flag in (("reclaim", T.STATUS_RECLAIMER), ("preempt", T.STATUS_PREEMPTOR)):
        mine = (gs["reserved0"] & flag) != 0
        out[f"{name}_admitted"] = int(mine.sum())
        out[f"{name}_victims"] = int(mine[victims["preemptor"]].sum()) if victims is not None and len(victims) else 0
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--share", type=float, default=0.6, help="leaf limits as a share of their members' demand (synth.c4_queues)")
    ap.add_argument("--spread", type=float, default=1.2, help="synth.c4_queue_quotas spread")
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    L, nodes, tables, qs, gq, running, holdings, rq = layout(a.share)
    quotas = synth.c4_queue_quotas(qs, running, holdings, rq, spread=a.spread)
    args = (L, nodes, tables, qs, gq, quotas, running, holdings, rq)
    prio = tables[0]["priority"]
    # the classes each pass considers: the reclaim pass's from the queue cycle, the preempt pass's from what is left rejected
    # before it (the queue cycle's rejected gangs for preempt_queues, the reclaim pass's for the new entry)
    _, _, qc, _ = run("queue_cycle", *args)
    _, _, rc, _ = run("reclaim_queues", *args)
    rej_q, rej_r = qc["state"] == T.GANG_REJECTED, rc["state"] == T.GANG_REJECTED
    classes = dict(reclaim=len({int(q) for q in gq[rej_q] if q != T.NONE_U32}), preempt_after_queue_cycle=len(set(prio[rej_q].tolist())),
                   preempt_after_reclaim=len(set(prio[rej_r].tolist())))
    res = {k: [] for k in FORMS}
    for i in range(a.warmup + a.steps):
        for k in FORMS:
            st, host_ms, gs, v = run(k, *args)
            if i < a.warmup:
                continue
            row = dict(ms=st["ms_total"], host_ms=host_ms, admitted=st["gangs_admitted"], kernel_launches=st["kernel_launches"])
            if v is not None:
                row.update(per_pass(gs, v), victims=int(len(v)))
            res[k].append(row)
    out = dict(workload="C4 with queue limits, deserved quotas and running gangs", nodes=int(len(nodes)), gangs=int(len(tables[0])),
               running=int(len(running)), members=int((gq != T.NONE_U32).sum()), classes=classes, share=a.share, spread=a.spread,
               steps=a.steps, **card())
    for k, rows in res.items():
        out[k] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows), ms_max=max(r["ms"] for r in rows),
                      host_ms_median=statistics.median(r["host_ms"] for r in rows),
                      **{x: rows[-1][x] for x in rows[-1] if x not in ("ms", "host_ms")})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
