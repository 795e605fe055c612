"""Fair-share order on the C4 workload: time grove_run_cycle with a fair-share set (grove_set_fair_share) on the C4 queue layout
(synth.c4_queues), alternating with the plain queue cycle on the same inputs, in two forms:

  empty    nothing runs yet; each leaf deserves 0.15 to 0.5 of its members' MinReplicas GPU demand (leaf i: 0.15 + 0.05 i), so
           the leaves' shares part early in the cycle and the order moves away from rank order;
  running  bench_reclaim_queues's layout (leaf limits at 0.6 of demand): the gangs a first queue cycle admitted run
           (synth.queue_running, counted in each queue's `used`) and the quotas are synth.c4_queue_quotas's, some leaves above
           their quota and some below.

Besides the two cycles, the plain queue cycle in the fair-share cycle's turn order (priority := G - turn position): the last
queue cycle of the fixed point with nothing left to re-run, which says what one iteration costs because of the order it runs in.

Each call runs on an engine of its own from the same node table.  Prints one JSON line: per form and cycle, ms per call (device
events, grove_cycle_stats_t.ms_total: for the fair-share cycle the sum over its queue cycles and its O(R) computations; and the host
clock around the blocking call), relaxation rounds, for the fair-share cycle the iterations and the turns re-run
(grove_get_fair_share_stats), the gangs admitted, and the card with its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_fair_share.py [--steps 5] [--warmup 1] [--share 0.3]
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
from scripts.bench_reclaim_queues import layout  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402


def empty_form(share):
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    qs, gq = synth.c4_queues(g, c, share=share)
    gpu = c["min_replicas"].astype(np.int64) * c["req_gpu"].astype(np.int64)
    per_gang = np.array([gpu[int(o): int(o) + int(k)].sum() for o, k in zip(g["clique_off"], g["n_cliques"])], dtype=np.int64)
    need = np.bincount(gq, weights=per_gang, minlength=len(qs))
    quotas = np.zeros(len(qs), dtype=T.queue_quota_dt)
    quotas["deserved"] = T.QUEUE_UNLIMITED
    for i in range(8):
        quotas["deserved"][2 + i, 2] = int(need[2 + i] * (0.15 + 0.05 * i))
    return cfg["n_levels"], cfg["nodes"], (g, c, s), qs, gq, quotas


def running_form(share):
    L, nodes, tables, qs, gq, running, holdings, rq = layout(0.6)   # (bench_reclaim_queues's layout: the running gangs fill the leaves)
    return L, nodes, tables, qs, gq, synth.c4_queue_quotas(qs, running, holdings, rq)


def run(form, L, nodes, tables, qs, gq, quotas, order=None):
    """one call -> (row, turn order of a fair-share cycle or None)"""
    g, c, s = tables
    if form == "in_turn_order":   # priority := G - turn position: a plain queue cycle takes the gangs in that order
        g = g.copy()
        g["priority"][order.astype(np.int64)] = len(g) - np.arange(len(g))
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(g, c, s); e.set_queues(qs, gq)
        if form == "fair_share":
            e.set_fair_share(quotas)
        t0 = time.perf_counter()
        st = e.run_cycle()
        host_ms = (time.perf_counter() - t0) * 1e3
        row = dict(ms=st["ms_total"], host_ms=host_ms, admitted=st["gangs_admitted"], rounds=st["rounds"])
        if form == "fair_share":
            row.update(e.fair_share_stats())
            return row, e.turn_order()
        return row, None


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--share", type=float, default=0.3, help="leaf limits as a share of their members' demand (synth.c4_queues)")
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    out = dict(workload="C4 in synth.c4_queues", share=a.share, steps=a.steps, **card())
    for name, make in (("empty", empty_form), ("running", running_form)):
        args = make(a.share)
        res = {"fair_share": [], "queue_cycle": [], "in_turn_order": []}
        order = None
        for i in range(a.warmup + a.steps):
            for k in res:
                row, o = run(k, *args, order=order)
                order = o if o is not None else order
                if i >= a.warmup:
                    res[k].append(row)
        form = dict(members=int((args[4] != T.NONE_U32).sum()), gangs=int(len(args[2][0])))
        for k, rows in res.items():
            form[k] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows),
                           ms_max=max(r["ms"] for r in rows), host_ms_median=statistics.median(r["host_ms"] for r in rows),
                           **{x: rows[-1][x] for x in rows[-1] if x not in ("ms", "host_ms")})
        out[name] = form
    print(json.dumps(out))


if __name__ == "__main__":
    main()
