"""Over-quota weight on the C4 workload: time grove_run_cycle_reclaim_queues on the C4 queue layout with running gangs
(scripts/bench_reclaim_queues.layout) and synth.c4_queue_quotas, with GPU over-quota weights by leaf (1 + leaf index mod 4) and
without weights, alternating, an engine per call from the same node table; then the fair-share kernels' own time in a
torch.profiler run of its own; then grove_run_cycle with a fair-share set on C4 with nothing running, with and without weights.

Prints one JSON line: per form, ms per call (device events summed over the cycles, grove_cycle_stats_t.ms_total, and the host
clock around the blocking call), reclaimers and victims; the k_oq_* kernels' summed device time per call; and the card with its
power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_over_quota.py [--steps 10] [--warmup 2]
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


def leaf_weights(n):
    w = np.zeros(n, dtype=T.queue_weight_dt)
    w["over_quota"] = 1
    w["over_quota"][2:, 2] = 1 + np.arange(n - 2) % 4
    return w


def fair_share_c4():
    """C4 with nothing running, synth.c4_queues, deserved GPU quotas 0.15-0.5 of each leaf's MinReplicas demand"""
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    qs, gq = synth.c4_queues(g, c)
    gpu = c["min_replicas"].astype(np.int64) * c["req_gpu"].astype(np.int64)
    per_gang = np.array([gpu[int(o): int(o) + int(k)].sum() for o, k in zip(g["clique_off"], g["n_cliques"])], dtype=np.int64)
    need = np.bincount(gq, weights=per_gang, minlength=len(qs))
    quotas = np.zeros(len(qs), dtype=T.queue_quota_dt)
    quotas["deserved"] = T.QUEUE_UNLIMITED
    for i in range(8):
        quotas["deserved"][2 + i, 2] = int(need[2 + i] * (0.15 + 0.05 * i))
    return cfg["n_levels"], cfg["nodes"], (g, c, s), qs, gq, quotas


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    L, nodes, (g, c, s), qs, gq, running, holdings, rq = layout(0.6)
    quotas = synth.c4_queue_quotas(qs, running, holdings, rq, spread=1.2)
    w = leaf_weights(len(qs))
    out = dict(workload="C4 with queue limits, deserved quotas, running gangs and GPU over-quota weights by leaf", nodes=int(len(nodes)),
               gangs=int(len(g)), running=int(len(running)), steps=a.steps, **card())

    def reclaim(weights):
        with PlacementEngine(L) as e:
            e.load_nodes(nodes); e.submit_gangs(g, c, s); e.set_queues(qs, gq)
            if weights is not None:
                e.set_over_quota(weights)
            t0 = time.perf_counter()
            st = e.run_cycle_reclaim_queues(quotas, running, holdings, rq)
            host_ms = (time.perf_counter() - t0) * 1e3
            gs = e.gang_status()
            row = dict(ms=st["ms_total"], host_ms=host_ms, reclaimers=int(((gs["reserved0"] & T.STATUS_RECLAIMER) != 0).sum()),
                       victims=int(len(e.victims())))
            if weights is not None:
                row["fair_gpu"] = e.fair_shares(len(qs))[:, 2].tolist()
            return row

    res = {"reclaim_weights": [], "reclaim_plain": []}
    for i in range(a.warmup + a.steps):
        for k, weights in (("reclaim_weights", w), ("reclaim_plain", None)):
            row = reclaim(weights)
            if i >= a.warmup:
                res[k].append(row)
    for k, rows in res.items():
        out[k] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows),
                      ms_max=max(r["ms"] for r in rows), host_ms_median=statistics.median(r["host_ms"] for r in rows),
                      **{x: rows[-1][x] for x in rows[-1] if x not in ("ms", "host_ms")})

    # the fair-share kernels' own time: a profiled run of the weighted form alone
    import torch
    from torch.profiler import ProfilerActivity, profile
    calls = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            reclaim(w)
        torch.cuda.synchronize()
    kern = {}
    for ev in prof.key_averages():
        if ev.key.startswith(("_Z11k_oq", "_Z13k_oq", "_Z9k_oq", "k_oq")):
            kern[ev.key] = dict(calls=ev.count, us_total=ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total)
    out["oq_kernels"] = kern
    out["oq_kernels_us_per_call"] = sum(v["us_total"] for v in kern.values()) / calls

    # the fair-share order, empty form (nothing running), with and without weights
    L2, nodes2, tb2, qs2, gq2, quotas2 = fair_share_c4()
    fs = {"fair_share_weights": [], "fair_share_plain": []}
    for i in range(a.warmup + a.steps):
        for k in fs:
            with PlacementEngine(L2) as e:
                e.load_nodes(nodes2); e.submit_gangs(*tb2); e.set_queues(qs2, gq2); e.set_fair_share(quotas2)
                if k == "fair_share_weights":
                    e.set_over_quota(leaf_weights(len(qs2)))
                t0 = time.perf_counter()
                st = e.run_cycle()
                host_ms = (time.perf_counter() - t0) * 1e3
                if i >= a.warmup:
                    fs[k].append(dict(ms=st["ms_total"], host_ms=host_ms, admitted=st["gangs_admitted"]))
    for k, rows in fs.items():
        out[k] = dict(ms_median=statistics.median(r["ms"] for r in rows), host_ms_median=statistics.median(r["host_ms"] for r in rows),
                      admitted=rows[-1]["admitted"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
