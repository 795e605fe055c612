"""Rolling update on the C4 cluster: time grove_run_cycle_reuse against grove_run_cycle on the same submission.

One ordinary cycle admits C4's gangs (they are RUNNING from then on).  The next submission carries the gangs that stayed pending
plus new versions of about --share of the running gangs: every other one the same shape, the others asking for twice the memory
per pod.  The two entries run on it alternately, from the same node table: reuse with replacements, the ordinary cycle with none
(the new versions then compete for the free table like everybody else).  Prints one JSON line: ms per cycle (device events,
grove_cycle_stats_t.ms_total, and the host clock around the blocking call), rounds, evaluations, what the new versions got, and
the card with its power limit and SM clock.  Needs a GPU; writes nothing.

    python scripts/bench_rolling.py [--steps 10] [--warmup 2] [--share 0.1]
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

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402


def holdings(placements, status, gangs, cliques):
    """running gangs (T.running_dt) and what each holds per node (T.holding_dt) after a cycle; running gang r = r-th admitted gang"""
    run, hold = [], []
    req = np.stack([cliques["req_cpu_milli"].astype(np.int64), cliques["req_mem_mib"].astype(np.int64), cliques["req_gpu"].astype(np.int64)], 1)
    for g in np.nonzero(status["state"] == T.GANG_ADMITTED)[0]:
        pl = placements[status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]]
        nodes, inv = np.unique(pl["node"], return_inverse=True)
        use = np.zeros((len(nodes), 4), dtype=np.int64)
        np.add.at(use[:, :3], inv, req[pl["clique"]])
        np.add.at(use[:, 3], inv, 1)
        run.append((int(gangs["priority"][g]), len(hold), len(nodes), 0))
        hold += [(int(n), *map(int, u)) for n, u in zip(nodes, use)]
    return np.array(run, dtype=T.running_dt), np.array(hold, dtype=T.holding_dt)


def rolling_submission(gangs, cliques, scopes, status, share, seed):
    """pending gangs + new versions of `share` of the admitted ones -> (tables, replaces)"""
    admitted = np.nonzero(status["state"] == T.GANG_ADMITTED)[0]
    rng = np.random.default_rng(seed)
    picks_r = np.sort(rng.choice(len(admitted), size=max(1, int(len(admitted) * share)), replace=False))
    keep = [int(g) for g in np.nonzero(status["state"] != T.GANG_ADMITTED)[0]]
    # a pending scaled gang whose base gang is running (or not carried over) is no longer gated behind it
    rows = keep + [int(admitted[r]) for r in picks_r]
    new_idx = {g: i for i, g in enumerate(keep)}
    ng, nq, ns = [], [], []
    for i, g in enumerate(rows):
        co, so = int(gangs["clique_off"][g]), int(gangs["scope_off"][g])
        q = cliques[co: co + int(gangs["n_cliques"][g])].copy()
        if i >= len(keep) and (i - len(keep)) % 2:
            q["req_mem_mib"] *= 2
        x = gangs[g: g + 1].copy()
        x["clique_off"] = sum(len(a) for a in nq); x["scope_off"] = sum(len(a) for a in ns)
        b = int(x["base_gang"][0])
        x["base_gang"] = new_idx.get(b, T.NONE_U32) if i < len(keep) and b != T.NONE_U32 else T.NONE_U32
        ng.append(x); nq.append(q); ns.append(scopes[so: so + int(gangs["n_scopes"][g])].copy())
    replaces = np.full(len(rows), T.NONE_U32, dtype=np.uint32)
    replaces[len(keep):] = picks_r
    return (np.concatenate(ng), np.concatenate(nq), np.concatenate(ns)), replaces


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=power, sm_clock_max=clock)
    except Exception as ex:  # the measurement stands without it; say so
        return dict(gpu="unknown", error=str(ex))


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--share", type=float, default=0.1)
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
        rep = replaces != T.NONE_U32
        res = {"reuse": [], "cycle": []}
        for i in range(a.warmup + a.steps):
            for kind in ("reuse", "cycle"):
                e.load_nodes(now); e.submit_gangs(*tables)
                t0 = time.perf_counter()
                st = e.run_cycle_reuse(replaces, running, held) if kind == "reuse" else e.run_cycle()
                wall = (time.perf_counter() - t0) * 1e3
                if i >= a.warmup:
                    got = e.gang_status()["state"][rep] == T.GANG_ADMITTED
                    res[kind].append(dict(ms=st["ms_total"], wall_ms=wall, rounds=st["rounds"], evaluations=st["evaluations"],
                                          admitted=st["gangs_admitted"], new_versions_admitted=int(got.sum())))
    out = dict(workload="C4 rolling update", nodes=int(len(cfg["nodes"])), gangs=int(len(replaces)), new_versions=int(rep.sum()),
               running=int(len(running)), steps=a.steps, **card())
    for kind, rows in res.items():
        out[kind] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows), ms_max=max(r["ms"] for r in rows),
                         wall_ms_median=statistics.median(r["wall_ms"] for r in rows), rounds=rows[-1]["rounds"],
                         evaluations=rows[-1]["evaluations"], gangs_admitted=rows[-1]["admitted"],
                         new_versions_admitted=rows[-1]["new_versions_admitted"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
