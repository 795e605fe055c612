"""Queue limits on the C4 workload: time grove_run_cycle with the reduced-C4 queue layout (synth.c4_queues: eight leaves under two
parents, each leaf's GPU limit 30 % of its members' MinReplicas GPU demand -- the cluster alone admits about 60 % of C4's gangs,
so at one half no limit would bind) and with every limit unlimited, on the same submission.

The two forms run alternately from the same node table, each on an engine of its own call.  Prints one JSON line: per form, ms per
cycle (device events, grove_cycle_stats_t.ms_total), rounds, evaluations, admitted gangs and OVER_LIMIT gangs, and the card with
its power limit and SM clock.  The cost of the two queue kernels per round is not measured here.  Needs a GPU; writes nothing.

    python scripts/bench_queues.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402
from scripts.bench_rolling import card  # noqa: E402


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if a.steps < 1:
        ap.error("--steps must be at least 1")
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    limited, gq = synth.c4_queues(g, c)
    unlimited = limited.copy()
    unlimited["limit"] = T.QUEUE_UNLIMITED
    kinds = {"limited": limited, "unlimited": unlimited}
    res = {k: [] for k in kinds}
    for i in range(a.warmup + a.steps):
        for k, qs in kinds.items():
            with PlacementEngine(cfg["n_levels"]) as e:
                e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
                e.set_queues(qs, gq)
                st = e.run_cycle()
                if i >= a.warmup:
                    over = int(((e.gang_status()["reserved0"] & T.STATUS_OVER_LIMIT) != 0).sum())
                    res[k].append(dict(ms=st["ms_total"], rounds=st["rounds"], evaluations=st["evaluations"],
                                       admitted=st["gangs_admitted"], over=over))
    out = dict(workload="C4 with queue limits", nodes=int(len(cfg["nodes"])), gangs=int(len(g)), members=int((gq != T.NONE_U32).sum()),
               steps=a.steps, **card())
    for k, rows in res.items():
        out[k] = dict(ms_median=statistics.median(r["ms"] for r in rows), ms_min=min(r["ms"] for r in rows),
                      ms_max=max(r["ms"] for r in rows), rounds=rows[-1]["rounds"], evaluations=rows[-1]["evaluations"],
                      gangs_admitted=rows[-1]["admitted"], over_limit=rows[-1]["over"])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
