"""Cost of grove_diagnose (why each rejected PodGang did not fit) after a C4 cycle and after the same cycle on a shrunken
node table.

For each workload: one grove_run_cycle, then --warmup + --steps grove_diagnose calls on its outputs (the call reads the cycle's
outputs and changes none of them, so every call does the same work).  Per workload it prints the rejected gangs, the median
ms per call by the host clock around the blocking call, and the device time per call: every kernel, copy and memset of the
timed calls as recorded by torch.profiler (CUPTI), divided by the calls.  One JSON line, with the card, its power limit and SM
clock read in the same run.  Needs a GPU; writes nothing.

    python scripts/bench_diagnose.py [--steps 20] [--warmup 3] [--shrunk-nodes 10080]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_rolling import card  # noqa: E402
from grove_b200 import synth, tables as T  # noqa: E402
from grove_b200.engine import PlacementEngine  # noqa: E402


def measure(cfg, steps: int, warmup: int) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile

    with PlacementEngine(cfg["n_levels"]) as e:
        e.load_nodes(cfg["nodes"])
        e.submit_gangs(*cfg["tables"])
        st = e.run_cycle()
        status = e.gang_status()
        for _ in range(warmup):
            gd, _ = e.diagnose()
        host = []
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                t0 = time.perf_counter()
                gd, _ = e.diagnose()
                host.append((time.perf_counter() - t0) * 1e3)
            torch.cuda.synchronize()
        dev_us = sum(ev.device_time_total for ev in prof.key_averages() if ev.device_time_total and ev.device_type.name == "CUDA")
        kern = {ev.key: ev.device_time_total / steps / 1e3 for ev in prof.key_averages() if "k_diag" in ev.key}
    rejected = int((status["state"] == T.GANG_REJECTED).sum())
    return dict(nodes=len(cfg["nodes"]), gangs=len(cfg["tables"][0]), admitted=int(st["gangs_admitted"]), rejected=rejected,
                verdicts={k: int((gd["verdict"] == v).sum()) for k, v in
                          (("clique_short", T.DIAG_CLIQUE_SHORT), ("no_domain", T.DIAG_NO_DOMAIN), ("no_joint_fit", T.DIAG_NO_JOINT_FIT))},
                ms_host=statistics.median(host), ms_device=dev_us / steps / 1e3,
                kernels_ms={k.split("(")[0].split("::")[-1]: round(v, 4) for k, v in kern.items()})


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--shrunk-nodes", type=int, default=10080)
    args = ap.parse_args()
    line = dict(bench="diagnose", steps=args.steps, **card())
    line["C4"] = measure(synth.config_c4(), args.steps, args.warmup)
    line["C4_shrunk"] = measure(synth.config_c4(n=args.shrunk_nodes), args.steps, args.warmup)
    print(json.dumps(line))


if __name__ == "__main__":
    main()
