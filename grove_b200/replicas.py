"""Multi-GPU = replicas only (DESIGN.md section 7).

One cluster is ONE sequential dependency chain over ~1.6 MB of node state: a cycle is bound by the latency of its
relaxation rounds, not by bytes or flops, so splitting it over GPUs would put a collective (>= 10-20 us on NVLink,
per round) on a critical path whose rounds cost a few tens of microseconds -- round 1 measured it: the cycle got
slower as GPUs were added.  What does scale is the number of clusters: a scheduler instance per cluster (or per
federated partition), one per GPU, no data-path collective.  This module is the thin orchestration of that: every
rank runs its own cycle, and the only communication is the bookkeeping reduction (max time over ranks, sum of
units) that bench.py reports.  It works with any torch.distributed backend (NCCL on the GPU box, gloo in the CPU
test, where the oracle stands in for the engine).
"""
from __future__ import annotations

import time


def run_replicas(dist, rank: int, world: int, make_cycle, steps: int, warmup: int, device=None):
    """make_cycle(rank) -> a zero-argument callable that runs ONE cycle on this rank's own cluster and returns
    (gangs_admitted, gangs_rejected).  Returns dict(seconds (max over ranks), admitted, rejected (summed over ranks),
    per_rank=[(admitted, rejected, seconds)...] on every rank)."""
    import torch

    cycle = make_cycle(rank)
    for _ in range(warmup):
        cycle()
    if world > 1:
        dist.barrier()
    t0 = time.perf_counter()
    adm = rej = 0
    for _ in range(steps):
        adm, rej = cycle()
    dt = time.perf_counter() - t0
    if world == 1:
        return dict(seconds=dt, admitted=adm, rejected=rej, per_rank=[(adm, rej, dt)])
    dev = device if device is not None else "cpu"
    mine = torch.tensor([float(adm), float(rej), dt], dtype=torch.float64, device=dev)
    every = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(every, mine)
    per_rank = [(int(t[0].item()), int(t[1].item()), float(t[2].item())) for t in every]
    return dict(seconds=max(p[2] for p in per_rank), admitted=sum(p[0] for p in per_rank),
                rejected=sum(p[1] for p in per_rank), per_rank=per_rank)
