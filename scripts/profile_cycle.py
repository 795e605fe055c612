#!/usr/bin/env python
"""profile_cycle.py -- where the device time of one scheduling cycle goes: per kernel, per relaxation round, and between kernels.

  python scripts/profile_cycle.py --out DIR [--config C4] [--warmup 3] [--cycles 5]

Builds the library, runs `--warmup` cycles exactly like bench.py's device-resident step (node table reset device->device, then
grove_run_cycle), then records `--cycles` more under torch.profiler with CUDA activities.  Writes to DIR:

  trace.pt.trace.json   the raw trace (Chrome trace format)
  summary.json          per cycle: time per kernel name (count / sum / min / median / max, us); per relaxation round the K3 duration
                        (first k_eval start to last k_eval end), k_apply and k_detect; the idle gaps on the device between the end of
                        one activity and the start of the next (the critical path is one stream, so an idle device is a serialisation
                        point); busy time against span for the admission phase (first k_eval to last k_detect).  Next to it one cycle
                        run with GROVE_DEBUG_ADMIT=1 (per-round evaluation cycles: the K3 tail against its median evaluation), and the
                        card's name, power limit and SM clocks read in the same run.

There is no CPU path: without a CUDA device the script stops with an error.
"""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return {"query": q, "raw": None}
    f = [x.strip() for x in out.split(",")]
    return {"query": q, "raw": out, **dict(zip(["name", "power_limit", "clocks_sm", "clocks_max_sm"], f))}


def short_name(n: str) -> str:
    """'void grove::k_eval<true, 8, true>(grove::Topo, ...)' -> 'k_eval<true, 8, true>'"""
    n = re.sub(r"^void ", "", n)
    depth = 0
    for i, ch in enumerate(n):   # cut at the parameter list (template arguments may hold parentheses)
        depth += ch == "<"
        depth -= ch == ">"
        if ch == "(" and depth == 0:
            n = n[:i]
            break
    return n.replace("grove::", "").strip()


def stats(v) -> dict:
    v = np.asarray(v, dtype=np.float64)
    if not len(v):
        return {"count": 0}
    return {"count": int(len(v)), "sum_us": float(v.sum()), "min_us": float(v.min()), "median_us": float(np.median(v)), "max_us": float(v.max())}


def device_activities(trace: dict) -> list[dict]:
    """kernels, memsets and copies in start order: {name, kind, start, end (us), stream}"""
    acts = []
    for ev in trace.get("traceEvents", []):
        cat = ev.get("cat", "")
        if ev.get("ph") != "X" or cat not in ("kernel", "gpu_memset", "gpu_memcpy"):
            continue
        ts, dur = float(ev["ts"]), float(ev.get("dur", 0.0))
        acts.append({"name": short_name(ev["name"]) if cat == "kernel" else ev["name"], "kind": cat, "start": ts, "end": ts + dur,
                     "stream": ev.get("args", {}).get("stream")})
    acts.sort(key=lambda a: a["start"])
    return acts


def idle_gaps(acts: list[dict]) -> tuple[float, float, list[dict]]:
    """-> (span, busy, gaps): busy = union of the activity intervals; a gap = the device idle between the end of everything
    started so far and the next start (labelled by the activity that ended last and the one that starts)"""
    if not acts:
        return 0.0, 0.0, []
    busy, gaps = 0.0, []
    cur_s, cur_e, last = acts[0]["start"], acts[0]["end"], acts[0]["name"]
    for a in acts[1:]:
        if a["start"] > cur_e:
            busy += cur_e - cur_s
            gaps.append({"after": last, "before": a["name"], "us": a["start"] - cur_e})
            cur_s, cur_e = a["start"], a["end"]
        elif a["end"] > cur_e:
            cur_e = a["end"]
        if a["end"] >= cur_e:
            last = a["name"]
    busy += cur_e - cur_s
    return acts[-1]["end"] - acts[0]["start"] if acts else 0.0, busy, gaps


def rounds_of(acts: list[dict]) -> list[dict]:
    """one entry per relaxation round: the k_eval launches, then k_apply, then k_detect"""
    out, evals, apply_ = [], [], None
    for a in acts:
        n = a["name"]
        if n.startswith("k_eval"):
            evals.append(a)
        elif n == "k_apply":
            apply_ = a
        elif n == "k_detect" and evals and apply_ is not None:
            k3_s, k3_e = min(e["start"] for e in evals), max(e["end"] for e in evals)
            out.append({"k3_us": k3_e - k3_s, "k3_launches": len(evals),
                        "k3_each_us": {e["name"]: e["end"] - e["start"] for e in evals},
                        "k_apply_us": apply_["end"] - apply_["start"], "k_detect_us": a["end"] - a["start"],
                        "gap_k3_to_apply_us": apply_["start"] - k3_e, "gap_apply_to_detect_us": a["start"] - apply_["end"],
                        "start": k3_s, "end": a["end"]})
            evals, apply_ = [], None
    for i in range(1, len(out)):
        out[i]["gap_from_previous_round_us"] = out[i]["start"] - out[i - 1]["end"]
    return out


def summarise_cycle(acts: list[dict]) -> dict:
    per = {}
    for a in acts:
        per.setdefault(a["name"], []).append(a["end"] - a["start"])
    span, busy, gaps = idle_gaps(acts)
    rnds = rounds_of(acts)
    adm = [a for a in acts if rnds and rnds[0]["start"] <= a["start"] and a["end"] <= rnds[-1]["end"]]
    a_span, a_busy, a_gaps = idle_gaps(adm)
    by_pair = {}
    for g in a_gaps:
        by_pair.setdefault(f'{g["after"]} -> {g["before"]}', []).append(g["us"])
    streams = sorted({a["stream"] for a in adm if a["kind"] == "kernel"}, key=str)
    return {
        "kernels": {k: stats(v) for k, v in sorted(per.items(), key=lambda kv: -sum(kv[1]))},
        "launches": sum(1 for a in acts if a["kind"] == "kernel"),
        "cycle": {"span_us": span, "busy_us": busy, "idle_us": span - busy, "gaps": len(gaps)},
        "admission": {"span_us": a_span, "busy_us": a_busy, "idle_us": a_span - a_busy, "idle_share": (a_span - a_busy) / a_span if a_span else 0.0,
                      "gaps": len(a_gaps), "gap_us": stats([g["us"] for g in a_gaps]),
                      "gaps_by_transition": {k: stats(v) for k, v in sorted(by_pair.items(), key=lambda kv: -sum(kv[1]))},
                      "kernel_streams": streams},
        "rounds": [{k: v for k, v in r.items() if k not in ("start", "end")} for r in rnds],
        "round_totals": {"rounds": len(rnds), "k3_us": stats([r["k3_us"] for r in rnds]), "k_apply_us": stats([r["k_apply_us"] for r in rnds]),
                         "k_detect_us": stats([r["k_detect_us"] for r in rnds]),
                         "gap_k3_to_apply_us": stats([r["gap_k3_to_apply_us"] for r in rnds]),
                         "gap_apply_to_detect_us": stats([r["gap_apply_to_detect_us"] for r in rnds]),
                         "gap_between_rounds_us": stats([r["gap_from_previous_round_us"] for r in rnds[1:]])},
    }


def split_cycles(acts: list[dict]) -> list[list[dict]]:
    """a device-resident step starts with the node-table reset (k_gather)"""
    cycles = []
    for a in acts:
        if a["name"] == "k_gather" or not cycles:
            cycles.append([])
        cycles[-1].append(a)
    return [c for c in cycles if any(a["name"].startswith("k_eval") for a in c)]


ROUND_RE = re.compile(r"^round (\d+): ")
EVALS_RE = re.compile(r"^\s+(\d+) packed evals, mean (\d+) cyc, median (\d+); slowest:(.*)$")
SLOW_RE = re.compile(r"\[g(\d+) rank\d+ st\d+ scopes\d+: (\d+) cyc, (\d+) plaus, (\d+) att\]")


def debug_admit_cycle(make_engine, step, sm_mhz) -> dict:
    """one cycle with GROVE_DEBUG_ADMIT=1 (the host looks at the control words after every round, so the rounds may be cut
    differently from a timed cycle): per round the evaluations' median and slowest cycles"""
    os.environ["GROVE_DEBUG_ADMIT"] = "1"
    eng = make_engine()
    del os.environ["GROVE_DEBUG_ADMIT"]
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            step(eng)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        lines = f.read().splitlines()
    eng.close()
    rounds, cur = [], None
    for ln in lines:
        m = ROUND_RE.match(ln)
        if m:
            cur = int(m.group(1))
            continue
        m = EVALS_RE.match(ln)
        if m and cur is not None:
            slow = [int(x[1]) for x in SLOW_RE.findall(m.group(4))]
            n, med = int(m.group(1)), int(m.group(3))
            mx = max(slow) if slow else med
            rounds.append({"round": cur, "evals": n, "median_cyc": med, "mean_cyc": int(m.group(2)), "slowest_cyc": mx,
                           "tail_over_median": mx / med if med else None})
    us = (lambda c: c / sm_mhz) if sm_mhz else (lambda c: None)
    return {"note": "evaluation cycles are clock64() on the SM; us at the SM clock read in this run",
            "sm_mhz": sm_mhz, "rounds": [{**r, "median_us": us(r["median_cyc"]), "slowest_us": us(r["slowest_cyc"])} for r in rounds],
            "median_tail_over_median": float(np.median([r["tail_over_median"] for r in rounds if r["tail_over_median"]])) if rounds else None}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--out", required=True, help="output directory (created)")
    ap.add_argument("--config", default="C4")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cycles", type=int, default=5)
    args = ap.parse_args()
    if args.cycles < 1:
        ap.error("--cycles must be at least 1")
    import bench
    from grove_b200 import synth
    if args.config not in synth.CONFIGS:
        ap.error(f"--config must be one of {sorted(synth.CONFIGS)}")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("profile_cycle.py: no CUDA device; the engine has no CPU path")
    from torch.profiler import ProfilerActivity, profile
    from grove_b200 import build
    from grove_b200.engine import PlacementEngine

    os.makedirs(args.out, exist_ok=True)
    build.build()
    torch.cuda.set_device(0)
    nodes, L, g, c, s = bench.make_workload(args.config)
    d_nodes = torch.from_numpy(nodes.view(np.uint8).reshape(-1)).cuda()

    def make_engine():
        e = PlacementEngine(L, device=0)
        e.load_nodes(nodes)
        e.submit_gangs(g, c, s)
        return e

    def step(e):   # bench.py step_dev
        e.load_nodes_device(d_nodes.data_ptr(), len(nodes))
        return e.run_cycle()

    info = gpu_info()
    eng = make_engine()
    for _ in range(args.warmup):
        step(eng)
    torch.cuda.synchronize()
    cyc_stats = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.cycles + 1):   # the first traced cycle pays the tracer's start-up and is dropped
            cyc_stats.append(step(eng))
            torch.cuda.synchronize()
    eng.close()
    trace_path = os.path.join(args.out, "trace.pt.trace.json")
    prof.export_chrome_trace(trace_path)
    with open(trace_path) as f:
        trace = json.load(f)
    acts = device_activities(trace)
    if not any(a["name"].startswith("k_eval") for a in acts):
        cats = sorted({str(e.get("cat")) for e in trace.get("traceEvents", [])})
        raise SystemExit(f"profile_cycle.py: the trace holds none of the engine's kernels ({len(acts)} device activities; "
                         f"event categories {cats}): CUPTI did not see the library's launches")
    cycles = split_cycles(acts)[1:]
    try:
        sm_mhz = float(info.get("clocks_sm", "").split()[0])
    except (ValueError, IndexError):
        sm_mhz = None
    dbg = debug_admit_cycle(make_engine, step, sm_mhz)
    per_cycle = [summarise_cycle(cy) for cy in cycles]
    engine_stats = [{k: st[k] for k in ("ms_total", "ms_admit", "rounds", "evaluations", "kernel_launches")} for st in cyc_stats[1:]]
    agg = {}
    if per_cycle:
        med = lambda f: float(np.median([f(p) for p in per_cycle]))
        agg = {"admission_span_us": med(lambda p: p["admission"]["span_us"]), "admission_busy_us": med(lambda p: p["admission"]["busy_us"]),
               "admission_idle_us": med(lambda p: p["admission"]["idle_us"]), "admission_idle_share": med(lambda p: p["admission"]["idle_share"]),
               "rounds": med(lambda p: p["round_totals"]["rounds"]), "launches": med(lambda p: p["launches"]),
               "k3_round_median_us": med(lambda p: p["round_totals"]["k3_us"].get("median_us", 0.0)),
               "k3_sum_us": med(lambda p: p["round_totals"]["k3_us"].get("sum_us", 0.0)),
               "k_apply_sum_us": med(lambda p: p["round_totals"]["k_apply_us"].get("sum_us", 0.0)),
               "k_detect_sum_us": med(lambda p: p["round_totals"]["k_detect_us"].get("sum_us", 0.0))}
    summary = {"config": args.config, "gpu": info, "warmup": args.warmup, "cycles_profiled": len(cycles),
               "engine_stats": engine_stats, "median_over_cycles": agg, "debug_admit": dbg, "per_cycle": per_cycle,
               "note": "timestamps from CUPTI through torch.profiler (CUDA activities only); tracing adds host overhead per launch"}
    with open(os.path.join(args.out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps({"gpu": info.get("raw"), **agg, "k3_tail_over_median": dbg["median_tail_over_median"]}))


if __name__ == "__main__":
    main()
