"""Packed table formats of the placement engine (numpy mirrors of include/grove_place.h).

The record layouts are the wire format between the host side (a scheduler backend's cycle loop)
and libgrove_place.so.  Field meanings follow the reference's PodGang schema
(ai-dynamo/grove scheduler/api/core/v1alpha1/podgang.go:51-131); see include/grove_place.h.
"""
from __future__ import annotations

import numpy as np

MAX_LEVELS = 4
LEVEL_NONE = 0xFF
DOM_ABSENT = 0xFFFFFFFF
NONE_U32 = 0xFFFFFFFF
MAX_GANG_PODS = 128
MAX_GANG_CLIQUES = 32
MAX_GANG_SCOPES = 32

NODE_SCHEDULABLE = 0x1
NODE_CLASS_SHIFT = 8

GANG_GATED = 0x1

GANG_PENDING, GANG_ADMITTED, GANG_REJECTED, GANG_GATED_SKIP, GANG_BASE_REJECTED = 0, 1, 2, 3, 4

node_dt = np.dtype([
    ("free_cpu_milli", "<u4"), ("free_mem_mib", "<u4"), ("free_gpu", "<u2"), ("free_pods", "<u2"),
    ("flags", "<u4"), ("dom", "<u4", (MAX_LEVELS,)),
])
clique_dt = np.dtype([
    ("req_cpu_milli", "<u4"), ("req_mem_mib", "<u4"), ("req_gpu", "<u2"), ("min_replicas", "u1"),
    ("replicas", "u1"), ("class_mask", "<u2"), ("level", "u1"), ("scope", "u1"),
])
# grove_submit_gangs_wide: MinReplicas / replicas of one clique, up to GROVE_MAX_WIDE_GANG_PODS
clique_count_dt = np.dtype([("min_replicas", "<u2"), ("replicas", "<u2")])
MAX_GANG_PODS, MAX_WIDE_GANG_PODS = 128, 2048
scope_dt = np.dtype([
    ("first_clique", "<u2"), ("n_cliques", "<u2"), ("level", "u1"), ("preferred1", "u1"), ("reserved", "u1", (2,)),
])
gang_dt = np.dtype([
    ("clique_off", "<u4"), ("scope_off", "<u4"), ("n_cliques", "<u2"), ("n_scopes", "<u2"),
    ("priority", "<i4"), ("anchor_node", "<u4"), ("base_gang", "<u4"), ("level", "u1"),
    ("preferred", "u1"), ("flags", "<u2"), ("reserved", "<u4"),
])
placement_dt = np.dtype([("clique", "<u4"), ("node", "<u4")])

# preemption / reclaim inputs and outputs (include/grove_place.h)
holding_dt = np.dtype([("node", np.uint32), ("cpu_milli", np.uint32), ("mem_mib", np.uint32), ("gpu", np.uint16), ("pods", np.uint16)])
running_dt = np.dtype([("priority", np.int32), ("holding_off", np.uint32), ("n_holdings", np.uint32), ("reserved", np.uint32)])
victim_dt = np.dtype([("running", np.uint32), ("preemptor", np.uint32)])
STATUS_PREEMPTOR = 0x1
status_dt = np.dtype([
    ("state", "u1"), ("level", "u1"), ("reserved0", "<u2"), ("score_num", "<u2"), ("score_den", "<u2"),
    ("n_pods", "<u4"), ("placement_off", "<u4"), ("domain_node", "<u4"), ("reserved1", "<u4", (3,)),
])
scope_status_dt = np.dtype([("level", "u1"), ("reserved", "u1", (3,)), ("domain_node", "<u4")])
config_dt = np.dtype([
    ("abi_version", "<u4"), ("device", "<i4"), ("n_levels", "<u4"), ("window", "<u4"),
    ("rank", "<u4"), ("world", "<u4"), ("reserved", "<u4", (2,)),
])
stats_dt = np.dtype([
    ("rounds", "<u4"), ("gangs_admitted", "<u4"), ("gangs_rejected", "<u4"), ("pods_bound", "<u4"),
    ("pairs_evaluated", "<u8"), ("kernel_launches", "<u8"), ("evaluations", "<u8"), ("ms_fit", "<f4"), ("ms_score", "<f4"),
    ("ms_admit", "<f4"), ("ms_commit", "<f4"), ("ms_total", "<f4"), ("reserved", "<f4"),
])
# grove_diagnose: why each REJECTED gang of the last grove_run_cycle did not fit (include/grove_place.h "diagnosis")
DIAG_NONE, DIAG_CLIQUE_SHORT, DIAG_NO_DOMAIN, DIAG_NO_JOINT_FIT = 0, 1, 2, 3
gang_diag_dt = np.dtype([
    ("verdict", "u1"), ("level", "u1"), ("clique", "<u2"), ("domains", "<u4"), ("domains_ok", "<u4"), ("reserved", "<u4"),
])
# the failure counts in the order a node is charged: the first predicate of fit(q, n) it fails
DIAG_FAILURES = ("unschedulable", "selector", "labels", "cpu", "mem", "gpu", "pods")
clique_diag_dt = np.dtype([("nodes_fit", "<u4")] + [(f, "<u4") for f in DIAG_FAILURES] + [("pods_fit", "<u8")])

# topology spread (grove_set_spread, include/grove_place.h "topology spread")
SPREAD_HARD, SPREAD_SOFT = 1, 2   # DoNotSchedule, ScheduleAnyway
STATUS_SPREAD_SKEWED = 0x2        # status reserved0: a SOFT member placed outside its allowed domains
spread_dt = np.dtype([("level", "u1"), ("mode", "u1"), ("max_skew", "<u2"), ("reserved", "<u4")])
spread_seed_dt = np.dtype([("group", "<u4"), ("node", "<u4")])

# fences (grove_set_fences, include/grove_place.h "fences")
MAX_FENCES = 64
STATUS_FENCING = 0x4              # status reserved0: a REJECTED gang whose fence held (level, domain_node name the fenced domain)

# ComputeDomain exclusivity (grove_set_compute_domains, include/grove_place.h "ComputeDomain exclusivity")
CD_NONE = NONE_U32                # a clique that is not enrolled / a node no CD holds
CD_NO_IMEX = 0xFFFFFFFE           # owner0: a node without an IMEX driver

# consolidation (grove_run_cycle_consolidate, include/grove_place.h "consolidation")
MAX_CONSOLIDATE_TARGETS = 16
CONSOLIDATE_TRIES = 4
STATUS_CONSOLIDATED = 0x8         # status reserved0: a target admitted by the consolidation pass
STATUS_MOVED = 0x10               # status reserved0: the spec row of a running gang that was relocated
move_dt = np.dtype([("running", np.uint32), ("target", np.uint32)])
MAX_QUEUES = 4096
MAX_QUEUE_DEPTH = 4
QUEUE_UNLIMITED = 0xFFFFFFFFFFFFFFFF   # a queue limit that is not set (KAI's -1)
STATUS_OVER_LIMIT = 0x20          # status reserved0: REJECTED by its queue chain's headroom, not evaluated
STATUS_SURPLUS_CAPPED = 0x40      # status reserved0: ADMITTED with fewer best-effort pods allowed than it asked for
queue_dt = np.dtype([("parent", np.uint32), ("reserved", np.uint32), ("limit", "<u8", (3,)), ("used", "<u8", (3,))])
STATUS_RECLAIMER = 0x80           # status reserved0: admitted by the class pass of grove_run_cycle_reclaim_queues (or
                                  # the reclaim pass of grove_run_cycle_reclaim_preempt_queues)
queue_quota_dt = np.dtype([("deserved", "<u8", (3,))])   # per resource, QUEUE_UNLIMITED = whatever the queue holds (KAI's -1)
fair_share_stats_dt = np.dtype([("iterations", "<u4"), ("turns_rerun", "<u4")])   # grove_get_fair_share_stats

assert node_dt.itemsize == 32 and clique_dt.itemsize == 16 and scope_dt.itemsize == 8
assert gang_dt.itemsize == 32 and placement_dt.itemsize == 8 and status_dt.itemsize == 32 and scope_status_dt.itemsize == 8
assert config_dt.itemsize == 32 and stats_dt.itemsize == 64
assert gang_diag_dt.itemsize == 16 and clique_diag_dt.itemsize == 40
assert spread_dt.itemsize == 8 and spread_seed_dt.itemsize == 8 and queue_dt.itemsize == 56
assert queue_quota_dt.itemsize == 24


def make_nodes(n: int) -> np.ndarray:
    nodes = np.zeros(n, dtype=node_dt)
    nodes["dom"][:] = DOM_ABSENT
    return nodes


class GangTableBuilder:
    """Accumulates PodGangs into the three packed tables.

    One `add_gang` call is one PodGang: `scopes` is a list of (level, [clique dict, ...]) or
    (level, [clique dict, ...], preferred); a scope with level None is the implicit scope of PodGroups
    that are in no TopologyConstraintGroupConfig.  Clique dict keys: cpu, mem, gpu (per-pod request),
    min, replicas (default = min), level, preferred, class_mask (default 0xFFFF).  `preferred` is the
    PackConstraint.Preferred level (podgang.go:110-117), deeper than the Required one.
    """

    def __init__(self) -> None:
        self.gangs: list[tuple] = []
        self.cliques: list[tuple] = []
        self.scopes: list[tuple] = []

    @staticmethod
    def _lvl(level) -> int:
        return LEVEL_NONE if level is None else int(level)

    @staticmethod
    def _pref1(level) -> int:
        return 0 if level is None else int(level) + 1

    def add_gang(self, scopes, level=None, priority=0, anchor=None, base=None, gated=False, preferred=None) -> int:
        clique_off, scope_off = len(self.cliques), len(self.scopes)
        rel = 0
        for si, scope in enumerate(scopes):
            slevel, cliques = scope[0], scope[1]
            spref = scope[2] if len(scope) > 2 else None
            self.scopes.append((rel, len(cliques), self._lvl(slevel), self._pref1(spref)))
            for c in cliques:
                mn = int(c.get("min", 1))
                self.cliques.append((
                    int(c.get("cpu", 0)), int(c.get("mem", 0)), int(c.get("gpu", 0)), mn,
                    int(c.get("replicas", mn)), int(c.get("class_mask", 0xFFFF)), self._lvl(c.get("level")),
                    si | (self._pref1(c.get("preferred")) << 5),
                ))
                rel += 1
        self.gangs.append((
            clique_off, scope_off, rel, len(scopes), int(priority),
            NONE_U32 if anchor is None else int(anchor), NONE_U32 if base is None else int(base),
            self._lvl(level), GANG_GATED if gated else 0, self._lvl(preferred),
        ))
        return len(self.gangs) - 1

    def build(self):
        gangs = np.zeros(len(self.gangs), dtype=gang_dt)
        cliques = np.zeros(len(self.cliques), dtype=clique_dt)
        scopes = np.zeros(len(self.scopes), dtype=scope_dt)
        for i, g in enumerate(self.gangs):
            (gangs["clique_off"][i], gangs["scope_off"][i], gangs["n_cliques"][i], gangs["n_scopes"][i],
             gangs["priority"][i], gangs["anchor_node"][i], gangs["base_gang"][i], gangs["level"][i],
             gangs["flags"][i], gangs["preferred"][i]) = g
        for i, c in enumerate(self.cliques):
            (cliques["req_cpu_milli"][i], cliques["req_mem_mib"][i], cliques["req_gpu"][i],
             cliques["min_replicas"][i], cliques["replicas"][i], cliques["class_mask"][i],
             cliques["level"][i], cliques["scope"][i]) = c
        for i, s in enumerate(self.scopes):
            scopes["first_clique"][i], scopes["n_cliques"][i], scopes["level"][i], scopes["preferred1"][i] = s
        return gangs, cliques, scopes

    def build_wide(self):
        """The tables of grove_submit_gangs_wide: (gangs, cliques, counts, scopes).  `counts` carries every clique's MinReplicas
        and replicas (up to MAX_WIDE_GANG_PODS); the clique records' 8-bit count fields, which that entry ignores, are zero."""
        counts = np.zeros(len(self.cliques), dtype=clique_count_dt)
        for i, c in enumerate(self.cliques):
            counts["min_replicas"][i], counts["replicas"][i] = c[3], c[4]
        narrow = GangTableBuilder()
        narrow.gangs, narrow.scopes = self.gangs, self.scopes
        narrow.cliques = [c[:3] + (0, 0) + c[5:] for c in self.cliques]
        gangs, cliques, scopes = narrow.build()
        return gangs, cliques, counts, scopes
