"""ctypes binding of libgrove_place.so -- the call a scheduler backend makes.

Mirrors the C ABI of include/grove_place.h one to one (the cgo stub in INTEGRATION.md binds the same
symbols).  Nothing here computes placements and nothing here falls back to a CPU path: if the
library is missing or no CUDA device is usable, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import tables as T

ABI_VERSION = 2
_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgrove_place.so")

ERRORS = {0: "OK", -1: "INVALID_ARG", -2: "NO_DEVICE", -3: "CUDA", -4: "LIMIT", -5: "STATE", -6: "OOM"}

# every symbol include/grove_place.h declares
SYMBOLS = [
    "grove_abi_version", "grove_engine_create", "grove_engine_destroy", "grove_last_error",
    "grove_load_nodes", "grove_update_nodes", "grove_get_nodes", "grove_submit_gangs", "grove_submit_gangs_wide", "grove_run_cycle",
    "grove_get_placements", "grove_get_gang_status", "grove_get_scope_domains", "grove_load_nodes_device",
    "grove_build_score_matrix", "grove_run_cycle_preempt", "grove_get_victims", "grove_run_cycle_reuse",
    "grove_run_cycle_reuse_preempt", "grove_diagnose", "grove_set_spread", "grove_set_fences", "grove_set_queues",
    "grove_run_cycle_consolidate", "grove_get_moves", "grove_run_cycle_preempt_queues",
    "grove_run_cycle_reclaim_queues", "grove_run_cycle_reclaim_preempt_queues",
    "grove_set_fair_share", "grove_get_turn_order", "grove_get_fair_share_stats",
    "grove_set_binpack", "grove_get_binpack_picks", "grove_set_compute_domains", "grove_get_compute_domain_owners",
    "grove_shard_range", "grove_run_score_pass", "grove_shard_summary_device",
    "grove_debug_get_perm", "grove_debug_get_fit_row", "grove_debug_get_score_row",
]


class GroveError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{ERRORS.get(code, code)}: {msg}")
        self.code = code


_lib = None


def load_library(path: str = LIB_PATH):
    """dlopen the engine.  Raises (never falls back) when the shared library has not been built."""
    global _lib
    if _lib is None:
        path = os.environ.get("GROVE_PLACE_LIB", path)  # experiments: another build of the same sources
        if not os.path.exists(path):
            raise GroveError(-2, f"{path} not built; run `python -m grove_b200.build` (needs nvcc)")
        lib = C.CDLL(path)
        for s in SYMBOLS:
            getattr(lib, s).restype = C.c_int32
        lib.grove_abi_version.restype = C.c_uint32
        lib.grove_last_error.restype = C.c_char_p
        lib.grove_engine_destroy.restype = None
        _lib = lib
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


class PlacementEngine:
    """One scheduler session on one GPU (not thread-safe; one cycle in flight)."""

    def __init__(self, n_levels: int, device: int = 0, window: int = 0, rank: int = 0, world: int = 1):
        self.lib = load_library()
        cfg = np.zeros(1, dtype=T.config_dt)
        cfg["abi_version"] = ABI_VERSION
        cfg["device"], cfg["n_levels"], cfg["window"] = device, n_levels, window
        cfg["rank"], cfg["world"] = rank, world
        self.h = C.c_void_p()
        rc = self.lib.grove_engine_create(_p(cfg), C.byref(self.h))
        if rc != 0:
            self.h = None
            raise GroveError(rc, "grove_engine_create failed (no CPU fallback exists)")
        self.n_levels = n_levels
        self.n = self.G = self.Q = self.S = 0
        self._cap_pods = 0
        self._pl_buf = self._st_buf = None

    def _check(self, rc: int):
        if rc != 0:
            raise GroveError(rc, (self.lib.grove_last_error(self.h) or b"").decode())

    def close(self):
        if getattr(self, "h", None):
            self.lib.grove_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # ---- inputs ----
    def load_nodes(self, nodes: np.ndarray):
        nodes = np.ascontiguousarray(nodes, dtype=T.node_dt)
        self._check(self.lib.grove_load_nodes(self.h, _p(nodes), C.c_uint32(len(nodes))))
        self.n = len(nodes)

    def load_nodes_device(self, dev_ptr: int, n: int):
        self._check(self.lib.grove_load_nodes_device(self.h, C.c_void_p(dev_ptr), C.c_uint32(n)))

    def update_nodes(self, idx: np.ndarray, recs: np.ndarray):
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        recs = np.ascontiguousarray(recs, dtype=T.node_dt)
        self._check(self.lib.grove_update_nodes(self.h, _p(idx), _p(recs), C.c_uint32(len(idx))))

    def submit_gangs(self, gangs: np.ndarray, cliques: np.ndarray, scopes: np.ndarray):
        gangs = np.ascontiguousarray(gangs, dtype=T.gang_dt)
        cliques = np.ascontiguousarray(cliques, dtype=T.clique_dt)
        scopes = np.ascontiguousarray(scopes, dtype=T.scope_dt)
        self._check(self.lib.grove_submit_gangs(self.h, _p(gangs), C.c_uint32(len(gangs)), _p(cliques),
                                                C.c_uint32(len(cliques)), _p(scopes), C.c_uint32(len(scopes))))
        self.G, self.Q, self.S = len(gangs), len(cliques), len(scopes)
        self._cap_pods = int(cliques["replicas"].astype(np.int64).sum()) if len(cliques) else 0

    def submit_gangs_wide(self, gangs: np.ndarray, cliques: np.ndarray, counts: np.ndarray, scopes: np.ndarray):
        """grove_submit_gangs_wide: `counts` (tables.clique_count_dt) holds every clique's MinReplicas / replicas, up to
        tables.MAX_WIDE_GANG_PODS pods per gang; the 8-bit count fields of `cliques` are ignored."""
        gangs = np.ascontiguousarray(gangs, dtype=T.gang_dt)
        cliques = np.ascontiguousarray(cliques, dtype=T.clique_dt)
        counts = np.ascontiguousarray(counts, dtype=T.clique_count_dt)
        scopes = np.ascontiguousarray(scopes, dtype=T.scope_dt)
        if len(counts) != len(cliques):
            raise ValueError("one count record per clique")
        self._check(self.lib.grove_submit_gangs_wide(self.h, _p(gangs), C.c_uint32(len(gangs)), _p(cliques), _p(counts),
                                                     C.c_uint32(len(cliques)), _p(scopes), C.c_uint32(len(scopes))))
        self.G, self.Q, self.S = len(gangs), len(cliques), len(scopes)
        self._cap_pods = int(counts["replicas"].astype(np.int64).sum()) if len(cliques) else 0

    def set_spread(self, groups: np.ndarray, gang_group: np.ndarray, seeds: np.ndarray | None = None):
        """grove_set_spread: topology spread groups (tables.spread_dt), the group of every submitted gang (tables.NONE_U32 = none)
        and the running replicas of each group (tables.spread_seed_dt, caller node indices).  Call after submit_gangs; the next
        submit / load_nodes clears it (include/grove_place.h "topology spread")."""
        groups = np.ascontiguousarray(groups, dtype=T.spread_dt)
        gang_group = np.ascontiguousarray(gang_group, dtype=np.uint32)
        seeds = np.ascontiguousarray(np.zeros(0, dtype=T.spread_seed_dt) if seeds is None else seeds, dtype=T.spread_seed_dt)
        self._check(self.lib.grove_set_spread(self.h, _p(groups), C.c_uint32(len(groups)), _p(gang_group), C.c_uint32(len(gang_group)),
                                              _p(seeds), C.c_uint32(len(seeds))))

    def set_fences(self, gangs):
        """grove_set_fences: the fencing gangs of the current submission (at most tables.MAX_FENCES, each with a gang Required
        level).  While one of them is REJECTED, the gangs ranked after it see the domain it picked at cycle start as unschedulable;
        its status then carries tables.STATUS_FENCING with that domain.  Call after submit_gangs; the next submit / load_nodes
        clears it (include/grove_place.h "fences")."""
        gangs = np.ascontiguousarray(gangs, dtype=np.uint32)
        self._check(self.lib.grove_set_fences(self.h, _p(gangs), C.c_uint32(len(gangs))))

    def set_queues(self, queues: np.ndarray, gang_queue: np.ndarray):
        """grove_set_queues: hierarchical queues (tables.queue_dt: parent, per-resource limit -- tables.QUEUE_UNLIMITED = none --
        and what the running gangs of exactly that queue hold) and the queue of every submitted gang (tables.NONE_U32 = none).
        A member is admitted only while its queue chain has room for its MinReplicas (else tables.STATUS_OVER_LIMIT), and its
        best-effort pods are capped to what is left (tables.STATUS_SURPLUS_CAPPED).  Call after submit_gangs; the next submit /
        load_nodes clears it (include/grove_place.h "queue limits")."""
        queues = np.ascontiguousarray(queues, dtype=T.queue_dt)
        gang_queue = np.ascontiguousarray(gang_queue, dtype=np.uint32)
        self._check(self.lib.grove_set_queues(self.h, _p(queues), C.c_uint32(len(queues)), _p(gang_queue), C.c_uint32(len(gang_queue))))

    def set_binpack(self, levels):
        """grove_set_binpack: the pack level of every submitted gang (tables.LEVEL_NONE = not a member; at or below the gang's
        Required level).  A member's anchor becomes the first node of the fullest level-b domain that holds it on the table the
        cycle starts from, so its search starts there; binpack_picks() reports the picks.  Call after submit_gangs; the next
        submit / load_nodes clears it (include/grove_place.h "bin-packing")."""
        levels = np.ascontiguousarray(levels, dtype=np.uint8)
        self._check(self.lib.grove_set_binpack(self.h, _p(levels), C.c_uint32(len(levels))))

    def set_fair_share(self, quotas: np.ndarray):
        """grove_set_fair_share: one quota row per queue of the set_queues set (tables.queue_quota_dt; QUEUE_UNLIMITED = KAI's
        quota -1).  run_cycle then gives the next turn to the gang at the head of the queue furthest below its deserved quota --
        priority orders gangs only inside a queue -- and turn_order() reports the order.  Every member must sit in a leaf queue.
        Cleared with the queue set (include/grove_place.h "fair-share order")."""
        quotas = np.ascontiguousarray(quotas, dtype=T.queue_quota_dt)
        self._check(self.lib.grove_set_fair_share(self.h, _p(quotas), C.c_uint32(len(quotas))))

    def turn_order(self) -> np.ndarray:
        """the gangs in the order they had their turn in the last fair-share cycle"""
        out = np.zeros(max(self.G, 1), dtype=np.uint32)
        self._check(self.lib.grove_get_turn_order(self.h, _p(out), C.c_uint32(len(out))))
        return out[: self.G]

    def fair_share_stats(self) -> dict:
        """{iterations, turns_rerun} of the last fair-share cycle: the queue cycles run to reach its order, and the turns the
        cycles after the first ran again"""
        st = np.zeros(1, dtype=T.fair_share_stats_dt)
        self._check(self.lib.grove_get_fair_share_stats(self.h, _p(st)))
        return {k: st[k][0].item() for k in T.fair_share_stats_dt.names}

    def binpack_picks(self) -> np.ndarray:
        """caller index of the first node of each gang's pick in the last cycle that ran with a set_binpack set (tables.NONE_U32:
        not a member, or no domain qualified)"""
        out = np.zeros(max(self.G, 1), dtype=np.uint32)
        self._check(self.lib.grove_get_binpack_picks(self.h, _p(out), C.c_uint32(len(out))))
        return out[: self.G]

    def set_compute_domains(self, cd, owner0):
        """grove_set_compute_domains: the ComputeDomain of every submitted clique's pods (tables.CD_NONE = not enrolled) and the
        CD holding every loaded node's IMEX channel when the cycle starts (tables.CD_NONE, or tables.CD_NO_IMEX for a node
        without an IMEX driver).  An enrolled clique's pods land only on nodes that no other CD holds at its gang's turn;
        compute_domain_owners() reports the owners after the cycle.  Call after submit_gangs; the next submit / load_nodes
        clears it (include/grove_place.h "ComputeDomain exclusivity")."""
        cd = np.ascontiguousarray(cd, dtype=np.uint32)
        owner0 = np.ascontiguousarray(owner0, dtype=np.uint32)
        self._check(self.lib.grove_set_compute_domains(self.h, _p(cd), C.c_uint32(len(cd)), _p(owner0), C.c_uint32(len(owner0))))

    def compute_domain_owners(self) -> np.ndarray:
        """per loaded node (caller order), the CD holding its IMEX channel after the last cycle that ran with a
        set_compute_domains set: owner0 plus the CD of every admitted gang's enrolled pods -- the next cycle's owner0"""
        out = np.zeros(max(self.n, 1), dtype=np.uint32)
        self._check(self.lib.grove_get_compute_domain_owners(self.h, _p(out), C.c_uint32(len(out))))
        return out[: self.n]

    # ---- the cycle ----
    def run_cycle(self) -> dict:
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle(self.h, _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def run_cycle_preempt(self, running: np.ndarray, holdings: np.ndarray) -> dict:
        """ordinary pass + reclaim pass: `running` (T.running_dt) are the gangs admitted by earlier cycles, `holdings`
        (T.holding_dt) what each holds per node; rejected gangs may evict running gangs of a lower priority"""
        running = np.ascontiguousarray(running, dtype=T.running_dt)
        holdings = np.ascontiguousarray(holdings, dtype=T.holding_dt)
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle_preempt(self.h, _p(running), C.c_uint32(len(running)), _p(holdings),
                                                     C.c_uint32(len(holdings)), _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def run_cycle_reuse(self, replaces: np.ndarray, running: np.ndarray, holdings: np.ndarray) -> dict:
        """the ordinary cycle in which gang g with replaces[g] = r != NONE_U32 is the new version of running gang r
        (PodGangSpec.ReuseReservationRef): it may use what r holds (`running` T.running_dt, `holdings` T.holding_dt), nobody else
        may, and when g is admitted r's leftovers return to the free table (include/grove_place.h "reservation reuse")"""
        replaces = np.ascontiguousarray(replaces, dtype=np.uint32)
        running = np.ascontiguousarray(running, dtype=T.running_dt)
        holdings = np.ascontiguousarray(holdings, dtype=T.holding_dt)
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle_reuse(self.h, _p(replaces), C.c_uint32(len(replaces)), _p(running),
                                                   C.c_uint32(len(running)), _p(holdings), C.c_uint32(len(holdings)), _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def run_cycle_reuse_preempt(self, replaces: np.ndarray, running: np.ndarray, holdings: np.ndarray) -> dict:
        """run_cycle_reuse, then the reclaim pass over the gangs it rejected: a rejected gang may evict running gangs of a lower
        priority, and a rejected new version still holds what its predecessor holds when that one ranks at or above it
        (include/grove_place.h "reuse with reclaim"); victims() lists the evictions"""
        replaces = np.ascontiguousarray(replaces, dtype=np.uint32)
        running = np.ascontiguousarray(running, dtype=T.running_dt)
        holdings = np.ascontiguousarray(holdings, dtype=T.holding_dt)
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle_reuse_preempt(self.h, _p(replaces), C.c_uint32(len(replaces)), _p(running),
                                                           C.c_uint32(len(running)), _p(holdings), C.c_uint32(len(holdings)), _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def run_cycle_preempt_queues(self, running: np.ndarray, holdings: np.ndarray, running_queue: np.ndarray) -> dict:
        """the queue cycle of the set_queues set, then the reclaim pass within queue limits: a gang it rejected (OVER_LIMIT ones
        included) may evict running gangs of a lower priority, node by node and then from its own queues until they are within
        their limits.  `running` / `holdings` as for run_cycle_preempt; running_queue[r] is the queue of running gang r
        (tables.NONE_U32 = none), and what the running gangs of a queue hold must not exceed its `used`
        (include/grove_place.h "reclaim within queue limits"); victims() lists the evictions"""
        running = np.ascontiguousarray(running, dtype=T.running_dt)
        holdings = np.ascontiguousarray(holdings, dtype=T.holding_dt)
        running_queue = np.ascontiguousarray(running_queue, dtype=np.uint32)
        if len(running_queue) != len(running):
            raise ValueError("one running_queue entry per running gang")
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle_preempt_queues(self.h, _p(running), C.c_uint32(len(running)), _p(holdings),
                                                            C.c_uint32(len(holdings)), _p(running_queue), _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def run_cycle_reclaim_queues(self, quotas: np.ndarray, running: np.ndarray, holdings: np.ndarray, running_queue: np.ndarray) -> dict:
        """the queue cycle of the set_queues set, then reclaim across queues: a queue below its deserved quota takes room back from
        queues above theirs, whatever the priorities.  `quotas` (tables.queue_quota_dt, one row per queue of the set; QUEUE_UNLIMITED =
        KAI's quota -1); the queues of the gangs the queue cycle rejected go in ascending order of their share, and a member
        admitted against its donor set carries tables.STATUS_RECLAIMER.  `running` / `holdings` / `running_queue` as for
        run_cycle_preempt_queues (include/grove_place.h "reclaim across queues"); victims() lists the evictions"""
        quotas = np.ascontiguousarray(quotas, dtype=T.queue_quota_dt)
        running = np.ascontiguousarray(running, dtype=T.running_dt)
        holdings = np.ascontiguousarray(holdings, dtype=T.holding_dt)
        running_queue = np.ascontiguousarray(running_queue, dtype=np.uint32)
        if len(running_queue) != len(running):
            raise ValueError("one running_queue entry per running gang")
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle_reclaim_queues(self.h, _p(quotas), C.c_uint32(len(quotas)), _p(running),
                                                            C.c_uint32(len(running)), _p(holdings), C.c_uint32(len(holdings)),
                                                            _p(running_queue), _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def run_cycle_reclaim_preempt_queues(self, quotas: np.ndarray, running: np.ndarray, holdings: np.ndarray,
                                         running_queue: np.ndarray) -> dict:
        """the queue cycle of the set_queues set, then both queue eviction passes in KAI-Scheduler's order: reclaim across queues
        (its admitted gangs carry tables.STATUS_RECLAIMER), then reclaim within queue limits for every gang still rejected, from
        the state the first pass left (tables.STATUS_PREEMPTOR).  Inputs as for run_cycle_reclaim_queues (include/grove_place.h
        "reclaim, then preempt"); victims() lists the evictions of both passes, the reclaim pass's first"""
        quotas = np.ascontiguousarray(quotas, dtype=T.queue_quota_dt)
        running = np.ascontiguousarray(running, dtype=T.running_dt)
        holdings = np.ascontiguousarray(holdings, dtype=T.holding_dt)
        running_queue = np.ascontiguousarray(running_queue, dtype=np.uint32)
        if len(running_queue) != len(running):
            raise ValueError("one running_queue entry per running gang")
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle_reclaim_preempt_queues(self.h, _p(quotas), C.c_uint32(len(quotas)), _p(running),
                                                                    C.c_uint32(len(running)), _p(holdings), C.c_uint32(len(holdings)),
                                                                    _p(running_queue), _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def victims(self) -> np.ndarray:
        """(running gang, preemptor gang) pairs of the last run_cycle_preempt / run_cycle_reuse_preempt /
        run_cycle_preempt_queues / run_cycle_reclaim_queues / run_cycle_reclaim_preempt_queues: the caller sets
        DisruptionTarget on them"""
        n = C.c_uint32(0)
        self._check(self.lib.grove_get_victims(self.h, None, C.c_uint32(0), C.byref(n)))
        out = np.zeros(max(n.value, 1), dtype=T.victim_dt)
        self._check(self.lib.grove_get_victims(self.h, _p(out), C.c_uint32(len(out)), C.byref(n)))
        return out[: n.value]

    def run_cycle_consolidate(self, targets, spec_of, running: np.ndarray, holdings: np.ndarray) -> dict:
        """the ordinary cycle, then the consolidation pass: every REJECTED target (at most tables.MAX_CONSOLIDATE_TARGETS, tried in
        rank order) may be admitted by relocating movable running gangs of its priority or below, and only when every relocated
        gang is admitted elsewhere.  spec_of[r] is the gated row of the submission that restates running gang r (tables.NONE_U32:
        not movable); `running` / `holdings` as for run_cycle_preempt.  Targets admitted this way carry
        tables.STATUS_CONSOLIDATED, relocated spec rows tables.STATUS_MOVED; moves() lists the relocations
        (include/grove_place.h "consolidation")"""
        targets = np.ascontiguousarray(targets, dtype=np.uint32)
        spec_of = np.ascontiguousarray(spec_of, dtype=np.uint32)
        running = np.ascontiguousarray(running, dtype=T.running_dt)
        holdings = np.ascontiguousarray(holdings, dtype=T.holding_dt)
        if len(spec_of) != len(running):
            raise ValueError("one spec_of entry per running gang")
        st = np.zeros(1, dtype=T.stats_dt)
        self._check(self.lib.grove_run_cycle_consolidate(self.h, _p(targets), C.c_uint32(len(targets)), _p(spec_of), _p(running),
                                                         C.c_uint32(len(running)), _p(holdings), C.c_uint32(len(holdings)), _p(st)))
        return {k: st[k][0].item() for k in T.stats_dt.names}

    def moves(self) -> np.ndarray:
        """(running gang, target gang) pairs of the last run_cycle_consolidate: the running gangs relocated to make room for each
        consolidated target"""
        n = C.c_uint32(0)
        self._check(self.lib.grove_get_moves(self.h, None, C.c_uint32(0), C.byref(n)))
        out = np.zeros(max(n.value, 1), dtype=T.move_dt)
        self._check(self.lib.grove_get_moves(self.h, _p(out), C.c_uint32(len(out)), C.byref(n)))
        return out[: n.value]

    # ---- outputs ----
    def placements(self, copy: bool = True) -> np.ndarray:
        """copy=False returns a view into a buffer the wrapper reuses (valid until the next call)."""
        cap = max(self._cap_pods, 1)
        if self._pl_buf is None or len(self._pl_buf) < cap:
            self._pl_buf = np.empty(cap, dtype=T.placement_dt)
        n = C.c_uint32(0)
        self._check(self.lib.grove_get_placements(self.h, _p(self._pl_buf), C.c_uint32(len(self._pl_buf)), C.byref(n)))
        out = self._pl_buf[: n.value]
        return out.copy() if copy else out

    def gang_status(self, copy: bool = True) -> np.ndarray:
        cap = max(self.G, 1)
        if self._st_buf is None or len(self._st_buf) < cap:
            self._st_buf = np.empty(cap, dtype=T.status_dt)
        self._check(self.lib.grove_get_gang_status(self.h, _p(self._st_buf), C.c_uint32(len(self._st_buf))))
        out = self._st_buf[: self.G]
        return out.copy() if copy else out

    def scope_domains(self) -> np.ndarray:
        """chosen topology domain of every scope (TopologyConstraintGroupConfig) of the submission"""
        out = np.zeros(max(self.S, 1), dtype=T.scope_status_dt)
        self._check(self.lib.grove_get_scope_domains(self.h, _p(out), C.c_uint32(len(out))))
        return out[: self.S]

    def diagnose(self) -> tuple[np.ndarray, np.ndarray]:
        """Why each REJECTED gang of the last run_cycle did not fit: (tables.gang_diag_dt[G], tables.clique_diag_dt[Q]), computed
        on the GPU against the node table each gang met at its turn (include/grove_place.h "diagnosis of rejected gangs").
        Other gangs and their cliques get zero records.  Raises GroveError STATE after a running-gang cycle or when nodes or
        gangs changed since the cycle."""
        g = np.zeros(max(self.G, 1), dtype=T.gang_diag_dt)
        q = np.zeros(max(self.Q, 1), dtype=T.clique_diag_dt)
        self._check(self.lib.grove_diagnose(self.h, _p(g), C.c_uint32(self.G), _p(q), C.c_uint32(self.Q)))
        return g[: self.G], q[: self.Q]

    def nodes(self) -> np.ndarray:
        out = np.zeros(self.n, dtype=T.node_dt)
        self._check(self.lib.grove_get_nodes(self.h, _p(out), C.c_uint32(self.n)))
        return out

    def build_score_matrix(self) -> float:
        """K2 over the last cycle's start snapshot; returns the kernel's device time in ms"""
        ms = C.c_float(0)
        self._check(self.lib.grove_build_score_matrix(self.h, C.byref(ms)))
        return ms.value

    # ---- multi-GPU score pass (node-range shards; grove_b200/sharded.py drives it) ----
    def shard_range(self) -> tuple[int, int]:
        """topology-sorted node range [lo, hi) this handle builds K1 / K2 for (the whole table when world <= 1)"""
        lo, hi = C.c_uint32(0), C.c_uint32(0)
        self._check(self.lib.grove_shard_range(self.h, C.byref(lo), C.byref(hi)))
        return lo.value, hi.value

    def run_score_pass(self) -> float:
        """K1 + K2 over the loaded snapshot for this handle's node range, no admission; returns device ms"""
        ms = C.c_float(0)
        self._check(self.lib.grove_run_score_pass(self.h, C.byref(ms)))
        return ms.value

    def shard_summary_into(self, dev_ptr: int, cap_words: int):
        """int32[G + Q] feasibility / capacity counts of this shard into a DEVICE buffer (all-reduced by the caller)"""
        self._check(self.lib.grove_shard_summary_device(self.h, C.c_void_p(dev_ptr), C.c_uint32(cap_words)))

    # ---- introspection (parity tests) ----
    def debug_perm(self) -> np.ndarray:
        out = np.zeros(self.n, dtype=np.uint32)
        self._check(self.lib.grove_debug_get_perm(self.h, _p(out), C.c_uint32(self.n)))
        return out

    def debug_fit_row(self, clique: int) -> np.ndarray:
        out = np.zeros((self.n + 31) // 32, dtype=np.uint32)
        self._check(self.lib.grove_debug_get_fit_row(self.h, C.c_uint32(clique), _p(out), C.c_uint32(len(out))))
        return out

    def debug_score_row(self, clique: int) -> np.ndarray:
        out = np.zeros(self.n, dtype=np.uint8)
        self._check(self.lib.grove_debug_get_score_row(self.h, C.c_uint32(clique), _p(out), C.c_uint32(self.n)))
        return out
