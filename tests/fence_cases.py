"""Fences (grove_set_fences, include/grove_place.h "fences") restated over the sequential oracle, and the scenarios the oracle
property tests and the GPU parity tests share.

The picks are computed here in numpy on F0, the table the cycle starts from.  The pass then walks the cycle's order (priority desc,
submission index asc) and hands the oracle one piece at a time: a run of gangs ranked between fencing gangs is one ordinary oracle
cycle with the nodes of the fences active so far marked unschedulable -- exact, because candidate order does not depend on fit --
and a fencing gang is one oracle call of its own with its anchor pinned.  Base gating across pieces is decided here, so every gang
meets exactly the state the definition gives it."""
import numpy as np

from grove_b200 import tables as T
from diagnose_cases import need_depth
from reuse_cases import free_table, _with_free
from spread_cases import _masked

ABSENT = T.DOM_ABSENT


def _fmix32(x):
    from oracle import oracle_py
    return oracle_py._fmix32(x)


def sorted_anchor(gangs, inv, g, N):
    a = int(gangs["anchor_node"][g])
    return int(inv[a]) if a != T.NONE_U32 else _fmix32(g) % N


def picks(oracle, nodes, n_levels, gangs, cliques, scopes, fencing):
    """-> {gang: (lo, hi) sorted node range of its pick, or None}, made in rank order on the table `nodes` (F0)"""
    perm, dom, ndom, _ = oracle.topology(nodes, n_levels)
    N = len(nodes)
    inv = np.empty(N, dtype=np.int64); inv[perm] = np.arange(N)
    sn = np.asarray(nodes)[perm]
    absent = dom[:, :n_levels] == ABSENT
    vdepth = np.where(absent.any(axis=1), absent.argmax(axis=1), n_levels)
    sched = (sn["flags"] & T.NODE_SCHEDULABLE) != 0
    ncls = (sn["flags"].astype(np.int64) >> T.NODE_CLASS_SHIFT) & 0xF
    free = [sn[f].astype(np.int64) for f in ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")]
    taken = np.zeros(N, dtype=bool)
    out = {}
    for g in sorted(fencing, key=lambda i: (-int(gangs["priority"][i]), i)):
        l, co = int(gangs["level"][g]), int(gangs["clique_off"][g])
        ids = dom[:, l].astype(np.int64)
        nd = int(ndom[l])
        short = np.zeros(nd, dtype=np.int64)
        has = ids != ABSENT
        for c in range(int(gangs["n_cliques"][g])):
            q = cliques[co + c]
            m = int(q["min_replicas"])
            if not m:
                continue
            req = [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"])]
            fit = sched & (((int(q["class_mask"]) >> ncls) & 1) != 0) & (vdepth >= need_depth(gangs, cliques, scopes, g, c))
            for f, rq in zip(free, req):
                fit &= f >= rq
            fit &= free[3] >= 1
            cap = free[3].copy()
            for f, rq in zip(free, req):
                if rq:
                    cap = np.minimum(cap, f // rq)
            cap = np.where(fit, np.minimum(cap, m), 0)
            have = np.zeros(nd, dtype=np.int64)
            np.add.at(have, ids[has], cap[has])
            short += np.maximum(0, m - have)
        a = sorted_anchor(gangs, inv, g, N)
        best = None
        for d in range(nd):
            members = np.nonzero(ids == d)[0]
            lo, hi = int(members[0]), int(members[-1]) + 1
            if taken[lo:hi].any():
                continue
            close = sum(1 for x in range(n_levels) if dom[lo, x] != ABSENT and dom[lo, x] == dom[a, x])
            key = (int(short[d]), -min(close, l + 1), (lo - a) % N)
            if best is None or key < best[0]:
                best = (key, lo, hi)
        out[g] = None if best is None else (best[1], best[2])
        if best is not None:
            taken[best[1]: best[2]] = True
    return out


def run_cycle_fences(oracle, nodes, n_levels, gangs, cliques, scopes, fencing, trace=None):
    """-> dict(placements, status, scope_status, nodes_after, perm, picks) of the fenced cycle, as its definition reads.
    trace (a dict): gets gang -> (lo, hi) of every fence that was active at the end."""
    G, N = len(gangs), len(nodes)
    fencing = [int(g) for g in fencing]
    pk = picks(oracle, nodes, n_levels, gangs, cliques, scopes, fencing)
    perm, _, _, _ = oracle.topology(nodes, n_levels)
    order = sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i))
    pieces, run = [], []
    for g in order:
        if g in pk:
            if run:
                pieces.append(run); run = []
            pieces.append([g])
        else:
            run.append(g)
    if run:
        pieces.append(run)
    F = free_table(nodes)
    status = np.zeros(G, dtype=T.status_dt)
    status["level"] = T.LEVEL_NONE; status["domain_node"] = T.NONE_U32
    sstat = np.zeros(len(scopes), dtype=T.scope_status_dt)
    sstat["level"] = T.LEVEL_NONE; sstat["domain_node"] = T.NONE_U32
    state = np.zeros(G, dtype=np.uint8)
    fenced = np.zeros(N, dtype=bool)   # caller order: nodes of the active fences
    active = {}
    per_gang = {}
    for piece in pieces:
        ids = []
        for g in sorted(piece):
            b = int(gangs["base_gang"][g])
            if gangs["flags"][g] & T.GANG_GATED:
                state[g] = T.GANG_GATED_SKIP
            elif b != T.NONE_U32 and b not in piece and state[b] != T.GANG_ADMITTED:
                state[g] = T.GANG_BASE_REJECTED
            else:
                ids.append(g)
        while True:   # a base gang of the piece that is gated (or waits for its own base) is never admitted
            out_ = [g for g in ids if int(gangs["base_gang"][g]) in piece and int(gangs["base_gang"][g]) not in ids]
            if not out_:
                break
            for g in out_:
                state[g] = T.GANG_BASE_REJECTED
            ids = [g for g in ids if g not in out_]
        if not ids:
            continue
        sub = {g: k for k, g in enumerate(ids)}
        sg = gangs[ids].copy()
        sq, ss = [], []
        for k, g in enumerate(ids):
            b = int(gangs["base_gang"][g])
            sg["base_gang"][k] = sub[b] if b in sub else T.NONE_U32
            if sg["anchor_node"][k] == T.NONE_U32:
                sg["anchor_node"][k] = perm[_fmix32(g) % N]
            sg["clique_off"][k] = sum(len(x) for x in sq); sg["scope_off"][k] = sum(len(x) for x in ss)
            co, so = int(gangs["clique_off"][g]), int(gangs["scope_off"][g])
            sq.append(cliques[co: co + int(gangs["n_cliques"][g])]); ss.append(scopes[so: so + int(gangs["n_scopes"][g])])
        sq, ss = np.concatenate(sq), np.concatenate(ss)
        out = oracle.run_cycle(_masked(nodes, F, fenced), n_levels, sg, sq, ss)
        for k, g in enumerate(ids):
            st = out["status"][k]
            state[g] = st["state"]
            so = int(gangs["scope_off"][g])
            sstat[so: so + int(gangs["n_scopes"][g])] = out["scope_status"][int(sg["scope_off"][k]): int(sg["scope_off"][k]) + int(sg["n_scopes"][k])]
            status[g] = st
            if st["state"] == T.GANG_ADMITTED:
                pl = out["placements"][st["placement_off"]: st["placement_off"] + st["n_pods"]].copy()
                pl["clique"] += int(gangs["clique_off"][g]) - int(sg["clique_off"][k])
                per_gang[g] = pl
            elif st["state"] == T.GANG_REJECTED and pk.get(g) is not None:
                lo, hi = pk[g]
                fenced[perm[lo:hi]] = True
                active[g] = (lo, hi)
        F = free_table(out["nodes_after"])
    status["state"] = state
    for g, (lo, hi) in active.items():
        status["reserved0"][g] = T.STATUS_FENCING
        status["level"][g] = gangs["level"][g]
        status["domain_node"][g] = perm[lo]
    if trace is not None:
        trace.update(active)
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off
        if state[g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F), perm=perm, picks=pk)


def fence_randomly(rng, gangs, k=None):
    """a few gangs with a gang Required level, at random -> uint32 array"""
    may = [g for g in range(len(gangs)) if int(gangs["level"][g]) != T.LEVEL_NONE]
    if not may:
        return np.zeros(0, dtype=np.uint32)
    k = int(rng.integers(1, min(len(may), 6) + 1)) if k is None else min(k, len(may))
    return np.array(sorted(rng.choice(may, k, replace=False)), dtype=np.uint32)


def blocks_case(blocks=4, per_block=8, gpus=8):
    """`blocks` blocks of `per_block` nodes of `gpus` GPUs (two levels: block, host), all free"""
    n = blocks * per_block
    nodes = T.make_nodes(n)
    nodes["dom"][:, 0] = np.arange(n) // per_block
    nodes["dom"][:, 1] = np.arange(n)
    nodes["free_cpu_milli"] = 64000; nodes["free_mem_mib"] = 1 << 20; nodes["free_gpu"] = gpus; nodes["free_pods"] = 110
    nodes["flags"] = T.NODE_SCHEDULABLE
    return nodes, 2


def hand_cases():
    """name -> (nodes, n_levels, tables, fencing): one case per rule of the definition"""

    def least_shortfall():     # block 2 has the most free GPUs: the big gang fences it, the small one after it goes elsewhere
        nodes, L = blocks_case(blocks=3, per_block=2)
        nodes["free_gpu"] = [4, 4, 4, 4, 8, 4]
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=2)   # needs a whole block: rejected
        b.add_gang([(None, [dict(gpu=4, min=1)])], level=0, priority=1, anchor=4)
        return nodes, L, b.build(), [0]

    def tie_order():           # every block is equally short: the anchor's block is the pick
        nodes, L = blocks_case(blocks=3, per_block=2)
        nodes["free_gpu"] = 4
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=2, anchor=5)
        b.add_gang([(None, [dict(gpu=4, min=1)])], level=0, priority=1, anchor=5)
        return nodes, L, b.build(), [0]

    def nested_overlap():      # a block-level fence takes block 0; the host-level gang after it cannot pick inside it
        nodes, L = blocks_case(blocks=2, per_block=2)
        nodes["free_gpu"] = [8, 4, 2, 2]
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=3)
        b.add_gang([(None, [dict(gpu=8, min=1)])], level=1, priority=2)
        b.add_gang([(None, [dict(gpu=2, min=1)])], level=1, priority=1, anchor=0)
        return nodes, L, b.build(), [0, 1]

    def admitted_fences_nothing():
        nodes, L = blocks_case(blocks=2, per_block=2)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=2)
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=1)
        return nodes, L, b.build(), [0]

    def gated_fences_nothing():
        nodes, L = blocks_case(blocks=2, per_block=2)
        nodes["free_gpu"] = 4
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=3, gated=True)
        base = b.add_gang([(None, [dict(gpu=16, min=1)])], level=0, priority=3)      # never fits: rejected, not fencing
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=3, base=base)   # BASE_REJECTED: fences nothing
        b.add_gang([(None, [dict(gpu=4, min=1)])], level=0, priority=1)
        return nodes, L, b.build(), [0, 2]

    def before_and_after():    # gangs ranked before the fencing gang are untouched; those after it avoid its domain
        nodes, L = blocks_case(blocks=3, per_block=2)
        nodes["free_gpu"] = 6
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=2, min=1)])], level=0, priority=3, anchor=0)
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=2)
        for a in (0, 2, 4, 1, 3):
            b.add_gang([(None, [dict(gpu=2, min=1)])], level=0, priority=1, anchor=a)
        return nodes, L, b.build(), [1]

    return {"least_shortfall": least_shortfall, "tie_order": tie_order, "nested_overlap": nested_overlap,
            "admitted_fences_nothing": admitted_fences_nothing, "gated_fences_nothing": gated_fences_nothing,
            "before_and_after": before_and_after}


class Starvation:
    """Four blocks of 8 x 8-GPU nodes.  Each cycle a stream of one-node gangs arrives, each living two cycles once admitted, and
    one gang that needs a whole block (8 pods of 8 GPUs) waits at equal priority, ranked first.  `run(cycle_fn, fence_after)`
    drives it: cycle_fn(nodes, L, tables, fencing) -> outputs; fence_after = None runs without fences, k fences the big gang
    once it has been rejected k cycles in a row.  Returns (cycle the big gang was admitted or None, per-cycle statuses of it)."""

    def __init__(self, cycles=20, small_per_cycle=14, seed=0):
        self.cycles, self.small, self.seed = cycles, small_per_cycle, seed
        self.nodes, self.L = blocks_case()

    def run(self, cycle_fn, fence_after=None):
        free = self.nodes["free_gpu"].astype(np.int64).copy()
        # the cluster is busy when the big gang arrives: one-node gangs on every node but one per block, leaving in cycle 1 or 2
        busy = [n for n in range(len(self.nodes)) if n % 8 != 7]
        running = [(n, int(c)) for n, c in zip(busy, np.random.default_rng(1).integers(1, 3, len(busy)))]   # (node, cycle it leaves)
        free[busy] -= 8
        rejected_for = 0
        history = []
        anchors = np.random.default_rng(self.seed).integers(0, len(self.nodes), size=(self.cycles, self.small))
        for cyc in range(self.cycles):
            for n, _ in [r for r in running if r[1] == cyc]:
                free[n] += 8
            running = [r for r in running if r[1] != cyc]
            nodes = self.nodes.copy()
            nodes["free_gpu"] = free
            b = T.GangTableBuilder()
            b.add_gang([(None, [dict(gpu=8, min=8)])], level=0, anchor=0)   # the big gang: submission index 0, ranked first
            for a in anchors[cyc]:
                b.add_gang([(None, [dict(gpu=8, min=1)])], level=0, anchor=int(a))
            tables = b.build()
            fencing = [0] if fence_after is not None and rejected_for >= fence_after else []
            out = cycle_fn(nodes, self.L, tables, fencing)
            st = out["status"]
            history.append(st[0].copy())
            if st["state"][0] == T.GANG_ADMITTED:
                return cyc, history
            rejected_for = rejected_for + 1 if st["state"][0] == T.GANG_REJECTED else rejected_for
            for g in range(1, len(tables[0])):
                if st["state"][g] == T.GANG_ADMITTED:
                    n = int(out["placements"][st["placement_off"][g]]["node"])
                    free[n] -= 8
                    running.append((n, cyc + 2))
        return None, history
