"""Bin-packing (grove_set_binpack, include/grove_place.h "bin-packing") restated over the sequential oracle, and the scenarios the
oracle property tests and the GPU parity tests share.

The picks are computed here in numpy on F0, the table the cycle starts from, every member on its own.  The cycle is then the
unchanged oracle cycle (or tests/queue_cases.py's queue cycle) on the same gangs, with each picked member's anchor_node pinned to
the caller index of its pick's first node: candidate order is a function of the anchor alone, so that is the whole definition."""
import numpy as np

from grove_b200 import tables as T
from diagnose_cases import need_depth
from fence_cases import blocks_case

ABSENT = T.DOM_ABSENT
RES = ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")


def _sorted_view(oracle, nodes, n_levels):
    perm, dom, ndom, _ = oracle.topology(nodes, n_levels)
    sn = np.asarray(nodes)[perm]
    absent = dom[:, :n_levels] == ABSENT
    vdepth = np.where(absent.any(axis=1), absent.argmax(axis=1), n_levels)
    sched = (sn["flags"] & T.NODE_SCHEDULABLE) != 0
    ncls = (sn["flags"].astype(np.int64) >> T.NODE_CLASS_SHIFT) & 0xF
    free = np.stack([sn[f].astype(np.int64) for f in RES])   # [4][N]
    return perm, dom, ndom, vdepth, sched, ncls, free


def capacity(view, gangs, cliques, scopes, g, c):
    """grove_diagnose's exact capacity of clique c of gang g on every sorted node (0 where K1 fit fails)"""
    _, _, _, vdepth, sched, ncls, free = view
    q = cliques[int(gangs["clique_off"][g]) + c]
    req = [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"])]
    fit = sched & (((int(q["class_mask"]) >> ncls) & 1) != 0) & (vdepth >= need_depth(gangs, cliques, scopes, g, c)) & (free[3] >= 1)
    cap = free[3].copy()
    for k, rq in enumerate(req):
        fit &= free[k] >= rq
        if rq:
            cap = np.minimum(cap, free[k] // rq)
    return np.where(fit, cap, 0)


def _need(gangs, cliques, g):
    co = int(gangs["clique_off"][g])
    q = cliques[co: co + int(gangs["n_cliques"][g])]
    m = q["min_replicas"].astype(np.int64)
    return np.array([(m * q["req_cpu_milli"].astype(np.int64)).sum(), (m * q["req_mem_mib"].astype(np.int64)).sum(),
                     (m * q["req_gpu"].astype(np.int64)).sum(), m.sum()])


def picks(oracle, nodes, n_levels, gangs, cliques, scopes, levels):
    """-> int64[G]: the sorted index of the first node of each member's pick, -1 for non-members and members without one"""
    view = _sorted_view(oracle, nodes, n_levels)
    _, dom, ndom, _, sched, _, free = view
    N = len(nodes)
    out = np.full(len(gangs), -1, dtype=np.int64)
    per_level = {}
    for b in sorted({int(x) for x in levels if x != T.LEVEL_NONE}):
        ids = dom[:, b].astype(np.int64)
        has = ids != ABSENT
        nd = int(ndom[b])
        S = np.zeros((nd, 4), dtype=np.int64)
        np.add.at(S, ids[has], (free * sched).T[has])
        first = np.full(nd, N, dtype=np.int64)
        np.minimum.at(first, ids[has], np.arange(N)[has])
        order = np.lexsort((first, S[:, 1], S[:, 0], S[:, 2]))   # (gpu, cpu, mem, first node), the last key primary
        per_level[b] = (ids, has, nd, S, first, order)
    for g in range(len(gangs)):
        b = int(levels[g])
        if b == T.LEVEL_NONE:
            continue
        ids, has, nd, S, first, order = per_level[b]
        ok = (S >= _need(gangs, cliques, g)).all(axis=1)
        for c in range(int(gangs["n_cliques"][g])):
            m = int(cliques[int(gangs["clique_off"][g]) + c]["min_replicas"])
            if m:
                have = np.zeros(nd, dtype=np.int64)
                np.add.at(have, ids[has], capacity(view, gangs, cliques, scopes, g, c)[has])
                ok &= have >= m
        q = ok[order]
        if q.any():
            out[g] = first[order[int(np.argmax(q))]]
    return out


def picks_brute(oracle, nodes, n_levels, gangs, cliques, scopes, levels):
    """the same picks by a plain loop over every domain and every node of it"""
    view = _sorted_view(oracle, nodes, n_levels)
    _, dom, ndom, _, sched, _, free = view
    out = np.full(len(gangs), -1, dtype=np.int64)
    for g in range(len(gangs)):
        b = int(levels[g])
        if b == T.LEVEL_NONE:
            continue
        need = _need(gangs, cliques, g)
        caps = [capacity(view, gangs, cliques, scopes, g, c) for c in range(int(gangs["n_cliques"][g]))]
        best = None
        for d in range(int(ndom[b])):
            members = [n for n in range(len(nodes)) if dom[n, b] == d]
            s = [sum(int(free[k][n]) for n in members if sched[n]) for k in range(4)]
            if any(s[k] < need[k] for k in range(4)):
                continue
            co = int(gangs["clique_off"][g])
            if any(sum(int(caps[c][n]) for n in members) < int(cliques[co + c]["min_replicas"]) for c in range(len(caps))):
                continue
            key = (s[2], s[0], s[1], members[0])
            if best is None or key < best:
                best = key
        if best is not None:
            out[g] = best[3]
    return out


def run_cycle_binpack(oracle, nodes, n_levels, gangs, cliques, scopes, levels, queues=None, gang_queue=None):
    """-> dict(placements, status, scope_status, nodes_after, perm, picks) of the bin-packing cycle, as its definition reads;
    picks in caller indices (NONE_U32: none).  With `queues` the cycle is the queue cycle."""
    pk = picks(oracle, nodes, n_levels, gangs, cliques, scopes, levels)
    perm = oracle.topology(nodes, n_levels)[0]
    pinned = gangs.copy()
    hit = pk >= 0
    pinned["anchor_node"][hit] = perm[pk[hit]]
    if queues is None:
        out = oracle.run_cycle(nodes, n_levels, pinned, cliques, scopes)
    else:
        from queue_cases import run_cycle_queues
        out = run_cycle_queues(oracle, nodes, n_levels, pinned, cliques, scopes, queues, gang_queue)
    out["picks"] = np.where(hit, perm[np.maximum(pk, 0)], T.NONE_U32).astype(np.uint32)
    return out


def random_levels(rng, gangs, n_levels, share=0.6):
    """pack levels for a random share of the gangs: any level at or below the Required one (any level without one)"""
    out = np.full(len(gangs), T.LEVEL_NONE, dtype=np.uint8)
    for g in range(len(gangs)):
        if rng.random() < share:
            req = int(gangs["level"][g])
            out[g] = int(rng.integers(0 if req == T.LEVEL_NONE else req, n_levels))
    return out


def hand_cases():
    """name -> (nodes, n_levels, tables, levels, expected picks in caller indices, NONE_U32 = none): one case per rule"""
    NONE = T.NONE_U32

    def fuller_wins():           # block 1 has fewer free GPUs and still holds the gang
        nodes, L = blocks_case(blocks=3, per_block=2)
        nodes["free_gpu"] = [8, 8, 4, 4, 8, 8]
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=4, min=1)])], level=0, anchor=5)
        return nodes, L, b.build(), [0], [2]

    def unschedulable_not_summed():   # node 1's GPUs do not count: block 0 is the fullest
        nodes, L = blocks_case(blocks=3, per_block=2)
        nodes["free_gpu"] = [8, 8, 4, 8, 8, 8]
        nodes["flags"][1] = 0
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=1)])], level=0, anchor=5)
        return nodes, L, b.build(), [0], [0]

    def unlabelled_node():       # node 2 has no block label: block 0 cannot count it, so only block 1 holds two 8-GPU pods
        nodes, L = blocks_case(blocks=2, per_block=3)
        nodes["free_gpu"] = [8, 0, 8, 8, 8, 8]
        nodes["dom"][2, :] = ABSENT
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, anchor=0)
        return nodes, L, b.build(), [0], [3]

    def class_mask():            # block 0 is fuller, but its nodes are of a class the clique does not accept
        nodes, L = blocks_case(blocks=2, per_block=2)
        nodes["free_gpu"] = [4, 4, 8, 8]
        nodes["flags"][:2] |= np.uint32(1 << T.NODE_CLASS_SHIFT)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=4, min=1, class_mask=0x1)])], level=0, anchor=0)
        return nodes, L, b.build(), [0], [2]

    def aggregate():             # each clique fits block 0 alone, not both together
        nodes, L = blocks_case(blocks=2, per_block=2)
        nodes["free_gpu"] = [8, 0, 8, 8]
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=1), dict(gpu=8, min=1)])], level=0, anchor=0)
        return nodes, L, b.build(), [0], [2]

    def no_domain_keeps_hash():  # nothing holds 16 GPUs on one node: the member keeps its hash anchor and is rejected
        nodes, L = blocks_case(blocks=2, per_block=2)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=16, min=1)])], level=0)
        b.add_gang([(None, [dict(gpu=2, min=1)])], level=0)
        return nodes, L, b.build(), [0, 0], [NONE, 0]

    def deeper_than_required():  # Required block, packed per host: the fullest host that holds the pod, in its block first
        nodes, L = blocks_case(blocks=3, per_block=2)
        nodes["free_gpu"] = [8, 8, 8, 2, 8, 6]
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=4, min=1)])], level=0, anchor=0)
        b.add_gang([(None, [dict(gpu=4, min=2)])], level=0, anchor=0)
        return nodes, L, b.build(), [1, 1], [5, 0]

    def host_without_required():  # no Required level: packed per host anyway
        nodes, L = blocks_case(blocks=2, per_block=2)
        nodes["free_gpu"] = [8, 3, 5, 8]
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=4, min=1)])], anchor=0)
        return nodes, L, b.build(), [1], [2]

    def ties_lowest_domain():    # a uniform cluster: every member picks block 0, fills it in index order, the rest spill
        nodes, L = blocks_case(blocks=3, per_block=2)
        b = T.GangTableBuilder()
        for a in (5, 3, 1, 4, 2):
            b.add_gang([(None, [dict(gpu=8, min=1)])], level=0, anchor=a)
        return nodes, L, b.build(), [0] * 5, [0] * 5

    return {f.__name__: f for f in (fuller_wins, unschedulable_not_summed, unlabelled_node, class_mask, aggregate,
                                    no_domain_keeps_hash, deeper_than_required, host_without_required, ties_lowest_domain)}


class Fragmentation:
    """Four blocks of 8 x 8-GPU nodes, two cycles.  Cycle 1: a stream of one-node gangs.  Cycle 2, on the table cycle 1 left: a gang
    that needs a whole block (8 pods of 8 GPUs), ranked first, and another stream of one-node gangs.  `run(cycle_fn, binpack)`:
    cycle_fn(nodes, L, tables, levels or None) -> outputs; returns (cycle 1 outputs, cycle 2 outputs, the blocks cycle 1 used)."""

    def __init__(self, small=8):
        self.small = small
        self.nodes, self.L = blocks_case()

    def tables(self, big):
        b = T.GangTableBuilder()
        if big:
            b.add_gang([(None, [dict(gpu=8, min=8)])], level=0, priority=1)
        for _ in range(self.small):
            b.add_gang([(None, [dict(gpu=8, min=1)])], level=0)
        return b.build()

    def run(self, cycle_fn, binpack):
        t1 = self.tables(False)
        o1 = cycle_fn(self.nodes, self.L, t1, np.zeros(len(t1[0]), np.uint8) if binpack else None)
        used = sorted({int(p["node"]) // 8 for p in o1["placements"]})
        t2 = self.tables(True)
        o2 = cycle_fn(o1["nodes_after"], self.L, t2, np.zeros(len(t2[0]), np.uint8) if binpack else None)
        return o1, o2, used
