"""Fair-share order (grove_set_fair_share, include/grove_place.h "fair-share order") restated over the sequential oracle, the
turn order O(R) two ways, and the scenarios the oracle property tests and the GPU parity tests share.

The restatement walks the definition one turn at a time: next(root) over the queue tree, shares as Python Fractions of the loads
at the turn.  A member's turn is decided as in tests/queue_cases.py -- gate and surplus caps in Python integers
(queue_cases.decide), then one oracle call with its anchor pinned and its replicas capped; a run of turns of the pseudo-queue of
the gangs without a queue is one oracle cycle (their admissions charge no queue, so the walk does not depend on them).

order_walk is the definition's order for given per-gang usages U; order_vec computes the same order the way the engine does --
per tree level a segmented exclusive scan of U, the key (share, rank), its prefix max along each sequence and a stable sort by
(parent, key).  fixed_point runs the engine's loop over the unchanged queue restatement: a queue cycle in order O_i, then
O_{i+1} = O(R_i), until the order stays."""
import math
from fractions import Fraction

import numpy as np

from grove_b200 import tables as T
from queue_cases import REQ, chain, decide, loads, make_queues, nodes_flat, assign_queues
from reclaim_queue_cases import make_quotas, share
from reuse_cases import free_table, _with_free

UNL = T.QUEUE_UNLIMITED
NONE = T.NONE_U32


def _tree(queues):
    NQ = len(queues)
    kids = {q: [] for q in range(NQ + 2)}   # NQ = the pseudo-queue of the gangs without a queue, NQ + 1 = the root
    for q in range(NQ):
        p = int(queues["parent"][q])
        kids[NQ + 1 if p == NONE else p].append(q)
    kids[NQ + 1].append(NQ)
    return kids


def ranks(gangs):
    order = sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))
    rank = [0] * len(gangs)
    for k, g in enumerate(order):
        rank[g] = k
    return order, rank


def share_value(quota, load):
    n, d = share(quota, load)
    return math.inf if d == 0 else Fraction(n, d)


def walk(queues, quotas, gangs, gang_queue, take, trace=None):
    """the turns of the definition: take(g) -> what gang g charges to its chain at its turn (None or zeros: nothing).
    trace (a list): gets (gang, loads of its chain before its turn, after it) for every member"""
    queues = np.asarray(queues, dtype=T.queue_dt)
    NQ = len(queues)
    kids = _tree(queues)
    order, rank = ranks(gangs)
    waiting = {q: [] for q in range(NQ + 1)}
    for g in order:
        waiting[NQ if gang_queue[g] == NONE else int(gang_queue[g])].append(g)
    ld = loads(queues)

    def shr(X):
        return Fraction(0) if X == NQ else share_value(quotas[X], ld[X])

    def nxt(X):
        if X <= NQ and not kids[X]:
            return waiting[X][0] if waiting[X] else None
        best = None
        for C in kids[X]:
            h = nxt(C)
            if h is not None and (best is None or (shr(C), rank[h]) < best[0]):
                best = ((shr(C), rank[h]), h)
        return None if best is None else best[1]

    turns = []
    while True:
        g = nxt(NQ + 1)
        if g is None:
            return turns
        q = NQ if gang_queue[g] == NONE else int(gang_queue[g])
        waiting[q].pop(0)
        turns.append(g)
        before = [list(ld[Q]) for Q in chain(queues, q)] if q != NQ else None
        u = take(g)
        if u is not None and q != NQ:
            for Q in chain(queues, q):
                for r in range(3):
                    ld[Q][r] += int(u[r])
        if trace is not None and q != NQ:
            trace.append((g, before, [list(ld[Q]) for Q in chain(queues, q)]))


def r_min_use(gangs, cliques, gang_queue):
    """U of the first order: R_min of every member, 0 for the others -> int64 [G, 3]"""
    from queue_cases import r_min
    U = np.zeros((len(gangs), 3), dtype=np.int64)
    for g in range(len(gangs)):
        if gang_queue[g] != NONE:
            U[g] = r_min(gangs, cliques, g)
    return U


def use_of(out, cliques):
    """U of every gang from a cycle's outputs: what its placements ask for, 0 when not admitted -> int64 [G, 3]"""
    st = out["status"]
    U = np.zeros((len(st), 3), dtype=np.int64)
    for g in np.nonzero(st["state"] == T.GANG_ADMITTED)[0]:
        pl = out["placements"][int(st["placement_off"][g]): int(st["placement_off"][g]) + int(st["n_pods"][g])]
        for r in range(3):
            U[g, r] = int(cliques[REQ[r]][pl["clique"]].astype(np.int64).sum())
    return U


def order_walk(queues, quotas, gangs, gang_queue, U):
    """O(U) by the definition's walk"""
    return np.array(walk(queues, quotas, gangs, gang_queue, lambda g: U[g]), dtype=np.uint32)


def order_vec(queues, quotas, gangs, gang_queue, U):
    """O(U) as the engine computes it: bottom-up over the tree levels, a segmented exclusive scan of U, the key (share, rank),
    its segmented prefix max and a stable sort by (parent, key).  Shares are numbered exactly (sorted distinct Fractions)."""
    queues = np.asarray(queues, dtype=T.queue_dt)
    G, NQ = len(gangs), len(queues)
    parent = np.full(NQ + 2, NQ + 1, dtype=np.int64)
    depth = np.ones(NQ + 2, dtype=np.int64)
    depth[NQ + 1] = 0
    for q in range(NQ):
        if queues["parent"][q] != NONE:
            parent[q] = int(queues["parent"][q]); depth[q] = depth[parent[q]] + 1
    ld = loads(queues) + [[0, 0, 0], [0, 0, 0]]
    _, rank = ranks(gangs)
    rank = np.asarray(rank, dtype=np.int64)
    leaf = np.where(gang_queue == NONE, NQ, gang_queue).astype(np.int64)
    seq = np.lexsort((rank, leaf))          # every leaf's sequence in rank order
    own = leaf[seq]
    U = np.asarray(U, dtype=np.int64)
    for d in range(int(depth.max()), 0, -1):
        seg = np.concatenate(([0], np.cumsum(own[1:] != own[:-1])))
        first = np.concatenate(([0], np.nonzero(own[1:] != own[:-1])[0] + 1))
        us = U[seq]
        excl = np.cumsum(us, axis=0) - us
        before = excl - excl[first][seg]                       # segmented exclusive scan
        at = depth[own] == d
        sh = [share_value(quotas[int(o)], [ld[int(o)][r] + int(before[i, r]) for r in range(3)]) if at[i] and o < NQ else Fraction(0)
              for i, o in enumerate(own)]
        ids = {v: k for k, v in enumerate(sorted(set(sh)))}
        key = np.array([ids[v] for v in sh], dtype=np.int64) * (G + 1) + rank[seq]
        big = int(key.max()) + 1
        pmax = np.maximum.accumulate(key + seg * big) - seg * big   # segmented prefix max
        new_own = np.where(at, parent[own], own)
        perm = np.lexsort((pmax, new_own))                            # stable
        seq, own = seq[perm], new_own[perm]
    return seq.astype(np.uint32)


def fixed_point(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, quotas, order=order_vec):
    """the engine's loop over the queue restatement: O_0 = O(R_min), then the queue cycle in order O_i (priority := G - turn
    position) and O_{i+1} = O(R_i) until it stays -> (outputs, order, iterations)"""
    from queue_cases import run_cycle_queues
    G = len(gangs)
    O = order(queues, quotas, gangs, gang_queue, r_min_use(gangs, cliques, gang_queue))
    it = 0
    while True:
        it += 1
        out = run_cycle_queues(oracle, nodes, n_levels, with_order(gangs, O), cliques, scopes, queues, gang_queue)
        O2 = order(queues, quotas, gangs, gang_queue, use_of(out, cliques))
        if np.array_equal(O, O2):
            return out, O, it
        assert it <= G + 1
        O = O2


def with_order(gangs, O):
    """the gangs with priority := G - turn position: a plain queue cycle takes them in order O"""
    g = gangs.copy()
    g["priority"][np.asarray(O, dtype=np.int64)] = len(gangs) - np.arange(len(gangs))
    return g


def run_fair_share(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, quotas):
    """-> dict(placements, status, scope_status, nodes_after, perm, order, trace) of the fair-share cycle, one turn at a time;
    trace: (member, its chain's loads before its turn, after it) per member turn"""
    G, N = len(gangs), len(nodes)
    queues = np.asarray(queues, dtype=T.queue_dt)
    gang_queue = np.asarray(gang_queue, dtype=np.uint32)
    perm = oracle.topology(nodes, n_levels)[0]
    ld = loads(queues)
    charged = [[0, 0, 0] for _ in range(len(queues))]
    status = np.zeros(G, dtype=T.status_dt)
    status["level"] = T.LEVEL_NONE; status["domain_node"] = T.NONE_U32
    sstat = np.zeros(len(scopes), dtype=T.scope_status_dt)
    sstat["level"] = T.LEVEL_NONE; sstat["domain_node"] = T.NONE_U32
    state = np.zeros(G, dtype=np.uint8)
    flags = np.zeros(G, dtype=np.uint16)
    per_gang = {}
    box = dict(F=free_table(nodes))

    def piece(run):   # the turns `run` (in turn order) as one oracle cycle; -> the oracle's output, the gangs it saw
        ids = []
        for g in sorted(run):   # submission order inside a piece: the oracle's order is then the turn order
            b = int(gangs["base_gang"][g])
            if gangs["flags"][g] & T.GANG_GATED:
                state[g] = T.GANG_GATED_SKIP
            elif b != NONE and b not in run and state[b] != T.GANG_ADMITTED:
                state[g] = T.GANG_BASE_REJECTED
            else:
                ids.append(g)
        while True:   # a base gang of the piece that is gated (or waits for its own base) is never admitted
            out_ = [g for g in ids if int(gangs["base_gang"][g]) in run and int(gangs["base_gang"][g]) not in ids]
            if not out_:
                break
            for g in out_:
                state[g] = T.GANG_BASE_REJECTED
            ids = [g for g in ids if g not in out_]
        if not ids:
            return None, ids, None
        sub = {g: k for k, g in enumerate(ids)}
        sg = gangs[ids].copy()
        sq, ss = [], []
        for k, g in enumerate(ids):
            b = int(gangs["base_gang"][g])
            sg["base_gang"][k] = sub[b] if b in sub else NONE
            if sg["anchor_node"][k] == NONE:
                sg["anchor_node"][k] = perm[oracle._fmix32(g) % N]
            sg["clique_off"][k] = sum(len(x) for x in sq); sg["scope_off"][k] = sum(len(x) for x in ss)
            co, so = int(gangs["clique_off"][g]), int(gangs["scope_off"][g])
            sq.append(cliques[co: co + int(gangs["n_cliques"][g])].copy()); ss.append(scopes[so: so + int(gangs["n_scopes"][g])])
        return sg, ids, (np.concatenate(sq), np.concatenate(ss))

    def record(out, ids, sg):
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
        box["F"] = free_table(out["nodes_after"])

    pending = []

    def flush():
        if not pending:
            return
        sg, ids, t = piece(list(pending))
        pending.clear()
        if sg is not None:
            record(oracle.run_cycle(_with_free(nodes, box["F"]), n_levels, sg, *t), ids, sg)

    def take(g):
        if gang_queue[g] == NONE:
            pending.append(g)
            return None
        flush()
        sg, ids, t = piece([g])
        if sg is None:
            return None
        sq, ss = t
        q = int(gang_queue[g])
        closed, caps = decide(queues, ld, charged, gangs, cliques, g, q)
        if closed:   # REJECTED without evaluation: the record of a gang that fits nowhere, and nothing changes
            blocked = _with_free(nodes, box["F"])
            blocked["flags"] &= ~np.uint32(T.NODE_SCHEDULABLE)
            out = oracle.run_cycle(blocked, n_levels, sg, sq, ss)
            out["nodes_after"] = _with_free(nodes, box["F"])
            flags[g] |= T.STATUS_OVER_LIMIT
            record(out, ids, sg)
            return None
        sq["replicas"] = sq["min_replicas"] + np.asarray(caps, dtype=np.uint8)
        out = oracle.run_cycle(_with_free(nodes, box["F"]), n_levels, sg, sq, ss)
        record(out, ids, sg)
        # what the gang's own placements ask for, admitted or not: its charge (a rejected gang's record binds nothing)
        st = out["status"][0]
        pl = out["placements"][int(st["placement_off"]): int(st["placement_off"]) + int(st["n_pods"])]
        U = [int(sum(int(sq[REQ[r]][int(e["clique"])]) for e in pl)) for r in range(3)]
        if st["state"] != T.GANG_ADMITTED:
            return U
        for Q in chain(queues, q):
            for r in range(3):
                charged[Q][r] += U[r]
        extra = (cliques["replicas"].astype(int) - cliques["min_replicas"].astype(int))[int(gangs["clique_off"][g]):][: len(caps)]
        if any(s < x for s, x in zip(caps, extra)):
            flags[g] |= T.STATUS_SURPLUS_CAPPED
        return U

    trace = []
    turns = walk(queues, quotas, gangs, gang_queue, take, trace)
    flush()
    status["state"] = state
    status["reserved0"] = flags
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off
        if state[g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, box["F"]), perm=perm,
                order=np.array(turns, dtype=np.uint32), trace=trace)


def random_snapshot(seed, pref=False):
    """a random contested snapshot: random_case's cluster and gangs, queue_cases.assign_queues's tree (limits tight, loose,
    unlimited or exceeded), every member moved to a leaf, and deserved quotas per queue and resource -- mostly GPU, around a share
    of the demand, some 0, some unlimited -> (nodes, n_levels, tables, queues, gang_queue, quotas)"""
    from test_random_parity_gpu import random_case
    nodes, L, tables = random_case(seed, pref=pref)
    rng = np.random.default_rng(seed + 77)
    qs, gq = assign_queues(rng, tables[0], tables[1], share=0.85)
    NQ = len(qs)
    inner = {int(p) for p in qs["parent"] if p != NONE}
    leaves = [q for q in range(NQ) if q not in inner]
    for g in range(len(gq)):
        if gq[g] != NONE and int(gq[g]) in inner:
            gq[g] = int(rng.choice(leaves))
    from queue_cases import demand
    D = demand(tables[1])
    quotas = np.zeros(NQ, dtype=T.queue_quota_dt)
    quotas["deserved"] = UNL
    for q in range(NQ):
        for r in range(3):
            x = rng.random()
            if r < 2 and x < 0.7:
                continue
            quotas["deserved"][q, r] = 0 if x > 0.95 else int(max(D[r], 1) * rng.uniform(0.02, 0.6))
    return nodes, L, tables, qs, gq, quotas


def _one(b, gpu, prio=0, n=1, replicas=None, level=None, base=None):
    cl = dict(gpu=gpu, min=n)
    if replicas is not None:
        cl["replicas"] = replicas
    return b.add_gang([(None, [cl])], priority=prio, level=level, base=base)


def hand_cases():
    """name -> (nodes, n_levels, tables, queues, gang_queue, quotas): one case per rule of the definition"""
    def starved_team_first():   # team-b holds its 16-GPU quota and submits at priority 5; team-a holds nothing: a's gangs go first
        nodes = nodes_flat(2)
        b = T.GangTableBuilder()
        for p in (5, 5, 0, 0):
            _one(b, 8, p)
        qs = make_queues([(None, (None, None, None), (0, 0, 16)), (None, (None, None, None), (0, 0, 0))])
        return nodes, 2, b.build(), qs, np.array([0, 0, 1, 1], np.uint32), make_quotas([(None, None, 16), (None, None, 16)])

    def parent_before_child():   # A's share is 0 but its parent is above its own quota; B's parent is below: B goes first
        nodes = nodes_flat(1)
        b = T.GangTableBuilder()
        _one(b, 8); _one(b, 8)
        qs = make_queues([(None, (None, None, None), (0, 0, 0)), (None, (None, None, None), (0, 0, 0)),
                          (0, (None, None, None), (0, 0, 0)), (0, (None, None, None), (0, 0, 8)), (1, (None, None, None), (0, 0, 4))])
        quotas = make_quotas([(None, None, 8), (None, None, 16), (None, None, 16), (None, None, None), (None, None, 8)])
        return nodes, 2, b.build(), qs, np.array([2, 4], np.uint32), quotas

    def share_tie_by_rank():   # equal shares: the head of better rank goes first
        nodes = nodes_flat(1)
        b = T.GangTableBuilder()
        _one(b, 8, 0); _one(b, 8, 5)
        qs = make_queues([(None, (None, None, None), (0, 0, 4)), (None, (None, None, None), (0, 0, 2))])
        return nodes, 2, b.build(), qs, np.array([0, 1], np.uint32), make_quotas([(None, None, 8), (None, None, 4)])

    def rejected_goes_again():   # a-1 asks for more than a node has: A's share stays 0 and a-2 goes before b-1
        nodes = nodes_flat(1)
        b = T.GangTableBuilder()
        _one(b, 8, 0, n=2, level=1); _one(b, 8, 0); _one(b, 8, 9)
        qs = make_queues([(None, (None, None, None), (0, 0, 0)), (None, (None, None, None), (0, 0, 2))])
        return nodes, 2, b.build(), qs, np.array([0, 0, 1], np.uint32), make_quotas([(None, None, 8), (None, None, 8)])

    def zero_quota_last():   # quota 0 with load is +inf: Z goes after Y, whatever the priorities
        nodes = nodes_flat(1)
        b = T.GangTableBuilder()
        _one(b, 8, 9); _one(b, 8, 0)
        qs = make_queues([(None, (None, None, None), (0, 0, 1)), (None, (None, None, None), (0, 0, 16))])
        return nodes, 2, b.build(), qs, np.array([0, 1], np.uint32), make_quotas([(None, None, 0), (None, None, 8)])

    def over_limit_member():   # A may hold 8 GPUs: its second gang is OVER_LIMIT, after B's gang has had its turn in between
        nodes = nodes_flat(3)
        b = T.GangTableBuilder()
        _one(b, 8, 3); _one(b, 8, 3); _one(b, 8, 0)
        qs = make_queues([(None, (None, None, 8), (0, 0, 0)), (None, (None, None, None), (0, 0, 2))])
        return nodes, 2, b.build(), qs, np.array([0, 0, 1], np.uint32), make_quotas([(None, None, 16), (None, None, 8)])

    def base_takes_turn_later():   # the scaled gang's queue is below its quota, its base's queue above: BASE_REJECTED
        nodes = nodes_flat(2)
        b = T.GangTableBuilder()
        x = _one(b, 8, 1)
        _one(b, 8, 1, base=x)
        qs = make_queues([(None, (None, None, None), (0, 0, 16)), (None, (None, None, None), (0, 0, 0))])
        return nodes, 2, b.build(), qs, np.array([0, 1], np.uint32), make_quotas([(None, None, 8), (None, None, 8)])

    def many_iterations():   # surplus pods make every A and B turn charge more than R_min: the first orders are wrong
        nodes = nodes_flat(6)
        b = T.GangTableBuilder()
        for i in range(3):
            _one(b, 1, 0, n=1, replicas=8)
            _one(b, 1, 0, n=1, replicas=6)
            _one(b, 2, 0, n=1, replicas=3)
        qs = make_queues([(None, (None, None, None), (0, 0, 0)), (None, (None, None, None), (0, 0, 3)),
                          (None, (None, None, None), (0, 0, 5))])
        return nodes, 2, b.build(), qs, np.array([0, 1, 2] * 3, np.uint32), make_quotas([(None, None, 8), (None, None, 9), (None, None, 10)])

    return {"starved_team_first": starved_team_first, "parent_before_child": parent_before_child,
            "share_tie_by_rank": share_tie_by_rank, "rejected_goes_again": rejected_goes_again, "zero_quota_last": zero_quota_last,
            "over_limit_member": over_limit_member, "base_takes_turn_later": base_takes_turn_later,
            "many_iterations": many_iterations}
