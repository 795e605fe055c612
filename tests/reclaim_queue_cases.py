"""Reclaim across queues (grove_run_cycle_reclaim_queues, include/grove_place.h "reclaim across queues") restated over the
sequential oracle, and the scenarios the oracle property tests and the GPU parity tests share.

The ordinary pass is queue_cases.run_cycle_queues.  The queues of the gangs it left REJECTED are the classes, in ascending order of
their share when the pass starts.  Per class Q the donor set E(Q) is computed here in Python integers, one inclusive prefix per
queue in victim order; the members then go one at a time in rank order: the gate and surplus caps come from queue_cases.decide
over load' (the loads without what the standing gangs of E(Q) hold) with cap = min(limit, deserved) in place of the limits, and a
gang that passes is one oracle call over the node view (free + what the standing gangs of E(Q) hold) with its anchor pinned and its
cliques' replicas capped.  Victims are chosen here, node by node and then queue by queue of its chain, leaf first, with the
helpers of preempt_queue_cases."""
import numpy as np

from grove_b200 import tables as T
from preempt_queue_cases import NODE_STEP, QUEUE_STEP, _running, _subtree_loads, _take, usage_of
from queue_cases import NONE, REQ, UNL, chain, decide, make_queues, nodes_flat, run_cycle_queues
from reuse_cases import _with_free, free_table, hold_table

__all__ = ["NODE_STEP", "QUEUE_STEP", "make_quotas", "share", "share_less", "donor_set", "caps_of", "run_cycle_reclaim_queues",
           "hand_cases", "random_snapshot"]


def make_quotas(rows):
    """rows: (cpu, mem, gpu) deserved with None = unlimited -> queue_quota_dt array"""
    out = np.zeros(len(rows), dtype=T.queue_quota_dt)
    for i, row in enumerate(rows):
        out["deserved"][i] = [UNL if x is None else x for x in row]
    return out


def share(quota, load):
    """share_Q as (num, den), den 0 = +inf: the max over resources with a finite quota of load / deserved; 0/0 and no finite quota 0"""
    best = (0, 1)
    for k in range(3):
        d = int(quota["deserved"][k])
        if d == UNL:
            continue
        l = max(int(load[k]), 0)
        x = (l, d) if d else ((1, 0) if l else (0, 1))
        if share_less(best, x):
            best = x
    return best


def share_less(a, b):
    if b[1] == 0:
        return a[1] != 0
    if a[1] == 0:
        return False
    return a[0] * b[1] < b[0] * a[1]


def caps_of(queues, quotas):
    """the queue set with cap = min(limit, deserved) in place of the limits"""
    q = queues.copy()
    q["limit"] = np.minimum(queues["limit"], quotas["deserved"])
    return q


def _victim_key(prio, r):
    return (prio[r], -r)


def donor_set(queues, quotas, ld, prio, use_r, running_queue, gone, Q):
    """E(Q) as a sorted list: one inclusive prefix per queue X with a finite quota, in victim order, over the standing running gangs
    of X's subtree gives ok_X / over_X; r is a donor when it stands, has a queue apart from chain(Q) both ways, and over
    D(r, Q) = chain(queue(r)) minus chain(Q) every X says ok and some X says over"""
    R = len(prio)
    order = sorted(range(R), key=lambda r: _victim_key(prio, r))
    ok, over = {}, {}
    for X in range(len(queues)):
        d = [int(x) for x in quotas["deserved"][X]]
        fin = [x != UNL for x in d]
        if not any(fin):
            continue
        P = [0, 0, 0]
        for r in order:
            if gone[r] or running_queue[r] == NONE or X not in chain(queues, int(running_queue[r])):
                continue
            P = [P[k] + use_r[r][k] for k in range(3)]
            held = [k for k in range(3) if fin[k] and use_r[r][k] > 0]
            ok[X, r] = all(ld[X][k] - P[k] >= d[k] for k in held)
            over[X, r] = bool(held)
    cq = chain(queues, Q)
    out = []
    for r in range(R):
        if gone[r] or running_queue[r] == NONE:
            continue
        cr = chain(queues, int(running_queue[r]))
        if int(running_queue[r]) in cq or Q in cr:
            continue
        D = [X for X in cr if X not in cq]
        if all(ok.get((X, r), True) for X in D) and any(over.get((X, r), False) for X in D):
            out.append(r)
    return out


def run_cycle_reclaim_queues(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, quotas, running, holdings,
                             running_queue):
    """-> dict(placements, status, scope_status, nodes_after, victims, steps, loads_after, perm, classes) of the cycle as its
    definition reads; steps[i] says which step chose victims[i]; classes lists, per class run in order, dict(queue, donors,
    members, victims, loads_end) (donors empty: skipped)"""
    queues = np.asarray(queues, dtype=T.queue_dt)
    quotas = np.asarray(quotas, dtype=T.queue_quota_dt)
    gang_queue = np.asarray(gang_queue, dtype=np.uint32)
    running_queue = np.asarray(running_queue, dtype=np.uint32)
    base = run_cycle_queues(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue)
    G, N, R, NQ = len(gangs), len(nodes), len(running), len(queues)
    capq = caps_of(queues, quotas)
    status = base["status"].copy()
    sstat = base["scope_status"].copy()
    per_gang = {g: base["placements"][status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]].copy()
                for g in range(G) if status["state"][g] == T.GANG_ADMITTED}
    F = free_table(base["nodes_after"])
    perm = base["perm"]
    H = [hold_table(N, running, holdings, r) for r in range(R)]
    use_r = usage_of(running, holdings)
    prio = [int(running["priority"][r]) for r in range(R)]
    own = [[int(x) for x in queues["used"][q]] for q in range(NQ)]
    for g in range(G):   # the ordinary pass's admitted members join their queue
        if status["state"][g] == T.GANG_ADMITTED and gang_queue[g] != NONE:
            for e in per_gang[g]:
                for k in range(3):
                    own[int(gang_queue[g])][k] += int(cliques[REQ[k]][int(e["clique"])])
    gone = np.zeros(R, dtype=bool)
    on_node = {}
    for r in range(R):
        for h in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
            on_node.setdefault(int(h["node"]), []).append(r)
    victims, steps, classes = [], [], []
    rank = sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i))
    rejected = [g for g in rank if status["state"][g] == T.GANG_REJECTED and gang_queue[g] != NONE]
    ld0 = _subtree_loads(queues, own)
    order = sorted({int(gang_queue[g]) for g in rejected})
    sh = {Q: share(quotas[Q], ld0[Q]) for Q in order}
    # ascending share, ties by queue index (a stable insertion sort over the exact comparison)
    ranked = []
    for Q in order:
        i = len(ranked)
        while i > 0 and share_less(sh[Q], sh[ranked[i - 1]]):
            i -= 1
        ranked.insert(i, Q)

    def evict(v, g, step, cls):
        nonlocal F
        gone[v] = True
        F = F + H[v]
        if running_queue[v] != NONE:
            for k in range(3):
                own[int(running_queue[v])][k] -= use_r[v][k]
        victims.append((v, g)); steps.append(step); cls["victims"].append(v)

    for Q in ranked:
        E = donor_set(queues, quotas, _subtree_loads(queues, own), prio, use_r, running_queue, gone, Q)
        members = [g for g in rejected if int(gang_queue[g]) == Q]
        cls = dict(queue=Q, donors=E, members=members, victims=[], loads_end=None)
        classes.append(cls)
        if not E:
            cls["loads_end"] = _subtree_loads(queues, own)
            continue
        for g in members:
            standing = [x for x in E if not gone[x]]
            o = [list(x) for x in own]
            for r in standing:
                if running_queue[r] != NONE:
                    for k in range(3):
                        o[int(running_queue[r])][k] -= use_r[r][k]
            closed, caps = decide(capq, _subtree_loads(queues, o), [[0, 0, 0]] * NQ, gangs, cliques, g, Q)
            if closed:
                continue
            view = F + sum((H[x] for x in standing), np.zeros_like(F))
            sg = gangs[g: g + 1].copy()
            co, so = int(sg["clique_off"][0]), int(sg["scope_off"][0])
            sq = cliques[co: co + int(sg["n_cliques"][0])].copy()
            ss = scopes[so: so + int(sg["n_scopes"][0])].copy()
            sq["replicas"] = sq["min_replicas"] + np.asarray(caps, dtype=np.uint8)
            if sg["anchor_node"][0] == T.NONE_U32:
                sg["anchor_node"][0] = perm[oracle._fmix32(g) % N]   # the anchor the ordinary pass derived for this gang
            sg["base_gang"][0] = T.NONE_U32; sg["clique_off"][0] = 0; sg["scope_off"][0] = 0
            out = oracle.run_cycle(_with_free(nodes, view), n_levels, sg, sq, ss)
            if out["status"]["state"][0] != T.GANG_ADMITTED:
                continue
            pl = out["placements"].copy()
            use, first, U = {}, [], [0, 0, 0]
            for e in pl:
                n, c = int(e["node"]), sq[int(e["clique"])]
                if n not in use:
                    use[n] = np.zeros(4, dtype=np.int64); first.append(n)
                use[n] += [int(c["req_cpu_milli"]), int(c["req_mem_mib"]), int(c["req_gpu"]), 1]
                for k in range(3):
                    U[k] += int(c[REQ[k]])
            for n in first:   # (a) the node step
                while not (F[n] >= use[n]).all():
                    v = min((x for x in on_node.get(n, []) if x in E and not gone[x]), key=lambda x: _victim_key(prio, x))
                    evict(v, g, NODE_STEP, cls)
                F[n] -= use[n]
            for k in range(3):   # (b) the queue step
                own[Q][k] += U[k]
            for X in chain(queues, Q):
                while True:
                    ld = _subtree_loads(queues, own)[X]
                    cap = [int(capq["limit"][X][r]) for r in range(3)]
                    over = [U[r] > 0 and cap[r] != UNL and ld[r] > cap[r] for r in range(3)]
                    if not any(over):
                        break
                    cand = [x for x in E if not gone[x] and X in chain(queues, int(running_queue[x]))
                            and any(over[r] and use_r[x][r] > 0 for r in range(3))]
                    v = min(cand, key=lambda x: _victim_key(prio, x))
                    evict(v, g, QUEUE_STEP, cls)
            pl["clique"] += co
            per_gang[g] = pl
            st = out["status"][0].copy()
            flags = T.STATUS_RECLAIMER
            if any(s < int(c["replicas"]) - int(c["min_replicas"]) for s, c in zip(caps, cliques[co: co + len(caps)])):
                flags |= T.STATUS_SURPLUS_CAPPED
            st["reserved0"] = flags
            status[g] = st
            sstat[so: so + len(ss)] = out["scope_status"]
        cls["loads_end"] = _subtree_loads(queues, own)
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off if status["state"][g] == T.GANG_ADMITTED else status["placement_off"][g]
        if status["state"][g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F),
                victims=np.array(victims, dtype=T.victim_dt) if victims else np.zeros(0, dtype=T.victim_dt),
                steps=steps, loads_after=_subtree_loads(queues, own), perm=perm, classes=classes)


# ---- scenarios -------------------------------------------------------------------------------------------------------------------

def _gang(b, gpu, prio=0, n=1):
    for _ in range(n):
        b.add_gang([(None, [dict(gpu=gpu, cpu=1000, mem=1000, min=1)])], priority=prio)


def _used(running, holdings, running_queue, nq):
    """each queue's used = what its running gangs hold"""
    use = usage_of(running, holdings)
    out = [[0, 0, 0] for _ in range(nq)]
    for r, q in enumerate(running_queue):
        if q != NONE:
            for k in range(3):
                out[int(q)][k] += use[r][k]
    return out


def _case(n_nodes, run_prios, run_nodes, run_queue, parents, limits, quotas, subs, gang_queue, gpu_nodes=None):
    """a cluster of n_nodes 8-GPU nodes (gpu_nodes: per-node GPUs instead), running gangs of 8 GPUs per node (run_nodes[r]) in
    run_queue[r], a queue tree (parents, limits) whose used is what its running gangs hold, quotas, and the submission subs =
    [(gpu, priority)] in gang_queue"""
    nodes = nodes_flat(n_nodes)
    if gpu_nodes is not None:
        nodes["free_gpu"] = gpu_nodes
    running, holdings = _running(8, run_prios, run_nodes)
    if gpu_nodes is not None:   # a running gang holds every GPU of its nodes
        holdings["gpu"] = [gpu_nodes[int(h["node"])] for h in holdings]
    rq = np.array(run_queue, dtype=np.uint32)
    used = _used(running, holdings, rq, len(parents))
    qs = make_queues([(p, lim, u) for p, lim, u in zip(parents, limits, used)])
    b = T.GangTableBuilder()
    for gpu, prio in subs:
        _gang(b, gpu, prio)
    return _take(nodes, running, holdings), 2, b.build(), qs, np.array(gang_queue, np.uint32), make_quotas(quotas), running, holdings, rq


UL = (None, None, None)


def hand_cases():
    """name -> (nodes, n_levels, tables, queues, gang_queue, quotas, running, holdings, running_queue): one case per rule"""
    return {
        # team-a deserves 8 GPUs and holds none; team-b deserves 8 and runs two 8-GPU gangs on a full cluster: one of them goes
        "starved_team": lambda: _case(2, [5, 5], [[0], [1]], [1, 1], [None, None], [UL, UL], [(None, None, 8)] * 2,
                                      [(8, 0)], [0]),
        # team-b holds exactly its quota: nothing is reclaimable
        "donor_at_quota": lambda: _case(2, [0, 0], [[0], [1]], [1, 1], [None, None], [UL, UL], [(None, None, 8), (None, None, 16)],
                                        [(8, 0)], [0]),
        # team-a already holds its quota of 8: its next gang is gated by its cap, nothing is evicted
        "reclaimer_at_quota": lambda: _case(3, [0, 0, 0], [[0], [1], [2]], [0, 1, 1], [None, None], [UL, UL],
                                            [(None, None, 8), (None, None, 8)], [(8, 0)], [0]),
        # siblings under a parent at its quota of 16: the parent is not asked, team-b's surplus goes to team-a
        "siblings": lambda: _case(2, [0, 0], [[0], [1]], [2, 2], [None, 0, 0], [UL, UL, UL],
                                  [(None, None, 16), (None, None, 8), (None, None, 8)], [(8, 0)], [1]),
        # a victim of a higher priority than its reclaimer
        "victim_outranks": lambda: _case(2, [9, 1], [[0], [1]], [1, 1], [None, None], [UL, UL], [(None, None, 8)] * 2,
                                         [(8, 0)], [0]),
        # team-b holds 24 against 8: only its two first gangs in victim order are donors, the third keeps it at its quota
        "partial_donor": lambda: _case(3, [0, 1, 2], [[0], [1], [2]], [1, 1, 1], [None, None], [UL, UL],
                                       [(None, None, 16), (None, None, 8)], [(8, 0), (8, 0)], [0, 0]),
        # quota 0: everything team-b runs is reclaimable
        "quota_zero": lambda: _case(2, [3, 3], [[0], [1]], [1, 1], [None, None], [UL, UL], [UL, (None, None, 0)],
                                    [(8, 0), (8, 0)], [0, 0]),
        # quota -1: nothing team-b runs is reclaimable
        "quota_unlimited": lambda: _case(2, [0, 0], [[0], [1]], [1, 1], [None, None], [UL, UL], [(None, None, 8), UL],
                                         [(8, 0)], [0]),
        # a running gang without a queue is never a victim: the second gang of team-a finds no room
        "no_queue_running": lambda: _case(2, [0, 0], [[0], [1]], [NONE, 1], [None, None], [UL, UL], [UL, (None, None, 0)],
                                          [(8, 0), (8, 0)], [0, 0]),
        # two starved queues compete for one donor gang: team-a (share 0) goes before team-c (share 1/2) despite its index
        "two_starved": lambda: _case(3, [0, 0, 0], [[0], [1], [2]], [0, 2, 2], [None, None, None], [UL, UL, UL],
                                     [(None, None, 16), (None, None, 8), (None, None, 8)], [(8, 0), (8, 0)], [0, 1]),
        # team-a's limit of 8 is below its quota of 16: it binds
        "limit_below_quota": lambda: _case(2, [0, 0], [[0], [1]], [1, 1], [None, None], [(None, None, 8), UL],
                                           [(None, None, 16), (None, None, 0)], [(8, 0), (8, 0)], [0, 0]),
        # the parent's limit of 16 turns team-a's gang away OVER_LIMIT; the class admits it on a free node and the queue step evicts
        # team-b's gang to bring the parent back within its limit
        "over_limit_shared_parent": lambda: _case(4, [0, 0], [[0], [1]], [2, 2], [None, 0, 0], [(None, None, 16), UL, UL],
                                                  [UL, (None, None, 8), (None, None, 8)], [(8, 0)], [1]),
        # the queue step evicts by the victim order, lowest priority first, then the highest index: 4-GPU nodes 0-2 each held by a
        # team-b gang, node 3 free; the parent's limit of 12 makes the queue step evict gangs 2 and 1, gang 0 stays
        "queue_step_order": lambda: _case(4, [3, 1, 1], [[0], [1], [2]], [2, 2, 2], [None, 0, 0], [(None, None, 12), UL, UL],
                                          [UL, UL, (None, None, 0)], [(8, 0)], [1], gpu_nodes=[4, 4, 4, 8]),
    }


def random_snapshot(seed, pref=False):
    """A random contested cluster: 8-GPU hosts in racks (two levels), most of them held by running gangs of random priorities in a
    random queue tree of depth 1-3, and a submission of 1-16-GPU gangs in those queues; limits mostly lifted, quotas random
    around each queue's load (some queues starved, some 0 or -1).  pref: some gangs ask for a Preferred host level.
    -> (nodes, n_levels, tables, queues, gang_queue, quotas, running, holdings, running_queue)"""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(6, 40))
    nodes = nodes_flat(n, per_block=int(rng.integers(2, 9)))
    n_roots, depth = int(rng.integers(1, 3)), int(rng.integers(1, 4))
    parents, frontier = [None] * n_roots, list(range(n_roots))
    for _ in range(depth - 1):
        nxt = []
        for p in frontier:
            for _ in range(int(rng.integers(1, 4))):
                parents.append(p); nxt.append(len(parents) - 1)
        frontier = nxt
    NQ = len(parents)
    # running gangs: 1-3 nodes each, 4 or 8 GPUs per node, over most of the nodes
    free = list(rng.permutation(n)[: int(n * rng.uniform(0.85, 1.0))])
    prios, on, gpus = [], [], []
    while free:
        k = min(len(free), int(rng.integers(1, 4)))
        on.append([int(x) for x in free[:k]]); free = free[k:]
        prios.append(int(rng.integers(0, 4))); gpus.append(int(rng.choice([4, 8, 8])))
    running = np.zeros(len(prios), dtype=T.running_dt)
    hold = []
    for r, (p, ns, gpu) in enumerate(zip(prios, on, gpus)):
        running["priority"][r] = p; running["holding_off"][r] = len(hold); running["n_holdings"][r] = len(ns)
        hold += [(x, int(rng.integers(500, 4000)), int(rng.integers(512, 8192)), gpu, 1) for x in ns]
    holdings = np.array(hold, dtype=T.holding_dt)
    # each queue plays a role: a donor runs most of the gangs and deserves part of its load, a starved queue deserves more than it
    # holds; cpu and memory quotas are rarer, parents deserve about what their subtree holds
    role = rng.choice(["donor", "starved", "unlimited", "zero"], NQ, p=[0.4, 0.4, 0.12, 0.08])
    donors = [q for q in range(NQ) if role[q] in ("donor", "zero")] or [int(rng.integers(0, NQ))]
    rq = np.array([NONE if rng.random() < 0.1 else int(rng.choice(donors)) if rng.random() < 0.8 else int(rng.integers(0, NQ))
                   for _ in range(len(running))], dtype=np.uint32)
    used = _used(running, holdings, rq, NQ)
    ld = [list(u) for u in used]
    for q in range(NQ - 1, -1, -1):
        if parents[q] is not None:
            for k in range(3):
                ld[parents[q]][k] += ld[q][k]
    limits = []
    for q in range(NQ):
        limits.append(tuple(None if rng.random() < 0.8 else int(ld[q][k] * rng.uniform(0.8, 1.3)) + int(rng.integers(0, 24)) * (1000, 2048, 1)[k]
                            for k in range(3)))
    qs = make_queues([(p, lim, u) for p, lim, u in zip(parents, limits, used)])
    quotas = np.zeros(NQ, dtype=T.queue_quota_dt)
    quotas["deserved"] = UNL
    kids = {p for p in parents if p is not None}
    for q in range(NQ):
        for k in range(3):
            if (k < 2 and rng.random() < 0.8) or role[q] == "unlimited" or (q in kids and rng.random() < 0.5):
                continue
            quotas["deserved"][q, k] = (0 if role[q] == "zero" else int(ld[q][k] * rng.uniform(0.9, 1.6)) if q in kids else
                                        int(ld[q][k] * rng.uniform(0.2, 0.9)) if role[q] == "donor" else ld[q][k] + int(rng.integers(4, 48)) * (1000, 2048, 1)[k])
    b = T.GangTableBuilder()
    gq = []
    for _ in range(int(rng.integers(2, 14))):
        cl = [dict(gpu=int(rng.choice([1, 2, 4, 8])), cpu=int(rng.integers(0, 4000)), mem=int(rng.integers(0, 8192)),
                   min=int(rng.integers(1, 3)))]
        if rng.random() < 0.3:
            cl[0]["replicas"] = cl[0]["min"] + int(rng.integers(1, 3))
        level = None if rng.random() < 0.5 else 0
        b.add_gang([(None, cl)], level=level, priority=int(rng.integers(0, 4)),
                   preferred=1 if pref and rng.random() < 0.5 else None)
        starved = [q for q in range(NQ) if role[q] == "starved"] or donors
        gq.append(NONE if rng.random() < 0.1 else int(rng.choice(starved)) if rng.random() < 0.85 else int(rng.integers(0, NQ)))
    return _take(nodes, running, holdings), 2, b.build(), qs, np.array(gq, np.uint32), quotas, running, holdings, rq
