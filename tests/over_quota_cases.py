"""Over-quota weight (grove_set_over_quota, include/grove_place.h "over-quota weight"): the fair shares restated in Python integers,
random weights for the snapshots of tests/fair_share_cases.py and tests/reclaim_queue_cases.py, random queue trees for the fair
shares alone, and the hand cases.  An entry with weights is its existing restatement fed the fair shares as the deserved quotas."""
import numpy as np

from grove_b200 import tables as T
from queue_cases import REQ, nodes_flat, make_queues
from reclaim_queue_cases import _case, make_quotas

UNL = T.QUEUE_UNLIMITED
NONE = T.NONE_U32
CLAMP = 1 << 62


def make_weights(rows):
    """rows: (cpu, mem, gpu) weights -> queue_weight_dt array"""
    out = np.zeros(len(rows), dtype=T.queue_weight_dt)
    for i, row in enumerate(rows):
        out["over_quota"][i] = row
    return out


def ones(n):
    return make_weights([(1, 1, 1)] * n)


def inputs(nodes, gangs, cliques, queues, gang_queue):
    """-> (C, load, demand): the capacity per resource, the starting load and the demand per queue and resource"""
    NQ = len(queues)
    par = [int(p) for p in queues["parent"]]
    load = [[min(int(queues["used"][q][r]), CLAMP) for r in range(3)] for q in range(NQ)]
    for q in range(NQ - 1, -1, -1):
        if par[q] != NONE:
            for r in range(3):
                load[par[q]][r] = min(load[par[q]][r] + load[q][r], CLAMP)
    sched = (nodes["flags"] & T.NODE_SCHEDULABLE) != 0
    free = [int(nodes[f][sched].astype(np.int64).sum()) for f in ("free_cpu_milli", "free_mem_mib", "free_gpu")]
    C = [min(free[r] + sum(load[q][r] for q in range(NQ) if par[q] == NONE), CLAMP) for r in range(3)]
    dem = [list(x) for x in load]
    for g in range(len(gangs)):
        q = int(gang_queue[g])
        if q == NONE or gangs["flags"][g] & T.GANG_GATED:
            continue
        co, nc = int(gangs["clique_off"][g]), int(gangs["n_cliques"][g])
        s = [sum(int(cliques["replicas"][i]) * int(cliques[REQ[r]][i]) for i in range(co, co + nc)) for r in range(3)]
        while q != NONE:
            for r in range(3):
                dem[q][r] += s[r]
            q = par[q]
    return C, load, [[min(x, CLAMP) for x in row] for row in dem]


def divide(P, kids, dem, lim, des, w, rounds=None):
    """one parent's division of pool P among kids (ascending) -> ({kid: fair}, {kid: pool of its own children}); rounds (a list):
    gets the number of water-fill rounds that gave something"""
    fair, pool, need = {}, {}, {}
    k = 0
    took = 0
    for c in kids:
        want = min(dem[c], lim[c])
        if des[c] == UNL:
            fair[c] = UNL; pool[c] = want; took += want
        else:
            base = min(des[c], want)
            fair[c] = base; need[c] = want - base; took += base
    R = max(0, P - took)
    while True:
        A = [c for c in kids if des[c] != UNL and need[c] > 0 and w[c] > 0]
        W = sum(w[c] for c in A)
        if not A or R == 0:
            break
        give = {c: min(need[c], R * w[c] // W) for c in A}
        if not sum(give.values()):
            break
        for c in A:
            fair[c] += give[c]; need[c] -= give[c]
        R -= sum(give.values())
        k += 1
    if R:
        A = sorted((c for c in kids if des[c] != UNL and need[c] > 0 and w[c] > 0), key=lambda c: (-w[c], c))
        assert not A or R < len(A)
        for c in A[:R]:
            fair[c] += 1
    for c in kids:
        if des[c] != UNL:
            pool[c] = fair[c]
    if rounds is not None:
        rounds.append(k)
    return fair, pool


def fair_shares(nodes, gangs, cliques, queues, gang_queue, quotas, weights):
    """-> (NQ, 3) list of Python integers: the fair shares, UNL where deserved is"""
    queues = np.asarray(queues, dtype=T.queue_dt)
    NQ = len(queues)
    C, _, dem = inputs(nodes, gangs, cliques, queues, gang_queue)
    kids = {q: [] for q in range(NQ + 1)}
    for q in range(NQ):
        p = int(queues["parent"][q])
        kids[NQ if p == NONE else p].append(q)
    out = [[0, 0, 0] for _ in range(NQ)]
    for r in range(3):
        pool = {NQ: C[r]}
        dm = [dem[q][r] for q in range(NQ)]
        lim = [int(queues["limit"][q][r]) for q in range(NQ)]
        des = [int(quotas["deserved"][q][r]) for q in range(NQ)]
        w = [int(weights["over_quota"][q][r]) for q in range(NQ)]
        for p in [NQ] + list(range(NQ)):   # parents come before their children
            if kids[p]:
                f, pl = divide(pool[p], kids[p], dm, lim, des, w)
                pool.update(pl)
                for c, x in f.items():
                    out[c][r] = x
    return out


def as_quotas(fair):
    out = np.zeros(len(fair), dtype=T.queue_quota_dt)
    out["deserved"] = np.array(fair, dtype=np.uint64).reshape(len(fair), 3)
    return out


def random_weights(rng, n):
    """mostly small weights, some 0, some up to 2^32 - 1"""
    w = np.zeros(n, dtype=T.queue_weight_dt)
    for q in range(n):
        for r in range(3):
            x = rng.random()
            w["over_quota"][q, r] = 0 if x < 0.12 else int(rng.integers(1, 1 << 32)) if x > 0.9 else int(rng.integers(1, 6))
    return w


def fair_share_snapshot(seed, pref=False):
    """fair_share_cases.random_snapshot plus random weights -> (nodes, n_levels, tables, queues, gang_queue, quotas, weights)"""
    from fair_share_cases import random_snapshot
    nodes, L, tables, qs, gq, quotas = random_snapshot(seed, pref=pref)
    return nodes, L, tables, qs, gq, quotas, random_weights(np.random.default_rng(seed + 991), len(qs))


def reclaim_snapshot(seed, pref=False):
    """reclaim_queue_cases.random_snapshot plus random weights -> (nodes, n_levels, tables, queues, gang_queue, quotas, running,
    holdings, running_queue, weights)"""
    from reclaim_queue_cases import random_snapshot
    case = random_snapshot(seed, pref=pref)
    return (*case, random_weights(np.random.default_rng(seed + 991), len(case[3])))


def tree_snapshot(seed):
    """a random queue tree of depth 1-4 for the fair shares alone: zero and unlimited quotas and limits, weights up to 2^32 - 1,
    loads and node tables whose capacity passes 2^40, gated gangs, surplus pods -> (nodes, tables, queues, gang_queue, quotas,
    weights)"""
    rng = np.random.default_rng(seed)
    big = rng.random() < 0.5
    n = int(rng.integers(1, 300))
    nodes = nodes_flat(n)
    if big:
        nodes["free_cpu_milli"] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
        nodes["free_mem_mib"] = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    nodes["free_gpu"] = rng.integers(0, 9, n)
    nodes["flags"][rng.random(n) < 0.1] = 0   # cordoned: not counted
    parents = [None] * int(rng.integers(1, 5))
    frontier = list(range(len(parents)))
    for _ in range(int(rng.integers(0, 4))):
        nxt = []
        for p in frontier:
            for _ in range(int(rng.integers(0, 4))):
                parents.append(p); nxt.append(len(parents) - 1)
        frontier = nxt
    NQ = len(parents)
    scale = (1 << 44) if big else 64

    def amount(r):
        return int(rng.integers(0, scale)) * (1000, 1024, 1)[r]

    rows = []
    for q in range(NQ):
        lim = tuple(None if rng.random() < 0.6 else (0 if rng.random() < 0.1 else amount(r)) for r in range(3))
        used = tuple(amount(r) if rng.random() < 0.7 else 0 for r in range(3))
        rows.append((parents[q], lim, used))
    qs = make_queues(rows)
    quotas = make_quotas([tuple(None if rng.random() < 0.25 else (0 if rng.random() < 0.15 else amount(r)) for r in range(3))
                          for _ in range(NQ)])
    b = T.GangTableBuilder()
    gq = []
    for _ in range(int(rng.integers(1, 40))):
        cl = [dict(gpu=int(rng.integers(0, 9)), cpu=int(rng.integers(0, 1 << 31)) if big else int(rng.integers(0, 8000)),
                   mem=int(rng.integers(0, 1 << 31)) if big else int(rng.integers(0, 65536)), min=int(rng.integers(1, 4)))
              for _ in range(int(rng.integers(1, 3)))]
        for x in cl:
            if rng.random() < 0.3:
                x["replicas"] = x["min"] + int(rng.integers(1, 5))
        b.add_gang([(None, cl)], priority=int(rng.integers(0, 4)))
        gq.append(NONE if rng.random() < 0.1 else int(rng.integers(0, NQ)))
    gangs, cliques, scopes = b.build()
    if len(gangs):
        gangs["flags"][rng.random(len(gangs)) < 0.15] |= T.GANG_GATED
    return nodes, (gangs, cliques, scopes), qs, np.array(gq, np.uint32), quotas, random_weights(rng, NQ)


# ---- hand cases ------------------------------------------------------------------------------------------------------------------

def _one(b, gpu, prio):
    return b.add_gang([(None, [dict(gpu=gpu, min=1)])], priority=prio)


def split_three_to_one():
    """six 8-GPU nodes; team-a (deserved 8 GPUs, weight 3) and team-b (deserved 8, weight 1) each run 8 GPUs on a node of their own
    and submit four 8-GPU gangs, team-b's at the higher priority.  Fair shares 32 / 16: the fair-share order admits three of
    team-a's gangs and one of team-b's (two and two without weights).
    -> (nodes, n_levels, tables, queues, gang_queue, quotas, weights)"""
    nodes = nodes_flat(6)
    nodes["free_gpu"][:2] = 0
    b = T.GangTableBuilder()
    for p in (0, 0, 0, 0, 5, 5, 5, 5):
        _one(b, 8, p)
    qs = make_queues([(None, (None, None, None), (0, 0, 8)), (None, (None, None, None), (0, 0, 8))])
    return (nodes, 2, b.build(), qs, np.array([0] * 4 + [1] * 4, np.uint32), make_quotas([(None, None, 8)] * 2),
            make_weights([(1, 1, 3), (1, 1, 1)]))


def reclaim_beyond_quota():
    """four full 8-GPU nodes; team-a runs 8 GPUs, team-b 24 in three gangs, both deserve 8 with weights 3 and 1, and team-a submits
    two 8-GPU gangs.  Fair shares 20 / 12: the reclaim pass admits one of team-a's gangs with one team-b victim (none without
    weights: team-a is at its quota).
    -> (nodes, n_levels, tables, queues, gang_queue, quotas, running, holdings, running_queue, weights)"""
    UL = (None, None, None)
    case = _case(4, [0, 0, 0, 0], [[0], [1], [2], [3]], [0, 1, 1, 1], [None, None], [UL, UL], [(None, None, 8)] * 2,
                 [(8, 0), (8, 0)], [0, 0])
    return (*case, make_weights([(1, 1, 3), (1, 1, 1)]))
