"""Queue limits (grove_set_queues, include/grove_place.h "queue limits") restated over the sequential oracle, and the scenarios
the oracle property tests and the GPU parity tests share.

The restatement walks the cycle's order (priority desc, submission index asc) and hands the oracle one piece at a time: a run of
gangs that belong to no queue is one ordinary oracle cycle over the free table F, a member is decided here.  Its gate and its
surplus caps come from the headroom of its chain, in Python integers; an admitted one is one oracle call with its anchor pinned
and its cliques' replicas set to MinReplicas + s_q, and its usage U is read from that call's placements.  Base gating across
pieces is decided here, so every gang meets exactly the state the definition gives it."""
import numpy as np

from grove_b200 import tables as T
from reuse_cases import free_table, _with_free

UNL = T.QUEUE_UNLIMITED
NONE = T.NONE_U32
REQ = ("req_cpu_milli", "req_mem_mib", "req_gpu")


def make_queues(rows):
    """rows: (parent or None, (cpu, mem, gpu) limits with None = unlimited, (cpu, mem, gpu) used) -> queue_dt array"""
    out = np.zeros(len(rows), dtype=T.queue_dt)
    for i, (parent, limit, used) in enumerate(rows):
        out["parent"][i] = NONE if parent is None else parent
        out["limit"][i] = [UNL if x is None else x for x in limit]
        out["used"][i] = used
    return out


def chain(queues, q):
    out = []
    while q != NONE:
        out.append(int(q)); q = int(queues["parent"][q])
    return out


def loads(queues):
    """[n][3] Python ints: own used + every descendant's"""
    ld = [[int(x) for x in queues["used"][q]] for q in range(len(queues))]
    for q in range(len(queues) - 1, -1, -1):
        p = int(queues["parent"][q])
        if p != NONE:
            for r in range(3):
                ld[p][r] += ld[q][r]
    return ld


def r_min(gangs, cliques, g):
    co = int(gangs["clique_off"][g])
    out = [0, 0, 0]
    for q in cliques[co: co + int(gangs["n_cliques"][g])]:
        for r in range(3):
            out[r] += int(q["min_replicas"]) * int(q[REQ[r]])
    return out


def decide(queues, ld, charged, gangs, cliques, g, q):
    """-> (closed, caps s_q per clique) of member g of queue q, given what the admitted members before it charged"""
    fin, H = [False] * 3, [None] * 3
    for Q in chain(queues, q):
        for r in range(3):
            lim = int(queues["limit"][Q][r])
            if lim == UNL:
                continue
            h = lim - ld[Q][r] - charged[Q][r]
            fin[r] = True
            H[r] = h if H[r] is None else min(H[r], h)
    R = r_min(gangs, cliques, g)
    if any(fin[r] and R[r] > 0 and R[r] > H[r] for r in range(3)):
        return True, None
    rem = [H[r] - R[r] if fin[r] else None for r in range(3)]
    caps = []
    co = int(gangs["clique_off"][g])
    for c in cliques[co: co + int(gangs["n_cliques"][g])]:
        s = int(c["replicas"]) - int(c["min_replicas"])
        for r in range(3):
            req = int(c[REQ[r]])
            if fin[r] and req > 0:
                s = min(s, rem[r] // req)
        s = max(s, 0)
        for r in range(3):
            if fin[r]:
                rem[r] -= s * int(c[REQ[r]])
        caps.append(s)
    return False, caps


def run_cycle_queues(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, trace=None):
    """-> dict(placements, status, scope_status, nodes_after, perm) of the queue cycle, as its definition reads.
    trace (a list): gets (gang, closed, caps, U or None) for every member that reached the gate."""
    G, N = len(gangs), len(nodes)
    queues = np.asarray(queues, dtype=T.queue_dt)
    gang_queue = np.asarray(gang_queue, dtype=np.uint32)
    perm = oracle.topology(nodes, n_levels)[0]
    ld = loads(queues)
    charged = [[0, 0, 0] for _ in range(len(queues))]
    F = free_table(nodes)
    order = sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i))
    pieces, run = [], []
    for g in order:
        if gang_queue[g] == NONE:
            run.append(g)
        else:
            if run:
                pieces.append(run); run = []
            pieces.append([g])
    if run:
        pieces.append(run)
    status = np.zeros(G, dtype=T.status_dt)
    status["level"] = T.LEVEL_NONE; status["domain_node"] = T.NONE_U32
    sstat = np.zeros(len(scopes), dtype=T.scope_status_dt)
    sstat["level"] = T.LEVEL_NONE; sstat["domain_node"] = T.NONE_U32
    state = np.zeros(G, dtype=np.uint8)
    flags = np.zeros(G, dtype=np.uint16)
    per_gang = {}
    for piece in pieces:
        ids = []
        for g in sorted(piece):   # submission order inside a piece: the oracle's order is then the cycle's
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
                sg["anchor_node"][k] = perm[oracle._fmix32(g) % N]
            sg["clique_off"][k] = sum(len(x) for x in sq); sg["scope_off"][k] = sum(len(x) for x in ss)
            co, so = int(gangs["clique_off"][g]), int(gangs["scope_off"][g])
            sq.append(cliques[co: co + int(gangs["n_cliques"][g])].copy()); ss.append(scopes[so: so + int(gangs["n_scopes"][g])])
        sq, ss = np.concatenate(sq), np.concatenate(ss)
        q = int(gang_queue[ids[0]])
        if q == NONE:
            out = oracle.run_cycle(_with_free(nodes, F), n_levels, sg, sq, ss)
        else:
            g = ids[0]
            closed, caps = decide(queues, ld, charged, gangs, cliques, g, q)
            if closed:   # REJECTED without evaluation: the record of a gang that fits nowhere, and nothing changes
                blocked = _with_free(nodes, F)
                blocked["flags"] &= ~np.uint32(T.NODE_SCHEDULABLE)
                out = oracle.run_cycle(blocked, n_levels, sg, sq, ss)
                assert out["status"]["state"][0] == T.GANG_REJECTED
                out["nodes_after"] = _with_free(nodes, F)
                flags[g] |= T.STATUS_OVER_LIMIT
                if trace is not None:
                    trace.append((g, True, None, None))
            else:
                sq["replicas"] = sq["min_replicas"] + np.asarray(caps, dtype=np.uint8)
                out = oracle.run_cycle(_with_free(nodes, F), n_levels, sg, sq, ss)
                U = None
                if out["status"]["state"][0] == T.GANG_ADMITTED:
                    pl = out["placements"][: int(out["status"]["n_pods"][0])]
                    U = [int(sum(int(sq[REQ[r]][int(e["clique"])]) for e in pl)) for r in range(3)]
                    for Q in chain(queues, q):
                        for r in range(3):
                            charged[Q][r] += U[r]
                    extra = (cliques["replicas"].astype(int) - cliques["min_replicas"].astype(int))[int(gangs["clique_off"][g]):][: len(caps)]
                    if any(s < x for s, x in zip(caps, extra)):
                        flags[g] |= T.STATUS_SURPLUS_CAPPED
                if trace is not None:
                    trace.append((g, False, caps, U))
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
        F = free_table(out["nodes_after"])
    status["state"] = state
    status["reserved0"] = flags
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off
        if state[g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F), perm=perm)


def diagnose_queue_cycle(nodes, n_levels, gangs, cliques, scopes, out):
    """grove_diagnose after a queue cycle: the ordinary restatement over the cycle's outputs (the gate never touches the node
    table, so every gang met the table it restates), with all-zero records for the OVER_LIMIT gangs and their cliques"""
    import diagnose_cases as D
    gd, qd = D.diagnose(nodes, n_levels, gangs, cliques, scopes, cliques["min_replicas"], out)
    for x in np.nonzero(out["status"]["reserved0"] & T.STATUS_OVER_LIMIT)[0]:
        gd[x] = 0
        co = int(gangs["clique_off"][x])
        qd[co: co + int(gangs["n_cliques"][x])] = 0
    return gd, qd


def demand(cliques):
    """[3] Python ints: what every clique asks for with all its replicas"""
    return [int((cliques["replicas"].astype(np.int64) * cliques[REQ[r]].astype(np.int64)).sum()) for r in range(3)]


def assign_queues(rng, gangs, cliques, share=0.8):
    """a random queue tree of depth 1-3 whose limits are tight, loose, unlimited or already exceeded, and a queue for most
    gangs -> (queues, gang_queue)"""
    D = demand(cliques)
    rows = []
    n_roots = int(rng.integers(1, 3))
    depth = int(rng.integers(1, 4))
    level = [None] * n_roots
    frontier = list(range(n_roots))
    for _ in range(n_roots):
        rows.append(None)
    for _ in range(depth - 1):
        nxt = []
        for p in frontier:
            for _ in range(int(rng.integers(1, 3))):
                rows.append(p); nxt.append(len(rows) - 1)
        frontier = nxt
    out = []
    for i, parent in enumerate(rows):
        limit, used = [], []
        for r in range(3):
            kind = rng.choice(["tight", "loose", "unlimited", "exceeded"], p=[0.45, 0.2, 0.2, 0.15])
            total = max(D[r], 1)
            if kind == "unlimited":
                limit.append(None); used.append(int(rng.integers(0, total // 4 + 1)))
            elif kind == "exceeded":
                lim = int(rng.integers(0, total // 4 + 1))
                limit.append(lim); used.append(lim + int(rng.integers(1, total // 8 + 2)))
            else:
                f = rng.uniform(0.2, 0.7) if kind == "tight" else rng.uniform(0.8, 1.5)
                limit.append(int(total * f)); used.append(int(rng.integers(0, max(int(total * f) // 5, 1))))
        out.append((parent, tuple(limit), tuple(used)))
    queues = make_queues(out)
    gq = np.full(len(gangs), NONE, dtype=np.uint32)
    for g in range(len(gangs)):
        if rng.random() < share:
            gq[g] = int(rng.integers(0, len(queues)))
    return queues, gq


def nodes_flat(n, gpu=8, cpu=64000, mem=512000, per_block=None):
    """n identical schedulable nodes in blocks of `per_block` (two levels: block, host)"""
    nodes = T.make_nodes(n)
    pb = per_block or n
    nodes["dom"][:, 0] = np.arange(n) // pb
    nodes["dom"][:, 1] = np.arange(n)
    nodes["free_cpu_milli"] = cpu; nodes["free_mem_mib"] = mem; nodes["free_gpu"] = gpu; nodes["free_pods"] = 110
    nodes["flags"] = T.NODE_SCHEDULABLE
    return nodes


def hand_cases():
    """name -> (nodes, n_levels, tables, queues, gang_queue): one case per rule of the definition"""
    def leaf_limit():        # team-a may hold 16 GPUs: two of three 8-GPU gangs
        nodes = nodes_flat(4)
        b = T.GangTableBuilder()
        for _ in range(3):
            b.add_gang([(None, [dict(gpu=8, min=1)])])
        return nodes, 2, b.build(), make_queues([(None, (None, None, 16), (0, 0, 0))]), np.zeros(3, np.uint32)

    def shared_parent():     # two children under a 24-GPU parent; each child alone would take 16
        nodes = nodes_flat(8)
        b = T.GangTableBuilder()
        for i in range(6):
            b.add_gang([(None, [dict(gpu=8, min=1)])], priority=i % 2)
        qs = make_queues([(None, (None, None, 24), (0, 0, 0)), (0, (None, None, 16), (0, 0, 0)), (0, (None, None, 16), (0, 0, 0))])
        return nodes, 2, b.build(), qs, np.array([1, 2, 1, 2, 1, 2], np.uint32)

    def over_limit_start():  # the queue already holds more than its limit: nothing is admitted
        nodes = nodes_flat(4)
        b = T.GangTableBuilder()
        for _ in range(3):
            b.add_gang([(None, [dict(gpu=1, cpu=1000, min=1)])])
        return nodes, 2, b.build(), make_queues([(None, (None, None, 8), (0, 0, 10))]), np.zeros(3, np.uint32)

    def zero_gpu_gang():     # over its GPU limit, a CPU-only gang still gets in; a GPU gang does not
        nodes = nodes_flat(4)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=1, min=1)])])
        b.add_gang([(None, [dict(cpu=2000, min=2)])])
        return nodes, 2, b.build(), make_queues([(None, (None, None, 4), (0, 0, 6))]), np.zeros(2, np.uint32)

    def surplus_two_cliques():   # 10 GPUs of headroom: MinReplicas 2 + 2 GPUs, 6 left: clique 0 takes 3 of its 4, clique 1 none
        nodes = nodes_flat(4)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=2, min=1, replicas=5), dict(gpu=1, min=2, replicas=6)])])
        return nodes, 2, b.build(), make_queues([(None, (None, None, 10), (0, 0, 0))]), np.zeros(1, np.uint32)

    def nonmember_takes():   # the gated-out member's node goes to the non-member after it
        nodes = nodes_flat(1)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, min=1)])], priority=1)
        b.add_gang([(None, [dict(gpu=8, min=1)])], priority=0)
        return nodes, 2, b.build(), make_queues([(None, (None, None, 4), (0, 0, 0))]), np.array([0, NONE], np.uint32)

    def scaled_base_gated():   # the base gang is gated out by its queue: its scaled gang comes back BASE_REJECTED
        nodes = nodes_flat(4)
        b = T.GangTableBuilder()
        x = b.add_gang([(None, [dict(gpu=8, min=1)])], priority=1)
        b.add_gang([(None, [dict(gpu=8, min=1)])], priority=1, base=x)
        return nodes, 2, b.build(), make_queues([(None, (None, None, 4), (0, 0, 0))]), np.array([0, NONE], np.uint32)

    def cpu_and_mem():       # limits on cpu and memory, a three-level chain
        nodes = nodes_flat(6, per_block=3)
        b = T.GangTableBuilder()
        for i in range(8):
            b.add_gang([(None, [dict(cpu=4000, mem=8000, min=2, replicas=4)])], level=0 if i % 2 else None, priority=i % 3)
        qs = make_queues([(None, (40000, None, None), (0, 0, 0)), (0, (None, 70000, None), (4000, 0, 0)),
                          (1, (20000, None, None), (0, 8000, 0))])
        return nodes, 2, b.build(), qs, np.array([2, 1, 0, 2, 1, 0, 2, NONE], np.uint32)

    return {"leaf_limit": leaf_limit, "shared_parent": shared_parent, "over_limit_start": over_limit_start,
            "zero_gpu_gang": zero_gpu_gang, "surplus_two_cliques": surplus_two_cliques, "nonmember_takes": nonmember_takes,
            "scaled_base_gated": scaled_base_gated, "cpu_and_mem": cpu_and_mem}
