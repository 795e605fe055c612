"""Reclaim, then preempt (grove_run_cycle_reclaim_preempt_queues, include/grove_place.h "reclaim, then preempt") restated over the
sequential oracle, and the scenarios the oracle property tests and the GPU parity tests share.

The ordinary pass is queue_cases.run_cycle_queues.  The two passes then run one after the other on one state (ordinary_pass): the
reclaim pass as reclaim_queue_cases restates reclaim across queues (classes by ascending share, donor sets from
reclaim_queue_cases.donor_set, queue_cases.decide on load' with the caps, one oracle call per member on the node view), and the
preempt pass as preempt_queue_cases restates reclaim within queue limits (every gang still rejected, one at a time in rank order,
against E(p) and the limits), from the free table, queue loads and standing set the reclaim pass left.  Inputs are those of
reclaim_queue_cases.run_cycle_reclaim_queues; random snapshots are reclaim_queue_cases.random_snapshot."""
import numpy as np

from grove_b200 import tables as T
from preempt_queue_cases import NODE_STEP, QUEUE_STEP, _running, _subtree_loads, _take, usage_of
from queue_cases import NONE, REQ, UNL, chain, decide, make_queues, nodes_flat, run_cycle_queues
from reclaim_queue_cases import UL, _used, _victim_key, caps_of, donor_set, make_quotas, random_snapshot, share, share_less
from reuse_cases import _with_free, free_table, hold_table

__all__ = ["NODE_STEP", "QUEUE_STEP", "run_cycle_reclaim_preempt_queues", "hand_cases", "random_snapshot"]


def run_cycle_reclaim_preempt_queues(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, quotas, running, holdings,
                                     running_queue):
    """-> dict(placements, status, scope_status, nodes_after, victims, steps, loads_after, perm, classes, n_reclaim) of the cycle as
    its definition reads; victims[:n_reclaim] are the reclaim pass's, classes its classes (reclaim_queue_cases)"""
    queues = np.asarray(queues, dtype=T.queue_dt)
    quotas = np.asarray(quotas, dtype=T.queue_quota_dt)
    gang_queue = np.asarray(gang_queue, dtype=np.uint32)
    running_queue = np.asarray(running_queue, dtype=np.uint32)
    s = ordinary_pass(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, running, holdings)
    classes = reclaim_pass(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, quotas, running_queue, s)
    n_reclaim = len(s["victims"])
    preempt_pass(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, running_queue, s)
    return dict(outputs(nodes, queues, s), classes=classes, n_reclaim=n_reclaim)


def ordinary_pass(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, running, holdings):
    """the queue cycle, and the state the two passes start from and change: dict(status, sstat, per_gang, F (free table), perm,
    H (each running gang's holdings as a table), use_r, prio, own (each queue's own used), gone, on_node, victims, steps)"""
    base = run_cycle_queues(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue)
    G, N, R, NQ = len(gangs), len(nodes), len(running), len(queues)
    status = base["status"].copy()
    per_gang = {g: base["placements"][status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]].copy()
                for g in range(G) if status["state"][g] == T.GANG_ADMITTED}
    own = [[int(x) for x in queues["used"][q]] for q in range(NQ)]
    for g in range(G):   # the ordinary pass's admitted members join their queue
        if status["state"][g] == T.GANG_ADMITTED and gang_queue[g] != NONE:
            for e in per_gang[g]:
                for k in range(3):
                    own[int(gang_queue[g])][k] += int(cliques[REQ[k]][int(e["clique"])])
    on_node = {}
    for r in range(R):
        for h in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
            on_node.setdefault(int(h["node"]), []).append(r)
    return dict(status=status, sstat=base["scope_status"].copy(), per_gang=per_gang, F=free_table(base["nodes_after"]),
                perm=base["perm"], H=[hold_table(N, running, holdings, r) for r in range(R)], use_r=usage_of(running, holdings),
                prio=[int(running["priority"][r]) for r in range(R)], own=own, gone=np.zeros(R, dtype=bool), on_node=on_node,
                victims=[], steps=[])


def evict(s, running_queue, v, g, step):
    """running gang v falls for gang g: its holdings return to the free table, its usage leaves its queue"""
    s["gone"][v] = True
    s["F"] = s["F"] + s["H"][v]
    if running_queue[v] != NONE:
        for k in range(3):
            s["own"][int(running_queue[v])][k] -= s["use_r"][v][k]
    s["victims"].append((v, g)); s["steps"].append(step)


def reclaim_pass(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, quotas, running_queue, s):
    """the reclaim pass: steps 2-5 of reclaim across queues (reclaim_queue_cases.run_cycle_reclaim_queues) from state s (ordinary_pass),
    which it changes -> the classes, as that restatement lists them"""
    G, N, R, NQ = len(gangs), len(nodes), len(s["prio"]), len(queues)
    capq = caps_of(queues, quotas)
    status, sstat, per_gang, perm, H, use_r, prio, own, gone, on_node = (
        s[k] for k in ("status", "sstat", "per_gang", "perm", "H", "use_r", "prio", "own", "gone", "on_node"))
    classes = []
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

    def evict_for(v, g, step, cls):
        evict(s, running_queue, v, g, step)
        cls["victims"].append(v)

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
            view = s["F"] + sum((H[x] for x in standing), np.zeros_like(s["F"]))
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
                while not (s["F"][n] >= use[n]).all():
                    v = min((x for x in on_node.get(n, []) if x in E and not gone[x]), key=lambda x: _victim_key(prio, x))
                    evict_for(v, g, NODE_STEP, cls)
                s["F"][n] -= use[n]
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
                    evict_for(v, g, QUEUE_STEP, cls)
            pl["clique"] += co
            per_gang[g] = pl
            st = out["status"][0].copy()
            flags = T.STATUS_RECLAIMER
            if any(s_ < int(c["replicas"]) - int(c["min_replicas"]) for s_, c in zip(caps, cliques[co: co + len(caps)])):
                flags |= T.STATUS_SURPLUS_CAPPED
            st["reserved0"] = flags
            status[g] = st
            sstat[so: so + len(ss)] = out["scope_status"]
        cls["loads_end"] = _subtree_loads(queues, own)
    return classes


def preempt_pass(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, running_queue, s):
    """the preempt pass: steps 2-3 of reclaim within queue limits (preempt_queue_cases.run_cycle_preempt_queues) from state s,
    which it changes"""
    G, N, R, NQ = len(gangs), len(nodes), len(s["prio"]), len(queues)
    status, sstat, per_gang, perm, H, use_r, prio, own, gone, on_node = (
        s[k] for k in ("status", "sstat", "per_gang", "perm", "H", "use_r", "prio", "own", "gone", "on_node"))
    for g in sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i)):
        if status["state"][g] != T.GANG_REJECTED:
            continue
        p = int(gangs["priority"][g])
        elig = [r for r in range(R) if not gone[r] and prio[r] < p]
        if not elig:
            continue
        q = int(gang_queue[g])
        caps = None
        if q != NONE:
            o = [list(x) for x in own]
            for r in elig:
                if running_queue[r] != NONE:
                    for k in range(3):
                        o[int(running_queue[r])][k] -= use_r[r][k]
            closed, caps = decide(queues, _subtree_loads(queues, o), [[0, 0, 0]] * NQ, gangs, cliques, g, q)
            if closed:
                continue
        view = s["F"] + sum(H[x] for x in elig)
        sg = gangs[g: g + 1].copy()
        co, so = int(sg["clique_off"][0]), int(sg["scope_off"][0])
        sq = cliques[co: co + int(sg["n_cliques"][0])].copy()
        ss = scopes[so: so + int(sg["n_scopes"][0])].copy()
        if caps is not None:
            sq["replicas"] = sq["min_replicas"] + np.asarray(caps, dtype=np.uint8)
        if sg["anchor_node"][0] == T.NONE_U32:
            sg["anchor_node"][0] = perm[oracle._fmix32(g) % N]   # the anchor the ordinary pass derived for this gang
        sg["base_gang"][0] = T.NONE_U32; sg["clique_off"][0] = 0; sg["scope_off"][0] = 0
        out = oracle.run_cycle(_with_free(nodes, view), n_levels, sg, sq, ss)
        if out["status"]["state"][0] != T.GANG_ADMITTED:
            continue
        pl = out["placements"].copy()
        use, order, U = {}, [], [0, 0, 0]
        for e in pl:
            n, c = int(e["node"]), sq[int(e["clique"])]
            if n not in use:
                use[n] = np.zeros(4, dtype=np.int64); order.append(n)
            use[n] += [int(c["req_cpu_milli"]), int(c["req_mem_mib"]), int(c["req_gpu"]), 1]
            for k in range(3):
                U[k] += int(c[REQ[k]])
        for n in order:   # (a) the node step
            while not (s["F"][n] >= use[n]).all():
                v = min((x for x in on_node.get(n, []) if not gone[x] and prio[x] < p), key=lambda x: (prio[x], -x))
                evict(s, running_queue, v, g, NODE_STEP)
            s["F"][n] -= use[n]
        if q != NONE:     # (b) the queue step
            for k in range(3):
                own[q][k] += U[k]
            for Q in chain(queues, q):
                while True:
                    ld = _subtree_loads(queues, own)[Q]
                    over = [U[r] > 0 and int(queues["limit"][Q][r]) != UNL and ld[r] > int(queues["limit"][Q][r]) for r in range(3)]
                    if not any(over):
                        break
                    cand = [x for x in range(R) if not gone[x] and prio[x] < p and running_queue[x] != NONE
                            and Q in chain(queues, int(running_queue[x])) and any(over[r] and use_r[x][r] > 0 for r in range(3))]
                    v = min(cand, key=lambda x: (prio[x], -x))
                    evict(s, running_queue, v, g, QUEUE_STEP)
        pl["clique"] += co
        per_gang[g] = pl
        st = out["status"][0].copy()
        flags = T.STATUS_PREEMPTOR
        if caps is not None and any(s_ < int(c["replicas"]) - int(c["min_replicas"]) for s_, c in zip(caps, cliques[co: co + len(caps)])):
            flags |= T.STATUS_SURPLUS_CAPPED
        st["reserved0"] = flags
        status[g] = st
        sstat[so: so + len(ss)] = out["scope_status"]


def outputs(nodes, queues, s):
    """the cycle's outputs from the state its passes left: placements grouped by gang in submission order"""
    status, per_gang = s["status"], s["per_gang"]
    merged, off = [], 0
    for g in range(len(status)):
        status["placement_off"][g] = off if status["state"][g] == T.GANG_ADMITTED else status["placement_off"][g]
        if status["state"][g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=s["sstat"], nodes_after=_with_free(nodes, s["F"]),
                victims=np.array(s["victims"], dtype=T.victim_dt) if s["victims"] else np.zeros(0, dtype=T.victim_dt),
                steps=s["steps"], loads_after=_subtree_loads(queues, s["own"]), perm=s["perm"])


# ---- scenarios -------------------------------------------------------------------------------------------------------------------

def _case(n_nodes, run_prios, run_nodes, run_queue, limits, quotas, subs, gang_queue, pin=None):
    """root queues (limits, quotas) on a full cluster of n_nodes 8-GPU nodes: running gangs of 8 GPUs on the nodes run_nodes[r] in
    run_queue[r], whose used is what they hold; the submission subs = [(gpu, priority)] in gang_queue.  pin = (gang, node): that
    gang fits only on that node (node class 1)."""
    nodes = nodes_flat(n_nodes)
    running, holdings = _running(8, run_prios, run_nodes)
    rq = np.array(run_queue, dtype=np.uint32)
    qs = make_queues([(None, lim, u) for lim, u in zip(limits, _used(running, holdings, rq, len(limits)))])
    b = T.GangTableBuilder()
    for i, (gpu, prio) in enumerate(subs):
        mask = 0x2 if pin is not None and pin[0] == i else 0xFFFF
        b.add_gang([(None, [dict(gpu=gpu, cpu=1000, mem=1000, min=1, class_mask=mask)])], priority=prio)
    if pin is not None:
        nodes["flags"][pin[1]] |= 1 << T.NODE_CLASS_SHIFT
    return (_take(nodes, running, holdings), 2, b.build(), qs, np.array(gang_queue, np.uint32), make_quotas(quotas), running, holdings,
            rq)


G8 = (None, None, 8)


def hand_cases():
    """name -> (nodes, n_levels, tables, queues, gang_queue, quotas, running, holdings, running_queue): one case per interaction"""
    return {
        # queues team-a (0), team-b (1), team-c (2) on three full 8-GPU nodes.  team-b (quota 8) runs b-0 and b-1 at priority 5,
        # team-c (limit 8, quota 8) runs c-low at priority 0.  team-a (quota 8) submits a-0 (priority 0), team-c c-high (priority
        # 9, pinned to c-low's node).  Reclaim admits a-0 with b-1 as victim; preemption admits c-high with c-low as victim.
        "three_teams": lambda: _case(3, [5, 5, 0], [[0], [1], [2]], [1, 1, 2], [UL, UL, G8], [G8, G8, G8], [(8, 0), (8, 9)], [0, 2],
                                     pin=(1, 2)),
        # team-a holds its quota of 8 with a-old (priority 0); its a-new (priority 5) is turned away by its cap in the reclaim
        # pass although team-b (quota 0, b-0 at priority 9) is a donor, and admitted by preemption under its unlimited limit
        "capped_then_preempted": lambda: _case(2, [0, 9], [[0], [1]], [0, 1], [UL, UL], [G8, (None, None, 0)], [(8, 5)], [0]),
        # a gang without a queue: no reclaim class, only the preempt pass considers it
        "no_queue_gang": lambda: _case(2, [0, 0], [[0], [1]], [1, 1], [UL, UL], [G8, UL], [(8, 5)], [NONE]),
        # the reclaim pass evicts b-0, the only running gang below priority 5: E(5) is then empty and x (no queue) stays rejected
        "reclaim_empties_e": lambda: _case(2, [0, 9], [[0], [1]], [1, 2], [UL, UL, UL], [G8, (None, None, 0), UL], [(8, 0), (8, 5)],
                                           [0, NONE]),
        # team-b holds exactly its quota: team-a's class has no donor and is skipped; its a-0 (priority 5) then preempts b-0
        "skipped_class_preempts": lambda: _case(2, [0, 9], [[0], [1]], [1, 2], [UL, UL, UL], [G8, G8, UL], [(8, 5)], [0]),
    }
