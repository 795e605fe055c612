"""Reclaim within queue limits (grove_run_cycle_preempt_queues, include/grove_place.h "reclaim within queue limits") restated over
the sequential oracle, and the scenarios the oracle property tests and the GPU parity tests share.

The ordinary pass is queue_cases.run_cycle_queues.  The reclaim pass then takes the gangs it left REJECTED one at a time, in order
rank, while E(p) (the standing running gangs of a priority below p) is non-empty.  A member's gate and surplus caps come from
queue_cases.decide over load' (the loads without what the gangs of E(p) hold); a gang that passes is one oracle call over the node
view (free + what E(p) holds) with its anchor pinned and its cliques' replicas set to MinReplicas + s_q.  Victims are chosen here:
node by node (the reclaim pass's rule), then queue by queue of its chain, leaf first."""
import numpy as np

from grove_b200 import synth, tables as T
from queue_cases import NONE, REQ, UNL, chain, decide, loads, make_queues, nodes_flat, run_cycle_queues
from reuse_cases import _with_free, free_table, hold_table

NODE_STEP, QUEUE_STEP = 0, 1


def usage_of(running, holdings):
    """[R][3] Python ints: what each running gang holds, summed over its holdings (cpu, mem, gpu)"""
    out = []
    for r in range(len(running)):
        h = holdings[int(running["holding_off"][r]): int(running["holding_off"][r]) + int(running["n_holdings"][r])]
        out.append([int(h["cpu_milli"].astype(np.int64).sum()), int(h["mem_mib"].astype(np.int64).sum()), int(h["gpu"].astype(np.int64).sum())])
    return out


def _subtree_loads(queues, own):
    q = queues.copy()
    q["used"] = np.asarray(own, dtype=np.uint64).reshape(len(queues), 3) if len(queues) else q["used"]
    return loads(q)


def run_cycle_preempt_queues(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue, running, holdings, running_queue):
    """-> dict(placements, status, scope_status, nodes_after, victims, steps, loads_after, perm) of the cycle as its definition
    reads; steps[i] says which step (NODE_STEP, QUEUE_STEP) chose victims[i], loads_after the queue loads the cycle leaves"""
    queues = np.asarray(queues, dtype=T.queue_dt)
    gang_queue = np.asarray(gang_queue, dtype=np.uint32)
    running_queue = np.asarray(running_queue, dtype=np.uint32)
    base = run_cycle_queues(oracle, nodes, n_levels, gangs, cliques, scopes, queues, gang_queue)
    G, N, R, NQ = len(gangs), len(nodes), len(running), len(queues)
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
    victims, steps = [], []

    def evict(v, g, step):
        nonlocal F
        gone[v] = True
        F = F + H[v]
        if running_queue[v] != NONE:
            for k in range(3):
                own[int(running_queue[v])][k] -= use_r[v][k]
        victims.append((v, g)); steps.append(step)

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
        view = F + sum(H[x] for x in elig)
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
            while not (F[n] >= use[n]).all():
                v = min((x for x in on_node.get(n, []) if not gone[x] and prio[x] < p), key=lambda x: (prio[x], -x))
                evict(v, g, NODE_STEP)
            F[n] -= use[n]
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
                    evict(v, g, QUEUE_STEP)
        pl["clique"] += co
        per_gang[g] = pl
        st = out["status"][0].copy()
        flags = T.STATUS_PREEMPTOR
        if caps is not None and any(s < int(c["replicas"]) - int(c["min_replicas"]) for s, c in zip(caps, cliques[co: co + len(caps)])):
            flags |= T.STATUS_SURPLUS_CAPPED
        st["reserved0"] = flags
        status[g] = st
        sstat[so: so + len(ss)] = out["scope_status"]
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off if status["state"][g] == T.GANG_ADMITTED else status["placement_off"][g]
        if status["state"][g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F),
                victims=np.array(victims, dtype=T.victim_dt) if victims else np.zeros(0, dtype=T.victim_dt),
                steps=steps, loads_after=_subtree_loads(queues, own), perm=perm)


# ---- scenarios -------------------------------------------------------------------------------------------------------------------

def _running(per_node_gpu, prios, nodes_of, gpu=8):
    """running gangs r of priority prios[r] holding `gpu` GPUs on each node of nodes_of[r] -> running, holdings"""
    running = np.zeros(len(prios), dtype=T.running_dt)
    hold = []
    for r, (p, ns) in enumerate(zip(prios, nodes_of)):
        running["priority"][r] = p; running["holding_off"][r] = len(hold); running["n_holdings"][r] = len(ns)
        hold += [(n, 1000, 1000, gpu, 1) for n in ns]
    return running, np.array(hold, dtype=T.holding_dt) if hold else np.zeros(0, dtype=T.holding_dt)


def _take(nodes, running, holdings):
    """the free table once the running gangs' holdings are taken off"""
    nodes = nodes.copy()
    for h in holdings:
        n = int(h["node"])
        nodes["free_cpu_milli"][n] -= h["cpu_milli"]; nodes["free_mem_mib"][n] -= h["mem_mib"]
        nodes["free_gpu"][n] -= h["gpu"]; nodes["free_pods"][n] -= h["pods"]
    return nodes


def hand_cases():
    """name -> (nodes, n_levels, tables, queues, gang_queue, running, holdings, running_queue): one case per rule"""
    def team_a():                # team-a at its 16-GPU limit with two low-priority gangs; a high-priority one arrives
        nodes = nodes_flat(6)
        running, holdings = _running(8, [0, 0], [[0], [1]])
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, cpu=1000, mem=1000, min=1)])], priority=5)
        qs = make_queues([(None, (None, None, 16), (2000, 2000, 16))])
        return _take(nodes, running, holdings), 2, b.build(), qs, np.zeros(1, np.uint32), running, holdings, np.zeros(2, np.uint32)

    def sibling_victim():        # a 24-GPU parent over two children: the room comes from the sibling's low-priority gang
        nodes = nodes_flat(6)
        running, holdings = _running(8, [1, 0, 3], [[0], [1], [2]])
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, cpu=1000, mem=1000, min=1)])], priority=2, level=0)
        qs = make_queues([(None, (None, None, 24), (0, 0, 0)), (0, (None, None, 16), (1000, 1000, 8)),
                          (0, (None, None, 16), (2000, 2000, 16))])
        return _take(nodes, running, holdings), 2, b.build(), qs, np.array([1], np.uint32), running, holdings, np.array([1, 2, 2], np.uint32)

    def other_queue_spared():    # a lower-priority gang of another queue frees no room in this one: it keeps running
        nodes = nodes_flat(6)
        running, holdings = _running(8, [0, 7], [[0], [1]])
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, cpu=1000, mem=1000, min=1)])], priority=5)
        qs = make_queues([(None, (None, None, 8), (1000, 1000, 8)), (None, (None, None, None), (1000, 1000, 8))])
        return _take(nodes, running, holdings), 2, b.build(), qs, np.array([0], np.uint32), running, holdings, np.array([1, 0], np.uint32)

    def victim_order():          # the lowest priority first, then the highest index; a gang without GPUs frees no GPU room
        nodes = nodes_flat(8)
        running = np.zeros(4, dtype=T.running_dt)
        running["priority"] = [1, 0, 0, 0]; running["holding_off"] = [0, 1, 2, 3]; running["n_holdings"] = 1
        holdings = np.array([(0, 1000, 1000, 4, 1), (1, 1000, 1000, 4, 1), (2, 1000, 1000, 4, 1), (3, 8000, 1000, 0, 1)], dtype=T.holding_dt)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=6, cpu=1000, mem=1000, min=1)])], priority=3)
        qs = make_queues([(None, (None, None, 12), (11000, 4000, 12))])
        return _take(nodes, running, holdings), 2, b.build(), qs, np.zeros(1, np.uint32), running, holdings, np.zeros(4, np.uint32)

    def surplus_capped():        # the reclaim pass admits it with only the best-effort pods its queue has room for
        nodes = nodes_flat(6)
        running, holdings = _running(8, [0], [[0]])
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=4, cpu=1000, mem=1000, min=1, replicas=4)])], priority=2)
        qs = make_queues([(None, (None, None, 12), (1000, 1000, 12))])   # (4 GPUs of it not handed in)
        return _take(nodes, running, holdings), 2, b.build(), qs, np.zeros(1, np.uint32), running, holdings, np.zeros(1, np.uint32)

    def no_queue_preemptor():    # a preemptor without a queue: the node step alone, as the reclaim pass
        nodes = nodes_flat(2)
        running, holdings = _running(8, [0, 0], [[0], [1]])
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=8, cpu=1000, mem=1000, min=1)])], priority=5)
        qs = make_queues([(None, (None, None, 16), (2000, 2000, 16))])
        return _take(nodes, running, holdings), 2, b.build(), qs, np.array([NONE], np.uint32), running, holdings, np.zeros(2, np.uint32)

    def runs_out():              # E(p) runs out part-way through a class: the later gangs stay as the ordinary pass left them
        nodes = nodes_flat(4)
        running, holdings = _running(8, [0], [[0]])
        b = T.GangTableBuilder()
        for _ in range(3):
            b.add_gang([(None, [dict(gpu=8, cpu=1000, mem=1000, min=1)])], priority=4)
        qs = make_queues([(None, (None, None, 8), (1000, 1000, 8))])
        return _take(nodes, running, holdings), 2, b.build(), qs, np.zeros(3, np.uint32), running, holdings, np.zeros(1, np.uint32)

    def starts_over():           # the queue already holds more than its limit (some of it not evictable)
        nodes = nodes_flat(6)
        running, holdings = _running(8, [0, 0], [[0], [1]])
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=4, cpu=1000, mem=1000, min=1)])], priority=5)
        b.add_gang([(None, [dict(gpu=8, cpu=1000, mem=1000, min=1)])], priority=5)
        qs = make_queues([(None, (None, None, 12), (2000, 2000, 24))])
        return _take(nodes, running, holdings), 2, b.build(), qs, np.zeros(2, np.uint32), running, holdings, np.zeros(2, np.uint32)

    return {"team_a": team_a, "sibling_victim": sibling_victim, "other_queue_spared": other_queue_spared,
            "victim_order": victim_order, "surplus_capped": surplus_capped, "no_queue_preemptor": no_queue_preemptor,
            "runs_out": runs_out, "starts_over": starts_over}


def running_layout(oracle, nodes, n_levels, tables, queues, gang_queue, seed):
    """synth.queue_running over the queue cycle restated: -> nodes (free now), tables, queues, gang_queue, running, holdings,
    running_queue"""
    first = run_cycle_queues(oracle, nodes, n_levels, *tables, queues, gang_queue)
    t2, q2, gq2, running, holdings, rq = synth.queue_running(tables, queues, gang_queue, first["placements"], first["status"], seed)
    return first["nodes_after"], t2, q2, gq2, running, holdings, rq
