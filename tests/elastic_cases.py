"""Elastic reclaim (grove_run_cycle_preempt_elastic, include/grove_place.h "elastic reclaim") restated over the sequential oracle, and
the scenarios the oracle property tests and the GPU parity tests share.

The restatement reads as the definition does, one gang at a time, beside oracle_py.run_cycle_preempt: the ordinary oracle cycle,
then every priority class of the gangs it rejected, descending, while E(p) stands.  Pass 1 evaluates each member with one oracle
call against F + the untaken surplus pods of E(p); pass 2 each member pass 1 did not admit against F + what the standing gangs of
E(p) still hold.  The node step takes surplus pods before it evicts any gang whole.  Small cases only (an oracle cycle per gang)."""
import numpy as np

from grove_b200 import synth, tables as T
from preempt_cases import holdings_of
from reuse_cases import _with_free, free_table, hold_table


def surplus_of(placements, status, gangs, cliques):
    """T.surplus_pod_dt: the surplus pods of the gangs a cycle admitted, running gangs numbered as holdings_of numbers them.  The
    r-th placement of a clique binds its r-th PodReference, so a gang gives up its pods at r >= MinReplicas highest r first,
    clique by clique."""
    out, r = [], 0
    for g in range(len(gangs)):
        if status["state"][g] != T.GANG_ADMITTED:
            continue
        pl = placements[status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]]
        co = int(gangs["clique_off"][g])
        for q in range(co, co + int(gangs["n_cliques"][g])):
            mine = [int(e["node"]) for e in pl if int(e["clique"]) == q]
            c = cliques[q]
            for k in range(len(mine) - 1, int(c["min_replicas"]) - 1, -1):
                out.append((r, mine[k], int(c["req_cpu_milli"]), int(c["req_mem_mib"]), int(c["req_gpu"]), 0))
        r += 1
    return np.array(out, dtype=T.surplus_pod_dt) if out else np.zeros(0, dtype=T.surplus_pod_dt)


def run_cycle_preempt_elastic(oracle, nodes, n_levels, gangs, cliques, scopes, running, holdings, surplus):
    """-> dict(placements, status, scope_status, nodes_after, victims, surplus_victims, perm) of the cycle as its definition
    reads"""
    base = oracle.run_cycle(nodes, n_levels, gangs, cliques, scopes)
    G, N, R = len(gangs), len(nodes), len(running)
    status = base["status"].copy()
    sstat = base["scope_status"].copy()
    per_gang = {g: base["placements"][status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]].copy()
                for g in range(G) if status["state"][g] == T.GANG_ADMITTED}
    F = free_table(base["nodes_after"])
    perm = base["perm"]
    H = [hold_table(N, running, holdings, r) for r in range(R)]
    prio = [int(running["priority"][r]) for r in range(R)]
    pod_run = [int(x["running"]) for x in surplus]
    pod_node = [int(x["node"]) for x in surplus]
    pod_use = [np.array([int(x["cpu_milli"]), int(x["mem_mib"]), int(x["gpu"]), 1], dtype=np.int64) for x in surplus]
    gone = np.zeros(R, dtype=bool)
    taken = np.zeros(len(surplus), dtype=bool)
    on_node = {}
    for r in range(R):
        for h in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
            on_node.setdefault(int(h["node"]), []).append(r)
    victims, surplus_victims = [], []

    def still_holds(r):   # [N, 4]: what running gang r holds once its taken pods are off
        h = H[r].copy()
        for i in range(len(surplus)):
            if taken[i] and pod_run[i] == r:
                h[pod_node[i]] -= pod_use[i]
        return h

    def takeable(i, p):
        return not taken[i] and not gone[pod_run[i]] and prio[pod_run[i]] < p

    def evaluate(g, view):
        sg = gangs[g: g + 1].copy()
        co, so = int(sg["clique_off"][0]), int(sg["scope_off"][0])
        sq = cliques[co: co + int(sg["n_cliques"][0])].copy()
        ss = scopes[so: so + int(sg["n_scopes"][0])].copy()
        if sg["anchor_node"][0] == T.NONE_U32:
            sg["anchor_node"][0] = perm[oracle._fmix32(g) % N]   # the anchor the ordinary pass derived for this gang
        sg["base_gang"][0] = T.NONE_U32; sg["clique_off"][0] = 0; sg["scope_off"][0] = 0
        out = oracle.run_cycle(_with_free(nodes, view), n_levels, sg, sq, ss)
        return out if out["status"]["state"][0] == T.GANG_ADMITTED else None, co, so, sq

    def admit(g, p, out, co, so, sq, flag, surplus_only):
        pl = out["placements"].copy()
        use, order = {}, []
        for e in pl:
            n, q = int(e["node"]), sq[int(e["clique"])]
            if n not in use:
                use[n] = np.zeros(4, dtype=np.int64); order.append(n)
            use[n] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
        for n in order:   # the node step
            need = use[n]
            while not (F[n] >= need).all():
                here = [i for i in range(len(surplus)) if pod_node[i] == n and takeable(i, p)]
                if (F[n] + sum((pod_use[i] for i in here), np.zeros(4, dtype=np.int64)) >= need).all():
                    while not (F[n] >= need).all():
                        v = min({pod_run[i] for i in here if not taken[i]}, key=lambda x: (prio[x], -x))
                        i = next(i for i in here if not taken[i] and pod_run[i] == v)
                        taken[i] = True
                        F[n] += pod_use[i]
                        surplus_victims.append((i, g))
                    break
                if surplus_only:
                    raise AssertionError("a surplus-only preemptor's node cannot be freed by surplus pods")
                v = min((x for x in on_node.get(n, []) if not gone[x] and prio[x] < p and still_holds(x)[n].any()),
                        key=lambda x: (prio[x], -x))
                F[:] += still_holds(v)
                gone[v] = True
                victims.append((v, g))
            F[n] -= need
        pl["clique"] += co
        per_gang[g] = pl
        st = out["status"][0].copy()
        st["reserved0"] = flag
        status[g] = st
        sstat[so: so + int(gangs["n_scopes"][g])] = out["scope_status"]

    classes = sorted({int(gangs["priority"][g]) for g in range(G) if status["state"][g] == T.GANG_REJECTED}, reverse=True)
    for p in classes:
        E = lambda: [r for r in range(R) if not gone[r] and prio[r] < p]   # noqa: E731
        if not E():
            break
        members = [g for g in range(G) if status["state"][g] == T.GANG_REJECTED and int(gangs["priority"][g]) == p]
        if any(takeable(i, p) for i in range(len(surplus))):   # pass 1: surplus pods only
            for g in members:
                up = [i for i in range(len(surplus)) if takeable(i, p)]
                if not up:
                    continue
                view = F.copy()
                for i in up:
                    view[pod_node[i]] += pod_use[i]
                out, co, so, sq = evaluate(g, view)
                if out is not None:
                    admit(g, p, out, co, so, sq, T.STATUS_PREEMPTOR | T.STATUS_SURPLUS_ONLY, True)
        for g in members:   # pass 2: whole gangs, for the members pass 1 did not admit
            if status["state"][g] != T.GANG_REJECTED:
                continue
            elig = E()
            if not elig:
                continue
            view = F + sum(still_holds(r) for r in elig)
            out, co, so, sq = evaluate(g, view)
            if out is not None:
                admit(g, p, out, co, so, sq, T.STATUS_PREEMPTOR, False)
    merged, off = [], 0
    for g in range(G):
        if status["state"][g] == T.GANG_ADMITTED:
            status["placement_off"][g] = off
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(base["nodes_after"], F),
                victims=np.array(victims, dtype=T.victim_dt) if victims else np.zeros(0, dtype=T.victim_dt),
                surplus_victims=(np.array(surplus_victims, dtype=T.surplus_victim_dt) if surplus_victims
                                 else np.zeros(0, dtype=T.surplus_victim_dt)), perm=perm)


def elastic_cluster(oracle, seed, n=1260, g_running=400, g_pending=200, boost=2, used_pct=80, share=0.5):
    """preempt_cases.churned_cluster with surplus: a `share` of the running submission's worker cliques ask for 1-3 pods above
    MinReplicas (synth.c4_surplus), which the first oracle cycle places best effort.
    -> nodes (free now), n_levels, pending tables, running, holdings, surplus"""
    first = synth.config_c4(n=n, g=g_running, seed=seed, max_used_pct=used_pct)
    g1, c1, s1 = first["tables"]
    c1 = synth.c4_surplus(c1, share=share, seed=seed)
    ref = oracle.run_cycle(first["nodes"], first["n_levels"], g1, c1, s1, threads=2)
    running, holdings = holdings_of(ref["placements"], ref["status"], g1, c1)
    surplus = surplus_of(ref["placements"], ref["status"], g1, c1)
    second = synth.config_c4(n=n, g=g_pending, seed=seed + 7919, max_used_pct=used_pct)
    g2, c2, s2 = (a.copy() for a in second["tables"])
    for i in range(len(g2)):   # a scaled gang keeps its base gang's priority (podgang/podgang.go:158)
        b = int(g2["base_gang"][i])
        root = i if b == T.NONE_U32 else b
        if root % 2 == 0:
            g2["priority"][i] += boost
    return ref["nodes_after"], first["n_levels"], (g2, c2, s2), running, holdings, surplus


def hand_case(p_gpu=4, b_priority=0):
    """Two 8-GPU nodes n0 and n1 of one block, nothing free.  Running gang A (priority 0) holds n0 with one 8-GPU pod, MinReplicas
    1; running gang B (priority b_priority) holds n1 with two 4-GPU pods, MinReplicas 1 and replicas 2, so its pod 1 is surplus.
    The submission is one preemptor P (priority 5) of one p_gpu-GPU pod.  -> nodes, n_levels, tables, running, holdings, surplus"""
    nodes = synth.kwok_nodes(2, [2, 2, 1, 1], gpu=8)
    nodes["free_gpu"] = 0; nodes["free_pods"] = [109, 108]
    running = np.zeros(2, dtype=T.running_dt)
    running["priority"] = [0, b_priority]; running["holding_off"] = [0, 1]; running["n_holdings"] = 1
    holdings = np.array([(0, 0, 0, 8, 1), (1, 0, 0, 8, 2)], dtype=T.holding_dt)
    surplus = np.array([(1, 1, 0, 0, 4, 0)], dtype=T.surplus_pod_dt)
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(gpu=p_gpu, min=1)])], priority=5)
    return nodes, 4, b.build(), running, holdings, surplus
