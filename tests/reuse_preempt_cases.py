"""Reuse with reclaim (grove_run_cycle_reuse_preempt, include/grove_place.h "reuse with reclaim") restated over the sequential
oracle, and the scenarios the oracle property tests and the GPU parity tests share.

The ordinary pass is reuse_cases.run_cycle_reuse.  The reclaim pass then takes the gangs it left REJECTED one at a time, in order
rank, as oracle_py.run_cycle_preempt does: one oracle call per gang, against the free table plus what the standing running gangs
of a lower priority hold (E(p)), plus the hold of its predecessor when that one stands at or above p.  Victims are chosen node by
node; a hold's leftovers return after the last gang of the class."""
import numpy as np

from grove_b200 import synth, tables as T
from reuse_cases import _with_free, free_table, hold_table, rolling_cluster, run_cycle_reuse


def run_cycle_reuse_preempt(oracle, nodes, n_levels, gangs, cliques, scopes, replaces, running, holdings):
    """-> dict(placements, status, scope_status, nodes_after, victims, released) of the cycle as its definition reads; `released`
    lists the running gangs whose new version was admitted (in the ordinary pass or the reclaim pass)"""
    base = run_cycle_reuse(oracle, nodes, n_levels, gangs, cliques, scopes, replaces, running, holdings)
    G, N, R = len(gangs), len(nodes), len(running)
    status = base["status"].copy()
    sstat = base["scope_status"].copy()
    per_gang = {g: base["placements"][status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]].copy()
                for g in range(G) if status["state"][g] == T.GANG_ADMITTED}
    F = free_table(base["nodes_after"])
    perm = base["perm"]
    H = [hold_table(N, running, holdings, r) for r in range(R)]
    prio = [int(running["priority"][r]) for r in range(R)]
    gone = np.zeros(R, dtype=bool)   # released or evicted
    released = []
    for g in range(G):
        if status["state"][g] == T.GANG_ADMITTED and replaces[g] != T.NONE_U32:
            gone[int(replaces[g])] = True; released.append(int(replaces[g]))
    on_node = {}
    for r in range(R):
        for h in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
            on_node.setdefault(int(h["node"]), []).append(r)
    victims = []
    cls, leftover = None, np.zeros((N, 4), dtype=np.int64)
    for g in sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i)):
        if status["state"][g] != T.GANG_REJECTED:
            continue
        p = int(gangs["priority"][g])
        if p != cls:   # the leftovers of the holds of the class before come back
            F += leftover; leftover[:] = 0; cls = p
        elig = [r for r in range(R) if not gone[r] and prio[r] < p]
        if not elig:
            continue
        r = int(replaces[g]) if replaces[g] != T.NONE_U32 else None
        holds = r is not None and not gone[r] and prio[r] >= p
        view = F + sum(H[x] for x in elig) + (H[r] if holds else 0)
        sg = gangs[g: g + 1].copy()
        co, so = int(sg["clique_off"][0]), int(sg["scope_off"][0])
        sq = cliques[co: co + int(sg["n_cliques"][0])].copy()
        ss = scopes[so: so + int(sg["n_scopes"][0])].copy()
        if sg["anchor_node"][0] == T.NONE_U32:
            sg["anchor_node"][0] = perm[oracle._fmix32(g) % N]   # the anchor the ordinary pass derived for this gang
        sg["base_gang"][0] = T.NONE_U32; sg["clique_off"][0] = 0; sg["scope_off"][0] = 0
        out = oracle.run_cycle(_with_free(nodes, view), n_levels, sg, sq, ss)
        if out["status"]["state"][0] != T.GANG_ADMITTED:
            continue
        if r is not None and not holds and not gone[r]:   # its predecessor is in E(p): released first, never its victim
            gone[r] = True; released.append(r); F += H[r]
        pl = out["placements"].copy()
        use, order = {}, []
        for e in pl:
            n, q = int(e["node"]), sq[int(e["clique"])]
            if n not in use:
                use[n] = np.zeros(4, dtype=np.int64); order.append(n)
            use[n] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
        for n in order:
            need = np.maximum(use[n] - H[r][n], 0) if holds else use[n]
            while not (F[n] >= need).all():
                v = min((x for x in on_node.get(n, []) if not gone[x] and prio[x] < p), key=lambda x: (prio[x], -x))
                gone[v] = True
                F += H[v]
                victims.append((v, g))
            F[n] -= need
        if holds:   # released; what it leaves of the hold comes back after the last gang of priority p
            gone[r] = True; released.append(r)
            U = np.zeros((N, 4), dtype=np.int64)
            for n in order:
                U[n] = use[n]
            leftover += np.maximum(H[r] - U, 0)
        pl["clique"] += co
        per_gang[g] = pl
        st = out["status"][0].copy()
        st["reserved0"] = T.STATUS_PREEMPTOR
        status[g] = st
        sstat[so: so + len(ss)] = out["scope_status"]
    F += leftover
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off if status["state"][g] == T.GANG_ADMITTED else status["placement_off"][g]
        if status["state"][g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F),
                victims=np.array(victims, dtype=T.victim_dt) if victims else np.zeros(0, dtype=T.victim_dt),
                released=sorted(released), perm=perm)


def one_gang(pods, mem=80, priority=0, b=None):
    """one gang of `pods` agent pods of `mem` MiB (appended to builder b)"""
    b = b or T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=mem, min=pods, class_mask=synth.AGENT)])], priority=priority)
    return b


def half_full(prios):
    """2 * len(prios) e2e nodes (150 MiB each); running gang r (priority prios[r]) holds one 80 MiB pod on each of nodes 2r and
    2r + 1, so 70 MiB are free everywhere -> free table, running, holdings"""
    k = len(prios)
    nodes = synth.e2e_cluster(2 * k)
    running = np.zeros(k, dtype=T.running_dt)
    running["priority"] = prios; running["holding_off"] = 2 * np.arange(k); running["n_holdings"] = 2
    holdings = np.zeros(2 * k, dtype=T.holding_dt)
    holdings["node"] = np.arange(2 * k); holdings["mem_mib"] = 80; holdings["pods"] = 1
    nodes["free_mem_mib"] -= 80; nodes["free_pods"] -= 1
    return nodes, running, holdings


def shared_nodes():
    """four e2e nodes; running gangs 0 (priority 0) and 1 (priority 1) each hold 40 MiB on every node: 70 MiB free"""
    nodes = synth.e2e_cluster(4)
    running = np.zeros(2, dtype=T.running_dt)
    running["priority"] = [0, 1]; running["holding_off"] = [0, 4]; running["n_holdings"] = 4
    holdings = np.zeros(8, dtype=T.holding_dt)
    holdings["node"] = np.tile(np.arange(4), 2); holdings["mem_mib"] = 40; holdings["pods"] = 1
    nodes["free_mem_mib"] -= 80; nodes["free_pods"] -= 2
    return nodes, running, holdings


def reclaim_rolling_cluster(oracle, seed, n=630, g_running=200, g_pending=60, share=0.2, used_pct=85, boost=2, **kw):
    """reuse_cases.rolling_cluster with pressure from above: every other pending gang (with its scaled gangs) and every other new
    version get `boost` added to their priority, so that part of the submission outranks part of what is running, and every
    new version asks for half as much memory again per pod, so that some need the reclaim pass.
    -> nodes, n_levels, tables, replaces, running, holdings"""
    nodes, L, (g, c, s), rep, running, holdings = rolling_cluster(oracle, seed, n=n, g_running=g_running, g_pending=g_pending,
                                                                 share=share, used_pct=used_pct, **kw)
    g, c = g.copy(), c.copy()
    new = np.nonzero(rep != T.NONE_U32)[0]
    for i in range(len(g)):
        b = int(g["base_gang"][i])
        root = i if b == T.NONE_U32 else b
        if rep[root] == T.NONE_U32 and root % 2 == 0:
            g["priority"][i] += boost
    g["priority"][new[0::2]] += boost
    for i in new:
        q = slice(int(g["clique_off"][i]), int(g["clique_off"][i]) + int(g["n_cliques"][i]))
        c["req_mem_mib"][q] = c["req_mem_mib"][q] * 3 // 2
    return nodes, L, (g, c, s), rep, running, holdings
