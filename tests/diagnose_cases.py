"""Numpy restatement of grove_diagnose (include/grove_place.h "diagnosis of rejected gangs", DESIGN.md section 1 "Diagnosis").

From the inputs and the outputs of a completed cycle it rebuilds the state each gang met at its turn,
    V_g = F_end + sum of U_h over the admitted gangs h ranked after g,
and computes, for every REJECTED gang, the clique and gang records the engine must equal exactly.  Nothing here knows how
the search works: only K1 fit, the exact capacity and the domains of the gang's Required level.  Shared by the CPU and GPU
tests."""
from __future__ import annotations

import numpy as np

from grove_b200 import tables as T
from oracle import oracle_py

ABSENT = 0xFFFFFFFF


def ranks(gangs):
    """order rank of every gang: (priority desc, submission index asc)"""
    order = sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))
    r = np.zeros(len(gangs), dtype=np.int64)
    r[order] = np.arange(len(gangs))
    return r


def usage(nodes, gangs, cliques, out):
    """per admitted gang: its usage as four int64 rows (cpu, mem, gpu, pods) over the caller's node order"""
    n = len(nodes)
    st, pl = out["status"], out["placements"]
    use = {}
    for g in range(len(gangs)):
        if st["state"][g] != T.GANG_ADMITTED:
            continue
        e = pl[int(st["placement_off"][g]): int(st["placement_off"][g]) + int(st["n_pods"][g])]
        u = np.zeros((4, n), dtype=np.int64)
        q = cliques[e["clique"].astype(np.int64)]
        for k, f in enumerate(("req_cpu_milli", "req_mem_mib", "req_gpu")):
            np.add.at(u[k], e["node"].astype(np.int64), q[f].astype(np.int64))
        np.add.at(u[3], e["node"].astype(np.int64), 1)
        use[g] = u
    return use


def _table(nodes):
    return np.stack([nodes[f].astype(np.int64) for f in ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")])


def views(nodes, gangs, cliques, out):
    """yields (g, the node table at g's turn in the caller's order) for every gang the pass evaluated (ADMITTED or REJECTED),
    highest rank first: F_end plus the usage of the admitted gangs ranked at or after g.  For a REJECTED gang (no usage of
    its own) that is V_g."""
    use = usage(nodes, gangs, cliques, out)
    end = out["nodes_after"]
    acc = _table(end)
    r = ranks(gangs)
    for g in sorted(range(len(gangs)), key=lambda i: -r[i]):
        s = int(out["status"]["state"][g])
        if s == T.GANG_ADMITTED:
            acc = acc + use[g]
        if s in (T.GANG_ADMITTED, T.GANG_REJECTED):
            v = end.copy()
            for k, f in enumerate(("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")):
                v[f] = acc[k]
            yield g, v


def need_depth(gangs, cliques, scopes, g, c):
    """labels a node must carry for clique c of gang g: the deepest Required level binding it (its own, its scope's, its
    gang's) + 1"""
    q = cliques[int(gangs["clique_off"][g]) + c]
    sc = scopes[int(gangs["scope_off"][g]) + (int(q["scope"]) & 0x1F)]
    need = 0
    for lv in (int(gangs["level"][g]), int(sc["level"]), int(q["level"])):
        if lv != T.LEVEL_NONE:
            need = max(need, lv + 1)
    return need


def diagnose(nodes, n_levels, gangs, cliques, scopes, min_replicas, out):
    """-> (gang_diag_dt[G], clique_diag_dt[Q]); min_replicas[q] is clique q's MinReplicas (the 16-bit count of a wide
    submission)"""
    G, Q = len(gangs), len(cliques)
    gd = np.zeros(G, dtype=T.gang_diag_dt)
    qd = np.zeros(Q, dtype=T.clique_diag_dt)
    perm, dom, ndom, _ = oracle_py.topology(nodes, n_levels)
    absent = dom[:, :n_levels] == ABSENT
    vdepth = np.where(absent.any(axis=1), absent.argmax(axis=1), n_levels)
    sn = np.asarray(nodes)[perm]
    sched = (sn["flags"] & T.NODE_SCHEDULABLE) != 0
    ncls = (sn["flags"].astype(np.int64) >> T.NODE_CLASS_SHIFT) & 0xF
    for g, v in views(nodes, gangs, cliques, out):
        if out["status"]["state"][g] != T.GANG_REJECTED:
            continue
        v = v[perm]
        free = [v[f].astype(np.int64) for f in ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")]
        gg = gangs[g]
        co, lv = int(gg["clique_off"]), int(gg["level"])
        if lv == T.LEVEL_NONE:
            ids, nd = np.zeros(len(sn), dtype=np.int64), 1
        else:
            ids, nd = dom[:, lv].astype(np.int64), int(ndom[lv])
        has = ids != ABSENT
        ok = np.ones(nd, dtype=bool)
        short = None
        for c in range(int(gg["n_cliques"])):
            q = cliques[co + c]
            need = need_depth(gangs, cliques, scopes, g, c)
            req = [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"])]
            fails = [~sched, ((int(q["class_mask"]) >> ncls) & 1) == 0, vdepth < need,
                     free[0] < req[0], free[1] < req[1], free[2] < req[2], free[3] < 1]
            first = np.full(len(sn), -1)
            for k in range(len(fails) - 1, -1, -1):
                first = np.where(fails[k], k, first)
            fit = first < 0
            cap = free[3].copy()
            for f, rq in zip(free, req):
                if rq:
                    cap = np.minimum(cap, f // rq)
            cap = np.where(fit, cap, 0)
            rec = qd[co + c]
            rec["nodes_fit"] = int(fit.sum())
            for k, name in enumerate(T.DIAG_FAILURES):
                rec[name] = int((first == k).sum())
            rec["pods_fit"] = int(cap.sum())
            qd[co + c] = rec
            m = int(min_replicas[co + c])
            if short is None and int(cap.sum()) < m:
                short = c
            if m:
                per_dom = np.zeros(nd, dtype=np.int64)
                np.add.at(per_dom, ids[has], cap[has])
                ok &= per_dom >= m
        d = gd[g]
        d["level"], d["domains"], d["domains_ok"] = lv, nd, int(ok.sum())
        if short is not None:
            d["verdict"], d["clique"] = T.DIAG_CLIQUE_SHORT, short
        elif lv != T.LEVEL_NONE and int(ok.sum()) == 0:
            d["verdict"] = T.DIAG_NO_DOMAIN
        else:
            d["verdict"] = T.DIAG_NO_JOINT_FIT
        gd[g] = d
    return gd, qd
