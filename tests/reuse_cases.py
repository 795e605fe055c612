"""Reservation reuse (grove_run_cycle_reuse, include/grove_place.h "reservation reuse") restated over the sequential oracle, and
the scenarios the oracle property tests and the GPU parity tests share.

The restatement walks the cycle's order (priority desc, submission index asc) and hands the oracle one piece at a time: a run of
gangs without a predecessor is one ordinary oracle cycle over the free table F (the sequential pass restricted to those gangs),
a gang with a predecessor is a cycle of its own over F + H_g.  Anchors are pinned to the ones the whole cycle derives and base
gating across pieces is decided here, so every gang meets exactly the state the definition gives it."""
import numpy as np

from grove_b200 import synth, tables as T
from preempt_cases import holdings_of

RES = ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")
HELD = ("cpu_milli", "mem_mib", "gpu", "pods")


def hold_table(n, running, holdings, r):
    """[n, 4] int64: what running gang r holds per node"""
    h = np.zeros((n, 4), dtype=np.int64)
    for x in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
        h[int(x["node"])] += [int(x[f]) for f in HELD]
    return h


def free_table(nodes):
    return np.stack([nodes[f].astype(np.int64) for f in RES], axis=1)


def usage(placements, status, cliques, g, n):
    """[n, 4] int64: what admitted gang g puts on every node"""
    u = np.zeros((n, 4), dtype=np.int64)
    for e in placements[status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]]:
        q = cliques[int(e["clique"])]
        u[int(e["node"])] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
    return u


def _with_free(nodes, F):
    out = nodes.copy()
    for k, f in enumerate(RES):
        out[f] = F[:, k]
    return out


def run_cycle_reuse(oracle, nodes, n_levels, gangs, cliques, scopes, replaces, running, holdings, one_per_call=False):
    """-> dict(placements, status, scope_status, nodes_after) of the reservation-reuse cycle, as its definition reads.
    one_per_call: every gang is a piece of its own (a check of the pieces: the result must not change)"""
    G, N = len(gangs), len(nodes)
    perm = oracle.topology(nodes, n_levels)[0]
    F = free_table(nodes)
    order = sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i))
    pieces, run = [], []
    for g in order:
        if replaces[g] == T.NONE_U32 and not one_per_call:
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
    per_gang = {}
    release = np.zeros((N, 4), dtype=np.int64)
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
            sq.append(cliques[co: co + int(gangs["n_cliques"][g])]); ss.append(scopes[so: so + int(gangs["n_scopes"][g])])
        sq, ss = np.concatenate(sq), np.concatenate(ss)
        H = hold_table(N, running, holdings, int(replaces[ids[0]])) if replaces[ids[0]] != T.NONE_U32 else None
        out = oracle.run_cycle(_with_free(nodes, F if H is None else F + H), n_levels, sg, sq, ss)
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
        if H is None:
            F = free_table(out["nodes_after"])
        elif state[ids[0]] == T.GANG_ADMITTED:
            U = (F + H) - free_table(out["nodes_after"])
            F = F - np.maximum(U - H, 0)
            release += np.maximum(H - U, 0)
    status["state"] = state
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off
        if state[g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F + release), perm=perm)


def new_versions(gangs, cliques, scopes, picks, grow=()):
    """the next versions of gangs `picks` of a submission (same shape; those in `grow` ask for twice the memory per pod),
    appended after `gangs` as a submission of their own: -> (gangs, cliques, scopes) of the new versions"""
    ng, nq, ns = [], [], []
    for i in picks:
        co, so = int(gangs["clique_off"][i]), int(gangs["scope_off"][i])
        q = cliques[co: co + int(gangs["n_cliques"][i])].copy()
        if i in grow:
            q["req_mem_mib"] *= 2
        x = gangs[i: i + 1].copy()
        x["clique_off"] = sum(len(a) for a in nq); x["scope_off"] = sum(len(a) for a in ns); x["base_gang"] = T.NONE_U32
        ng.append(x); nq.append(q); ns.append(scopes[so: so + int(gangs["n_scopes"][i])].copy())
    return np.concatenate(ng), np.concatenate(nq), np.concatenate(ns)


def concat_tables(a, b):
    """submission a followed by submission b (b's offsets and base gangs shifted)"""
    (g1, c1, s1), (g2, c2, s2) = a, b
    g2 = g2.copy()
    g2["clique_off"] += len(c1); g2["scope_off"] += len(s1)
    has = g2["base_gang"] != T.NONE_U32
    g2["base_gang"][has] += len(g1)
    return np.concatenate([g1, g2]), np.concatenate([c1, c2]), np.concatenate([s1, s2])


def rolling_cluster(oracle, seed, n=1260, g_running=400, g_pending=120, share=0.1, used_pct=80, config=synth.config_c4):
    """A rolling update on a churned cluster: an ordinary cycle admits gangs (now RUNNING); the next submission carries other
    pending gangs plus new versions of about `share` of the running gangs, every other one asking for more memory.
    -> nodes (free now), n_levels, tables, replaces, running, holdings"""
    first = config(n=n, g=g_running, seed=seed, max_used_pct=used_pct)
    g1, c1, s1 = first["tables"]
    ref = oracle.run_cycle(first["nodes"], first["n_levels"], g1, c1, s1, threads=2)
    running, holdings = holdings_of(ref["placements"], ref["status"], g1, c1)
    admitted = np.nonzero(ref["status"]["state"] == T.GANG_ADMITTED)[0]   # running gang r is gang admitted[r] of the first cycle
    rng = np.random.default_rng(seed)
    k = max(1, int(len(admitted) * share))
    picks_r = np.sort(rng.choice(len(admitted), size=k, replace=False))
    picks = [int(admitted[r]) for r in picks_r]
    nv = new_versions(g1, c1, s1, picks, grow=set(picks[1::2]))
    second = config(n=n, g=g_pending, seed=seed + 7919, max_used_pct=used_pct)
    tables = concat_tables(second["tables"], nv)
    replaces = np.full(len(tables[0]), T.NONE_U32, dtype=np.uint32)
    replaces[len(second["tables"][0]):] = picks_r
    return ref["nodes_after"], first["n_levels"], tables, replaces, running, holdings
