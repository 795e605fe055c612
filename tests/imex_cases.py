"""ComputeDomain exclusivity (grove_set_compute_domains, include/grove_place.h "ComputeDomain exclusivity") restated over the
sequential oracle, and the scenarios the oracle property tests and the GPU parity tests share.

The pass walks the cycle's order (priority desc, submission index asc) and hands the oracle one piece at a time.  A run of gangs
without enrolled cliques is one ordinary oracle cycle: ownership cannot affect them.  A gang with enrolled cliques is one oracle
call of its own with its anchor pinned, on a table where every node whose owner is foreign to the gang's CD carries the shadow
selector class c + 8.  Its enrolled cliques accept only classes 0-7, its other cliques also the shadow classes.  That is exact
while the test nodes use classes 0-7, and candidate order does not depend on fit.  Base gating across pieces is decided here, as
in fence_cases.py, so every gang meets exactly the state the definition gives it."""
import numpy as np

from grove_b200 import tables as T
from fence_cases import _fmix32, blocks_case
from reuse_cases import free_table, _with_free

NONE, NO_IMEX = T.CD_NONE, T.CD_NO_IMEX


def gang_cds(gangs, cd):
    """-> [G] the CD of each gang's enrolled cliques (CD_NONE: none enrolled); raises on two CDs in one gang"""
    out = np.full(len(gangs), NONE, dtype=np.uint32)
    for g in range(len(gangs)):
        co = int(gangs["clique_off"][g])
        cds = {int(x) for x in cd[co: co + int(gangs["n_cliques"][g])]} - {NONE}
        assert len(cds) <= 1, f"gang {g} names two CDs"
        if cds:
            out[g] = cds.pop()
    return out


def _shadowed(nodes, F, owner, c):
    """the node table with free resources F and every node whose owner is foreign to CD c in shadow class + 8"""
    out = _with_free(nodes, F)
    foreign = (owner != NONE) & (owner != c)
    cls = (out["flags"] >> T.NODE_CLASS_SHIFT) & 0xF
    assert (cls < 8).all(), "the restatement needs node classes 0-7"
    out["flags"] = np.where(foreign, (out["flags"] & ~np.uint32(0xF << T.NODE_CLASS_SHIFT)) | ((cls + 8) << T.NODE_CLASS_SHIFT), out["flags"])
    return out


def run_cycle_imex(oracle, nodes, n_levels, gangs, cliques, scopes, cd, owner0):
    """-> dict(placements, status, scope_status, nodes_after, perm, owners) of the cycle with ComputeDomains, as its definition
    reads"""
    G, N = len(gangs), len(nodes)
    cd = np.asarray(cd, dtype=np.uint32)
    owner = np.asarray(owner0, dtype=np.uint32).copy()
    gcd = gang_cds(gangs, cd)
    perm, _, _, _ = oracle.topology(nodes, n_levels)
    order = sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i))
    pieces, run = [], []
    for g in order:
        if gcd[g] != NONE:
            if run:
                pieces.append(run); run = []
            pieces.append([g])
        else:
            run.append(g)
    if run:
        pieces.append(run)
    F = free_table(nodes)
    status = np.zeros(G, dtype=T.status_dt)
    status["level"] = T.LEVEL_NONE; status["domain_node"] = T.NONE_U32
    sstat = np.zeros(len(scopes), dtype=T.scope_status_dt)
    sstat["level"] = T.LEVEL_NONE; sstat["domain_node"] = T.NONE_U32
    state = np.zeros(G, dtype=np.uint8)
    per_gang = {}
    for piece in pieces:
        ids = []
        for g in sorted(piece):
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
                sg["anchor_node"][k] = perm[_fmix32(g) % N]
            sg["clique_off"][k] = sum(len(x) for x in sq); sg["scope_off"][k] = sum(len(x) for x in ss)
            co, so = int(gangs["clique_off"][g]), int(gangs["scope_off"][g])
            sq.append(cliques[co: co + int(gangs["n_cliques"][g])].copy()); ss.append(scopes[so: so + int(gangs["n_scopes"][g])])
        sq, ss = np.concatenate(sq), np.concatenate(ss)
        c = int(gcd[piece[0]]) if len(piece) == 1 else NONE
        if c != NONE:   # one enrolled gang: its enrolled cliques avoid the shadow classes, its other cliques take them too
            g = piece[0]
            co = int(gangs["clique_off"][g])
            enr = cd[co: co + int(gangs["n_cliques"][g])] != NONE
            m = sq["class_mask"].astype(np.uint32) & 0xFF
            sq["class_mask"] = np.where(enr, m, m | (m << 8))
            table = _shadowed(nodes, F, owner, c)
        else:
            table = _with_free(nodes, F)
        out = oracle.run_cycle(table, n_levels, sg, sq, ss)
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
                for e in pl:
                    q = int(cd[int(e["clique"])])
                    if q != NONE:
                        n = int(e["node"])
                        assert owner[n] in (NONE, q), "an enrolled pod on a node another CD holds"
                        owner[n] = q
        F = free_table(out["nodes_after"])
    status["state"] = state
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off
        if state[g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F), perm=perm, owners=owner)


def enroll_randomly(rng, gangs, cliques, nodes, n_cds=None):
    """-> (cd [Q], owner0 [N]): a random CD for some gangs, shared by a base gang and the gangs scaled from it, their GPU cliques
    enrolled at random; some nodes owned by random CDs or without an IMEX driver"""
    G, Q, N = len(gangs), len(cliques), len(nodes)
    n_cds = int(rng.integers(1, 5)) if n_cds is None else n_cds
    gcd = np.full(G, NONE, dtype=np.int64)
    for g in range(G):
        b = int(gangs["base_gang"][g])
        if b != T.NONE_U32 and b < g and gcd[b] != NONE:
            gcd[g] = gcd[b] if rng.random() < 0.8 else NONE
        elif rng.random() < 0.6:
            gcd[g] = int(rng.integers(0, n_cds))
    cd = np.full(Q, NONE, dtype=np.uint32)
    for g in range(G):
        if gcd[g] == NONE:
            continue
        co = int(gangs["clique_off"][g])
        for c in range(int(gangs["n_cliques"][g])):
            if cliques["req_gpu"][co + c] > 0 and rng.random() < 0.75:
                cd[co + c] = gcd[g]
    owner0 = np.full(N, NONE, dtype=np.uint32)
    r = rng.random(N)
    owner0[r < 0.15] = rng.integers(0, n_cds, int((r < 0.15).sum()))
    owner0[(r >= 0.15) & (r < 0.2)] = NO_IMEX
    return cd, owner0


def _workers(b, k, anchor=None, base=None, level=None, frontend=False, extra=0):
    """a PCS replica: k enrolled 1-GPU workers (clique 0), optionally a CPU frontend (clique 1) -> gang index"""
    cl = [dict(gpu=1, cpu=1000, mem=1024, min=k, replicas=k + extra)]
    if frontend:
        cl.append(dict(gpu=0, cpu=1000, mem=1024, min=1))
    return b.add_gang([(None, cl)], level=level, priority=1, anchor=anchor, base=base)


def _enrolled(tables, gang_cd):
    """cd [Q]: the GPU cliques of every gang g in gang_cd enrolled in gang_cd[g]"""
    gangs, cliques, _ = tables
    cd = np.full(len(cliques), NONE, dtype=np.uint32)
    for g, c in gang_cd.items():
        co = int(gangs["clique_off"][g])
        for q in range(co, co + int(gangs["n_cliques"][g])):
            if cliques["req_gpu"][q] > 0:
                cd[q] = c
    return cd


def hand_cases():
    """name -> (nodes, n_levels, tables, cd, owner0): one case per rule of the definition"""

    def two_replicas():        # both anchored at node 0: the plain cycle stacks them there, exclusivity splits them
        nodes, L = blocks_case(blocks=1, per_block=2)
        b = T.GangTableBuilder()
        _workers(b, 4, anchor=0); _workers(b, 4, anchor=0)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 7, 1: 8}), np.full(len(nodes), NONE, np.uint32)

    def third_rejected():      # three replicas, two nodes: the third waits
        nodes, L = blocks_case(blocks=1, per_block=2)
        b = T.GangTableBuilder()
        for _ in range(3):
            _workers(b, 4, anchor=0)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 1, 1: 2, 2: 3}), np.full(len(nodes), NONE, np.uint32)

    def after_delete():        # the next cycle after replica 0 is deleted: node 0 is free again, replica 2 lands there
        nodes, L = blocks_case(blocks=1, per_block=2)
        nodes["free_gpu"] = [8, 4]   # replica 1 still runs on node 1
        b = T.GangTableBuilder()
        _workers(b, 4, anchor=1)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 3}), np.array([NONE, 2], np.uint32)

    def frontend_shares():     # the frontend is not enrolled: it may sit on a node another CD holds
        nodes, L = blocks_case(blocks=1, per_block=2)
        nodes["free_gpu"] = [8, 0]
        b = T.GangTableBuilder()
        _workers(b, 4, anchor=0, frontend=True)
        b.add_gang([(None, [dict(gpu=0, cpu=1000, mem=1024, min=1)])], priority=1, anchor=1)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 5}), np.array([NONE, 9], np.uint32)

    def scaled_joins_base():   # a scaled gang carries its base's CD: it joins the node its base took in this cycle
        nodes, L = blocks_case(blocks=1, per_block=2)
        b = T.GangTableBuilder()
        base = _workers(b, 4, anchor=0)
        _workers(b, 4, anchor=0)
        _workers(b, 2, anchor=0, base=base)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 1, 1: 2, 2: 1}), np.full(len(nodes), NONE, np.uint32)

    def no_imex_node():        # a node without an IMEX driver takes only pods that are not enrolled
        nodes, L = blocks_case(blocks=1, per_block=2)
        b = T.GangTableBuilder()
        _workers(b, 4, anchor=0)
        b.add_gang([(None, [dict(gpu=1, cpu=1000, mem=1024, min=2)])], priority=1, anchor=0)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 4}), np.array([NO_IMEX, NONE], np.uint32)

    def surplus_blocked():     # 4 workers and 4 best-effort ones: MinReplicas fit on the free node, the surplus may not spill
                               # onto the nodes other CDs hold
        nodes, L = blocks_case(blocks=1, per_block=3)
        nodes["free_gpu"] = [4, 8, 8]
        b = T.GangTableBuilder()
        _workers(b, 4, anchor=0, level=0, extra=4)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 1}), np.array([NONE, 2, 3], np.uint32)

    def preferred_levels():    # two blocks, host level preferred: the anchor's host is held by another CD, the next host is taken
        nodes, L = blocks_case(blocks=2, per_block=2)
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=1, cpu=1000, mem=1024, min=6)])], level=0, preferred=1, priority=1, anchor=1)
        b.add_gang([(None, [dict(gpu=2, cpu=1000, mem=1024, min=2)])], level=0, preferred=1, priority=1, anchor=0)
        t = b.build()
        return nodes, L, t, _enrolled(t, {0: 1, 1: 2}), np.array([NONE, 3, NONE, NONE], np.uint32)

    return {"two_replicas": two_replicas, "third_rejected": third_rejected, "after_delete": after_delete,
            "frontend_shares": frontend_shares, "scaled_joins_base": scaled_joins_base, "no_imex_node": no_imex_node,
            "surplus_blocked": surplus_blocked, "preferred_levels": preferred_levels}
