"""Topology spread (grove_set_spread, include/grove_place.h "topology spread") restated over the sequential oracle, and the
scenarios the oracle property tests and the GPU parity tests share.

The restatement walks the cycle's order (priority desc, submission index asc) and hands the oracle one piece at a time: a run of
gangs that belong to no spread group is one ordinary oracle cycle over the free table F, a member is a cycle of its own.  For a
member the nodes outside its allowed level-l_s domains are marked unschedulable -- exact, because a member has a clique with
MinReplicas > 0 (a candidate inside a masked domain cannot hold it) and the candidate order does not depend on fit.  A SOFT member
that this leaves rejected gets a second call with only the allowed domains masked.  Anchors are pinned to the ones the whole cycle
derives and base gating across pieces is decided here, so every gang meets exactly the state the definition gives it."""
import numpy as np

from grove_b200 import tables as T
from reuse_cases import free_table, _with_free


def domains(oracle, nodes, n_levels):
    """-> (perm, dom [n, MAX_LEVELS] tree-ified domain ids in CALLER order, n_dom per level)"""
    perm, dom_sorted, n_dom, _ = oracle.topology(nodes, n_levels)
    dom = np.empty_like(dom_sorted)
    dom[perm] = dom_sorted
    return perm, dom, n_dom


def domain_classes(nodes, dom, n_dom, level):
    """[n_dom[level]] the OR of the selector classes of the schedulable nodes of every level-`level` domain"""
    out = np.zeros(int(n_dom[level]), dtype=np.uint32)
    d = dom[:, level]
    ok = ((nodes["flags"] & T.NODE_SCHEDULABLE) != 0) & (d != T.DOM_ABSENT)
    bits = np.uint32(1) << ((nodes["flags"] >> T.NODE_CLASS_SHIFT) & 0xF).astype(np.uint32)
    np.bitwise_or.at(out, d[ok].astype(np.int64), bits[ok])
    return out


def gang_classes(gangs, cliques, g):
    co = int(gangs["clique_off"][g])
    return int(np.bitwise_or.reduce(cliques["class_mask"][co: co + int(gangs["n_cliques"][g])].astype(np.uint32)))


def allowed_domains(counts, dcls, cmask, max_skew):
    """the allowed level-l_s domains of a member: eligible (a schedulable node of a class it accepts) and c + 1 - m <= max_skew"""
    elig = (dcls & np.uint32(cmask)) != 0
    if not elig.any():
        return elig
    m = counts[elig].min()
    return elig & (counts + 1 - m <= max_skew)


def _masked(nodes, F, node_out):
    """the node table with free resources F and the nodes of node_out marked unschedulable"""
    out = _with_free(nodes, F)
    out["flags"][node_out] &= ~np.uint32(T.NODE_SCHEDULABLE)
    return out


def run_cycle_spread(oracle, nodes, n_levels, gangs, cliques, scopes, groups, gang_group, seeds=None, trace=None):
    """-> dict(placements, status, scope_status, nodes_after, perm) of the spread cycle, as its definition reads.
    trace (a list): gets (gang, group, counts at its turn, m, allowed domains, A(g) or None) for every member evaluated."""
    G, N = len(gangs), len(nodes)
    groups = np.asarray(groups, dtype=T.spread_dt)
    gang_group = np.asarray(gang_group, dtype=np.uint32)
    perm, dom, n_dom = domains(oracle, nodes, n_levels)
    counts = []
    for s in range(len(groups)):
        c = np.zeros(int(n_dom[int(groups["level"][s])]), dtype=np.int64)
        for x in (seeds if seeds is not None else []):
            if int(x["group"]) == s:
                d = dom[int(x["node"]), int(groups["level"][s])]
                if d != T.DOM_ABSENT:
                    c[int(d)] += 1
        counts.append(c)
    dcls = {int(l): domain_classes(nodes, dom, n_dom, int(l)) for l in set(groups["level"].tolist())}
    F = free_table(nodes)
    order = sorted(range(G), key=lambda i: (-int(gangs["priority"][i]), i))
    pieces, run = [], []
    for g in order:
        if gang_group[g] == T.NONE_U32:
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
    skewed = np.zeros(G, dtype=bool)
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
            sq.append(cliques[co: co + int(gangs["n_cliques"][g])]); ss.append(scopes[so: so + int(gangs["n_scopes"][g])])
        sq, ss = np.concatenate(sq), np.concatenate(ss)
        s = int(gang_group[ids[0]])
        if s == T.NONE_U32:
            out = oracle.run_cycle(_with_free(nodes, F), n_levels, sg, sq, ss)
        else:
            g = ids[0]
            l, mode, skew = int(groups["level"][s]), int(groups["mode"][s]), int(groups["max_skew"][s])
            cm = gang_classes(gangs, cliques, g)
            al = allowed_domains(counts[s], dcls[l], cm, skew)
            d = dom[:, l]
            in_allowed = (d != T.DOM_ABSENT) & al[np.where(d == T.DOM_ABSENT, 0, d).astype(np.int64)]
            out = oracle.run_cycle(_masked(nodes, F, ~in_allowed), n_levels, sg, sq, ss)
            if mode == T.SPREAD_SOFT and out["status"]["state"][0] == T.GANG_REJECTED:
                out = oracle.run_cycle(_masked(nodes, F, in_allowed), n_levels, sg, sq, ss)
                skewed[g] = out["status"]["state"][0] == T.GANG_ADMITTED
            A = None
            if out["status"]["state"][0] == T.GANG_ADMITTED:
                A = int(dom[int(out["status"]["domain_node"][0]), l])
            if trace is not None:
                elig = (dcls[l] & np.uint32(cm)) != 0
                trace.append((g, s, counts[s].copy(), int(counts[s][elig].min()) if elig.any() else None, al.copy(), A))
            if A is not None:
                counts[s][A] += 1
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
    status["reserved0"] = np.where(skewed, T.STATUS_SPREAD_SKEWED, 0)
    merged, off = [], 0
    for g in range(G):
        status["placement_off"][g] = off
        if state[g] == T.GANG_ADMITTED:
            merged.append(per_gang[g]); off += len(per_gang[g])
    placements = np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt)
    return dict(placements=placements, status=status, scope_status=sstat, nodes_after=_with_free(nodes, F), perm=perm)


def spread_groups(levels, modes, skews):
    out = np.zeros(len(levels), dtype=T.spread_dt)
    out["level"], out["mode"], out["max_skew"] = levels, modes, skews
    return out


def eligible_members(gangs, cliques, level):
    """gangs that may join a group of level `level`: a gang Required level at or below it and a clique with MinReplicas > 0"""
    out = []
    for g in range(len(gangs)):
        lv = int(gangs["level"][g])
        co = int(gangs["clique_off"][g])
        if lv != T.LEVEL_NONE and lv >= level and (cliques["min_replicas"][co: co + int(gangs["n_cliques"][g])] > 0).any():
            out.append(g)
    return out


def group_randomly(rng, nodes, n_levels, gangs, cliques, n_groups=None, share=0.8, seeds=True):
    """spread groups at random levels over the gangs that may join them -> (groups, gang_group, seeds)"""
    n_groups = int(rng.integers(1, 4)) if n_groups is None else n_groups
    levels = rng.integers(0, n_levels, n_groups)
    groups = spread_groups(levels, rng.choice([T.SPREAD_HARD, T.SPREAD_SOFT], n_groups), rng.choice([1, 1, 2, 3], n_groups))
    gang_group = np.full(len(gangs), T.NONE_U32, dtype=np.uint32)
    may = [set(eligible_members(gangs, cliques, int(levels[s]))) for s in range(n_groups)]
    for g in range(len(gangs)):
        fits = [s for s in range(n_groups) if g in may[s] and rng.random() < share]
        if fits:
            gang_group[g] = int(rng.choice(fits))
    sd = np.zeros(int(rng.integers(0, 6)) if seeds else 0, dtype=T.spread_seed_dt)
    sd["group"] = rng.integers(0, n_groups, len(sd)); sd["node"] = rng.integers(0, len(nodes), len(sd))
    return groups, gang_group, sd


def zones_case(zones=4, nodes_per_zone=4, replicas=8, pods=1, free_mem=100, mem=80, level=0, gang_level=None):
    """`zones` zones of `nodes_per_zone` hosts (two levels: zone, host), `replicas` identical one-clique gangs of `pods` pods at
    gang level `gang_level` (default the zone level) -> nodes, n_levels, tables"""
    n = zones * nodes_per_zone
    nodes = T.make_nodes(n)
    nodes["dom"][:, 0] = np.arange(n) // nodes_per_zone
    nodes["dom"][:, 1] = np.arange(n)
    nodes["free_cpu_milli"] = 64000; nodes["free_mem_mib"] = free_mem; nodes["free_gpu"] = 8; nodes["free_pods"] = 110
    nodes["flags"] = T.NODE_SCHEDULABLE
    b = T.GangTableBuilder()
    for _ in range(replicas):
        b.add_gang([(None, [dict(mem=mem, min=pods)])], level=level if gang_level is None else gang_level)
    return nodes, 2, b.build()


def hand_cases():
    """name -> (nodes, n_levels, tables, groups, gang_group, seeds): one case per rule of the definition"""
    H, S = T.SPREAD_HARD, T.SPREAD_SOFT

    def all_in(G, s=0):
        return np.full(G, s, dtype=np.uint32)

    def seeds_at(pairs):
        sd = np.zeros(len(pairs), dtype=T.spread_seed_dt)
        for i, (grp, node) in enumerate(pairs):
            sd[i] = (grp, node)
        return sd

    def four_zones(mode):   # 4 zones, 8 replicas, max skew 1: two per zone
        nodes, L, tb = zones_case()
        return nodes, L, tb, spread_groups([0], [mode], [1]), all_in(8), None

    def full_zone(mode):    # zone 1 is full after one replica: the fourth one has to skew (SOFT) or wait (HARD)
        nodes, L, tb = zones_case(zones=2, nodes_per_zone=2, replicas=4, pods=2)
        nodes["free_mem_mib"][:2] = 240   # zone 0 holds three gangs, zone 1 (2 x 100 MiB) one
        return nodes, L, tb, spread_groups([0], [mode], [1]), all_in(4), None

    def ineligible_zone():  # zone 3 only has class-1 nodes, which the gangs do not accept: it does not hold m at 0
        nodes, L, (g, c, s) = zones_case(replicas=6)
        nodes["flags"][12:] = T.NODE_SCHEDULABLE | (1 << T.NODE_CLASS_SHIFT)
        c["class_mask"] = 0x1
        return nodes, L, (g, c, s), spread_groups([0], [H], [1]), all_in(6), None

    def cordoned_zone():    # zone 2 is cordoned: not eligible either
        nodes, L, tb = zones_case(replicas=6)
        nodes["flags"][8:12] = 0
        return nodes, L, tb, spread_groups([0], [H], [1]), all_in(6), None

    def seeded(mode):       # zones 0 and 1 already run two replicas each: the scale-out fills 2 and 3 first
        nodes, L, tb = zones_case(replicas=4)
        return nodes, L, tb, spread_groups([0], [mode], [1]), all_in(4), seeds_at([(0, 0), (0, 1), (0, 5), (0, 6)])

    def skew_two():
        nodes, L, tb = zones_case(replicas=8)
        return nodes, L, tb, spread_groups([0], [H], [2]), all_in(8), None

    def host_level():       # spread over hosts: one replica per host while hosts last
        nodes, L, tb = zones_case(zones=2, nodes_per_zone=3, replicas=8, free_mem=200, gang_level=1)
        return nodes, L, tb, spread_groups([1], [S], [1]), all_in(8), None

    def preferred():        # Required zone, Preferred host: the spread decides the zone, the preference the host
        nodes, L, _ = zones_case()
        b = T.GangTableBuilder()
        for _ in range(6):
            b.add_gang([(None, [dict(mem=30, min=2)])], level=0, preferred=1)
        return nodes, L, b.build(), spread_groups([0], [H], [1]), all_in(6), None

    def scaled():           # base gangs in one group, their scaled gangs in another; a scaled gang waits for its base
        nodes, L, _ = zones_case()
        b = T.GangTableBuilder()
        bases = [b.add_gang([(None, [dict(mem=60, min=1)])], level=0, priority=1) for _ in range(3)]
        for x in bases:
            b.add_gang([(None, [dict(mem=60, min=1)])], level=0, priority=1, base=x)
        gg = np.array([0, 0, 0, 1, 1, 1], dtype=np.uint32)
        return nodes, L, b.build(), spread_groups([0, 0], [H, H], [1, 1]), gg, None

    def mixed():            # non-members before, between and after the members, two groups with their own levels
        nodes, L, _ = zones_case()
        b = T.GangTableBuilder()
        gg = []
        for i in range(10):
            b.add_gang([(None, [dict(mem=40, min=1, replicas=2)])], level=0 if i % 3 else None, priority=i % 2)
            gg.append(T.NONE_U32 if i % 3 == 0 else i % 2)
        return nodes, L, b.build(), spread_groups([0, 0], [H, S], [1, 1]), np.array(gg, dtype=np.uint32), None

    return {"four_zones_hard": lambda: four_zones(H), "four_zones_soft": lambda: four_zones(S),
            "full_zone_hard": lambda: full_zone(H), "full_zone_soft": lambda: full_zone(S),
            "ineligible_zone": ineligible_zone, "cordoned_zone": cordoned_zone, "seeded_hard": lambda: seeded(H),
            "seeded_soft": lambda: seeded(S), "skew_two": skew_two, "host_level": host_level, "preferred": preferred,
            "scaled": scaled, "mixed": mixed}

