"""Consolidation (grove_run_cycle_consolidate, include/grove_place.h "consolidation") restated over the unchanged sequential
oracle, and the scenarios the oracle property tests and the GPU parity tests share.

The ordinary pass is one oracle cycle.  Every REJECTED target is then taken in rank order: the candidate domains are ranked here
in numpy with the fences' shortfall (fence_cases) over F and over W; each try is one oracle call for the target alone, its anchor
pinned to the ordinary pass's and every node outside the domain unschedulable, against W; the relocation is one oracle cycle over
the displaced gangs' spec rows against F + what they hold - U."""
import numpy as np

from grove_b200 import synth, tables as T
from diagnose_cases import need_depth
from fence_cases import blocks_case, sorted_anchor
from preempt_cases import holdings_of
from reuse_cases import _with_free, free_table, hold_table
from spread_cases import _masked

ABSENT = T.DOM_ABSENT


def _rank_key(gangs):
    return lambda i: (-int(gangs["priority"][i]), i)


def shortfalls(topo, nodes, n_levels, gangs, cliques, scopes, g, F):
    """per level-l domain of gang g (l its gang Required level): sum over its cliques with MinReplicas m > 0 of
    max(0, m - sum over the domain of min(cap, m)), cap = grove_diagnose's exact capacity over the free table F (caller order)"""
    perm, dom, ndom, _ = topo
    N = len(nodes)
    sn = np.asarray(nodes)[perm]
    absent = dom[:, :n_levels] == ABSENT
    vdepth = np.where(absent.any(axis=1), absent.argmax(axis=1), n_levels)
    sched = (sn["flags"] & T.NODE_SCHEDULABLE) != 0
    ncls = (sn["flags"].astype(np.int64) >> T.NODE_CLASS_SHIFT) & 0xF
    free = [F[perm, k] for k in range(4)]
    l, co = int(gangs["level"][g]), int(gangs["clique_off"][g])
    ids = dom[:, l].astype(np.int64)
    has = ids != ABSENT
    short = np.zeros(int(ndom[l]), dtype=np.int64)
    for c in range(int(gangs["n_cliques"][g])):
        q = cliques[co + c]
        m = int(q["min_replicas"])
        if not m:
            continue
        req = [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"])]
        fit = sched & (((int(q["class_mask"]) >> ncls) & 1) != 0) & (vdepth >= need_depth(gangs, cliques, scopes, g, c)) & (free[3] >= 1)
        cap = free[3].copy()
        for f, rq in zip(free, req):
            fit &= f >= rq
            if rq:
                cap = np.minimum(cap, f // rq)
        cap = np.where(fit, np.minimum(cap, m), 0)
        have = np.zeros(len(short), dtype=np.int64)
        np.add.at(have, ids[has], cap[has])
        short += np.maximum(0, m - have)
    assert N == len(sn)
    return short


def candidates(topo, nodes, n_levels, gangs, cliques, scopes, b, F, W, qualify=True):
    """the sorted node ranges (lo, hi) a target tries, in order: the level-l domains without shortfall over W, by shortfall over F,
    ties by the fences' candidate order; at most CONSOLIDATE_TRIES.  Without a Required level: the whole cluster.
    qualify=False: every level-l domain, in that order (what the fences' pick takes the first of)."""
    perm, dom, _, _ = topo
    N = len(nodes)
    l = int(gangs["level"][b])
    if l == T.LEVEL_NONE:
        return [(0, N)]
    sf = shortfalls(topo, nodes, n_levels, gangs, cliques, scopes, b, F)
    sw = shortfalls(topo, nodes, n_levels, gangs, cliques, scopes, b, W)
    inv = np.empty(N, dtype=np.int64); inv[perm] = np.arange(N)
    a = sorted_anchor(gangs, inv, b, N)
    keyed = []
    for d in range(len(sf)):
        if qualify and sw[d]:
            continue
        members = np.nonzero(dom[:, l] == d)[0]
        lo, hi = int(members[0]), int(members[-1]) + 1
        close = sum(1 for x in range(n_levels) if dom[lo, x] != ABSENT and dom[lo, x] == dom[a, x])
        keyed.append(((int(sf[d]), -min(close, l + 1), (lo - a) % N), lo, hi))
    return [(lo, hi) for _, lo, hi in sorted(keyed)[: T.CONSOLIDATE_TRIES]]


def _sub(gangs, cliques, scopes, rows, perm, N, priority=None):
    """the gangs `rows` as a submission of their own: anchors pinned to the ones the whole submission derives, no gating, no base"""
    from oracle import oracle_py
    sg = gangs[list(rows)].copy()
    sq, ss = [], []
    for k, g in enumerate(rows):
        if sg["anchor_node"][k] == T.NONE_U32:
            sg["anchor_node"][k] = perm[oracle_py._fmix32(g) % N]
        sg["base_gang"][k] = T.NONE_U32
        sg["flags"][k] &= ~np.uint16(T.GANG_GATED)
        if priority is not None:
            sg["priority"][k] = priority[k]
        sg["clique_off"][k] = sum(len(x) for x in sq); sg["scope_off"][k] = sum(len(x) for x in ss)
        co, so = int(gangs["clique_off"][g]), int(gangs["scope_off"][g])
        sq.append(cliques[co: co + int(gangs["n_cliques"][g])]); ss.append(scopes[so: so + int(gangs["n_scopes"][g])])
    return sg, np.concatenate(sq), np.concatenate(ss)


def run_cycle_consolidate(oracle, nodes, n_levels, gangs, cliques, scopes, targets, spec_of, running, holdings, trace=None):
    """-> dict(placements, status, scope_status, nodes_after, moves, perm) of the cycle as its definition reads.
    trace (a dict): gets tries (count), commits (count) and tried (target -> the ranges it tried)."""
    G, N, R = len(gangs), len(nodes), len(running)
    base = oracle.run_cycle(nodes, n_levels, gangs, cliques, scopes)
    perm = base["perm"]
    topo = oracle.topology(nodes, n_levels)
    status, sstat = base["status"].copy(), base["scope_status"].copy()
    per_gang = {g: base["placements"][status["placement_off"][g]: status["placement_off"][g] + status["n_pods"][g]].copy()
                for g in range(G) if status["state"][g] == T.GANG_ADMITTED}
    F = free_table(base["nodes_after"])
    H = [hold_table(N, running, holdings, r) for r in range(R)]
    prio = [int(running["priority"][r]) for r in range(R)]
    gone = [int(spec_of[r]) == T.NONE_U32 for r in range(R)]   # not movable, or moved
    on_node = {}
    for r in range(R):
        for h in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
            on_node.setdefault(int(h["node"]), []).append(r)
    moves, tries, commits, tried = [], 0, 0, {}
    for b in sorted((int(t) for t in targets), key=_rank_key(gangs)):
        if status["state"][b] != T.GANG_REJECTED:
            continue
        p = int(gangs["priority"][b])
        M = [r for r in range(R) if not gone[r] and prio[r] <= p]
        if not M:
            continue
        W = F + sum(H[r] for r in M)
        sg, sq, ss = _sub(gangs, cliques, scopes, [b], perm, N)
        tried[b] = candidates(topo, nodes, n_levels, gangs, cliques, scopes, b, F, W)
        for lo, hi in tried[b]:
            tries += 1
            outside = np.ones(N, dtype=bool); outside[perm[lo:hi]] = False
            ob = oracle.run_cycle(_masked(nodes, W, outside), n_levels, sg, sq, ss)
            if ob["status"]["state"][0] != T.GANG_ADMITTED:
                continue
            U, order = np.zeros((N, 4), dtype=np.int64), []
            for e in ob["placements"]:
                n, q = int(e["node"]), sq[int(e["clique"])]
                if n not in order:
                    order.append(n)
                U[n] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
            X = []
            for n in order:
                while not (F[n] + sum((H[x][n] for x in X), np.zeros(4, np.int64)) >= U[n]).all():
                    X.append(min((r for r in on_node.get(n, []) if r in M and r not in X), key=lambda r: (prio[r], -r)))
            Fp = F + sum((H[x] for x in X), np.zeros((N, 4), np.int64)) - U
            xs = sorted(X, key=lambda r: (-prio[r], r))
            if xs:
                xg, xq, xsc = _sub(gangs, cliques, scopes, [int(spec_of[r]) for r in xs], perm, N, priority=[prio[r] for r in xs])
                ox = oracle.run_cycle(_with_free(nodes, Fp), n_levels, xg, xq, xsc)
                if not (ox["status"]["state"] == T.GANG_ADMITTED).all():
                    continue
                F = free_table(ox["nodes_after"])
                for k, r in enumerate(xs):
                    s = int(spec_of[r])
                    st = ox["status"][k].copy()
                    pl = ox["placements"][st["placement_off"]: st["placement_off"] + st["n_pods"]].copy()
                    pl["clique"] += int(gangs["clique_off"][s]) - int(xg["clique_off"][k])
                    per_gang[s] = pl
                    st["reserved0"] = T.STATUS_MOVED
                    status[s] = st
                    so = int(gangs["scope_off"][s])
                    sstat[so: so + int(gangs["n_scopes"][s])] = ox["scope_status"][int(xg["scope_off"][k]): int(xg["scope_off"][k]) + int(xg["n_scopes"][k])]
            else:
                F = Fp
            pl = ob["placements"].copy()
            pl["clique"] += int(gangs["clique_off"][b])
            per_gang[b] = pl
            st = ob["status"][0].copy()
            st["reserved0"] = T.STATUS_CONSOLIDATED
            status[b] = st
            so = int(gangs["scope_off"][b])
            sstat[so: so + len(ss)] = ob["scope_status"]
            for r in X:
                gone[r] = True
                moves.append((r, b))
            commits += 1
            break
    merged, off = [], 0
    for g in range(G):
        if status["state"][g] == T.GANG_ADMITTED:
            status["placement_off"][g] = off
            merged.append(per_gang[g]); off += len(per_gang[g])
    if trace is not None:
        trace.update(tries=tries, commits=commits, tried=tried)
    return dict(placements=np.concatenate(merged) if merged else np.zeros(0, dtype=T.placement_dt), status=status,
                scope_status=sstat, nodes_after=_with_free(nodes, F),
                moves=np.array(moves, dtype=T.move_dt) if moves else np.zeros(0, dtype=T.move_dt), perm=perm)


# ---- scenarios --------------------------------------------------------------------------------------------------------------
def with_specs(pending, source, rows):
    """the submission `pending` (gangs, cliques, scopes) followed by a gated spec row restating each gang `rows` of the
    submission `source` -> (tables, spec row index of each)"""
    g, c, s = (np.asarray(x).copy() for x in pending)
    sg, sc, ss = source
    add_g, add_c, add_s, idx = [], [len(c)], [len(s)], []
    nq, ns = len(c), len(s)
    for k, r in enumerate(rows):
        x = sg[r: r + 1].copy()
        co, so = int(x["clique_off"][0]), int(x["scope_off"][0])
        add_c.append(sc[co: co + int(x["n_cliques"][0])]); add_s.append(ss[so: so + int(x["n_scopes"][0])])
        x["clique_off"] = nq; x["scope_off"] = ns
        nq += int(x["n_cliques"][0]); ns += int(x["n_scopes"][0])
        x["base_gang"] = T.NONE_U32
        x["flags"] |= T.GANG_GATED
        add_g.append(x); idx.append(len(g) + k)
    if add_g:
        g = np.concatenate([g] + add_g); c = np.concatenate([c] + add_c[1:]); s = np.concatenate([s] + add_s[1:])
    return (g, c, s), np.array(idx, dtype=np.uint32)


def top_rejected(out, gangs, k=T.MAX_CONSOLIDATE_TARGETS, level_only=False):
    """the k highest-ranked gangs an ordinary cycle rejected (with a gang Required level only, if level_only)"""
    return np.array([g for g in sorted(range(len(gangs)), key=_rank_key(gangs)) if out["status"]["state"][g] == T.GANG_REJECTED
                     and (not level_only or gangs["level"][g] != T.LEVEL_NONE)][:k], dtype=np.uint32)


def snapshot(oracle, nodes, n_levels, first, second, movable=1.0, rng=None):
    """`first` (gangs, cliques, scopes) admitted by an ordinary oracle cycle on `nodes` is RUNNING; the submission is `second`
    followed by the spec rows of a share `movable` of them.  -> nodes (free now), tables, spec_of, running, holdings"""
    g1, c1, s1 = first
    ref = oracle.run_cycle(nodes, n_levels, g1, c1, s1)
    running, holdings = holdings_of(ref["placements"], ref["status"], g1, c1)
    admitted = [g for g in range(len(g1)) if ref["status"]["state"][g] == T.GANG_ADMITTED]
    pick = [k for k in range(len(admitted)) if movable >= 1.0 or rng.random() < movable]
    tables, idx = with_specs(second, first, [admitted[k] for k in pick])
    spec_of = np.full(len(running), T.NONE_U32, dtype=np.uint32)
    spec_of[pick] = idx
    return ref["nodes_after"], tables, spec_of, running, holdings


def random_snapshot(oracle, seed):
    """a random_case split in two: the first part runs, the second is submitted with the spec rows of most of the first; the
    targets are the highest-ranked gangs the ordinary cycle rejects -> nodes, L, tables, targets, spec_of, running, holdings"""
    from test_random_parity_gpu import random_case
    rng = np.random.default_rng(seed + 4099)
    nodes, L, (g, c, s) = random_case(seed, pref=seed % 2 == 1)
    cut = max(1, len(g) // 2)
    first = _slice((g, c, s), range(cut))
    second = _slice((g, c, s), range(cut, len(g)))
    free, tables, spec_of, running, holdings = snapshot(oracle, nodes, L, first, second, movable=0.8, rng=rng)
    running["priority"] -= rng.integers(0, 2, len(running)).astype(np.int32)   # some below their spec rows' targets
    plain = oracle.run_cycle(free, L, *tables)
    targets = top_rejected(plain, tables[0], k=int(rng.integers(0, T.MAX_CONSOLIDATE_TARGETS + 1)))
    return free, L, tables, targets, spec_of, running, holdings


def _slice(tables, rows):
    """gangs `rows` of a submission as a submission of their own (base gangs outside it dropped, inside it re-indexed)"""
    g, c, s = tables
    rows = list(rows)
    if not rows:
        return g[:0].copy(), c[:0].copy(), s[:0].copy()
    sub = {r: k for k, r in enumerate(rows)}
    sg = g[rows].copy()
    sq, ss = [], []
    for k, r in enumerate(rows):
        b = int(g["base_gang"][r])
        sg["base_gang"][k] = sub[b] if b in sub else T.NONE_U32
        sg["clique_off"][k] = sum(len(x) for x in sq); sg["scope_off"][k] = sum(len(x) for x in ss)
        co, so = int(g["clique_off"][r]), int(g["scope_off"][r])
        sq.append(c[co: co + int(g["n_cliques"][r])]); ss.append(s[so: so + int(g["n_scopes"][r])])
    return sg, np.concatenate(sq), np.concatenate(ss)


class Runner:
    """running one-node gangs on a blocks_case cluster: add(node, gpu, priority, movable, pods, level) holds `gpu` GPUs on each
    of `node` (an index or a list) and, when movable, restates itself as a gated spec row of the submission"""

    def __init__(self, blocks, per_block, gpus=8):
        self.nodes, self.L = blocks_case(blocks=blocks, per_block=per_block, gpus=gpus)
        self.b = T.GangTableBuilder()
        self.run, self.hold, self.spec = [], [], []

    def add(self, node, gpu=8, priority=0, movable=True, level=None):
        nodes = [node] if np.isscalar(node) else list(node)
        spec = self.b.add_gang([(None, [dict(gpu=gpu, min=len(nodes))])], level=level, priority=priority, gated=True) if movable else None
        self.run.append((priority, len(self.hold), len(nodes), 0))
        for n in nodes:
            self.hold.append((n, 0, 0, gpu, 1))
            self.nodes["free_gpu"][n] -= gpu; self.nodes["free_pods"][n] -= 1
        self.spec.append(T.NONE_U32 if spec is None else spec)

    def build(self, targets):
        return (self.nodes, self.L, self.b.build(), np.array(targets, dtype=np.uint32), np.array(self.spec, dtype=np.uint32),
                np.array(self.run, dtype=T.running_dt), np.array(self.hold, dtype=T.holding_dt))


def hand_cases():
    """name -> () -> (nodes, n_levels, tables, targets, spec_of, running, holdings): one case per rule of the definition.  In
    each, gang 0 is the target unless said otherwise."""

    def priority_bar():        # block 0 is closest to the anchor, but what blocks it runs above the target: block 1 instead
        c = Runner(3, 2)
        t = c.b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=3, anchor=0)
        c.add(0, priority=5); c.add(2, priority=3); c.add(4, priority=4)
        return c.build([t])

    def f_shortfall_order():   # block 1 is short by one node over F, the others by two: it is tried first although farther away
        c = Runner(4, 2)
        t = c.b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, anchor=0)
        for n in (0, 1, 2, 4, 5, 6, 7):
            c.add(n, gpu=4)
        return c.build([t])

    def try_limit(traps):      # `traps` blocks qualify and come first but cannot hold both cliques; the good block comes last
        c = Runner(traps + 1, 2)
        t = c.b.add_gang([(None, [dict(gpu=8, min=1), dict(gpu=8, min=1)])], level=0, anchor=0)
        for k in range(traps):
            c.add(2 * k + 1, movable=False)
        c.add(2 * traps, gpu=4); c.add(2 * traps + 1, gpu=4)
        return c.build([t])

    def rollback_fits_nowhere():   # the only qualifying block's runner has nowhere else to go: nothing changes
        c = Runner(2, 2)
        t = c.b.add_gang([(None, [dict(gpu=8, min=2)])], level=0)
        c.add(0); c.add(2, movable=False); c.add(3, movable=False)
        return c.build([t])

    def mover_required_level():    # the runner of block 0 needs a whole block itself: the two free nodes are in different blocks
        c = Runner(3, 2)
        t = c.b.add_gang([(None, [dict(gpu=8, min=2)])], level=0)
        c.add([0, 1], level=0); c.add(3, movable=False); c.add(5, movable=False)
        return c.build([t])

    def lands_back():          # the target leaves 2 GPUs on each node of its block; the runner's two pods land there again
        c = Runner(1, 2)
        t = c.b.add_gang([(None, [dict(gpu=6, min=2)])], level=0)
        c.add([0, 0], gpu=2)
        return c.build([t])

    def no_level():            # a target without a Required level: the whole cluster is the one candidate
        c = Runner(2, 3)
        t = c.b.add_gang([(None, [dict(gpu=8, min=5)])])
        c.add(0, gpu=4); c.add(1, gpu=4)
        return c.build([t])

    def two_targets():         # the higher-ranked target moves first; the other finds what is left
        c = Runner(3, 2)
        t0 = c.b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=2)
        t1 = c.b.add_gang([(None, [dict(gpu=8, min=2)])], level=0, priority=1)
        c.add(0, priority=1); c.add(2, priority=1); c.add(4, priority=1)
        return c.build([t1, t0])

    return {"priority_bar": priority_bar, "f_shortfall_order": f_shortfall_order, "try_limit_3": lambda: try_limit(3),
            "try_limit_4": lambda: try_limit(4), "rollback_fits_nowhere": rollback_fits_nowhere,
            "mover_required_level": mover_required_level, "lands_back": lands_back, "no_level": no_level, "two_targets": two_targets}


class Starvation:
    """fence_cases' starvation case with its one-node gangs running: four blocks of 8 x 8-GPU nodes, busy on every node but one per
    block when the block-sized gang arrives, and a stream of one-node gangs each cycle, each living two cycles once admitted.  Every
    running one-node gang is movable.  run(cycle_fn, target_after): cycle_fn(nodes, L, tables, targets, spec_of, running,
    holdings) -> outputs; target_after = None never names a target, k names the block gang once it was rejected k cycles in a row.
    Returns (cycle it was admitted or None, per-cycle records: (targeted, admitted, moves))."""

    def __init__(self, cycles=12, small_per_cycle=6, seed=0):
        self.cycles, self.small, self.seed = cycles, small_per_cycle, seed
        self.nodes, self.L = blocks_case()

    def run(self, cycle_fn, target_after=None):
        N = len(self.nodes)
        busy = [n for n in range(N) if n % 8 != 7]
        running = [(n, int(c)) for n, c in zip(busy, np.random.default_rng(1).integers(1, 3, len(busy)))]   # (node, leaves)
        rejected_for, history = 0, []
        anchors = np.random.default_rng(self.seed).integers(0, N, size=(self.cycles, self.small))
        for cyc in range(self.cycles):
            running = [r for r in running if r[1] != cyc]
            nodes = self.nodes.copy()
            b = T.GangTableBuilder()
            b.add_gang([(None, [dict(gpu=8, min=8)])], level=0, anchor=0)
            for a in anchors[cyc]:
                b.add_gang([(None, [dict(gpu=8, min=1)])], level=0, anchor=int(a))
            n_new = 1 + self.small
            spec = [b.add_gang([(None, [dict(gpu=8, min=1)])], level=0, anchor=n, gated=True) for n, _ in running]
            for n, _ in running:
                nodes["free_gpu"][n] -= 8; nodes["free_pods"][n] -= 1
            run = np.array([(0, k, 1, 0) for k in range(len(running))], dtype=T.running_dt).reshape(-1)
            hold = np.array([(n, 0, 0, 8, 1) for n, _ in running], dtype=T.holding_dt).reshape(-1)
            targeted = target_after is not None and rejected_for >= target_after
            tables = b.build()
            out = cycle_fn(nodes, self.L, tables, np.array([0] if targeted else [], dtype=np.uint32),
                           np.array(spec, dtype=np.uint32), run, hold)
            st = out["status"]
            history.append((targeted, int(st["state"][0]) == T.GANG_ADMITTED, len(out.get("moves", []))))
            new_running = []
            for k, (n, leaves) in enumerate(running):
                s = spec[k]
                if st["state"][s] == T.GANG_ADMITTED:   # moved: it runs on in its new place
                    n = int(out["placements"][st["placement_off"][s]]["node"])
                new_running.append((n, leaves))
            for g in range(1, n_new):
                if st["state"][g] == T.GANG_ADMITTED:
                    new_running.append((int(out["placements"][st["placement_off"][g]]["node"]), cyc + 2))
            running = new_running
            if st["state"][0] == T.GANG_ADMITTED:
                return cyc, history
            rejected_for = rejected_for + 1 if st["state"][0] == T.GANG_REJECTED else rejected_for
        return None, history


def reduced_c4(oracle, n=5040, g_running=400, g_pending=400, seed=41):
    """a C4-shaped cluster on which an earlier cycle admitted gangs (now running, all movable) and a new C4-shaped submission;
    targets: the 16 highest-ranked gangs with a Required level that the ordinary cycle rejects
    -> nodes, L, tables, targets, spec_of, running, holdings"""
    first = synth.config_c4(n=n, g=g_running, seed=seed, max_used_pct=85)
    second = synth.config_c4(n=n, g=g_pending, seed=seed + 7919, max_used_pct=85)
    free, tables, spec_of, running, holdings = snapshot(oracle, first["nodes"], first["n_levels"], first["tables"], second["tables"])
    plain = oracle.run_cycle(free, first["n_levels"], *tables)
    return free, first["n_levels"], tables, top_rejected(plain, tables[0], level_only=True), spec_of, running, holdings
