"""Synthetic cluster snapshots and pending-gang tables (measurement fixtures + e2e shapes).

Node side restates the reference's KWOK fake-node generator: topology labels by integer division of
the node index and a fixed allocatable (ai-dynamo/grove operator/hack/infra_manager/kwok.py:55-117,
constants.py:65-67,195-197).  Gang side restates the structure the operator's PodGang builder emits
for a PodCliqueSet -- a base gang per PCS replica holding standalone cliques plus the first
minAvailable replicas of each scaling group, and one scaled gang per further scaling-group replica
(operator/internal/controller/podcliqueset/components/podgang/syncflow.go:145-345).

All randomness is counter-based splitmix64 so that every config is reproducible from its seed
(0x6407E + config number, SURVEY.md section 8d) without sequential state.
"""
from __future__ import annotations

import numpy as np

from . import tables as T

SEED_BASE = 0x6407E


def splitmix64(seed: int, idx: np.ndarray) -> np.ndarray:
    """Counter-based hash: value i depends only on (seed, idx[i])."""
    with np.errstate(over="ignore"):
        z = idx.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(seed & 0xFFFFFFFFFFFFFFFF)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z


def _rand_below(seed: int, stream: int, n: int, bound: int) -> np.ndarray:
    return (splitmix64(seed * 1000003 + stream, np.arange(n)) % np.uint64(bound)).astype(np.int64)


def kwok_nodes(n: int, per_level: list[int], cpu_milli=64000, mem_mib=524288, gpu=8, pods=110,
               node_class=0) -> np.ndarray:
    """KWOK-shaped nodes: dom[l] = i // per_level[l] (kwok.py:64-68), all free, all schedulable."""
    nodes = T.make_nodes(n)
    i = np.arange(n, dtype=np.uint32)
    nodes["free_cpu_milli"] = cpu_milli
    nodes["free_mem_mib"] = mem_mib
    nodes["free_gpu"] = gpu
    nodes["free_pods"] = pods
    nodes["flags"] = T.NODE_SCHEDULABLE | (node_class << T.NODE_CLASS_SHIFT)
    for l, size in enumerate(per_level):
        nodes["dom"][:, l] = i // np.uint32(size)
    return nodes


def pre_use(nodes: np.ndarray, seed: int, max_frac_pct: int) -> None:
    """Uniform random 0..max_frac_pct % of every resource dimension already taken."""
    n = len(nodes)
    for k, f in enumerate(("free_cpu_milli", "free_mem_mib", "free_pods")):
        used = _rand_below(seed, 10 + k, n, max_frac_pct + 1)
        nodes[f] = (nodes[f].astype(np.int64) * (100 - used) // 100).astype(nodes[f].dtype)
    # GPUs are taken in whole units
    g = nodes["free_gpu"].astype(np.int64)
    used = _rand_below(seed, 13, n, max_frac_pct + 1)
    nodes["free_gpu"] = (g - (g * used + 99) // 100).clip(0).astype(np.uint16)


def cordon(nodes: np.ndarray, idx) -> None:
    nodes["flags"][idx] &= ~np.uint32(T.NODE_SCHEDULABLE)


# ------------------------------------------------------------------------------------------------
# e2e shapes (operator/e2e): 150 MiB nodes, 80 MiB pods => one pod per node
# ------------------------------------------------------------------------------------------------
E2E_LEVELS = 4  # zone / block / rack / host


def e2e_cluster(n: int, cordoned: int = 0) -> np.ndarray:
    """hack/e2e.yaml: kwok.nodes 30, node_cpu 4, node_memory 150Mi.  Nested variant of the label
    arithmetic (zone 28 / block 14 / rack 7 / host 1, create-e2e-cluster.py:137-139)."""
    nodes = kwok_nodes(n, [28, 14, 7, 1], cpu_milli=4000, mem_mib=150, gpu=0, pods=110, node_class=1)
    if cordoned:
        cordon(nodes, np.arange(n - cordoned, n))
    return nodes


AGENT = 0x2  # class_mask: only class-1 ("agent" role: nodeAffinity + toleration in e2e YAMLs)


def _clq(mem, mn, replicas=None, level=None):
    return dict(mem=mem, min=mn, replicas=mn if replicas is None else replicas, level=level, class_mask=AGENT)


def workload1(b: T.GangTableBuilder, pcsg_replicas=2, pcs_replicas=1, level=None) -> list[int]:
    """e2e/yaml/workload1.yaml: pc-a x2, sg-x x2 x (pc-b x1 + pc-c x3); minAvailable == replicas.
    Returns gang indices: per PCS replica one base gang, then scaled gangs for sg-x replicas >= 2."""
    out = []
    for _ in range(pcs_replicas):
        scopes = [(None, [_clq(80, 2)])]
        for _r in range(2):  # sg-x minAvailable = 2 -> both replicas in the base gang
            scopes.append((None, [_clq(80, 1), _clq(80, 3)]))
        base = b.add_gang(scopes, level=level)
        out.append(base)
        for _r in range(2, pcsg_replicas):
            out.append(b.add_gang([(None, [_clq(80, 1), _clq(80, 3)])], level=level, base=base))
    return out


def workload2(b: T.GangTableBuilder, pcsg_replicas=2, pcs_replicas=1) -> list[int]:
    """e2e/yaml/workload2.yaml: same shape, every minAvailable = 1 (sg-x minAvailable 1):
    base gang = pc-a (2, min 1) + sg-x-0 (pc-b 1/1, pc-c 3/1); scaled gang per sg-x replica >= 1."""
    out = []
    for _ in range(pcs_replicas):
        base = b.add_gang([(None, [_clq(80, 1, 2)]), (None, [_clq(80, 1, 1), _clq(80, 1, 3)])])
        out.append(base)
        for _r in range(1, pcsg_replicas):
            out.append(b.add_gang([(None, [_clq(80, 1, 1), _clq(80, 1, 3)])], base=base))
    return out


# ------------------------------------------------------------------------------------------------
# BASELINE.json configs
# ------------------------------------------------------------------------------------------------
def config_c1():
    """simple1.yaml on 4 kind fake nodes (kind-up.sh:303-316), 1 level (host)."""
    nodes = kwok_nodes(4, [1], cpu_milli=64000, mem_mib=524288, gpu=0, pods=110)
    b = T.GangTableBuilder()
    c = lambda n: dict(cpu=10, min=n)  # noqa: E731  -- 10m CPU each, MinReplicas = replicas after defaulting
    b.add_gang([(None, [c(3), c(2)]), (None, [c(2), c(2)])])
    return dict(name="C1", n_levels=1, nodes=nodes, tables=b.build())


def config_c2(n=1000, g=100, seed=SEED_BASE + 2):
    """1k nodes / 100 gangs, flat topology, no constraints, 1-3 cliques, replicas 1-8, gpu in {1,2,4,8}."""
    nodes = kwok_nodes(n, [1])
    pre_use(nodes, seed, 75)
    b = T.GangTableBuilder()
    ncl = _rand_below(seed, 1, g, 3) + 1
    for gi in range(g):
        cl = []
        for c in range(int(ncl[gi])):
            r = int(_rand_below(seed, 100 + c, g, 8)[gi]) + 1
            gp = 1 << int(_rand_below(seed, 200 + c, g, 4)[gi])
            cl.append(dict(cpu=1000 * gp, mem=8192 * gp, gpu=gp, min=r))
        b.add_gang([(None, cl)])
    return dict(name="C2", n_levels=1, nodes=nodes, tables=b.build())


def config_c3(n=10000, g=1000, seed=SEED_BASE + 3):
    """10k nodes / 1k gangs, 3 levels block 126 / rack 18 / host 1; prefill+decode PodCliques:
    gang Required=block, one scope per role Required=rack, leader cliques Required=host
    (shape of docs/proposals/244-topology-aware-scheduling/README.md:752-830)."""
    nodes = kwok_nodes(n, [126, 18, 1])
    pre_use(nodes, seed, 75)
    b = T.GangTableBuilder()
    gp = _rand_below(seed, 1, g, 4)
    for gi in range(g):
        w = 1 << int(gp[gi])
        lead = dict(cpu=2000, mem=16384, gpu=1, min=1, level=2)
        b.add_gang([
            (1, [lead, dict(cpu=1000 * w, mem=8192 * w, gpu=w, min=4)]),  # prefill leader + 4 workers
            (1, [lead, dict(cpu=1000 * w, mem=8192 * w, gpu=w, min=2)]),  # decode leader + 2 workers
        ], level=0)
    return dict(name="C3", n_levels=3, nodes=nodes, tables=b.build())


def config_c4(n=50000, g=10000, seed=SEED_BASE + 4, max_used_pct=90):
    """50k nodes / 10k gangs, 4 levels zone 2520 / block 126 / rack 18 / host 1, 2 % cordoned,
    3 selector classes, 3 priority classes.  A quarter of the gangs are base gangs
    (router x2 + 2 scaling groups x (leader x1 + worker x4)), the rest scaled gangs (one scaling-group
    replica each) gated behind a base gang: the hierarchical PodCliqueScalingGroup structure of
    syncflow.go:189-333.  Gang Required=block, scaling-group scope Required=rack, leaders Required=host.
    Every PodGang of a PodCliqueSet carries the set's PriorityClassName (podgang/podgang.go:158), so a
    scaled gang has its base gang's priority."""
    nodes = kwok_nodes(n, [2520, 126, 18, 1])
    pre_use(nodes, seed, max_used_pct)
    cls = _rand_below(seed, 20, n, 3)
    nodes["flags"] = T.NODE_SCHEDULABLE | (cls.astype(np.uint32) << T.NODE_CLASS_SHIFT)
    cordon(nodes, np.nonzero(_rand_below(seed, 21, n, 50) == 0)[0])
    b = T.GangTableBuilder()
    n_base = g // 4
    gp = _rand_below(seed, 1, g, 4)
    pr = _rand_below(seed, 2, g, 3)
    cm = _rand_below(seed, 3, g, 4)  # 0: any class, 1..3: exactly one class
    for gi in range(g):
        w = 1 << int(gp[gi])
        mask = 0xFFFF if cm[gi] == 0 else (1 << int(cm[gi] - 1))
        lead = dict(cpu=2000, mem=16384, gpu=1, min=1, level=3, class_mask=mask)
        work = dict(cpu=1000 * w, mem=8192 * w, gpu=w, min=4, class_mask=mask)
        if gi < n_base:
            router = dict(cpu=4000, mem=8192, gpu=0, min=2, class_mask=mask)
            b.add_gang([(None, [router]), (2, [lead, work]), (2, [dict(lead), dict(work)])],
                       level=1, priority=int(pr[gi]))
        else:
            base = (gi - n_base) % n_base
            b.add_gang([(2, [lead, work])], level=1, priority=int(pr[base]), base=base)
    return dict(name="C4", n_levels=4, nodes=nodes, tables=b.build())


def c4_spread_groups(gangs, cliques, size=8, level=0, mode=T.SPREAD_HARD, max_skew=1):
    """Topology spread groups over a C4-style submission (grove_set_spread): its base gangs whose Required level is `level` or
    deeper, in groups of `size` by (priority, template) -- the replicas of one PodCliqueSet.  -> (T.spread_dt groups, gang_group)"""
    gang_group = np.full(len(gangs), T.NONE_U32, dtype=np.uint32)
    by_key = {}
    for g in range(len(gangs)):
        if gangs["base_gang"][g] != T.NONE_U32 or gangs["level"][g] == T.LEVEL_NONE or gangs["level"][g] < level:
            continue
        co = int(gangs["clique_off"][g]); n = int(gangs["n_cliques"][g])
        q = cliques[co: co + n]
        key = (int(gangs["priority"][g]), n, tuple(q["req_cpu_milli"]), tuple(q["req_mem_mib"]), tuple(q["req_gpu"]),
               tuple(q["min_replicas"]), tuple(q["class_mask"]), int(gangs["level"][g]))
        by_key.setdefault(key, []).append(g)
    n_groups = 0
    for key in sorted(by_key):
        members = by_key[key]
        for i in range(0, len(members), size):
            gang_group[members[i: i + size]] = n_groups
            n_groups += 1
    groups = np.zeros(n_groups, dtype=T.spread_dt)
    groups["level"], groups["mode"], groups["max_skew"] = level, mode, max_skew
    return groups, gang_group


def binpack_levels(gangs, level=None):
    """Pack levels for grove_set_binpack over a C4-style submission: every gang is a member, at its Required level, or at `level`
    when that is deeper (a gang without a Required level packs at `level`, and is no member when `level` is None)."""
    req = gangs["level"].astype(np.int64)
    if level is None:
        return np.where(req == T.LEVEL_NONE, T.LEVEL_NONE, req).astype(np.uint8)
    return np.where(req == T.LEVEL_NONE, level, np.maximum(req, level)).astype(np.uint8)


def c4_compute_domains(nodes, gangs, cliques, owned=0.5, seed=SEED_BASE + 417):
    """ComputeDomains for grove_set_compute_domains over a C4-style submission, as Grove's auto-MNNVL makes them: one CD per PCS
    replica, i.e. per base gang and the gangs scaled from it, with every GPU clique enrolled; the CD id is the base gang's index.
    A share `owned` of the pre-used nodes (fewer free GPUs than the fullest node) is held by CDs of replicas that already run,
    ids from len(gangs) up.  -> (cd [Q], owner0 [N])"""
    cd = np.full(len(cliques), T.CD_NONE, dtype=np.uint32)
    for g in range(len(gangs)):
        b = int(gangs["base_gang"][g])
        co, nq = int(gangs["clique_off"][g]), int(gangs["n_cliques"][g])
        q = np.arange(co, co + nq)
        cd[q[cliques["req_gpu"][q] > 0]] = g if b == T.NONE_U32 else b
    rng = np.random.default_rng(seed)
    used = nodes["free_gpu"] < nodes["free_gpu"].max()
    owner0 = np.full(len(nodes), T.CD_NONE, dtype=np.uint32)
    pick = used & (rng.random(len(nodes)) < owned)
    owner0[pick] = len(gangs) + rng.integers(0, max(1, len(gangs) // 4), int(pick.sum()))
    return cd, owner0


def config_c4_large(n=50000, g=10000, n_large=24, seed=SEED_BASE + 44, max_used_pct=90):
    """C4 (config_c4) plus `n_large` PodGangs of 256-2048 pods, for grove_submit_gangs_wide: a leader (Required host) and a
    worker PodGroup of 255-2047 one-GPU pods under a Required zone with a Preferred block, priorities drawn from C4's three
    classes so that they interleave with the ordinary gangs.  tables = (gangs, cliques, counts, scopes); `ordinary` = the C4
    part alone, as grove_submit_gangs takes it."""
    base = config_c4(n=n, g=g, seed=seed, max_used_pct=max_used_pct)
    og, oc, os_ = base["tables"]
    b = T.GangTableBuilder()
    size = 256 + _rand_below(seed, 30, n_large, T.MAX_WIDE_GANG_PODS - 256 + 1)
    pr = _rand_below(seed, 31, n_large, 3)
    for i in range(n_large):
        lead = dict(cpu=2000, mem=16384, gpu=1, min=1, level=3)
        work = dict(cpu=1000, mem=8192, gpu=1, min=int(size[i]) - 1)
        b.add_gang([(None, [lead, work])], level=0, preferred=1, priority=int(pr[i]))
    lg, lc, lcnt, ls = b.build_wide()
    lg["clique_off"] += len(oc)
    lg["scope_off"] += len(os_)
    counts = np.zeros(len(oc) + len(lc), dtype=T.clique_count_dt)
    counts["min_replicas"][: len(oc)], counts["replicas"][: len(oc)] = oc["min_replicas"], oc["replicas"]
    counts[len(oc):] = lcnt
    tables = (np.concatenate([og, lg]), np.concatenate([oc, lc]), counts, np.concatenate([os_, ls]))
    return dict(name="C4+large", n_levels=4, nodes=base["nodes"], tables=tables, ordinary=base["tables"])


class ChurnC5:
    """BASELINE.json config 5: steady-state churn on the C4 cluster.  Every tick (100 ms of scheduler
    time) `arrivals` new PodGangs join the gangs still pending from earlier ticks, one cycle runs, and
    the pods of ~`release_pct` % of the running gangs finish (their resources return to their nodes
    through grove_update_nodes).  Deterministic from the seed; the oracle and the engine are driven
    with identical inputs tick by tick."""

    def __init__(self, n=50000, arrivals=100, seed=SEED_BASE + 5, release_pct=1, max_used_pct=60):
        self.n, self.arrivals, self.seed, self.release_pct = n, arrivals, seed, release_pct
        self.nodes = kwok_nodes(n, [2520, 126, 18, 1])
        pre_use(self.nodes, seed, max_used_pct)
        self.n_levels = 4
        self.tick = 0
        self.pending = []   # gang specs carried over: (uid, scopes, level, priority)
        self.running = []   # (uid, placements ndarray, clique table rows) of admitted gangs
        self.next_uid = 0

    def _new_gangs(self):
        t = self.tick
        w_ = _rand_below(self.seed + t, 1, self.arrivals, 4)
        pr = _rand_below(self.seed + t, 2, self.arrivals, 3)
        out = []
        for i in range(self.arrivals):
            w = 1 << int(w_[i])
            lead = dict(cpu=2000, mem=16384, gpu=1, min=1, level=3)
            work = dict(cpu=1000 * w, mem=8192 * w, gpu=w, min=4)
            out.append((self.next_uid, [(2, [lead, work])], 1, int(pr[i])))
            self.next_uid += 1
        return out

    def begin_tick(self):
        """-> (gang specs of this tick in submission order, packed tables)"""
        specs = self.pending + self._new_gangs()
        b = T.GangTableBuilder()
        for uid, scopes, level, prio in specs:
            b.add_gang(scopes, level=level, priority=prio, anchor=int(splitmix64(self.seed, np.array([uid]))[0] % np.uint64(self.n)))
        return specs, b.build()

    def end_tick(self, specs, tables, status, placements, nodes_after):
        """Book-keeping after the cycle: rejected gangs stay pending, admitted ones run; then some
        running gangs finish.  Returns (idx, recs) for grove_update_nodes and the new node table."""
        g, c, s = tables
        self.pending = []
        for i, sp in enumerate(specs):
            st = int(status["state"][i])
            if st == T.GANG_ADMITTED:
                pl = placements[status["placement_off"][i]: status["placement_off"][i] + status["n_pods"][i]]
                self.running.append((sp[0], pl["node"].copy(), c[pl["clique"]].copy()))
            else:
                self.pending.append(sp)
        nodes = nodes_after.copy()
        touched = set()
        keep = []
        for k, (uid, pnodes, pcl) in enumerate(self.running):
            h = int(splitmix64(self.seed * 7919 + self.tick, np.array([uid]))[0] % np.uint64(100))
            if h < self.release_pct:
                np.add.at(nodes["free_cpu_milli"], pnodes, pcl["req_cpu_milli"])
                np.add.at(nodes["free_mem_mib"], pnodes, pcl["req_mem_mib"])
                np.add.at(nodes["free_gpu"], pnodes, pcl["req_gpu"])
                np.add.at(nodes["free_pods"], pnodes, 1)
                touched.update(pnodes.tolist())
            else:
                keep.append((uid, pnodes, pcl))
        self.running = keep
        self.tick += 1
        idx = np.array(sorted(touched), dtype=np.uint32)
        self.nodes = nodes
        return idx, nodes[idx]


CONFIGS = {"C1": config_c1, "C2": config_c2, "C3": config_c3, "C4": config_c4}


def c4_queues(gangs, cliques, share=0.3):
    """eight leaf queues under two parents (queue indices 0-1 the parents, 2-9 the leaves) for the gangs of a C4 submission: a base
    gang and its scaled gangs share a leaf (by base index mod 8).  Each leaf's GPU limit is `share` of its members' MinReplicas GPU
    demand, each parent's 90 % of the sum of its leaves'; nothing runs yet -> (tables.queue_dt[10], gang_queue).  C4's cluster
    admits about 60 % of the gangs by itself, so at one half no limit binds; at 0.3 the limits turn away about one gang in six."""
    G = len(gangs)
    base = gangs["base_gang"].astype(np.int64)
    gq = (2 + np.where(base == T.NONE_U32, np.arange(G), base) % 8).astype(np.uint32)
    gpu = cliques["min_replicas"].astype(np.int64) * cliques["req_gpu"].astype(np.int64)
    per_gang = np.array([gpu[int(o): int(o) + int(n)].sum() for o, n in zip(gangs["clique_off"], gangs["n_cliques"])], dtype=np.int64)
    need = np.bincount(gq, weights=per_gang, minlength=10)
    q = np.zeros(10, dtype=T.queue_dt)
    q["limit"] = T.QUEUE_UNLIMITED
    q["parent"][:2] = T.NONE_U32
    q["parent"][2:] = np.arange(8) // 4
    q["limit"][2:, 2] = (share * need[2:]).astype(np.uint64)
    q["limit"][0, 2] = int(share * need[2:6].sum() * 0.9)
    q["limit"][1, 2] = int(share * need[6:10].sum() * 0.9)
    return q, gq



def queue_running(tables, queues, gang_queue, placements, status, seed=0, boost=2, share=0.5):
    """A running-gang layout for a queue set (synth.c4_queues): the gangs a queue cycle over `tables` admitted (its placements and
    statuses) run in their queues at priorities 0-2, and the submission is the same gangs again at priorities 0-2, about `share` of
    them (and every third base gang, with its scaled gangs) `boost` higher.  Each queue's `used` becomes what its running gangs
    hold plus, at random, a little that is not handed in (0.5 cores, 1 GiB, one GPU).
    -> (tables, queues, gang_queue, running, holdings, running_queue) for grove_run_cycle_preempt_queues"""
    g, c, s = tables
    rng = np.random.default_rng(seed)
    run, hold, rq = [], [], []
    for i in np.nonzero(status["state"] == T.GANG_ADMITTED)[0]:
        per = {}
        for e in placements[status["placement_off"][i]: status["placement_off"][i] + status["n_pods"][i]]:
            q = c[int(e["clique"])]
            u = per.setdefault(int(e["node"]), [0, 0, 0, 0])
            u[0] += int(q["req_cpu_milli"]); u[1] += int(q["req_mem_mib"]); u[2] += int(q["req_gpu"]); u[3] += 1
        run.append((int(rng.integers(0, 3)), len(hold), len(per), 0))
        hold += [(n, *u) for n, u in per.items()]
        rq.append(int(gang_queue[i]))
    running = np.array(run, dtype=T.running_dt) if run else np.zeros(0, dtype=T.running_dt)
    holdings = np.array(hold, dtype=T.holding_dt) if hold else np.zeros(0, dtype=T.holding_dt)
    running_queue = np.array(rq, dtype=np.uint32)
    q2 = np.asarray(queues, dtype=T.queue_dt).copy()
    q2["used"] = 0
    for r in range(len(running)):
        if running_queue[r] != T.NONE_U32:
            h = holdings[int(running["holding_off"][r]): int(running["holding_off"][r]) + int(running["n_holdings"][r])]
            q2["used"][int(running_queue[r])] += np.array([h["cpu_milli"].astype(np.uint64).sum(), h["mem_mib"].astype(np.uint64).sum(),
                                                           h["gpu"].astype(np.uint64).sum()], dtype=np.uint64)
    q2["used"] += rng.integers(0, 2, (len(q2), 3)).astype(np.uint64) * np.array([500, 1024, 1], np.uint64)
    g2 = g.copy()
    for i in range(len(g2)):
        b = int(g2["base_gang"][i])
        root = i if b == T.NONE_U32 else b
        g2["priority"][i] = int(rng.integers(0, 3)) + (boost if rng.random() < share or root % 3 == 0 else 0)
    for i in range(len(g2)):   # a scaled gang keeps its base gang's priority
        b = int(g2["base_gang"][i])
        if b != T.NONE_U32:
            g2["priority"][i] = g2["priority"][b]
    return (g2, c, s), q2, np.asarray(gang_queue, dtype=np.uint32), running, holdings, running_queue
