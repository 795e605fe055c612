"""The oracle against the only placement OUTCOMES the reference pins: the live-cluster e2e suites
(ai-dynamo/grove operator/e2e/tests/gang_scheduling_test.go GS1-GS12, topology_test.go TAS2-TAS17),
restated as properties over synthetic snapshots of the same shape (150 MiB nodes, 80/40/20/500 MiB
pods, zone/block/rack/host labels).  Node-level choices below these properties are unpinned
(DESIGN.md "Oracle").
"""
import numpy as np
import pytest

from grove_b200 import synth, tables as T

A = synth.AGENT
ZONE, BLOCK, RACK, HOST = 0, 1, 2, 3


def run(oracle, nodes, b, **kw):
    g, c, s = b.build()
    return oracle.run_cycle(nodes, synth.E2E_LEVELS, g, c, s, **kw), (g, c, s)


def clq(mem, n, level=None, replicas=None):
    return dict(mem=mem, min=n, replicas=n if replicas is None else replicas, level=level, class_mask=A)


def doms(nodes, pl, level):
    return set(int(nodes["dom"][int(n), level]) for n in pl["node"])


def pods_of(r, tabs, gang, clique_rel=None):
    g, c, s = tabs
    st = r["status"][gang]
    pl = r["placements"][st["placement_off"]: st["placement_off"] + st["n_pods"]]
    if clique_rel is not None:
        pl = pl[pl["clique"] == g["clique_off"][gang] + clique_rel]
    return pl


# ---------------------------------------------------------------- gang scheduling (GS) ----------
def test_gs1_all_or_nothing(oracle):
    """gang_scheduling_test.go:34-74: 9 schedulable nodes -> 0 of 10 pods; 10 -> 10 on 10 distinct nodes."""
    b = T.GangTableBuilder(); synth.workload1(b)
    r, _ = run(oracle, synth.e2e_cluster(10, cordoned=1), b)
    assert r["status"]["state"][0] == T.GANG_REJECTED and len(r["placements"]) == 0
    assert np.array_equal(r["nodes_after"], synth.e2e_cluster(10, cordoned=1))  # nothing partially bound
    b = T.GangTableBuilder(); synth.workload1(b)
    r, _ = run(oracle, synth.e2e_cluster(10), b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    assert len(r["placements"]) == 10 and len(set(r["placements"]["node"])) == 10


@pytest.mark.parametrize("free,scaled_ok", [(10, 0), (14, 1), (18, 2)])
def test_gs2_scaled_gangs_are_their_own_gangs(oracle, free, scaled_ok):
    """gang_scheduling_test.go:85-275: base gang of 10 is all-or-nothing; each further sg-x replica
    (4 pods) is admitted as its own gang when capacity appears."""
    b = T.GangTableBuilder(); ids = synth.workload1(b, pcsg_replicas=4)
    r, _ = run(oracle, synth.e2e_cluster(28, cordoned=28 - free), b)
    st = r["status"]["state"]
    assert st[ids[0]] == T.GANG_ADMITTED
    assert int((st[ids[1:]] == T.GANG_ADMITTED).sum()) == scaled_ok
    assert len(r["placements"]) == 10 + 4 * scaled_ok


def test_gs_new_pcs_replica_is_a_separate_gang(oracle):
    b = T.GangTableBuilder(); ids = synth.workload1(b, pcs_replicas=2)
    r, _ = run(oracle, synth.e2e_cluster(28, cordoned=12), b)  # 16 free: one replica (10) fits, two (20) do not
    assert sorted(r["status"]["state"][ids].tolist()) == [T.GANG_ADMITTED, T.GANG_REJECTED]
    assert len(r["placements"]) == 10


@pytest.mark.parametrize("free,placed", [(2, 0), (3, 3), (10, 10)])
def test_gs5_min_replicas_then_best_effort(oracle, free, placed):
    """gang_scheduling_test.go:285-337 (workload2, every minAvailable 1): 2 free nodes -> 0 pods;
    3 -> exactly sum(MinReplicas)=3 (pc-a 1, pc-b 1, pc-c 1); 10 -> all 10 (surplus is best effort)."""
    b = T.GangTableBuilder(); ids = synth.workload2(b)
    r, tabs = run(oracle, synth.e2e_cluster(10, cordoned=10 - free), b)
    assert len(r["placements"]) == placed
    if free == 3:
        assert [len(pods_of(r, tabs, ids[0], c)) for c in range(3)] == [1, 1, 1]
        assert r["status"]["state"][ids[1]] == T.GANG_REJECTED  # scaled gang needs 2 more nodes
    if free == 2:
        assert r["status"]["state"][ids[0]] == T.GANG_REJECTED
        assert r["status"]["state"][ids[1]] == T.GANG_BASE_REJECTED  # gated behind the base gang


def test_gs6_scaled_gang_minimum_is_two(oracle):
    """gang_scheduling_test.go:340-352: a scaled sg-x replica of workload2 needs pc-b 1 + pc-c 1 = 2 nodes."""
    b = T.GangTableBuilder(); ids = synth.workload2(b, pcsg_replicas=3)
    # base takes 6 pods on 6 nodes when it can; give 6 + 1 nodes: second scaled gang cannot get its 2
    r, _ = run(oracle, synth.e2e_cluster(10, cordoned=1), b)  # 9 free: base 6 (with surplus) ... scaled need >= 2 each
    st = r["status"]["state"]
    assert st[ids[0]] == T.GANG_ADMITTED
    placed_scaled = [int(r["status"]["n_pods"][i]) for i in ids[1:]]
    assert all(p == 0 or p >= 2 for p in placed_scaled)


def test_gated_gangs_are_skipped(oracle):
    """pods still carrying grove.io/podgang-pending-creation never reach a scheduler (pod.go:70,164)."""
    b = T.GangTableBuilder()
    b.add_gang([(None, [clq(80, 2)])], gated=True)
    b.add_gang([(None, [clq(80, 2)])])
    r, _ = run(oracle, synth.e2e_cluster(4), b)
    assert r["status"]["state"].tolist() == [T.GANG_GATED_SKIP, T.GANG_ADMITTED]


def test_priority_wins_conflicts(oracle):
    b = T.GangTableBuilder()
    lo = b.add_gang([(None, [clq(80, 3)])], priority=0, anchor=0)
    hi = b.add_gang([(None, [clq(80, 3)])], priority=10, anchor=0)
    r, _ = run(oracle, synth.e2e_cluster(4), b)  # only one gang of 3 fits on 4 one-pod nodes
    assert r["status"]["state"][hi] == T.GANG_ADMITTED and r["status"]["state"][lo] == T.GANG_REJECTED


# ---------------------------------------------------------------- topology (TAS) ----------------
def test_tas2_independent_clique_constraints(oracle):
    """topology_test.go:159-216: worker-rack x3 share a rack, worker-block x4 share a block."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    b.add_gang([(None, [clq(20, 3, level=RACK)]), (None, [clq(20, 4, level=BLOCK)])])
    r, tabs = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and len(r["placements"]) == 7
    assert len(doms(nodes, pods_of(r, tabs, 0, 0), RACK)) == 1
    assert len(doms(nodes, pods_of(r, tabs, 0, 1), BLOCK)) == 1


@pytest.mark.parametrize("level", [RACK, ZONE, BLOCK])
def test_tas3_6_gang_level_constraint(oracle, level):
    """topology_test.go:218-274, 398-450: every pod of the gang shares the PCS-level domain."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    b.add_gang([(None, [clq(80, 2)]), (None, [clq(80, 1)]), (None, [clq(80, 1)])], level=level)
    r, tabs = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    assert len(doms(nodes, pods_of(r, tabs, 0), level)) == 1


def test_tas4_scope_only_constraint(oracle):
    """topology_test.go:276-340: each PCSG replica (a group config) shares a rack; routers unconstrained."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    b.add_gang([(None, [clq(80, 2)]), (RACK, [clq(80, 1)]), (RACK, [clq(80, 1)])])
    r, tabs = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and len(r["placements"]) == 4
    for c in (1, 2):
        assert len(doms(nodes, pods_of(r, tabs, 0, c), RACK)) == 1


def test_tas5_host_level(oracle):
    """topology_test.go:342-396: 2 x 40 MiB pods with packDomain host land on the same node."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(40, 2, level=HOST)])])
    r, tabs = run(oracle, nodes, b)
    assert len(set(pods_of(r, tabs, 0)["node"])) == 1 and r["status"]["n_pods"][0] == 2
    assert r["status"]["score_num"][0] >= 1


def test_tas7_no_constraint(oracle):
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(80, 1)]) for _ in range(4)])
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and len(r["placements"]) == 4


def _tas8(b, level=BLOCK):
    return b.add_gang([(RACK, [clq(40, 2, level=HOST), clq(40, 2, level=HOST)]),
                       (RACK, [clq(40, 2, level=HOST), clq(40, 2, level=HOST)])], level=level)


def test_tas8_full_hierarchy(oracle):
    """topology_test.go:501-578 (tas-hierarchy.yaml): PCS block -> PCSG replica rack -> PCLQ host on 8
    nodes: 4 host groups, 2 rack groups, 1 block."""
    nodes = synth.e2e_cluster(8)
    b = T.GangTableBuilder(); _tas8(b)
    r, tabs = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and r["status"]["n_pods"][0] == 8
    for c in range(4):
        assert len(set(pods_of(r, tabs, 0, c)["node"])) == 1
    for cs in ((0, 1), (2, 3)):
        pl = np.concatenate([pods_of(r, tabs, 0, c) for c in cs])
        assert len(doms(nodes, pl, RACK)) == 1
    assert len(doms(nodes, pods_of(r, tabs, 0), BLOCK)) == 1


def test_tas9_gang_block_clique_host(oracle):
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(40, 2, level=HOST)])], level=BLOCK)
    r, tabs = run(oracle, nodes, b)
    assert len(set(pods_of(r, tabs, 0)["node"])) == 1


def test_tas10_scaled_gangs_carry_the_constraint(oracle):
    """topology_test.go:628-708: 3 PCSG replicas with rack constraint (base: minAvailable 1, 2 scaled
    gangs); each replica's 2 pods share a rack and, with the PCS-level rack constraint, its gang's rack."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    base = b.add_gang([(RACK, [clq(80, 2)])], level=RACK)
    sc = [b.add_gang([(RACK, [clq(80, 2)])], level=RACK, base=base) for _ in range(2)]
    r, tabs = run(oracle, nodes, b)
    assert all(r["status"]["state"][[base] + sc] == T.GANG_ADMITTED) and len(r["placements"]) == 6
    for g in [base] + sc:
        assert len(doms(nodes, pods_of(r, tabs, g), RACK)) == 1


def test_tas11_scope_rack_clique_host_no_gang_constraint(oracle):
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    b.add_gang([(RACK, [clq(40, 2, level=HOST)]), (RACK, [clq(40, 2, level=HOST)])])
    r, tabs = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    for c in (0, 1):
        assert len(set(pods_of(r, tabs, 0, c)["node"])) == 1


def test_tas12_large_scaling_ratio(oracle):
    """topology_test.go:767-860: replicas 10, minAvailable 3, PCSG host constraint, PCS block: base gang
    holds 3 replicas x 2 pods, 7 scaled gangs x 2 pods; every replica on one host, every gang in one block."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    base = b.add_gang([(HOST, [clq(40, 2)]) for _ in range(3)], level=BLOCK)
    sc = [b.add_gang([(HOST, [clq(40, 2)])], level=BLOCK, base=base) for _ in range(7)]
    r, tabs = run(oracle, nodes, b)
    assert all(r["status"]["state"] == T.GANG_ADMITTED) and len(r["placements"]) == 20
    for c in range(3):
        assert len(set(pods_of(r, tabs, base, c)["node"])) == 1
    for g in [base] + sc:
        assert len(doms(nodes, pods_of(r, tabs, g), BLOCK)) == 1
    for g in sc:
        assert len(set(pods_of(r, tabs, g)["node"])) == 1


def test_tas13_unsatisfiable_constraint_places_nothing(oracle):
    """topology_test.go:862-920 (tas-insuffic.yaml): 10 x 500 MiB pods, rack constraint, 150 MiB nodes:
    0 placed, no partial assignment."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(500, 10)])], level=RACK)
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_REJECTED and len(r["placements"]) == 0
    assert np.array_equal(r["nodes_after"], nodes)
    # also unsatisfiable by count alone: 10 one-per-node pods in a 7-node rack
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(80, 10)])], level=RACK)
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_REJECTED and len(r["placements"]) == 0


def test_tas14_each_pcs_replica_in_one_rack(oracle):
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    for _ in range(2):
        b.add_gang([(None, [clq(80, 2)])], level=RACK)
    r, tabs = run(oracle, nodes, b)
    assert all(r["status"]["state"] == T.GANG_ADMITTED)
    for g in (0, 1):
        assert len(doms(nodes, pods_of(r, tabs, g), RACK)) == 1


@pytest.mark.parametrize("pcs_replicas", [1, 2])
def test_tas15_16_disaggregated_multi_pcsg(oracle, pcs_replicas):
    """topology_test.go:977-1190: PCS block; decoder and prefill PCSGs (2 replicas, minAvailable 1, rack
    constraint; TAS16 adds a host constraint on the prefill worker) + 2 standalone routers.  Base gang:
    router + replica 0 of each PCSG; one scaled gang per replica 1."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder(); bases, scaled = [], []
    for _ in range(pcs_replicas):
        pw = HOST if pcs_replicas == 2 else None
        base = b.add_gang([(None, [clq(40, 2)]), (RACK, [clq(40, 1), clq(40, 1)]),
                           (RACK, [clq(40, 1), clq(40, 1, level=pw)])], level=BLOCK)
        bases.append(base)
        scaled.append(b.add_gang([(RACK, [clq(40, 1), clq(40, 1)])], level=BLOCK, base=base))
        scaled.append(b.add_gang([(RACK, [clq(40, 1), clq(40, 1, level=pw)])], level=BLOCK, base=base))
    r, tabs = run(oracle, nodes, b)
    assert all(r["status"]["state"] == T.GANG_ADMITTED) and len(r["placements"]) == 10 * pcs_replicas
    for g in bases:
        assert len(doms(nodes, pods_of(r, tabs, g), BLOCK)) == 1
        for cs in ((1, 2), (3, 4)):
            pl = np.concatenate([pods_of(r, tabs, g, c) for c in cs])
            assert len(doms(nodes, pl, RACK)) == 1
    for g in scaled:
        assert len(doms(nodes, pods_of(r, tabs, g), RACK)) == 1


def test_tas17_nodes_without_the_label_are_not_candidates(oracle):
    """topology_test.go:1192-1370 / GREP-244 README.md:65: a gang packed on a level only lands on nodes
    that carry that level's label."""
    nodes = synth.e2e_cluster(28)
    nodes["dom"][14:, RACK] = T.DOM_ABSENT  # second half lacks the rack label (and everything below it)
    b = T.GangTableBuilder()
    for _ in range(6):
        b.add_gang([(None, [clq(80, 2)])], level=RACK)
    r, tabs = run(oracle, nodes, b)
    assert (r["placements"]["node"] < 14).all()
    assert int((r["status"]["state"] == T.GANG_ADMITTED).sum()) == 6  # 14 labelled one-pod nodes, 2 racks of 7: 3 gangs each
    # block-level gangs may still use the unlabelled-rack half
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(80, 14)])], level=BLOCK, anchor=20)
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and (r["placements"]["node"] >= 14).all()


def test_kwok_label_arithmetic_is_not_a_tree(oracle):
    """kwok.py:64-68 with constants.py:65-67 (zone 28 / block 20 / rack 7): 20 does not divide 28, so
    block-1 straddles zone-0 and zone-1; path semantics splits it and reports it."""
    nodes = synth.kwok_nodes(56, [28, 20, 7, 1])
    perm, dom, ndom, non_tree = oracle.topology(nodes, 4)
    assert non_tree > 0
    assert ndom[1] > 56 // 20 + 1  # more tree domains than raw block ids
    nodes = synth.kwok_nodes(56, [28, 14, 7, 1])
    assert oracle.topology(nodes, 4)[3] == 0


def test_placement_score_range_and_meaning(oracle):
    """podgang.go:187-189: 1.0 = the best possible placement.  Best possible = every pack constraint held at the level
    it asked for (Preferred if set, else Required), wherever in the cluster the gang landed."""
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    same_host = b.add_gang([(None, [clq(40, 2, level=HOST)])], anchor=3)
    far = b.add_gang([(None, [clq(40, 2, level=HOST)])], anchor=27)          # perfectly packed far from anybody else: still 1.0
    loose = b.add_gang([(None, [clq(80, 20)])], anchor=3)                     # nothing asked: 1.0
    pref_ok = b.add_gang([(None, [clq(40, 3)])], preferred=RACK, anchor=10)   # fits the Preferred rack: 1.0
    pref_wide = b.add_gang([(None, [clq(80, 6)])], preferred=HOST, level=BLOCK, anchor=14)  # one pod per node: falls back
    r, _ = run(oracle, nodes, b)
    st = r["status"]
    assert (st["state"] == T.GANG_ADMITTED).all()
    for gi in (same_host, far, loose, pref_ok):
        assert st["score_num"][gi] == st["score_den"][gi] > 0
    assert 0 < st["score_num"][pref_wide] < st["score_den"][pref_wide]
    assert st["level"][pref_wide] < HOST and st["level"][pref_ok] == RACK
