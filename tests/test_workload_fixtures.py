"""The reference's own workload files, end to end: tests/golden/workloads.json (extracted from
ai-dynamo/grove operator/e2e/yaml/*.yaml and samples/simple/simple1.yaml by tests/golden/make_workload_fixtures.py)
-> producer (grove_b200/ingest.podgangs_from_pcs, the Python counterpart of ComputeExpectedPodGangs) -> PodGang
manifests -> packed tables -> oracle, with the outcome each e2e suite asserts for its file."""
import json
import os

import numpy as np
import pytest

from grove_b200 import ingest, synth, tables as T

HERE = os.path.dirname(os.path.abspath(__file__))
FX = json.load(open(os.path.join(HERE, "golden", "workloads.json")))
LEVELS = [("zone", "topology.kubernetes.io/zone"), ("block", "topology.kubernetes.io/block"),
          ("rack", "topology.kubernetes.io/rack"), ("host", "kubernetes.io/hostname")]
ZONE, BLOCK, RACK, HOST = range(4)


def pcs_of(name):
    (p,) = FX[name]
    return p


# ---- the producer, on the reference's unit-test vectors (syncflow_test.go:740-953) ---------------------------
def _pcs(replicas, cliques, groups=()):
    return dict(name="test-pcs", replicas=replicas, packDomain=None,
                cliques=[dict(name=n, replicas=r, minAvailable=m, requests={}, packDomain=None) for n, r, m in cliques],
                podCliqueScalingGroups=[dict(name=n, replicas=r, minAvailable=m, cliqueNames=list(cn), packDomain=None) for n, r, m, cn in groups])


PRODUCER = [
    ("standalone PCLQs only", _pcs(2, [("worker", 3, 2)]), ["test-pcs-0", "test-pcs-1"], []),
    ("PCSG with minAvailable=1", _pcs(1, [("sg-worker", 2, 2)], [("scaling-group", 3, 1, ["sg-worker"])]), ["test-pcs-0"],
     ["test-pcs-0-scaling-group-0", "test-pcs-0-scaling-group-1"]),
    ("mixed standalone PCLQ and PCSG", _pcs(1, [("standalone", 2, 1), ("scalable", 3, 2)], [("sg", 4, 2, ["scalable"])]), ["test-pcs-0"],
     ["test-pcs-0-sg-0", "test-pcs-0-sg-1"]),
    ("multiple PCS replicas with PCSG", _pcs(2, [("worker", 2, 1)], [("worker-sg", 2, 1, ["worker"])]), ["test-pcs-0", "test-pcs-1"],
     ["test-pcs-0-worker-sg-0", "test-pcs-1-worker-sg-0"]),
    ("PCSG with minAvailable equals replicas", _pcs(1, [("worker", 2, 2)], [("sg", 2, 2, ["worker"])]), ["test-pcs-0"], []),
    ("multiple PCSGs in one PCS replica", _pcs(1, [("worker-a", 2, 2), ("worker-b", 2, 2)], [("sg-a", 3, 1, ["worker-a"]), ("sg-b", 2, 1, ["worker-b"])]),
     ["test-pcs-0"], ["test-pcs-0-sg-a-0", "test-pcs-0-sg-a-1", "test-pcs-0-sg-b-0"]),
    ("multiple cliques in one PCSG", _pcs(1, [("worker", 2, 2), ("helper", 1, 1)], [("sg", 3, 1, ["worker", "helper"])]), ["test-pcs-0"],
     ["test-pcs-0-sg-0", "test-pcs-0-sg-1"]),
]


@pytest.mark.parametrize("name,pcs,base,scaled", PRODUCER, ids=[p[0] for p in PRODUCER])
def test_producer_vectors(name, pcs, base, scaled):
    gangs, _, base_of = ingest.podgangs_from_pcs(pcs, LEVELS)
    names = [g["metadata"]["name"] for g in gangs]
    assert len(names) == len(base) + len(scaled)
    assert sorted(n for n in names if n not in base_of) == sorted(base)
    assert sorted(base_of) == sorted(scaled)
    for g in gangs:   # podgang.go:165-186: MinReplicas = minAvailable, PodReferences sorted by name
        for pg in g["spec"]["podgroups"]:
            refs = [r["name"] for r in pg["podReferences"]]
            assert refs == sorted(refs) and 0 <= pg["minReplicas"] <= len(refs)


def test_topology_keys_land_where_the_reference_puts_them():
    """syncflow_test.go:965-1420 in short: PCS constraint -> PodGang, PCSG constraint -> one group config per base
    replica and the scaled PodGang's own constraint (PCS's if the PCSG has none), PCLQ constraint -> PodGroup;
    TAS disabled or an unknown domain -> nothing."""
    gangs, _, base_of = ingest.podgangs_from_pcs(pcs_of("e2e/yaml/tas-hierarchy.yaml"), LEVELS)
    (g,) = gangs
    assert g["spec"]["topologyConstraint"]["packConstraint"]["required"] == LEVELS[BLOCK][1]
    assert [c["topologyConstraint"]["packConstraint"]["required"] for c in g["spec"]["topologyConstraintGroupConfigs"]] == [LEVELS[RACK][1]] * 2
    assert all(p["topologyConstraint"]["packConstraint"]["required"] == LEVELS[HOST][1] for p in g["spec"]["podgroups"])
    gangs, _, base_of = ingest.podgangs_from_pcs(pcs_of("e2e/yaml/tas-pcsg-scale.yaml"), LEVELS)
    assert [x["spec"]["topologyConstraint"]["packConstraint"]["required"] for x in gangs] == [LEVELS[BLOCK][1], LEVELS[RACK][1], LEVELS[RACK][1]]
    gangs, _, _ = ingest.podgangs_from_pcs(pcs_of("e2e/yaml/tas-large-scale.yaml"), LEVELS)   # PCSG without a constraint: scaled gangs inherit the PCS's
    assert len(gangs) == 8 and all(x["spec"]["topologyConstraint"]["packConstraint"]["required"] == LEVELS[BLOCK][1] for x in gangs)
    gangs, _, _ = ingest.podgangs_from_pcs(pcs_of("e2e/yaml/tas-hierarchy.yaml"), LEVELS, tas_enabled=False)
    assert "topologyConstraint" not in gangs[0]["spec"] and "topologyConstraintGroupConfigs" not in gangs[0]["spec"]
    gangs, _, _ = ingest.podgangs_from_pcs(pcs_of("e2e/yaml/tas-hierarchy.yaml"), LEVELS[:1] + LEVELS[2:])   # no "block" level any more
    assert "topologyConstraint" not in gangs[0]["spec"]


# ---- the synthetic workload shapes used all over the test-suite are the reference's files ----------------------
@pytest.mark.parametrize("wl,path", [(1, "e2e/yaml/workload1.yaml"), (2, "e2e/yaml/workload2.yaml")])
def test_synth_workloads_are_the_reference_yaml(wl, path):
    g, c, s, names, gangs = ingest.tables_from_pcs(pcs_of(path), LEVELS, class_mask=synth.AGENT)
    b = T.GangTableBuilder()
    (synth.workload1 if wl == 1 else synth.workload2)(b)
    g2, c2, s2 = b.build()
    assert len(g) == len(g2) and g["base_gang"].tolist() == g2["base_gang"].tolist()
    key = lambda cc, gg: [sorted(zip(cc["min_replicas"][o:o + n].tolist(), cc["replicas"][o:o + n].tolist(), cc["req_mem_mib"][o:o + n].tolist()))
                          for o, n in zip(gg["clique_off"], gg["n_cliques"])]
    assert key(c, g) == key(c2, g2)
    assert all(cl["agentOnly"] and cl["tolerations"] == 1 and cl["schedulerName"] == "kai-scheduler" for cl in pcs_of(path)["cliques"])


# ---- every TAS workload through the oracle, with the outcome its suite asserts ---------------------------------
def check_pack_constraints(nodes, tabs, r):
    """every unit with a Required level has all its pods in one domain of that level (topology_test.go's
    VerifyPodsInSameTopologyDomain); returns pods placed"""
    g, c, s = tabs
    for gi in range(len(g)):
        st = r["status"][gi]
        if st["state"] != T.GANG_ADMITTED:
            continue
        pl = r["placements"][st["placement_off"]: st["placement_off"] + st["n_pods"]]
        rel = pl["clique"] - g["clique_off"][gi]
        dom = lambda sel, lvl: {int(nodes["dom"][int(n), lvl]) for n in pl["node"][sel]}
        if g["level"][gi] != T.LEVEL_NONE:
            assert len(dom(slice(None), g["level"][gi])) == 1
        for si in range(g["n_scopes"][gi]):
            sc = s[g["scope_off"][gi] + si]
            members = (rel >= sc["first_clique"]) & (rel < sc["first_clique"] + sc["n_cliques"])
            if sc["level"] != T.LEVEL_NONE and members.any():
                assert len(dom(members, sc["level"])) == 1
        for ci in range(g["n_cliques"][gi]):
            lvl = c["level"][g["clique_off"][gi] + ci]
            if lvl != T.LEVEL_NONE and (rel == ci).any():
                assert len(dom(rel == ci, lvl)) == 1
    return len(r["placements"])


TAS = {   # file -> (nodes, expected running pods) as the suite sets up / waits for (topology_test.go)
    "e2e/yaml/tas-indep-clq.yaml": (28, 7),                       # TAS2 :168
    "e2e/yaml/tas-sl-pcs-only.yaml": (28, 4),                     # TAS3 :227
    "e2e/yaml/tas-sl-pcsg-only.yaml": (28, 4),                    # TAS4 :281
    "e2e/yaml/tas-host-level.yaml": (28, 2),                      # TAS5 :346
    "e2e/yaml/tas-standalone-pclq-only-pcs-zone.yaml": (28, 4),   # TAS6 :408
    "e2e/yaml/tas-no-constraint.yaml": (28, 4),                   # TAS7 :456
    "e2e/yaml/tas-hierarchy.yaml": (28, 8),                       # TAS8 :508
    "e2e/yaml/tas-pcs-pclq.yaml": (28, 2),                        # TAS9 :585
    "e2e/yaml/tas-pcsg-scale.yaml": (28, 6),                      # TAS10 :635
    "e2e/yaml/tas-pcsg-pclq.yaml": (28, 4),                       # TAS11 :715
    "e2e/yaml/tas-large-scale.yaml": (28, 20),                    # TAS12 :774
    "e2e/yaml/tas-insuffic.yaml": (28, 0),                        # TAS13 :868: ten 500 MiB pods, nothing may be bound
    "e2e/yaml/tas-multirep.yaml": (28, 4),                        # TAS14 :927
    "e2e/yaml/tas-pcs-multi-pcsg.yaml": (28, 10),                 # TAS15 :985
    "e2e/yaml/tas-pcs-multi-pcsg-multi-replica.yaml": (28, 20),   # TAS16 :1099
}


@pytest.mark.parametrize("path", sorted(TAS))
def test_tas_workload_files_end_to_end(placer, path):
    n_nodes, expect = TAS[path]
    g, c, s, names, gangs = ingest.tables_from_pcs(pcs_of(path), LEVELS, class_mask=synth.AGENT)
    assert int(c["replicas"].sum()) == (expect if expect else 10)
    nodes = synth.e2e_cluster(n_nodes)
    r = placer.run_cycle(nodes, synth.E2E_LEVELS, g, c, s)
    assert check_pack_constraints(nodes, (g, c, s), r) == expect
    if expect:
        assert (r["status"]["state"] == T.GANG_ADMITTED).all()
    else:
        assert (r["status"]["state"] == T.GANG_REJECTED).all() and np.array_equal(r["nodes_after"], nodes)


def test_tas8_shape_from_the_file(placer):
    """topology_test.go:508-578 on the file itself: 4 host groups, 2 rack groups, 1 block"""
    g, c, s, names, _ = ingest.tables_from_pcs(pcs_of("e2e/yaml/tas-hierarchy.yaml"), LEVELS, class_mask=synth.AGENT)
    nodes = synth.e2e_cluster(28)
    pl = placer.run_cycle(nodes, synth.E2E_LEVELS, g, c, s)["placements"]
    assert len({int(n) for n in pl["node"]}) == 4                                             # each PodClique's two pods share a host
    by_replica = {}
    for q, n in zip(pl["clique"], pl["node"]):
        by_replica.setdefault(names[int(q)][1].rsplit("-", 1)[0], set()).add(int(nodes["dom"][int(n), RACK]))
    assert len(by_replica) == 2 and all(len(v) == 1 for v in by_replica.values())             # each PCSG replica in one rack
    assert len({int(nodes["dom"][int(n), BLOCK]) for n in pl["node"]}) == 1


def test_simple1_is_config_c1():
    """BASELINE.json config 1 = samples/simple/simple1.yaml after defaulting: one base gang {pca x3, pcd x2, sga-0: pcb x2 + pcc x2}"""
    g, c, s, names, gangs = ingest.tables_from_pcs(pcs_of("samples/simple/simple1.yaml"), LEVELS)
    cfg = synth.config_c1()
    g1, c1, _ = cfg["tables"]
    assert len(g) == len(g1) == 1
    assert sorted(zip(c["min_replicas"].tolist(), c["replicas"].tolist())) == sorted(zip(c1["min_replicas"].tolist(), c1["replicas"].tolist()))
    assert sorted(n for _, n in names) == ["simple1-0-pca", "simple1-0-pcd", "simple1-0-sga-0-pcb", "simple1-0-sga-0-pcc"]


def test_tas17_two_topologies_on_one_cluster(placer):
    """topology_test.go:1192-1370 on the reference's own files and its own node manifests: 28 nodes, the last 14
    relabelled as GB200 (no kubernetes.io/rack, example.com/nvl-block + example.com/nvlink-domain instead); the domain
    name "block" means kubernetes.io/rack in h100-topology and example.com/nvl-block in gb200-topology.  Each workload
    must land on the segment that carries ITS topology's labels, packed in one block of that topology."""
    kwok = json.load(open(os.path.join(HERE, "golden", "kwok_nodes_60.json")))
    K = kwok["label_keys"]
    ms = json.loads(json.dumps(kwok["manifests_e2e"][:28]))
    for idx, m in enumerate(ms[14:]):
        lab = m["metadata"]["labels"]
        del lab[K["rack"]]
        lab["example.com/nvl-block"] = f"block-{idx // 7}"
        lab["example.com/nvlink-domain"] = f"nvl-domain-{idx}"
    topologies = {
        "e2e/yaml/tas-multi-topology-h100.yaml": [("block", K["rack"]), ("host", K["host"])],
        "e2e/yaml/tas-multi-topology-gb200.yaml": [("block", "example.com/nvl-block"), ("rack", "example.com/nvlink-domain"), ("host", K["host"])],
    }
    used = {}
    for path, levels in topologies.items():
        pcs = pcs_of(path)
        nodes, names, *_ = ingest.nodes_from_manifests(ms, [k for _, k in levels], used=used)
        g, c, s, _, gangs = ingest.tables_from_pcs(pcs, levels)
        assert gangs[0]["spec"]["topologyConstraint"]["packConstraint"]["required"] == levels[0][1]
        r = placer.run_cycle(nodes, len(levels), g, c, s)
        assert (r["status"]["state"] == T.GANG_ADMITTED).all() and len(r["placements"]) == 2
        where = [int(n) for n in r["placements"]["node"]]
        segment = range(0, 14) if "h100" in path else range(14, 28)
        assert all(n in segment for n in where), (path, where)
        assert len({ms[n]["metadata"]["labels"][levels[0][1]] for n in where}) == 1     # one block of ITS topology
        for n in where:
            u = used.setdefault(names[n], {"memory": "0Mi", "pods": 0})
            u["memory"] = f"{ingest.parse_mem_mib(u['memory']) + 10}Mi"; u["pods"] += 1
