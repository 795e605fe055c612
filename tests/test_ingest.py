"""Manifests -> tables, pinned on output of the reference's own KWOK node generator
(tests/golden/kwok_nodes_60.json, made by tests/golden/make_kwok_fixture.py importing
ai-dynamo/grove operator/hack/infra_manager/kwok.py in the build container)."""
import json
import os

import numpy as np
import pytest

from grove_b200 import ingest, synth, tables as T

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def kwok():
    with open(os.path.join(HERE, "golden", "kwok_nodes_60.json")) as f:
        return json.load(f)


def test_quantities():
    assert ingest.parse_cpu_milli("64") == 64000 and ingest.parse_cpu_milli("500m") == 500 and ingest.parse_cpu_milli(4) == 4000
    assert ingest.parse_mem_mib("512Gi") == 524288 and ingest.parse_mem_mib("150Mi") == 150 and ingest.parse_mem_mib("80Mi") == 80
    assert ingest.parse_mem_mib("1G") == 953


def test_quantities_round_requests_up_and_offers_down():
    """resource.Quantity suffix set (m, k, M, G, T, P, E, Ki..Ei); a request is rounded up, what a node offers down (ADVICE
    round 1: flooring requests under-counts them and over-commits nodes)"""
    c, m = ingest.parse_cpu_milli, ingest.parse_mem_mib
    assert c("2k") == 2_000_000 and c("1e3") == 1_000_000 and c("0.0005") == 0 and c("0.0005", request=True) == 1
    assert m("100M") == 95 and m("100M", request=True) == 96
    assert m("500Ki") == 0 and m("500Ki", request=True) == 1
    assert m("1500m", request=True) == 1 and m("1Ei") == 2 ** 40 and m("1P") == 10 ** 15 // 2 ** 20 and m("2E") == 2 * 10 ** 18 // 2 ** 20


def test_reference_kwok_manifests_match_the_synthetic_generator(kwok):
    """our label arithmetic (synth.kwok_nodes) == what the reference generator labels its nodes with"""
    keys = [kwok["label_keys"][k] for k in ("zone", "block", "rack", "host")]
    nodes, names, intern, classes = ingest.nodes_from_manifests(kwok["manifests"], keys, class_key="node_role.e2e.grove.nvidia.com")
    per = kwok["nodes_per"]
    assert (per["zone"], per["block"], per["rack"]) == (28, 20, 7)  # constants.py:65-67
    ours = synth.kwok_nodes(60, [per["zone"], per["block"], per["rack"], 1], cpu_milli=64000, mem_mib=524288, gpu=0, pods=110, node_class=1)
    assert names[57] == "kwok-node-57"
    for f in ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods", "flags"):
        assert np.array_equal(nodes[f], ours[f]), f
    # interning assigns ids in first-seen order == the integer division for this generator
    assert np.array_equal(nodes["dom"], ours["dom"])
    assert classes == {"agent": 1}


def test_reference_e2e_preset(kwok):
    keys = [kwok["label_keys"][k] for k in ("zone", "block", "rack", "host")]
    nodes, *_ = ingest.nodes_from_manifests(kwok["manifests_e2e"], keys)
    assert (nodes["free_cpu_milli"] == 4000).all() and (nodes["free_mem_mib"] == 150).all() and (nodes["free_pods"] == 110).all()


def test_reference_labels_are_not_a_tree(kwok, oracle):
    """28/20/7: block-1 straddles zone-0 and zone-1 (20 does not divide 28); path semantics splits it"""
    keys = [kwok["label_keys"][k] for k in ("zone", "block", "rack", "host")]
    nodes, *_ = ingest.nodes_from_manifests(kwok["manifests"], keys)
    perm, dom, ndom, non_tree = oracle.topology(nodes, 4)
    assert non_tree > 0 and ndom[0] == 3 and ndom[1] > 3


def test_used_and_cordon_and_missing_labels(kwok):
    ms = json.loads(json.dumps(kwok["manifests"][:4]))
    ms[1]["spec"]["unschedulable"] = True
    del ms[2]["metadata"]["labels"][kwok["label_keys"]["rack"]]
    keys = [kwok["label_keys"][k] for k in ("zone", "block", "rack", "host")]
    nodes, names, *_ = ingest.nodes_from_manifests(ms, keys, used={"kwok-node-0": {"cpu": "1500m", "memory": "2Gi", "pods": 3}})
    assert nodes["free_cpu_milli"][0] == 62500 and nodes["free_mem_mib"][0] == 524288 - 2048 and nodes["free_pods"][0] == 107
    assert not nodes["flags"][1] & T.NODE_SCHEDULABLE and nodes["flags"][0] & T.NODE_SCHEDULABLE
    assert nodes["dom"][2, 2] == T.DOM_ABSENT and nodes["dom"][2, 3] != T.DOM_ABSENT


def _podgang(name, groups, gang_key=None, configs=()):
    tc = lambda k: {"packConstraint": {"required": k}} if k else None  # noqa: E731
    spec = {"podgroups": [dict(name=n, podReferences=[{"namespace": "default", "name": f"{n}-{i}"} for i in range(r)], minReplicas=m,
                               **({"topologyConstraint": tc(k)} if k else {})) for n, r, m, k in groups]}
    if gang_key:
        spec["topologyConstraint"] = tc(gang_key)
    if configs:
        spec["topologyConstraintGroupConfigs"] = [dict(name=cn, podGroupNames=list(members), topologyConstraint=tc(k)) for cn, members, k in configs]
    return {"apiVersion": "scheduler.grove.io/v1alpha1", "kind": "PodGang", "metadata": {"name": name, "namespace": "default"}, "spec": spec}


def test_podgang_manifest_to_tables_and_oracle(kwok, placer):
    """tas-hierarchy.yaml as the operator would emit it: PCS block -> PCSG replica rack -> PCLQ host"""
    Z, B, R, H = (kwok["label_keys"][k] for k in ("zone", "block", "rack", "host"))
    pg = _podgang("tas-hierarchy-0",
                  [("r0-prefill", 2, 2, H), ("r0-decode", 2, 2, H), ("r1-prefill", 2, 2, H), ("r1-decode", 2, 2, H), ("router", 1, 1, None)],
                  gang_key=B, configs=[("ig-0", ("r0-prefill", "r0-decode"), R), ("ig-1", ("r1-prefill", "r1-decode"), R)])
    req = {n: {"memory": "40Mi"} for n in ("r0-prefill", "r0-decode", "r1-prefill", "r1-decode", "router")}
    g, c, s, names = ingest.podgangs_from_manifests([pg], req, [Z, B, R, H])
    assert len(g) == 1 and g["level"][0] == 1 and g["n_scopes"][0] == 3 and g["n_cliques"][0] == 5
    assert names[0] == ("tas-hierarchy-0", "router") and s["level"].tolist() == [T.LEVEL_NONE, 2, 2]
    assert c["level"].tolist() == [T.LEVEL_NONE, 3, 3, 3, 3] and c["req_mem_mib"].tolist() == [40] * 5
    # 14/7 arithmetic nests (unlike 28/20/7): relabel a 14-node block of the reference manifests accordingly
    ms = json.loads(json.dumps(kwok["manifests_e2e"][:14]))
    for i, m in enumerate(ms):
        m["metadata"]["labels"][B] = f"block-{i // 14}"
    nodes, node_names, *_ = ingest.nodes_from_manifests(ms, [Z, B, R, H])
    r = placer.run_cycle(nodes, 4, g, c, s)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and r["status"]["n_pods"][0] == 9
    pl = r["placements"]
    for row in range(1, 5):
        assert len(set(pl["node"][pl["clique"] == row])) == 1        # each clique on one host
    for rows in ((1, 2), (3, 4)):
        racks = {int(nodes["dom"][n, 2]) for n in pl["node"][np.isin(pl["clique"], rows)]}
        assert len(racks) == 1                                        # each PCSG replica in one rack
    with pytest.raises(ValueError):
        ingest.podgangs_from_manifests([_podgang("x", [("a", 1, 1, "example.com/nope")])], {}, [Z, B, R, H])


def test_preferred_keys_become_preferred_levels(kwok, placer):
    """packConstraint.preferred (podgang.go:110-117) at PodGang, group-config and PodGroup level"""
    Z, B, R, H = (kwok["label_keys"][k] for k in ("zone", "block", "rack", "host"))
    pg = _podgang("p", [("a", 2, 2, None), ("b", 3, 3, None), ("c", 1, 1, None)], configs=[("cfg", ("b", "c"), B)])
    pg["spec"]["topologyConstraint"] = {"packConstraint": {"preferred": R}}
    pg["spec"]["podgroups"][0]["topologyConstraint"] = {"packConstraint": {"preferred": H}}
    pg["spec"]["topologyConstraintGroupConfigs"][0]["topologyConstraint"]["packConstraint"]["preferred"] = R
    pg["spec"]["podgroups"][1]["topologyConstraint"] = {"packConstraint": {"required": R, "preferred": B}}  # not deeper: dropped
    g, c, s, _ = ingest.podgangs_from_manifests([pg], {n: {"memory": "40Mi"} for n in "abc"}, [Z, B, R, H])
    assert g["level"][0] == T.LEVEL_NONE and g["preferred"][0] == 2
    assert s["level"].tolist() == [T.LEVEL_NONE, 1] and s["preferred1"].tolist() == [0, 3]
    assert (c["scope"] & 0x1F).tolist() == [0, 1, 1] and (c["scope"] >> 5).tolist() == [4, 0, 0]
    assert c["level"].tolist() == [T.LEVEL_NONE, 2, T.LEVEL_NONE]
    nodes, *_ = ingest.nodes_from_manifests(kwok["manifests_e2e"][:14], [Z, B, R, H])
    r = placer.run_cycle(nodes, 4, g, c, s)
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    pl = r["placements"]
    assert len(set(pl["node"][pl["clique"] == 0])) == 1                      # a: both pods on one host
    assert len({int(nodes["dom"][n, 2]) for n in pl["node"]}) == 1           # the gang in one rack
    with pytest.raises(ValueError):
        bad = _podgang("x", [("a", 1, 1, None)]); bad["spec"]["topologyConstraint"] = {"packConstraint": {"preferred": "example.com/nope"}}
        ingest.podgangs_from_manifests([bad], {}, [Z, B, R, H])


def test_reuse_reservation_ref_bindings_and_status(kwok, placer):
    """spec.reuseReservationRef -> anchor; placements -> (pod, node) bindings; status rows -> PodGang.status"""
    Z, B, R, H = (kwok["label_keys"][k] for k in ("zone", "block", "rack", "host"))
    nodes, node_names, *_ = ingest.nodes_from_manifests(kwok["manifests_e2e"][:28], [Z, B, R, H])
    first = _podgang("first", [("a", 2, 2, None)], gang_key=R)
    again = _podgang("again", [("w", 3, 3, None)], gang_key=R)
    again["spec"]["reuseReservationRef"] = {"namespace": "default", "name": "first"}
    huge = _podgang("huge", [("x", 9, 9, H)])           # nine 40 MiB pods on one 150 MiB host: unschedulable
    req = {"a": {"memory": "40Mi"}, "w": {"memory": "40Mi"}, "x": {"memory": "40Mi"}}
    g, c, s, names = ingest.podgangs_from_manifests([first], req, [Z, B, R, H])
    r = placer.run_cycle(nodes, 4, g, c, s)
    b1 = ingest.bindings(r["placements"], [first], names, node_names)
    assert [p for _, p, _ in b1] == ["a-0", "a-1"] and all(n.startswith("kwok-node-") for _, _, n in b1)
    landed = int(r["placements"]["node"][0])
    g, c, s, names = ingest.podgangs_from_manifests([again, huge], req, [Z, B, R, H], placed_on={"first": landed})
    assert g["anchor_node"].tolist() == [landed, T.NONE_U32]
    r2 = placer.run_cycle(r["nodes_after"], 4, g, c, s)
    b2 = ingest.bindings(r2["placements"], [again, huge], names, node_names)
    assert len(b2) == 3 and {int(nodes["dom"][node_names.index(n), 2]) for _, _, n in b2} == {int(nodes["dom"][landed, 2])}   # same rack as "first"
    st = [ingest.podgang_status(row) for row in r2["status"]]
    assert st[0]["phase"] == "Starting" and st[0]["conditions"][0]["status"] == "True" and 0 < st[0]["placementScore"] <= 1.0
    assert st[1] == {"phase": "Pending", "conditions": [{"type": "Scheduled", "status": "False", "reason": "Unschedulable"}]}
