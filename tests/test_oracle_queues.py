"""Queue limits as their definition reads (tests/queue_cases.py, over the unchanged sequential oracle): the properties the
definition promises on random snapshots, and one hand case per rule."""
import copy
import json
import os

import numpy as np
import pytest

from grove_b200 import ingest, tables as T
from queue_cases import assign_queues, chain, diagnose_queue_cycle, hand_cases, loads, make_queues, run_cycle_queues
from test_random_parity_gpu import random_case

NONE = T.NONE_U32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RES = ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")
REQ = ("req_cpu_milli", "req_mem_mib", "req_gpu")


def _case(seed):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    queues, gq = assign_queues(np.random.default_rng(seed + 91), tables[0], tables[1])
    return nodes, L, tables, queues, gq


def _order(gangs):
    return sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))


def _same(a, b):
    for k in ("status", "placements", "scope_status", "nodes_after"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("seed", range(0, 30))
def test_no_members_or_no_limits_is_the_ordinary_cycle(oracle, seed):
    nodes, L, tables, queues, gq = _case(seed)
    ref = oracle.run_cycle(nodes, L, *tables)
    _same(run_cycle_queues(oracle, nodes, L, *tables, queues, np.full(len(gq), NONE, np.uint32)), ref)
    unlimited = queues.copy()
    unlimited["limit"] = T.QUEUE_UNLIMITED
    _same(run_cycle_queues(oracle, nodes, L, *tables, unlimited, gq), ref)


@pytest.mark.parametrize("seed", range(30, 100))
def test_properties(oracle, seed):
    nodes, L, tables, queues, gq = _case(seed)
    gangs, cliques, _ = tables
    trace = []
    got = run_cycle_queues(oracle, nodes, L, *tables, queues, gq, trace=trace)
    st = got["status"]
    # gangs ranked before every member keep their ordinary outcome
    plain = oracle.run_cycle(nodes, L, *tables)
    for g in _order(gangs):
        if gq[g] != NONE:
            break
        a, r = st[g], plain["status"][g]
        for f in ("state", "level", "reserved0", "score_num", "score_den", "n_pods", "domain_node"):
            assert a[f] == r[f], (g, f)
    # flags only on members, OVER_LIMIT only on REJECTED ones, SURPLUS_CAPPED only on ADMITTED ones
    assert not st["reserved0"][gq == NONE].any()
    assert (st["state"][(st["reserved0"] & T.STATUS_OVER_LIMIT) != 0] == T.GANG_REJECTED).all()
    assert (st["state"][(st["reserved0"] & T.STATUS_SURPLUS_CAPPED) != 0] == T.GANG_ADMITTED).all()
    # only surplus is trimmed: every admitted gang bound at least its MinReplicas of every clique, and a member no more than its cap
    for g, closed, caps, U in trace:
        assert closed == bool(st["reserved0"][g] & T.STATUS_OVER_LIMIT)
        if U is None:
            continue
        co = int(gangs["clique_off"][g])
        pl = got["placements"][st["placement_off"][g]: st["placement_off"][g] + st["n_pods"][g]]
        for c in range(int(gangs["n_cliques"][g])):
            n = int((pl["clique"] == co + c).sum())
            assert int(cliques["min_replicas"][co + c]) <= n <= int(cliques["min_replicas"][co + c]) + caps[c]
    # a queue that starts within its limit never exceeds it
    ld = loads(queues)
    held = [[0, 0, 0] for _ in range(len(queues))]
    for g in range(len(gangs)):
        if gq[g] == NONE or st["state"][g] != T.GANG_ADMITTED:
            continue
        pl = got["placements"][st["placement_off"][g]: st["placement_off"][g] + st["n_pods"][g]]
        for Q in chain(queues, int(gq[g])):
            for r in range(3):
                held[Q][r] += int(cliques[REQ[r]][pl["clique"]].astype(np.int64).sum())
    for Q in range(len(queues)):
        for r in range(3):
            lim = int(queues["limit"][Q][r])
            if lim != T.QUEUE_UNLIMITED and ld[Q][r] <= lim:
                assert ld[Q][r] + held[Q][r] <= lim, (Q, r)
    # resources are conserved
    used = np.zeros((len(nodes), 4), dtype=np.int64)
    perm_inv = np.arange(len(nodes))
    for e in got["placements"]:
        q = cliques[int(e["clique"])]
        used[perm_inv[int(e["node"])]] += (int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1)
    for k, f in enumerate(RES):
        assert np.array_equal(nodes[f].astype(np.int64) - used[:, k], got["nodes_after"][f].astype(np.int64)), f


def _states(got):
    return got["status"]["state"].tolist(), got["status"]["reserved0"].tolist()


A, R, B = T.GANG_ADMITTED, T.GANG_REJECTED, T.GANG_BASE_REJECTED
OL, SC = T.STATUS_OVER_LIMIT, T.STATUS_SURPLUS_CAPPED


def test_leaf_limit(oracle):
    nodes, L, tb, qs, gq = hand_cases()["leaf_limit"]()
    assert _states(run_cycle_queues(oracle, nodes, L, *tb, qs, gq)) == ([A, A, R], [0, 0, OL])


def test_parent_limit_shared_by_two_children(oracle):
    nodes, L, tb, qs, gq = hand_cases()["shared_parent"]()
    # rank: priority 1 first (gangs 1, 3, 5 in queue 2), then 0, 2, 4 in queue 1; the parent holds 24 GPUs, each child 16
    assert _states(run_cycle_queues(oracle, nodes, L, *tb, qs, gq)) == ([A, A, R, A, R, R], [0, 0, OL, 0, OL, OL])


def test_queue_over_its_limit_admits_nothing(oracle):
    nodes, L, tb, qs, gq = hand_cases()["over_limit_start"]()
    assert _states(run_cycle_queues(oracle, nodes, L, *tb, qs, gq)) == ([R, R, R], [OL, OL, OL])


def test_zero_gpu_gang_is_not_stopped_by_a_gpu_limit(oracle):
    nodes, L, tb, qs, gq = hand_cases()["zero_gpu_gang"]()
    assert _states(run_cycle_queues(oracle, nodes, L, *tb, qs, gq)) == ([R, A], [OL, 0])


def test_exact_surplus_cap_across_two_cliques(oracle):
    nodes, L, tb, qs, gq = hand_cases()["surplus_two_cliques"]()
    trace = []
    got = run_cycle_queues(oracle, nodes, L, *tb, qs, gq, trace=trace)
    assert _states(got) == ([A], [SC])
    assert trace[0][2] == [3, 0]
    assert sorted(got["placements"]["clique"].tolist()) == [0, 0, 0, 0, 1, 1]


def test_gated_out_member_leaves_its_nodes_to_a_nonmember(oracle):
    nodes, L, tb, qs, gq = hand_cases()["nonmember_takes"]()
    assert oracle.run_cycle(nodes, L, *tb)["status"]["state"].tolist() == [A, R]
    assert _states(run_cycle_queues(oracle, nodes, L, *tb, qs, gq)) == ([R, A], [OL, 0])


def test_scaled_gang_of_a_gated_out_base(oracle):
    nodes, L, tb, qs, gq = hand_cases()["scaled_base_gated"]()
    assert _states(run_cycle_queues(oracle, nodes, L, *tb, qs, gq)) == ([R, B], [OL, 0])


def test_cpu_and_memory_limits_along_a_chain(oracle):
    nodes, L, tb, qs, gq = hand_cases()["cpu_and_mem"]()
    got = run_cycle_queues(oracle, nodes, L, *tb, qs, gq)
    # rank: gangs 2, 5 (queue 0), then 1 (queue 1), 4 (queue 2), 7 (none), then 0, 3, 6.  The root holds 4 000 millicores of its
    # 40 000; gangs 2 and 5 take 16 000 each with their surplus (4 pods of 4 000), which leaves 4 000: every later member of the
    # tree needs 8 000 for its MinReplicas and is turned away at the root, whatever its own queue allows
    assert _states(got) == ([R, R, A, R, R, A, R, A], [OL, OL, 0, OL, OL, 0, OL, 0])
    assert got["status"]["n_pods"].tolist() == [0, 0, 4, 0, 0, 4, 0, 4]


def test_diagnosis_of_a_queue_cycle(oracle):
    """grove_diagnose's restatement after a queue cycle: OVER_LIMIT gangs get all-zero records, every other record is the
    ordinary restatement's over the cycle's outputs"""
    import diagnose_cases as D
    for seed in range(500, 510):
        nodes, L, (g, c, s), qs, gq = _case(seed)
        out = run_cycle_queues(oracle, nodes, L, g, c, s, qs, gq)
        gd, qd = diagnose_queue_cycle(nodes, L, g, c, s, out)
        rg, rq = D.diagnose(nodes, L, g, c, s, c["min_replicas"], out)
        over = (out["status"]["reserved0"] & T.STATUS_OVER_LIMIT) != 0
        for x in range(len(g)):
            co, n = int(g["clique_off"][x]), int(g["n_cliques"][x])
            if over[x]:
                assert not gd[x].tobytes().strip(b"\0") and not qd[co: co + n].tobytes().strip(b"\0")
            else:
                assert gd[x] == rg[x] and np.array_equal(qd[co: co + n], rq[co: co + n])


def _workload(path, queue_docs):
    """the reference workload file `path` with the queue labels of its PodClique templates -> nodes, L, tables, queues, gang_queue"""
    fx = json.load(open(os.path.join(GOLDEN, "workloads.json")))
    labels = json.load(open(os.path.join(GOLDEN, "queues.json")))["labels"][path]
    (pcs,) = fx[path]
    levels = [("zone", "topology.kubernetes.io/zone"), ("host", "kubernetes.io/hostname")]
    g, c, s, _, manifests = ingest.tables_from_pcs(pcs, levels)
    qs, gq, _ = ingest.queues_from_manifests(queue_docs, manifests, ingest.podgroup_queues(manifests, labels[pcs["name"]]))
    nodes = T.make_nodes(8)
    nodes["dom"][:, 0] = np.arange(8) // 4; nodes["dom"][:, 1] = np.arange(8)
    nodes["free_cpu_milli"] = 8000; nodes["free_mem_mib"] = 1024; nodes["free_gpu"] = 0; nodes["free_pods"] = 110
    nodes["flags"] = T.NODE_SCHEDULABLE
    return nodes, 2, (g, c, s), qs, gq


@pytest.mark.parametrize("path", ["e2e/yaml/workload1.yaml", "e2e/yaml/workload2.yaml"])
def test_reference_workloads_in_their_queues(oracle, path):
    docs = json.load(open(os.path.join(GOLDEN, "queues.json")))["queues"]
    nodes, L, tb, qs, gq = _workload(path, docs)
    assert [d["metadata"]["name"] for d in docs] == ["default", "test"]
    assert (qs["limit"] == T.QUEUE_UNLIMITED).all() and qs["parent"].tolist() == [NONE, 0]
    assert (gq == 1).all()   # every PodGroup's template is labelled kai.scheduler/queue: test
    ref = oracle.run_cycle(nodes, L, *tb)
    assert (ref["status"]["state"] == A).any()
    _same(run_cycle_queues(oracle, nodes, L, *tb, qs, gq), ref)
    # a finite memory limit on `test` below what the first gang asks for: it is turned away by its queue
    tight = copy.deepcopy(docs)
    tight[1]["spec"]["resources"]["memory"]["limit"] = 100
    nodes, L, tb, qs, gq = _workload(path, tight)
    assert qs["limit"][1].tolist() == [T.QUEUE_UNLIMITED, 100, T.QUEUE_UNLIMITED]
    got = run_cycle_queues(oracle, nodes, L, *tb, qs, gq)
    first = _order(tb[0])[0]
    assert got["status"]["state"][first] == R and got["status"]["reserved0"][first] == OL


def test_queue_ingest():
    docs = [{"kind": "Queue", "metadata": {"name": "team-a"}, "spec": {"parentQueue": "org", "resources": {"cpu": {"limit": 2.5}, "gpu": {"limit": 16}}}},
            {"kind": "Queue", "metadata": {"name": "org"}, "spec": {"resources": {"gpu": {"limit": -1}, "memory": {"limit": 2048}}}}]
    pgs = [{"metadata": {"name": "a"}, "spec": {"podgroups": [{"name": "a-w"}, {"name": "a-x"}]}},
           {"metadata": {"name": "b"}, "spec": {"podgroups": [{"name": "b-w"}]}},
           {"metadata": {"name": "c"}, "spec": {"podgroups": [{"name": "c-w"}]}}]
    qs, gq, names = ingest.queues_from_manifests(docs, pgs, {"a-w": "team-a", "a-x": None, "b-w": "nobody", "c-w": None})
    assert names == ["org", "team-a"] and qs["parent"].tolist() == [NONE, 0]
    assert qs["limit"].tolist() == [[T.QUEUE_UNLIMITED, 2048, T.QUEUE_UNLIMITED], [2500, T.QUEUE_UNLIMITED, 16]]   # cores -> millicores
    assert gq.tolist() == [1, NONE, NONE]   # an unknown queue: not a member
    with pytest.raises(ValueError, match="different queues"):
        ingest.queues_from_manifests(docs, pgs, {"a-w": "team-a", "a-x": "org"})
    with pytest.raises(ValueError, match="does not exist"):
        ingest.queues_from_manifests(docs[:1], pgs, {})
    assert ingest.podgroup_queues(pgs[:1], {"w": "team-a", "x": None}) == {"a-w": "team-a", "a-x": None}


def test_unlimited_queue_tree_is_the_ordinary_cycle(oracle):
    nodes, L, tb, _, gq = hand_cases()["shared_parent"]()
    qs = make_queues([(None, (None, None, None), (0, 0, 0)), (0, (None, None, None), (0, 0, 5)), (0, (None, None, None), (0, 0, 0))])
    _same(run_cycle_queues(oracle, nodes, L, *tb, qs, gq), oracle.run_cycle(nodes, L, *tb))
