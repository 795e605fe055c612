"""Elastic reclaim as its definition reads (tests/elastic_cases.py run_cycle_preempt_elastic, over the sequential oracle): the
degenerate case, the hand cases, and the invariants every cycle keeps on churned clusters whose running gangs carry surplus pods."""
import numpy as np
import pytest

from elastic_cases import elastic_cluster, hand_case, run_cycle_preempt_elastic, surplus_of
from grove_b200 import tables as T
from preempt_cases import churned_cluster
from reuse_cases import free_table, hold_table

_CASES = {}


def _churned(oracle, seed):
    if seed not in _CASES:
        nodes, L, tabs, running, holdings, surplus = elastic_cluster(oracle, seed, n=252, g_running=80, g_pending=40)
        ref = run_cycle_preempt_elastic(oracle, nodes, L, *tabs, running, holdings, surplus)
        _CASES[seed] = (nodes, L, tabs, running, holdings, surplus, ref)
    return _CASES[seed]


def _same(a, b, keys=("status", "placements", "scope_status", "nodes_after", "victims")):
    for k in keys:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("seed", [3, 11])
def test_no_surplus_is_the_reclaim_pass(oracle, seed):
    nodes, L, (g, c, s), running, holdings = churned_cluster(oracle, seed, n=252, g_running=80, g_pending=40)
    ref = oracle.run_cycle_preempt(nodes, L, g, c, s, running, holdings)
    got = run_cycle_preempt_elastic(oracle, nodes, L, g, c, s, running, holdings, np.zeros(0, dtype=T.surplus_pod_dt))
    _same(got, ref)
    assert len(got["surplus_victims"]) == 0


def test_surplus_case(oracle):
    """P takes B's surplus pod on n1; A and B keep running"""
    nodes, L, (g, c, s), running, holdings, surplus = hand_case(4)
    whole = oracle.run_cycle_preempt(nodes, L, g, c, s, running, holdings)
    assert whole["status"]["reserved0"][0] == T.STATUS_PREEMPTOR and len(whole["victims"]) == 1
    got = run_cycle_preempt_elastic(oracle, nodes, L, g, c, s, running, holdings, surplus)
    assert got["status"]["state"][0] == T.GANG_ADMITTED
    assert got["status"]["reserved0"][0] == T.STATUS_PREEMPTOR | T.STATUS_SURPLUS_ONLY
    assert list(got["placements"]["node"]) == [1]
    assert len(got["victims"]) == 0
    assert [tuple(v) for v in got["surplus_victims"]] == [(0, 0)]
    assert list(got["nodes_after"]["free_gpu"]) == [0, 0]


def test_whole_case(oracle):
    """an 8-GPU P does not fit on the surplus: pass 2 evicts whole, exactly as the reclaim pass does"""
    nodes, L, (g, c, s), running, holdings, surplus = hand_case(8)
    whole = oracle.run_cycle_preempt(nodes, L, g, c, s, running, holdings)
    got = run_cycle_preempt_elastic(oracle, nodes, L, g, c, s, running, holdings, surplus)
    _same(got, whole)
    assert got["status"]["reserved0"][0] == T.STATUS_PREEMPTOR and len(got["victims"]) == 1
    assert len(got["surplus_victims"]) == 0


def test_surplus_ahead_of_lower_priority(oracle):
    """B outranks A, yet P takes B's surplus pod rather than evicting A whole"""
    nodes, L, (g, c, s), running, holdings, surplus = hand_case(4, b_priority=3)
    got = run_cycle_preempt_elastic(oracle, nodes, L, g, c, s, running, holdings, surplus)
    assert got["status"]["reserved0"][0] == T.STATUS_PREEMPTOR | T.STATUS_SURPLUS_ONLY
    assert len(got["victims"]) == 0 and [tuple(v) for v in got["surplus_victims"]] == [(0, 0)]


def test_surplus_of_lists_pods_above_min_highest_first():
    g = np.zeros(1, dtype=T.gang_dt); g["n_cliques"] = 2
    c = np.zeros(2, dtype=T.clique_dt)
    c["min_replicas"] = [1, 2]; c["replicas"] = [1, 5]; c["req_gpu"] = [0, 2]
    st = np.zeros(1, dtype=T.status_dt); st["state"] = T.GANG_ADMITTED; st["n_pods"] = 5
    pl = np.array([(0, 9), (1, 10), (1, 11), (1, 12), (1, 13)], dtype=T.placement_dt)
    got = surplus_of(pl, st, g, c)
    assert list(got["node"]) == [13, 12] and list(got["gpu"]) == [2, 2] and list(got["running"]) == [0, 0]


@pytest.mark.parametrize("seed", [3, 11, 29])
def test_invariants(oracle, seed):
    nodes, L, (g, c, s), running, holdings, surplus, ref = _churned(oracle, seed)
    assert len(surplus) > 0
    st, R = ref["status"], len(running)
    rank = lambda x: int(g["priority"][x])   # noqa: E731
    whole = {int(v["running"]) for v in ref["victims"]}
    # pass-1 preemptors evict no whole gang
    only = {x for x in range(len(g)) if st["reserved0"][x] & T.STATUS_SURPLUS_ONLY}
    assert all(st["reserved0"][x] & T.STATUS_PREEMPTOR for x in only)
    assert not any(int(v["preemptor"]) in only for v in ref["victims"])
    # no pod is taken twice, and none from a gang evicted whole before
    pods = [int(v["pod"]) for v in ref["surplus_victims"]]
    assert len(pods) == len(set(pods))
    # every victim ranks strictly below its preemptor
    for v in ref["victims"]:
        assert int(running["priority"][v["running"]]) < rank(int(v["preemptor"]))
    for v in ref["surplus_victims"]:
        assert int(running["priority"][surplus["running"][v["pod"]]]) < rank(int(v["preemptor"]))
    # resources are conserved: F_final + what the admitted gangs use + what the standing gangs hold = F0 + every holding
    N = len(nodes)
    taken = np.zeros((N, 4), dtype=np.int64)
    for v in ref["surplus_victims"]:
        x = surplus[int(v["pod"])]
        if int(x["running"]) not in whole:
            taken[int(x["node"])] += [int(x["cpu_milli"]), int(x["mem_mib"]), int(x["gpu"]), 1]
    lhs = free_table(ref["nodes_after"]) - taken
    for r in range(R):
        if r not in whole:
            lhs += hold_table(N, running, holdings, r)
    base = oracle.run_cycle(nodes, L, g, c, s)
    rhs = free_table(base["nodes_after"]) + sum(hold_table(N, running, holdings, r) for r in range(R))
    new = [x for x in range(len(g)) if st["state"][x] == T.GANG_ADMITTED and base["status"]["state"][x] != T.GANG_ADMITTED]
    for x in new:
        for e in ref["placements"][st["placement_off"][x]: st["placement_off"][x] + st["n_pods"][x]]:
            q = c[int(e["clique"])]
            rhs[int(e["node"])] -= [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
    assert np.array_equal(lhs, rhs)
    # the order of events: a pod is never taken from a gang after that gang was evicted whole (the restatement records both in
    # one order per preemptor; the gang's eviction must not come from an earlier preemptor)
    first_whole = {}
    for v in ref["victims"]:
        first_whole.setdefault(int(v["running"]), int(v["preemptor"]))
    order = sorted(range(len(g)), key=lambda x: (-rank(x), x))
    pos = {x: i for i, x in enumerate(order)}
    for v in ref["surplus_victims"]:
        r = int(surplus["running"][v["pod"]])
        if r in first_whole:
            assert pos[int(v["preemptor"])] <= pos[first_whole[r]]
