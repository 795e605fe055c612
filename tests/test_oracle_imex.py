"""ComputeDomain exclusivity as its definition reads (tests/imex_cases.py, over the unchanged sequential oracle): the properties the
definition promises on random snapshots, and one hand case per rule, the first of which the plain cycle gets wrong."""
import numpy as np
import pytest

from grove_b200 import tables as T
from imex_cases import NO_IMEX, NONE, enroll_randomly, gang_cds, hand_cases, run_cycle_imex
from test_random_parity_gpu import random_case

RES = ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")


def _order(gangs):
    return sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))


def _case(seed):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    cd, owner0 = enroll_randomly(np.random.default_rng(seed + 417), tables[0], tables[1], nodes)
    return nodes, L, tables, cd, owner0


def _gang_out(out, g):
    s = out["status"][g]
    return s, out["placements"][s["placement_off"]: s["placement_off"] + s["n_pods"]]


@pytest.mark.parametrize("seed", range(0, 30))
def test_no_enrolled_clique_is_the_ordinary_cycle(oracle, seed):
    nodes, L, tables, _, owner0 = _case(seed)
    got = run_cycle_imex(oracle, nodes, L, *tables, np.full(len(tables[1]), NONE, np.uint32), owner0)
    ref = oracle.run_cycle(nodes, L, *tables)
    for k in ("status", "placements", "scope_status", "nodes_after"):
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(got["owners"], owner0)


def check_consequences(nodes, tables, cd, owner0, got):
    """what the definition promises at the end of the cycle, whatever computed `got`"""
    gangs, cliques, _ = tables
    N = len(nodes)
    st = got["status"]
    holders = [set() for _ in range(N)]
    use = np.zeros((N, 4), dtype=np.int64)
    owners = np.asarray(owner0, dtype=np.uint32).copy()
    for g in range(len(gangs)):
        if st["state"][g] != T.GANG_ADMITTED:
            continue
        _, pl = _gang_out(got, g)
        for e in pl:
            q, n = int(e["clique"]), int(e["node"])
            c = cliques[q]
            use[n] += (int(c["req_cpu_milli"]), int(c["req_mem_mib"]), int(c["req_gpu"]), 1)
            if cd[q] != NONE:
                holders[n].add(int(cd[q]))
                # no enrolled pod on a node whose owner0 is foreign or has no IMEX driver
                assert owner0[n] in (NONE, cd[q]), (g, n, int(owner0[n]), int(cd[q]))
                owners[n] = cd[q]
    # no node holds enrolled pods of two CDs
    assert all(len(h) <= 1 for h in holders)
    # resources are conserved
    for k, f in enumerate(RES):
        assert np.array_equal(got["nodes_after"][f].astype(np.int64), nodes[f].astype(np.int64) - use[:, k]), f
    # the owners are owner0 plus the admitted enrolled placements
    assert np.array_equal(got["owners"], owners)


@pytest.mark.parametrize("seed", range(30, 110))
def test_properties(oracle, seed):
    nodes, L, tables, cd, owner0 = _case(seed)
    gangs = tables[0]
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    # gangs ranked before the first enrolled gang keep their ordinary outcome
    plain = oracle.run_cycle(nodes, L, *tables)
    gcd = gang_cds(gangs, cd)
    for g in _order(gangs):
        if gcd[g] != NONE:
            break
        a, pa = _gang_out(got, g)
        r, pr = _gang_out(plain, g)
        for f in ("state", "level", "reserved0", "score_num", "score_den", "n_pods", "domain_node"):
            assert a[f] == r[f], (g, f)
        assert np.array_equal(pa, pr)
    check_consequences(nodes, tables, cd, owner0, got)


def _nodes_of(out, g):
    return [int(e["node"]) for e in _gang_out(out, g)[1]]


def test_two_replicas_get_a_node_each(oracle):
    nodes, L, tables, cd, owner0 = hand_cases()["two_replicas"]()
    plain = oracle.run_cycle(nodes, L, *tables)
    assert set(_nodes_of(plain, 0)) == set(_nodes_of(plain, 1)) == {0}   # the plain cycle stacks them: the second cannot start
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    assert (got["status"]["state"] == T.GANG_ADMITTED).all()
    assert set(_nodes_of(got, 0)) == {0} and set(_nodes_of(got, 1)) == {1}
    assert got["owners"].tolist() == [7, 8]
    check_consequences(nodes, tables, cd, owner0, got)


def test_third_replica_waits_until_one_is_deleted(oracle):
    nodes, L, tables, cd, owner0 = hand_cases()["third_rejected"]()
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    assert got["status"]["state"].tolist() == [T.GANG_ADMITTED, T.GANG_ADMITTED, T.GANG_REJECTED]
    assert got["owners"].tolist() == [1, 2]
    nodes, L, tables, cd, owner0 = hand_cases()["after_delete"]()   # replica 0 deleted: node 0 free and unowned
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    assert got["status"]["state"][0] == T.GANG_ADMITTED and set(_nodes_of(got, 0)) == {0}
    assert got["owners"].tolist() == [3, 2]


def test_frontend_shares_an_owned_node(oracle):
    nodes, L, tables, cd, owner0 = hand_cases()["frontend_shares"]()
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    assert (got["status"]["state"] == T.GANG_ADMITTED).all()
    assert set(_nodes_of(got, 1)) == {1}   # a plain CPU gang on the node CD 9 holds
    pl = _gang_out(got, 0)[1]
    assert {int(e["node"]) for e in pl if cd[int(e["clique"])] != NONE} == {0}
    check_consequences(nodes, tables, cd, owner0, got)


def test_scaled_gang_joins_its_base(oracle):
    nodes, L, tables, cd, owner0 = hand_cases()["scaled_joins_base"]()
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    assert (got["status"]["state"] == T.GANG_ADMITTED).all()
    assert set(_nodes_of(got, 0)) == set(_nodes_of(got, 2)) == {0} and set(_nodes_of(got, 1)) == {1}
    check_consequences(nodes, tables, cd, owner0, got)


def test_no_imex_node_takes_only_plain_pods(oracle):
    nodes, L, tables, cd, owner0 = hand_cases()["no_imex_node"]()
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    assert (got["status"]["state"] == T.GANG_ADMITTED).all()
    assert set(_nodes_of(got, 0)) == {1} and set(_nodes_of(got, 1)) == {0}
    assert got["owners"].tolist() == [NO_IMEX, 4]
    check_consequences(nodes, tables, cd, owner0, got)


def test_surplus_is_blocked_while_min_replicas_fit(oracle):
    nodes, L, tables, cd, owner0 = hand_cases()["surplus_blocked"]()
    plain = oracle.run_cycle(nodes, L, *tables)
    assert plain["status"]["n_pods"][0] == 8
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    assert got["status"]["state"][0] == T.GANG_ADMITTED and got["status"]["n_pods"][0] == 4
    assert set(_nodes_of(got, 0)) == {0}
    check_consequences(nodes, tables, cd, owner0, got)


def test_preferred_levels(oracle):
    nodes, L, tables, cd, owner0 = hand_cases()["preferred_levels"]()
    plain = oracle.run_cycle(nodes, L, *tables)
    assert set(_nodes_of(plain, 0)) == {1}
    got = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    check_consequences(nodes, tables, cd, owner0, got)
    st = got["status"]
    # gang 0's anchor host is held by CD 3: its host-level Preferred domain is the next host of the block
    assert st["state"][0] == T.GANG_ADMITTED and set(_nodes_of(got, 0)) == {0} and st["level"][0] == 1
    # gang 1 (anchored at node 0, now CD 1's) keeps its Preferred level on the first host of the other block
    assert st["state"][1] == T.GANG_ADMITTED and set(_nodes_of(got, 1)) == {2} and st["level"][1] == 1


def test_restatement_refuses_two_cds_in_a_gang():
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(gpu=1, min=1), dict(gpu=1, min=1)])])
    gangs, cliques, _ = b.build()
    with pytest.raises(AssertionError):
        gang_cds(gangs, np.array([1, 2], np.uint32))
