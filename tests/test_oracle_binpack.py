"""Bin-packing as its definition reads (tests/binpack_cases.py, over the unchanged sequential oracle): the vectorised picks against a
brute-force loop, the properties the definition promises on random snapshots, one hand case per rule, and the two-cycle
fragmentation case the feature exists for."""
import numpy as np
import pytest

from grove_b200 import tables as T
from binpack_cases import Fragmentation, hand_cases, picks, picks_brute, random_levels, run_cycle_binpack
from test_random_parity_gpu import random_case

RES = ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")


def _case(seed):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    return nodes, L, tables, random_levels(np.random.default_rng(seed + 77), tables[0], L)


def _same(a, b):
    for k in ("placements", "status", "scope_status", "nodes_after", "perm"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("seed", range(40))
def test_picks_equal_a_brute_force_loop(oracle, seed):
    nodes, L, tables, levels = _case(seed)
    assert np.array_equal(picks(oracle, nodes, L, *tables, levels), picks_brute(oracle, nodes, L, *tables, levels))


@pytest.mark.parametrize("seed", range(20))
def test_no_members_is_the_ordinary_cycle(oracle, seed):
    nodes, L, tables, _ = _case(seed)
    got = run_cycle_binpack(oracle, nodes, L, *tables, np.full(len(tables[0]), T.LEVEL_NONE, np.uint8))
    _same(got, oracle.run_cycle(nodes, L, *tables))
    assert (got["picks"] == T.NONE_U32).all()


@pytest.mark.parametrize("seed", range(30))
def test_gangs_ranked_before_every_member_keep_their_outcome(oracle, seed):
    nodes, L, tables, levels = _case(seed)
    gangs = tables[0]
    order = sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))
    first = next((k for k, g in enumerate(order) if levels[g] != T.LEVEL_NONE), len(order))
    got, plain = run_cycle_binpack(oracle, nodes, L, *tables, levels), oracle.run_cycle(nodes, L, *tables)
    for g in order[:first]:
        a, b = got["status"][g], plain["status"][g]
        assert a["state"] == b["state"] and a["n_pods"] == b["n_pods"] and a["domain_node"] == b["domain_node"]
        pa = got["placements"][a["placement_off"]: a["placement_off"] + a["n_pods"]]
        pb = plain["placements"][b["placement_off"]: b["placement_off"] + b["n_pods"]]
        assert np.array_equal(pa, pb)


@pytest.mark.parametrize("seed", range(30))
def test_resources_are_conserved(oracle, seed):
    nodes, L, tables, levels = _case(seed)
    _, cliques, _ = tables
    got = run_cycle_binpack(oracle, nodes, L, *tables, levels)
    use = np.zeros((4, len(nodes)), dtype=np.int64)
    for p in got["placements"]:
        q = cliques[p["clique"]]
        use[:, p["node"]] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
    for k, f in enumerate(RES):
        assert np.array_equal(nodes[f].astype(np.int64) - use[k], got["nodes_after"][f].astype(np.int64)), f
    admitted = got["status"]["state"] == T.GANG_ADMITTED
    assert got["status"]["n_pods"][admitted].sum() == len(got["placements"])


@pytest.mark.parametrize("case", sorted(hand_cases()))
def test_hand_case(oracle, case):
    nodes, L, tables, levels, want = hand_cases()[case]()
    levels = np.array(levels, np.uint8)
    got = run_cycle_binpack(oracle, nodes, L, *tables, levels)
    assert got["picks"].tolist() == want
    assert np.array_equal(picks_brute(oracle, nodes, L, *tables, levels), picks(oracle, nodes, L, *tables, levels))


def test_picked_member_starts_in_its_pick(oracle):
    """fuller_wins: the hash anchor and the caller's anchor point elsewhere; the gang lands on the first node of its pick"""
    nodes, L, tables, levels, want = hand_cases()["fuller_wins"]()
    got = run_cycle_binpack(oracle, nodes, L, *tables, np.array(levels, np.uint8))
    assert got["status"]["state"][0] == T.GANG_ADMITTED and got["placements"]["node"].tolist() == want
    plain = oracle.run_cycle(nodes, L, *tables)
    assert plain["placements"]["node"].tolist() != want


def test_ties_fill_the_lowest_domain_then_spill(oracle):
    nodes, L, tables, levels, _ = hand_cases()["ties_lowest_domain"]()
    got = run_cycle_binpack(oracle, nodes, L, *tables, np.array(levels, np.uint8))
    assert got["placements"]["node"].tolist() == [0, 1, 2, 3, 4]


def test_no_domain_keeps_the_hash_anchor(oracle):
    nodes, L, tables, levels, _ = hand_cases()["no_domain_keeps_hash"]()
    got = run_cycle_binpack(oracle, nodes, L, *tables, np.array(levels, np.uint8))
    plain = oracle.run_cycle(nodes, L, *tables)
    assert got["status"]["state"][0] == plain["status"]["state"][0] == T.GANG_REJECTED
    assert got["placements"]["node"].tolist() == [0]


def test_fragmentation(oracle):
    def cycle(nodes, L, tables, levels):
        if levels is None:
            return oracle.run_cycle(nodes, L, *tables)
        return run_cycle_binpack(oracle, nodes, L, *tables, levels)

    f = Fragmentation()
    _, o2, used = f.run(cycle, binpack=False)
    assert used == [0, 1, 2, 3]                                   # the hash anchors leave a small gang in every block
    assert o2["status"]["state"][0] == T.GANG_REJECTED
    o1, o2, used = f.run(cycle, binpack=True)
    assert used == [0] and (o1["status"]["state"] == T.GANG_ADMITTED).all()
    assert o2["status"]["state"][0] == T.GANG_ADMITTED
    assert {int(p["node"]) // 8 for p in o2["placements"][:8]} == {1}
    small = o2["placements"][8:]["node"] // 8
    assert (o2["status"]["state"][1:] == T.GANG_ADMITTED).all() and set(small.tolist()) == {2}
