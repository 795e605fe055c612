"""Fences as their definition reads (tests/fence_cases.py, over the unchanged sequential oracle): the properties the definition
promises on random snapshots, one hand case per rule, and the multi-cycle starvation case the feature exists for."""
import numpy as np
import pytest

from grove_b200 import tables as T
from fence_cases import Starvation, fence_randomly, hand_cases, run_cycle_fences
from test_random_parity_gpu import random_case

RES = ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")


def _order(gangs):
    return sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))


def _case(seed):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    return nodes, L, tables, fence_randomly(np.random.default_rng(seed + 91), tables[0])


def _gang_out(out, g):
    s = out["status"][g]
    return s, out["placements"][s["placement_off"]: s["placement_off"] + s["n_pods"]]


@pytest.mark.parametrize("seed", range(0, 30))
def test_empty_set_is_the_ordinary_cycle(oracle, seed):
    nodes, L, tables, _ = _case(seed)
    got = run_cycle_fences(oracle, nodes, L, *tables, [])
    ref = oracle.run_cycle(nodes, L, *tables)
    for k in ("status", "placements", "scope_status", "nodes_after"):
        assert np.array_equal(got[k], ref[k]), k


@pytest.mark.parametrize("seed", range(30, 100))
def test_properties(oracle, seed):
    nodes, L, tables, fencing = _case(seed)
    gangs, cliques, _ = tables
    active = {}
    got = run_cycle_fences(oracle, nodes, L, *tables, fencing, trace=active)
    st, perm = got["status"], got["perm"]
    order = _order(gangs)
    # gangs ranked before the first fencing gang keep their ordinary outcome
    plain = oracle.run_cycle(nodes, L, *tables)
    for g in order:
        if g in set(fencing.tolist()):
            break
        a, pa = _gang_out(got, g)
        r, pr = _gang_out(plain, g)
        for f in ("state", "level", "reserved0", "score_num", "score_den", "n_pods", "domain_node"):
            assert a[f] == r[f], (g, f)
        assert np.array_equal(pa, pr)
    # no gang ranked after an active fence has a pod in the fenced domain
    rank = {g: k for k, g in enumerate(order)}
    for f, (lo, hi) in active.items():
        inside = set(perm[lo:hi].tolist())
        for g in order[rank[f] + 1:]:
            if st["state"][g] == T.GANG_ADMITTED:
                _, pl = _gang_out(got, g)
                assert not inside & set(pl["node"].tolist()), (f, g)
        assert st["reserved0"][f] == T.STATUS_FENCING and st["state"][f] == T.GANG_REJECTED
        assert st["domain_node"][f] == perm[lo] and st["level"][f] == gangs["level"][f]
    flagged = set(np.nonzero(st["reserved0"])[0].tolist())
    assert flagged == set(active)
    # picks never overlap
    ranges = sorted(p for p in got["picks"].values() if p is not None)
    for (a0, a1), (b0, b1) in zip(ranges, ranges[1:]):
        assert a1 <= b0
    # resources are conserved, and the node table is the arithmetic of what the admitted gangs bound
    used = np.zeros((len(nodes), 4), dtype=np.int64)
    for e in got["placements"]:
        q = cliques[int(e["clique"])]
        used[int(e["node"])] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
    for k, f in enumerate(RES):
        assert np.array_equal(nodes[f].astype(np.int64) - used[:, k], got["nodes_after"][f].astype(np.int64)), f
    assert np.array_equal(got["nodes_after"]["flags"], nodes["flags"])


def _hand(oracle, name):
    nodes, L, tables, fencing = hand_cases()[name]()
    return nodes, L, tables, run_cycle_fences(oracle, nodes, L, *tables, fencing)


def test_least_shortfall_wins(oracle):
    nodes, L, tables, got = _hand(oracle, "least_shortfall")
    st = got["status"]
    assert st["state"].tolist() == [T.GANG_REJECTED, T.GANG_ADMITTED]
    assert got["picks"][0] == (4, 6) and st["reserved0"][0] == T.STATUS_FENCING and st["domain_node"][0] == 4
    plain = oracle.run_cycle(nodes, L, *tables)
    assert plain["placements"]["node"].tolist() == [4]                     # without the fence it takes the big gang's block
    assert got["placements"]["node"][0] < 4


def test_ties_follow_candidate_order(oracle):
    _, _, _, got = _hand(oracle, "tie_order")
    assert got["picks"][0] == (4, 6)                                         # the anchor's block
    assert got["status"]["state"][1] == T.GANG_ADMITTED and got["placements"]["node"][0] < 4


def test_nested_overlap_is_skipped(oracle):
    _, _, _, got = _hand(oracle, "nested_overlap")
    assert got["picks"][0] == (0, 2)
    assert got["picks"][1] is not None and got["picks"][1][0] >= 2           # no host inside block 0
    st = got["status"]
    assert st["state"].tolist() == [T.GANG_REJECTED, T.GANG_REJECTED, T.GANG_ADMITTED]
    assert int(got["placements"]["node"][0]) not in (0, 1, got["picks"][1][0])


def test_admitted_gang_fences_nothing(oracle):
    nodes, L, tables, got = _hand(oracle, "admitted_fences_nothing")
    ref = oracle.run_cycle(nodes, L, *tables)
    assert got["status"]["state"][0] == T.GANG_ADMITTED
    for k in ("status", "placements", "nodes_after"):
        assert np.array_equal(got[k], ref[k]), k


def test_gated_or_base_rejected_gang_fences_nothing(oracle):
    nodes, L, tables, got = _hand(oracle, "gated_fences_nothing")
    ref = oracle.run_cycle(nodes, L, *tables)
    assert got["status"]["state"].tolist()[:3] == [T.GANG_GATED_SKIP, T.GANG_REJECTED, T.GANG_BASE_REJECTED]
    for k in ("status", "placements", "nodes_after"):
        assert np.array_equal(got[k], ref[k]), k


def test_before_and_after(oracle):
    nodes, L, tables, got = _hand(oracle, "before_and_after")
    plain = oracle.run_cycle(nodes, L, *tables)
    st = got["status"]
    assert np.array_equal(st[0], plain["status"][0])
    assert st["reserved0"][1] == T.STATUS_FENCING
    lo, hi = got["picks"][1]
    for g in range(2, len(tables[0])):
        if st["state"][g] == T.GANG_ADMITTED:
            n = got["placements"][st["placement_off"][g]]["node"]
            assert not lo <= n < hi


def test_starvation(oracle):
    """Without fences the block-sized gang is never admitted in 20 cycles; with a fence after one rejected cycle it is admitted
    within 4 (the fence empties its block as the one-node gangs in it finish, two cycles at most)."""
    def cycle(nodes, L, tables, fencing):
        return run_cycle_fences(oracle, nodes, L, *tables, fencing)
    never, hist = Starvation().run(cycle, fence_after=None)
    assert never is None and all(s["state"] == T.GANG_REJECTED for s in hist)
    at, hist = Starvation().run(cycle, fence_after=1)
    assert at is not None and at <= 4, at
    assert all(s["reserved0"] == T.STATUS_FENCING for s in hist[1:-1])
