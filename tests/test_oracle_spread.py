"""Topology spread as its definition reads (tests/spread_cases.py, over the unchanged sequential oracle): the properties the
definition promises on random snapshots, and one hand case per rule."""
import numpy as np
import pytest

from grove_b200 import tables as T
from spread_cases import domains, group_randomly, hand_cases, run_cycle_spread
from test_random_parity_gpu import random_case

NONE = T.NONE_U32
RES = ("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")


def _case(seed, **kw):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    groups, gg, seeds = group_randomly(np.random.default_rng(seed + 77), nodes, L, tables[0], tables[1], **kw)
    return nodes, L, tables, groups, gg, seeds


def _order(gangs):
    return sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))


@pytest.mark.parametrize("seed", range(0, 40))
def test_no_groups_is_the_ordinary_cycle(oracle, seed):
    nodes, L, tables, groups, _, seeds = _case(seed)
    none = np.full(len(tables[0]), NONE, np.uint32)
    got = run_cycle_spread(oracle, nodes, L, *tables, groups, none, seeds)
    ref = oracle.run_cycle(nodes, L, *tables)
    for k in ("status", "placements", "scope_status", "nodes_after"):
        assert np.array_equal(got[k], ref[k]), k


@pytest.mark.parametrize("seed", range(40, 100))
def test_properties(oracle, seed):
    nodes, L, tables, groups, gg, seeds = _case(seed)
    gangs, cliques, _ = tables
    trace = []
    got = run_cycle_spread(oracle, nodes, L, *tables, groups, gg, seeds, trace=trace)
    st = got["status"]
    # gangs ranked before every member keep their ordinary outcome
    plain = oracle.run_cycle(nodes, L, *tables)
    for g in _order(gangs):
        if gg[g] != NONE:
            break
        a, r = st[g], plain["status"][g]
        for f in ("state", "level", "reserved0", "score_num", "score_den", "n_pods", "domain_node"):
            assert a[f] == r[f], (g, f)
        assert np.array_equal(got["placements"][a["placement_off"]: a["placement_off"] + a["n_pods"]],
                              plain["placements"][r["placement_off"]: r["placement_off"] + r["n_pods"]])
    # every admitted member of a HARD group: the skew inequality held at its turn, in an eligible domain
    for g, s, counts, m, allowed, A in trace:
        if A is not None and groups["mode"][s] == T.SPREAD_HARD:
            assert allowed[A] and counts[A] + 1 - m <= groups["max_skew"][s]
        if A is not None and st["reserved0"][g]:
            assert groups["mode"][s] == T.SPREAD_SOFT and not allowed[A]
    assert not (st["reserved0"][gg == NONE]).any()
    # resources are conserved: what the admitted gangs bound is what left the free table
    used = np.zeros((len(nodes), 4), dtype=np.int64)
    for e in got["placements"]:
        q = cliques[int(e["clique"])]
        used[int(e["node"])] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
    for k, f in enumerate(RES):
        assert np.array_equal(nodes[f].astype(np.int64) - used[:, k], got["nodes_after"][f].astype(np.int64)), f


@pytest.mark.parametrize("seed", range(100, 140))
def test_soft_is_hard_when_hard_admits_every_member(oracle, seed):
    nodes, L, tables, groups, gg, seeds = _case(seed)
    hard, soft = groups.copy(), groups.copy()
    hard["mode"] = T.SPREAD_HARD; soft["mode"] = T.SPREAD_SOFT
    h = run_cycle_spread(oracle, nodes, L, *tables, hard, gg, seeds)
    s = run_cycle_spread(oracle, nodes, L, *tables, soft, gg, seeds)
    members = gg != NONE
    evaluated = members & (h["status"]["state"] != T.GANG_GATED_SKIP) & (h["status"]["state"] != T.GANG_BASE_REJECTED)
    if (h["status"]["state"][evaluated] == T.GANG_ADMITTED).all():
        for k in ("status", "placements", "scope_status", "nodes_after"):
            assert np.array_equal(h[k], s[k]), k


def _zones_of(oracle, nodes, L, out, level=0):
    _, dom, _ = domains(oracle, nodes, L)
    return [int(dom[int(d), level]) if d != NONE else None for d in out["status"]["domain_node"]]


def _hand(oracle, name):
    nodes, L, tables, groups, gg, seeds = hand_cases()[name]()
    return nodes, L, tables, run_cycle_spread(oracle, nodes, L, *tables, groups, gg, seeds)


def test_four_zones_eight_replicas_two_per_zone(oracle):
    for name in ("four_zones_hard", "four_zones_soft"):
        nodes, L, tables, out = _hand(oracle, name)
        assert (out["status"]["state"] == T.GANG_ADMITTED).all()
        assert sorted(_zones_of(oracle, nodes, L, out)) == [0, 0, 1, 1, 2, 2, 3, 3]
        assert not out["status"]["reserved0"].any()
        plain = oracle.run_cycle(nodes, L, *tables)
        assert sorted(_zones_of(oracle, nodes, L, plain)) != [0, 0, 1, 1, 2, 2, 3, 3]   # packing alone does not spread them


def test_full_zone_hard_waits_soft_skews(oracle):
    nodes, L, _, hard = _hand(oracle, "full_zone_hard")
    assert hard["status"]["state"].tolist() == [1, 1, 1, T.GANG_REJECTED]
    assert not hard["status"]["reserved0"].any()
    _, _, _, soft = _hand(oracle, "full_zone_soft")
    assert soft["status"]["state"].tolist() == [1, 1, 1, 1]
    assert soft["status"]["reserved0"].tolist() == [0, 0, 0, T.STATUS_SPREAD_SKEWED]
    assert _zones_of(oracle, nodes, L, soft).count(0) == 3


def test_ineligible_domains_are_not_counted(oracle):
    for name, out_zone in (("ineligible_zone", 3), ("cordoned_zone", 2)):
        nodes, L, _, out = _hand(oracle, name)
        z = _zones_of(oracle, nodes, L, out)
        assert (out["status"]["state"] == T.GANG_ADMITTED).all(), name
        assert out_zone not in z and sorted(z) == sorted([x for x in range(4) if x != out_zone] * 2), name


def test_seeds_shift_placements(oracle):
    for name in ("seeded_hard", "seeded_soft"):
        nodes, L, _, out = _hand(oracle, name)
        assert sorted(_zones_of(oracle, nodes, L, out)) == [2, 2, 3, 3]


def test_max_skew_two(oracle):
    nodes, L, _, out = _hand(oracle, "skew_two")
    z = _zones_of(oracle, nodes, L, out)
    counts = [z.count(x) for x in range(4)]
    assert sum(counts) == 8 and max(counts) - min(counts) <= 2


def test_host_level(oracle):
    nodes, L, _, out = _hand(oracle, "host_level")
    hosts = _zones_of(oracle, nodes, L, out, level=1)
    assert sorted(hosts[:6]) == list(range(6)) and len(set(hosts)) == 6


def test_preferred_levels(oracle):
    nodes, L, tables, out = _hand(oracle, "preferred")
    z = _zones_of(oracle, nodes, L, out)
    assert sorted(z.count(x) for x in range(4)) == [1, 1, 2, 2]
    assert (out["status"]["level"] == 1).all()   # every replica got its Preferred host


def test_scaled_gangs_as_members(oracle):
    nodes, L, tables, out = _hand(oracle, "scaled")
    z = _zones_of(oracle, nodes, L, out)
    assert (out["status"]["state"] == T.GANG_ADMITTED).all()
    assert len(set(z[:3])) == 3 and len(set(z[3:])) == 3


def test_mixed_members_and_non_members(oracle):
    nodes, L, tables, groups, gg, seeds = hand_cases()["mixed"]()
    out = run_cycle_spread(oracle, nodes, L, *tables, groups, gg, seeds)
    z = _zones_of(oracle, nodes, L, out)
    for s in (0, 1):
        zs = [z[g] for g in range(len(gg)) if gg[g] == s]
        assert max(zs.count(x) for x in range(4)) - min(zs.count(x) for x in range(4)) <= 1
