"""-m "not gpu": wide submissions (include/grove_place.h grove_submit_gangs_wide) on the CPU oracle's wide build: it equals the
ordinary oracle within the old limits, keeps the pass's properties beyond them, and hand cases of 600-pod PodGroups."""
import numpy as np
import pytest

from grove_b200 import tables as T
from test_random_parity_gpu import random_case
from wide_cases import pods_per_gang, wide_case
import wide_oracle as W

NONE = T.NONE_U32


def _counts_of(cliques):
    counts = np.zeros(len(cliques), dtype=T.clique_count_dt)
    counts["min_replicas"], counts["replicas"] = cliques["min_replicas"], cliques["replicas"]
    return counts


@pytest.mark.parametrize("seed", range(100))
def test_wide_build_equals_the_oracle_within_the_old_limits(oracle, seed):
    nodes, L, (g, c, s) = random_case(5000 + seed, pref=seed % 2 == 1)
    ref = oracle.run_cycle(nodes, L, g, c, s)
    q = c.copy(); q["min_replicas"] = 0; q["replicas"] = 0   # the wide entry reads the counts only
    got = W.run_cycle_wide(nodes, L, g, q, _counts_of(c), s)
    for k in ("placements", "status", "scope_status", "nodes_after", "perm"):
        assert np.array_equal(got[k], ref[k]), k


def _usage(nodes, tables, placements):
    gangs, cliques, counts, scopes = tables
    u = np.zeros((len(nodes), 4), dtype=np.int64)
    for p in placements:
        q = cliques[p["clique"]]
        u[p["node"]] += (int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1)
    return u


@pytest.mark.parametrize("seed", range(24))
def test_wide_pass_properties(seed):
    nodes, L, tables = wide_case(7000 + seed, pref=seed % 2 == 1, big_nodes=seed % 3 == 0)
    gangs, cliques, counts, scopes = tables
    assert pods_per_gang(gangs, counts).max() > T.MAX_GANG_PODS or counts["replicas"].max() > 255 or seed % 5   # mostly wide
    out = W.run_cycle_wide(nodes, L, *tables)
    st, pl = out["status"], out["placements"]
    # resources conserved: what is left plus what was bound is what there was, and nothing goes below zero
    u = _usage(nodes, tables, pl)
    for k, f in enumerate(("free_cpu_milli", "free_mem_mib", "free_gpu", "free_pods")):
        assert np.array_equal(out["nodes_after"][f].astype(np.int64) + u[:, k], nodes[f].astype(np.int64)), f
    # all or nothing, MinReplicas <= bound <= replicas, every Required level inside one labelled domain
    per_clique = np.bincount(pl["clique"], minlength=len(cliques)) if len(pl) else np.zeros(len(cliques), int)
    for gi, g in enumerate(gangs):
        qs = range(g["clique_off"], g["clique_off"] + g["n_cliques"])
        if st[gi]["state"] != T.GANG_ADMITTED:
            assert all(per_clique[q] == 0 for q in qs)
            continue
        for q in qs:
            assert counts["min_replicas"][q] <= per_clique[q] <= counts["replicas"][q]
        mine = pl[st[gi]["placement_off"]: st[gi]["placement_off"] + st[gi]["n_pods"]]
        if g["level"] != T.LEVEL_NONE:
            doms = nodes["dom"][mine["node"], g["level"]]
            assert len(set(doms.tolist())) <= 1 and T.DOM_ABSENT not in doms
        for si in range(g["scope_off"], g["scope_off"] + g["n_scopes"]):   # each scope's cliques share one domain of its level
            lv, sc = scopes["level"][si], scopes[si]
            if lv != T.LEVEL_NONE:
                qs_s = range(g["clique_off"] + sc["first_clique"], g["clique_off"] + sc["first_clique"] + sc["n_cliques"])
                doms = nodes["dom"][mine["node"][np.isin(mine["clique"], list(qs_s))], lv]
                assert len(set(doms.tolist())) <= 1 and T.DOM_ABSENT not in doms
        for q in qs:
            lv = cliques["level"][q]
            if lv != T.LEVEL_NONE:
                doms = nodes["dom"][mine["node"][mine["clique"] == q], lv]
                assert len(set(doms.tolist())) <= 1 and T.DOM_ABSENT not in doms


def _one_clique_gang(reps, level=None, anchor=0, mn=None):
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(cpu=100, mem=64, min=reps if mn is None else mn, replicas=reps, level=level)])], anchor=anchor)
    return b.build_wide()


def test_600_pods_on_110_pod_nodes():
    """no level: the pods fill the nodes in visiting order from the anchor, 110 each, 50 on the sixth"""
    nodes = T.make_nodes(8)
    nodes["free_cpu_milli"], nodes["free_mem_mib"], nodes["free_pods"], nodes["flags"] = 64000, 524288, 110, T.NODE_SCHEDULABLE
    nodes["dom"][:, 0] = 0
    out = W.run_cycle_wide(nodes, 1, *_one_clique_gang(600))
    assert out["status"][0]["state"] == T.GANG_ADMITTED and out["status"][0]["n_pods"] == 600
    assert np.bincount(out["placements"]["node"], minlength=8).tolist() == [110, 110, 110, 110, 110, 50, 0, 0]
    assert out["nodes_after"]["free_pods"].tolist() == [0, 0, 0, 0, 0, 60, 110, 110]


def test_600_pods_on_one_node_of_more_than_255():
    """Required host level: the first node in visiting order that takes all 600 pods (a capacity byte would say 255)"""
    nodes = T.make_nodes(4)
    nodes["free_cpu_milli"], nodes["free_mem_mib"], nodes["flags"] = 4_000_000, 4_000_000, T.NODE_SCHEDULABLE
    nodes["free_pods"] = [300, 599, 700, 1000]
    nodes["dom"][:, 0] = 0
    nodes["dom"][:, 1] = np.arange(4)
    out = W.run_cycle_wide(nodes, 2, *_one_clique_gang(600, level=1))
    assert out["status"][0]["state"] == T.GANG_ADMITTED
    assert np.bincount(out["placements"]["node"], minlength=4).tolist() == [0, 0, 600, 0]
    # 1000 pods of which 700 are guaranteed: the guaranteed ones need one node, the surplus stays on it (best effort)
    out = W.run_cycle_wide(nodes, 2, *_one_clique_gang(1000, level=1, mn=700))
    assert np.bincount(out["placements"]["node"], minlength=4).tolist() == [0, 0, 700, 0]
    out = W.run_cycle_wide(nodes, 2, *_one_clique_gang(1001, level=1))
    assert out["status"][0]["state"] == T.GANG_REJECTED and len(out["placements"]) == 0


def test_more_than_2048_pods_is_a_limit():
    nodes = T.make_nodes(4)
    nodes["free_pods"], nodes["flags"] = 1000, T.NODE_SCHEDULABLE
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(min=1024, replicas=1024), dict(min=1, replicas=1025)])])
    with pytest.raises(RuntimeError, match="-4"):
        W.run_cycle_wide(nodes, 1, *b.build_wide())
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(min=1024, replicas=1024), dict(min=1, replicas=1024)])])
    assert W.run_cycle_wide(nodes, 1, *b.build_wide())["status"][0]["state"] == T.GANG_ADMITTED
