"""-m "not gpu": the fair-share order (include/grove_place.h "fair-share order") as restated in tests/fair_share_cases.py -- the
consequences of the definition, O(R) computed the engine's way against the definition's walk, the fixed-point loop against the
one-turn-at-a-time restatement, and one hand case per rule."""
import numpy as np
import pytest

from grove_b200 import tables as T
from fair_share_cases import (UNL, NONE, fixed_point, hand_cases, order_vec, order_walk, random_snapshot, ranks, run_fair_share,
                              share_value, use_of, with_order, _tree)
from queue_cases import chain, loads, make_queues, run_cycle_queues
from reclaim_queue_cases import make_quotas

KEYS = ("status", "placements", "scope_status", "nodes_after")


def _same(a, b):
    return all(np.array_equal(a[k], b[k]) for k in KEYS)


@pytest.mark.parametrize("seed", range(12))
def test_zero_shares_are_the_queue_cycle(oracle, seed):
    """1. no finite quota anywhere: the merge by head rank is rank order, and the result is the queue cycle's"""
    nodes, L, tb, qs, gq, quotas = random_snapshot(seed)
    quotas["deserved"] = UNL
    got = run_fair_share(oracle, nodes, L, *tb, qs, gq, quotas)
    assert got["order"].tolist() == ranks(tb[0])[0]
    assert _same(got, run_cycle_queues(oracle, nodes, L, *tb, qs, gq))


@pytest.mark.parametrize("seed", range(6))
def test_no_members_is_the_ordinary_cycle(oracle, seed):
    """2. no members: grove_run_cycle's result"""
    nodes, L, tb, qs, gq, quotas = random_snapshot(seed)
    gq[:] = NONE
    got = run_fair_share(oracle, nodes, L, *tb, qs, gq, quotas)
    assert _same(got, oracle.run_cycle(nodes, L, *tb))


def _share_of(queues, quotas, ld, X):
    return share_value(quotas[X], ld[X])


@pytest.mark.parametrize("seed", range(40))
def test_properties(oracle, seed):
    nodes, L, tb, qs, gq, quotas = random_snapshot(seed, pref=seed % 2 == 1)
    gangs, cliques = tb[0], tb[1]
    got = run_fair_share(oracle, nodes, L, *tb, qs, gq, quotas)
    order = got["order"].tolist()
    G, NQ = len(gangs), len(qs)
    _, rank = ranks(gangs)
    # 4. a permutation of all gangs
    assert sorted(order) == list(range(G))
    # 3. inside a leaf, rank order
    pos = {g: p for p, g in enumerate(order)}
    for q in range(NQ + 1):
        mine = [g for g in order if (NQ if gq[g] == NONE else int(gq[g])) == q]
        assert mine == sorted(mine, key=lambda g: rank[g])
    # 5. at every turn the chosen path minimises (share, rank of head) among siblings at each level
    U = use_of(got, cliques)
    ld = loads(qs)
    kids = _tree(qs)
    waiting = {q: sorted([g for g in range(G) if (NQ if gq[g] == NONE else int(gq[g])) == q], key=lambda g: rank[g]) for q in range(NQ + 1)}

    def head(X):
        if X <= NQ and not kids[X]:
            return waiting[X][0] if waiting[X] else None
        hs = [(( _share_of(qs, quotas, ld, C) if C < NQ else 0), rank[h], h) for C in kids[X] for h in [head(C)] if h is not None]
        return min(hs)[2] if hs else None

    for g in order:
        q = NQ if gq[g] == NONE else int(gq[g])
        path = [q] + (chain(qs, q)[1:] if q < NQ else [])
        for X in path:   # every node on g's path: among its siblings, the smallest key
            p = int(qs["parent"][X]) if X < NQ and qs["parent"][X] != NONE else NQ + 1
            sib = [C for C in kids[p] if head(C) is not None]
            keys = {C: ((_share_of(qs, quotas, ld, C) if C < NQ else 0), rank[head(C)]) for C in sib}
            assert min(keys, key=keys.get) == X
        waiting[q].pop(0)
        if q < NQ:
            for Q in chain(qs, q):
                for r in range(3):
                    ld[Q][r] += int(U[g][r])
    # 6. a queue that starts within its limit ends within it
    start, end = loads(qs), [list(x) for x in ld]
    for Q in range(NQ):
        for r in range(3):
            lim = int(qs["limit"][Q][r])
            if lim != UNL and start[Q][r] <= lim:
                assert end[Q][r] <= lim
    # 7. a rejected member leaves its queue's share unchanged: in the walk, the loads of its chain after its turn are those
    # before it (the walk charges what the oracle bound for the gang at its turn)
    st = got["status"]["state"]
    for g, before, after in got["trace"]:
        if st[g] != T.GANG_ADMITTED:
            assert before == after and got["status"]["n_pods"][g] == 0
    assert len(got["trace"]) == int((gq != NONE).sum())


@pytest.mark.parametrize("seed", range(60))
def test_vectorised_order_is_the_walk(seed):
    """O(U) by scans, prefix maxima and stable sorts equals the walk, on random trees up to depth 4 with random usages"""
    rng = np.random.default_rng(seed)
    parents = [None] * int(rng.integers(1, 4))
    frontier = list(range(len(parents)))
    for _ in range(int(rng.integers(0, 4))):
        nxt = []
        for p in frontier:
            for _ in range(int(rng.integers(1, 3))):
                parents.append(p); nxt.append(len(parents) - 1)
        frontier = nxt
    NQ = len(parents)
    qs = make_queues([(p, (None, None, None), tuple(int(x) for x in rng.integers(0, 20, 3))) for p in parents])
    quotas = make_quotas([tuple(None if rng.random() < 0.3 else int(rng.integers(0, 30)) for _ in range(3)) for _ in range(NQ)])
    inner = {p for p in parents if p is not None}
    leaves = [q for q in range(NQ) if q not in inner]
    G = int(rng.integers(1, 60))
    b = T.GangTableBuilder()
    for _ in range(G):
        b.add_gang([(None, [dict(gpu=1, min=1)])], priority=int(rng.integers(0, 4)))
    gangs = b.build()[0]
    gq = np.array([NONE if rng.random() < 0.2 else int(rng.choice(leaves)) for _ in range(G)], np.uint32)
    U = rng.integers(0, 12, (G, 3)) * (rng.random((G, 1)) < 0.7)
    assert np.array_equal(order_vec(qs, quotas, gangs, gq, U), order_walk(qs, quotas, gangs, gq, U))


@pytest.mark.parametrize("seed", range(30))
def test_fixed_point_converges_to_the_walk(oracle, seed):
    nodes, L, tb, qs, gq, quotas = random_snapshot(seed, pref=seed % 2 == 1)
    ref = run_fair_share(oracle, nodes, L, *tb, qs, gq, quotas)
    for order in (order_vec, order_walk):
        out, O, it = fixed_point(oracle, nodes, L, *tb, qs, gq, quotas, order=order)
        assert np.array_equal(O, ref["order"]) and _same(out, ref)
        assert it <= int((gq != NONE).sum()) + 1


def _case(name, oracle):
    nodes, L, tb, qs, gq, quotas = hand_cases()[name]()
    got = run_fair_share(oracle, nodes, L, *tb, qs, gq, quotas)
    out, O, it = fixed_point(oracle, nodes, L, *tb, qs, gq, quotas)
    assert np.array_equal(O, got["order"]) and _same(out, got)
    return got, it, (nodes, L, tb, qs, gq)


def test_starved_low_priority_team_goes_first(oracle):
    got, _, (nodes, L, tb, qs, gq) = _case("starved_team_first", oracle)
    assert got["status"]["state"].tolist() == [T.GANG_REJECTED] * 2 + [T.GANG_ADMITTED] * 2
    plain = run_cycle_queues(oracle, nodes, L, *tb, qs, gq)   # by priority, team-b's gangs would take both nodes
    assert plain["status"]["state"].tolist() == [T.GANG_ADMITTED] * 2 + [T.GANG_REJECTED] * 2


def test_parent_share_decides_before_the_child(oracle):
    got, _, _ = _case("parent_before_child", oracle)
    assert got["order"].tolist() == [1, 0] and got["status"]["state"].tolist() == [T.GANG_REJECTED, T.GANG_ADMITTED]


def test_share_tie_goes_to_the_better_rank(oracle):
    got, _, _ = _case("share_tie_by_rank", oracle)
    assert got["order"].tolist() == [1, 0]


def test_rejected_member_leaves_its_share_and_goes_again(oracle):
    got, _, _ = _case("rejected_goes_again", oracle)
    assert got["order"].tolist() == [0, 1, 2]
    assert got["status"]["state"].tolist() == [T.GANG_REJECTED, T.GANG_ADMITTED, T.GANG_REJECTED]


def test_zero_quota_with_load_goes_last(oracle):
    got, _, _ = _case("zero_quota_last", oracle)
    assert got["order"].tolist() == [1, 0] and got["status"]["state"].tolist() == [T.GANG_REJECTED, T.GANG_ADMITTED]


def test_over_limit_member(oracle):
    got, _, _ = _case("over_limit_member", oracle)
    assert got["order"].tolist() == [0, 2, 1]
    assert got["status"]["reserved0"].tolist() == [0, T.STATUS_OVER_LIMIT, 0]


def test_scaled_gang_whose_base_goes_later_is_base_rejected(oracle):
    got, _, _ = _case("base_takes_turn_later", oracle)
    assert got["order"].tolist() == [1, 0]
    assert got["status"]["state"].tolist() == [T.GANG_ADMITTED, T.GANG_BASE_REJECTED]


def test_case_that_needs_three_iterations(oracle):
    _, it, _ = _case("many_iterations", oracle)
    assert it >= 3


def test_with_order_gives_the_order():
    b = T.GangTableBuilder()
    for p in (3, 1, 2):
        b.add_gang([(None, [dict(gpu=1, min=1)])], priority=p)
    g = b.build()[0]
    assert ranks(with_order(g, [2, 0, 1]))[0] == [2, 0, 1]


def test_abi_layout():
    assert T.fair_share_stats_dt.itemsize == 8
