"""-m "not gpu": the consolidation pass as restated in tests/consolidate_cases.py over the sequential oracle: the consequences
its definition names, on random snapshots; one hand case per rule; and the starvation case of fence_cases with its one-node
gangs running and movable."""
import numpy as np
import pytest

from grove_b200 import tables as T
from consolidate_cases import Starvation, candidates, hand_cases, random_snapshot, run_cycle_consolidate
from fence_cases import picks
from reuse_cases import free_table, hold_table, usage

OUT = ("status", "placements", "scope_status", "nodes_after")


def _same(a, b):
    for k in OUT:
        assert np.array_equal(a[k], b[k]), k


def _run(oracle, case, trace=None):
    nodes, L, tables, targets, spec_of, running, holdings = case
    return run_cycle_consolidate(oracle, nodes, L, *tables, targets, spec_of, running, holdings, trace=trace)


@pytest.mark.parametrize("seed", range(60))
def test_consequences_on_random_snapshots(oracle, seed):
    case = random_snapshot(oracle, seed)
    nodes, L, (g, c, s), targets, spec_of, running, holdings = case
    out = _run(oracle, case)
    plain = oracle.run_cycle(nodes, L, g, c, s)
    st, pst = out["status"], plain["status"]
    G, N, R = len(g), len(nodes), len(running)
    specs = {int(x) for x in spec_of if x != T.NONE_U32}
    moved = {int(m["running"]): int(m["target"]) for m in out["moves"]}
    assert len(moved) == len(out["moves"])                                       # a running gang moves at most once
    for gi in range(G):
        if gi in specs or gi in set(targets.tolist()):
            continue
        assert st[gi]["state"] == pst[gi]["state"] and st[gi]["reserved0"] == 0   # everyone else keeps the ordinary outcome
        if st[gi]["state"] == T.GANG_ADMITTED:                                     # ... its placement and its scope domains
            a = out["placements"][st[gi]["placement_off"]: st[gi]["placement_off"] + st[gi]["n_pods"]]
            b0 = plain["placements"][pst[gi]["placement_off"]: pst[gi]["placement_off"] + pst[gi]["n_pods"]]
            assert np.array_equal(a, b0)
        so, ns = int(g["scope_off"][gi]), int(g["n_scopes"][gi])
        assert np.array_equal(out["scope_status"][so: so + ns], plain["scope_status"][so: so + ns])
    for r, b in moved.items():
        assert int(running["priority"][r]) <= int(g["priority"][b])              # the priority bar
        assert st["reserved0"][b] == T.STATUS_CONSOLIDATED and st["state"][b] == T.GANG_ADMITTED
        x = int(spec_of[r])                                                       # no running gang is lost
        assert st["state"][x] == T.GANG_ADMITTED and st["reserved0"][x] == T.STATUS_MOVED
    for x in specs:
        if st["reserved0"][x] != T.STATUS_MOVED:
            assert st["state"][x] == T.GANG_GATED_SKIP
    for gi in range(G):
        if st["reserved0"][gi] == T.STATUS_CONSOLIDATED:                           # admitted only with its movers placed
            assert all(st["state"][int(spec_of[r])] == T.GANG_ADMITTED for r, b in moved.items() if b == gi)
    # resources: F_end + sum U(admitted) = F0 + sum H(moved)
    lhs = free_table(out["nodes_after"]).copy()
    for gi in range(G):
        if st["state"][gi] == T.GANG_ADMITTED:
            lhs += usage(out["placements"], st, c, gi, N)
    rhs = free_table(nodes) + sum((hold_table(N, running, holdings, r) for r in moved), np.zeros((N, 4), np.int64))
    assert np.array_equal(lhs, rhs)
    if not len(targets) or spec_of.size == 0 or (spec_of == T.NONE_U32).all() or not (pst["state"][targets] == T.GANG_REJECTED).any():
        _same(out, plain)


def test_nothing_to_do_is_the_ordinary_cycle(oracle):
    for seed in range(12):
        nodes, L, tables, targets, spec_of, running, holdings = random_snapshot(oracle, seed)
        plain = oracle.run_cycle(nodes, L, *tables)
        for t, so in ((targets[:0], spec_of), (targets, np.full_like(spec_of, T.NONE_U32))):
            _same(run_cycle_consolidate(oracle, nodes, L, *tables, t, so, running, holdings), plain)


@pytest.mark.parametrize("block", range(4))
def test_domain_order_matches_the_fence_pick(oracle, block):
    """the shortfall arithmetic here restates the fences': over the same table, the first domain in the order candidates are
    tried in is the domain fence_cases.picks picks, for every gang with a Required level of random snapshots"""
    from test_random_parity_gpu import random_case
    checked = 0
    for seed in range(block * 25, block * 25 + 25):
        nodes, L, (g, c, s) = random_case(seed, pref=seed % 2 == 1)
        topo = oracle.topology(nodes, L)
        F = free_table(nodes)
        for b in range(len(g)):
            if g["level"][b] == T.LEVEL_NONE:
                continue
            order = candidates(topo, nodes, L, g, c, s, b, F, F, qualify=False)
            assert order[0] == picks(oracle, nodes, L, g, c, s, [b])[b], (seed, b)
            checked += 1
    assert checked


def _case(name):
    return hand_cases()[name]()


def test_priority_bar(oracle):
    case = _case("priority_bar")
    tr = {}
    out = _run(oracle, case, tr)
    assert tr["tried"][0] == [(2, 4)]        # block 0 (closest to the anchor) holds a gang above the target: it never qualifies
    assert out["moves"].tolist() == [(1, 0)]


def test_order_by_shortfall_over_f(oracle):
    case = _case("f_shortfall_order")
    tr = {}
    out = _run(oracle, case, tr)
    assert tr["tried"][0][0] == (2, 4) and tr["tries"] == 1
    assert out["moves"].tolist() == [(2, 0)]
    nodes, L, (g, c, s) = case[0], case[1], case[2]
    Fmask = picks(oracle, nodes, L, g, c, s, [0])[0]   # the fences' pick over the same table is the first domain tried
    assert Fmask == tr["tried"][0][0]


@pytest.mark.parametrize("traps,admitted", [(3, True), (4, False)])
def test_try_limit(oracle, traps, admitted):
    tr = {}
    out = _run(oracle, _case(f"try_limit_{traps}"), tr)
    assert tr["tries"] == T.CONSOLIDATE_TRIES
    assert (out["status"]["state"][0] == T.GANG_ADMITTED) == admitted


@pytest.mark.parametrize("name", ["rollback_fits_nowhere", "mover_required_level"])
def test_rollback(oracle, name):
    case = _case(name)
    nodes, L, tables = case[:3]
    out = _run(oracle, case)
    _same(out, oracle.run_cycle(nodes, L, *tables))
    assert not len(out["moves"])


def test_mover_lands_back(oracle):
    out = _run(oracle, _case("lands_back"))
    st = out["status"]
    assert st["reserved0"][0] == T.STATUS_CONSOLIDATED and st["reserved0"][1] == T.STATUS_MOVED
    pl = out["placements"]
    assert set(pl[st["placement_off"][1]: st["placement_off"][1] + 2]["node"].tolist()) == {0, 1}


def test_no_required_level(oracle):
    tr = {}
    out = _run(oracle, _case("no_level"), tr)
    assert tr["tried"][0] == [(0, 6)] and out["status"]["reserved0"][0] == T.STATUS_CONSOLIDATED
    assert sorted(out["moves"]["running"].tolist()) == [0, 1]


def test_two_targets_in_rank_order(oracle):
    out = _run(oracle, _case("two_targets"))
    st = out["status"]
    assert st["reserved0"][0] == T.STATUS_CONSOLIDATED and st["state"][1] == T.GANG_REJECTED
    assert out["moves"]["target"].tolist() == [0]


def test_starvation(oracle):
    """the block gang is admitted in the first cycle it is a target in which the one-node gangs of the block it tries first have
    room elsewhere; without targets it waits longer"""
    seen = []

    def cycle(nodes, L, tables, targets, spec_of, running, holdings):
        tr = {}
        out = run_cycle_consolidate(oracle, nodes, L, *tables, targets, spec_of, running, holdings, trace=tr)
        if 0 in tr["tried"] and tr["tried"][0]:
            F = oracle.run_cycle(nodes, L, *tables)["nodes_after"]
            lo, hi = tr["tried"][0][0]   # blocks_case is in sorted order already: node = sorted index
            movers = int((F["free_gpu"][lo:hi] < 8).sum())
            room = int((F["free_gpu"][:lo] == 8).sum() + (F["free_gpu"][hi:] == 8).sum())
            seen.append((room >= movers, out["status"]["state"][0] == T.GANG_ADMITTED))
        return out

    plain, _ = Starvation(small_per_cycle=10).run(cycle, target_after=None)
    at, hist = Starvation(small_per_cycle=10).run(cycle, target_after=1)
    assert at is not None and plain is not None and at < plain
    assert seen and all(admitted for room, admitted in seen if room)
    assert hist[at][2] > 0
