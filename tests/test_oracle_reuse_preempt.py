"""-m "not gpu": reuse with reclaim (include/grove_place.h "reuse with reclaim") as its definition reads, on the CPU oracle: the
properties DESIGN.md section 1 pins, and a hand case for every way a rejected new version can meet its predecessor."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from preempt_cases import churned_cluster, holdings_of
from reuse_cases import free_table, hold_table, run_cycle_reuse, usage
from reuse_preempt_cases import half_full, one_gang as _one_gang, reclaim_rolling_cluster, run_cycle_reuse_preempt, shared_nodes

NONE = T.NONE_U32


def _running(oracle, nodes, tables, prios):
    """an ordinary cycle admits `tables`; running gang r then gets priority prios[r] -> free table, running, holdings"""
    ref = oracle.run_cycle(nodes, 4, *tables)
    running, holdings = holdings_of(ref["placements"], ref["status"], tables[0], tables[1])
    assert len(running) == len(prios)
    running["priority"] = prios
    return ref["nodes_after"], running, holdings


def _same(a, b, keys=("placements", "status", "scope_status", "nodes_after")):
    for k in keys:
        assert np.array_equal(a[k], b[k]), k


def _pairs(out):
    return [(int(v["running"]), int(v["preemptor"])) for v in out["victims"]]


@pytest.mark.parametrize("seed", [11, 12])
def test_without_replacements_it_is_the_reclaim_pass(oracle, seed):
    nodes, L, (g, c, s), running, holdings = churned_cluster(oracle, seed, n=630, g_running=200, g_pending=80)
    none = np.full(len(g), NONE, dtype=np.uint32)
    a = run_cycle_reuse_preempt(oracle, nodes, L, g, c, s, none, running, holdings)
    b = oracle.run_cycle_preempt(nodes, L, g, c, s, running, holdings)
    _same(a, b, keys=("placements", "status", "scope_status", "nodes_after", "victims"))
    assert len(a["victims"]) > 0


@pytest.mark.parametrize("seed", [3, 4])
def test_without_reclaim_work_it_is_the_reuse_cycle(oracle, seed):
    nodes, L, (g, c, s), rep, running, holdings = reclaim_rolling_cluster(oracle, seed, boost=0)
    g = g.copy()
    g["priority"] = running["priority"].min()   # nobody outranks anything that runs: E(p) is empty for every rejected gang
    a = run_cycle_reuse_preempt(oracle, nodes, L, g, c, s, rep, running, holdings)
    b = run_cycle_reuse(oracle, nodes, L, g, c, s, rep, running, holdings)
    _same(a, b)
    assert len(a["victims"]) == 0


def test_without_rejections_it_is_the_reuse_cycle(oracle):
    nodes = synth.e2e_cluster(8)
    now, running, holdings = _running(oracle, nodes, _one_gang(4).build(), [0])
    g, c, s = _one_gang(4, priority=3, b=_one_gang(2, priority=5)).build()
    rep = np.array([NONE, 0], dtype=np.uint32)
    a = run_cycle_reuse_preempt(oracle, now, 4, g, c, s, rep, running, holdings)
    assert (a["status"]["state"] == T.GANG_ADMITTED).all()
    _same(a, run_cycle_reuse(oracle, now, 4, g, c, s, rep, running, holdings))


@pytest.mark.parametrize("seed", [21, 22, 23])
def test_victims_released_and_conservation(oracle, seed):
    nodes, L, (g, c, s), rep, running, holdings = reclaim_rolling_cluster(oracle, seed)
    out = run_cycle_reuse_preempt(oracle, nodes, L, g, c, s, rep, running, holdings)
    pairs = _pairs(out)
    assert pairs, "the scenario must make the reclaim pass evict"
    vs = [v for v, _ in pairs]
    assert len(vs) == len(set(vs))                                              # evicted at most once
    for v, pre in pairs:
        assert int(running["priority"][v]) < int(g["priority"][pre])           # strictly below its preemptor
        assert rep[pre] != v                                                    # never its own new version's victim
        assert out["status"]["reserved0"][pre] & T.STATUS_PREEMPTOR
    assert not set(vs) & set(out["released"])                                   # released gangs are never victims
    N = len(nodes)
    lhs, rhs = free_table(out["nodes_after"]), free_table(nodes)
    for i in np.nonzero(out["status"]["state"] == T.GANG_ADMITTED)[0]:
        lhs = lhs + usage(out["placements"], out["status"], c, i, N)
    for r in set(vs) | set(out["released"]):
        rhs = rhs + hold_table(N, running, holdings, r)
    assert np.array_equal(lhs, rhs)


def test_predecessor_at_or_above_the_class_holds(oracle):
    # running: 0 (priority 5) on nodes 0-1, 1..3 (priority 0) on nodes 2-7; 70 MiB free everywhere.  The new version of 0 asks
    # for 4 pods of 100 MiB: its hold (80 MiB on nodes 0 and 1) gives it two in the ordinary pass.  In the reclaim pass it sees
    # 150 MiB on every node, uses the hold first where it lands on 0 or 1, and evicts elsewhere.
    now, running, holdings = half_full([5, 0, 0, 0])
    b = _one_gang(4, mem=100, priority=5)       # the new version of 0
    _one_gang(1, mem=100, priority=5, b=b)      # ranks after it in the class
    g, c, s = b.build()
    rep = np.array([0, NONE], dtype=np.uint32)
    assert run_cycle_reuse(oracle, now, 4, g, c, s, rep, running, holdings)["status"]["state"][0] == T.GANG_REJECTED
    out = run_cycle_reuse_preempt(oracle, now, 4, g, c, s, rep, running, holdings)
    assert out["status"]["state"][0] == T.GANG_ADMITTED and out["status"]["reserved0"][0] & T.STATUS_PREEMPTOR
    assert 0 in out["released"] and _pairs(out) and all(v != 0 for v, _ in _pairs(out))


def test_predecessor_below_the_class_is_released_not_evicted(oracle):
    # the new version (priority 5) of running gang 0 (priority 1): 0 is in E(5) and evictable.  Admitted, the new version
    # releases it first; it is not a victim.
    now, running, holdings = half_full([1, 0, 2, 2])
    g, c, s = _one_gang(4, mem=80, priority=5).build()
    rep = np.array([0], dtype=np.uint32)
    out = run_cycle_reuse_preempt(oracle, now, 4, g, c, s, rep, running, holdings)
    assert out["status"]["state"][0] == T.GANG_ADMITTED and out["status"]["reserved0"][0] & T.STATUS_PREEMPTOR
    assert out["released"] == [0] and all(v != 0 for v, _ in _pairs(out))


def test_predecessor_evicted_by_an_earlier_preemptor(oracle):
    # gang 0 (priority 9) puts 100 MiB on two nodes: it evicts running 0, the lowest priority.  Gang 1 (priority 9) is the new
    # version of running 0 (its hold, 40 MiB a node, is not enough in the ordinary pass) and finds it gone by its turn: a plain
    # preemptor, it evicts running 1.
    now, running, holdings = shared_nodes()
    b = _one_gang(2, mem=100, priority=9)
    _one_gang(1, mem=120, priority=9, b=b)
    g, c, s = b.build()
    rep = np.array([NONE, 0], dtype=np.uint32)
    out = run_cycle_reuse_preempt(oracle, now, 4, g, c, s, rep, running, holdings)
    assert list(out["status"]["state"]) == [T.GANG_ADMITTED, T.GANG_ADMITTED]
    assert _pairs(out) == [(0, 0), (1, 1)] and out["released"] == []


def test_new_version_outranks_its_predecessor(oracle):
    # the new version (priority 4) of running gang 2 (priority 0) asks for three whole nodes: its hold gives it two in the
    # ordinary pass.  The reclaim pass admits it: it releases its predecessor and evicts one more running gang.
    now, running, holdings = half_full([3, 3, 0, 3])
    g, c, s = _one_gang(3, mem=150, priority=4).build()
    rep = np.array([2], dtype=np.uint32)
    out = run_cycle_reuse_preempt(oracle, now, 4, g, c, s, rep, running, holdings)
    assert out["status"]["state"][0] == T.GANG_ADMITTED and out["status"]["reserved0"][0] & T.STATUS_PREEMPTOR
    assert out["released"] == [2] and len(_pairs(out)) == 1 and _pairs(out)[0][0] != 2
