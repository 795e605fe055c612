"""Reclaim within queue limits restated over the oracle (tests/preempt_queue_cases.py): the consequences of the definition on random
queue trees with running gangs in two to four priority classes, and one exact hand case per rule."""
import numpy as np
import pytest

from grove_b200 import tables as T
from preempt_queue_cases import (NODE_STEP, QUEUE_STEP, hand_cases, run_cycle_preempt_queues, running_layout, usage_of)
from queue_cases import NONE, REQ, UNL, assign_queues, chain, loads, run_cycle_queues
from reuse_cases import free_table
from test_random_parity_gpu import random_case


def random_snapshot(oracle, seed):
    """a random cluster whose first cycle's admitted gangs run in their queues, in two to four priority classes, and a submission
    of copies of every gang of that cycle at priorities 0-4 -> (nodes, L, tables, queues, gang_queue, running, holdings, running_queue)"""
    nodes, L, tables = random_case(seed)
    rng = np.random.default_rng(seed + 4242)
    qs, gq = assign_queues(rng, tables[0], tables[1])
    n2, t2, q2, gq2, running, holdings, rq = running_layout(oracle, nodes, L, tables, qs, gq, seed)
    running["priority"] = rng.integers(0, int(rng.integers(2, 5)), len(running))
    return n2, L, t2, q2, gq2, running, holdings, rq


def _gang_usage(out, cliques, g):
    pl = out["placements"][out["status"]["placement_off"][g]: out["status"]["placement_off"][g] + out["status"]["n_pods"][g]]
    return [sum(int(cliques[REQ[r]][int(e["clique"])]) for e in pl) for r in range(3)]


def check_consequences(oracle, case):
    nodes, L, (g, c, s), qs, gq, running, holdings, rq = case
    out = run_cycle_preempt_queues(oracle, nodes, L, g, c, s, qs, gq, running, holdings, rq)
    st = out["status"]
    use_r = usage_of(running, holdings)
    ld0 = loads(qs)
    # victims rank strictly below their preemptor and fall at most once
    v = out["victims"]
    assert len(set(v["running"].tolist())) == len(v)
    for x in v:
        assert int(running["priority"][x["running"]]) < int(g["priority"][x["preemptor"]])
        assert st["reserved0"][x["preemptor"]] & T.STATUS_PREEMPTOR
    # node resources are conserved: F_end + U(admitted) = F_0 + holdings(victims)
    F0, Fend = free_table(nodes), free_table(out["nodes_after"])
    lhs = Fend.copy()
    for x in np.nonzero(st["state"] == T.GANG_ADMITTED)[0]:
        for e in out["placements"][st["placement_off"][x]: st["placement_off"][x] + st["n_pods"][x]]:
            q = c[int(e["clique"])]
            lhs[int(e["node"])] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
    rhs = F0.copy()
    for r in v["running"]:
        for h in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
            rhs[int(h["node"])] += [int(h["cpu_milli"]), int(h["mem_mib"]), int(h["gpu"]), int(h["pods"])]
    assert np.array_equal(lhs, rhs)
    # queue loads are conserved the same way
    want = [list(x) for x in ld0]
    for x in np.nonzero((st["state"] == T.GANG_ADMITTED) & (gq != NONE))[0]:
        u = _gang_usage(out, c, x)
        for Q in chain(qs, int(gq[x])):
            for r in range(3):
                want[Q][r] += u[r]
    for r_ in v["running"]:
        if rq[r_] != NONE:
            for Q in chain(qs, int(rq[r_])):
                for r in range(3):
                    want[Q][r] -= use_r[r_][r]
    assert want == out["loads_after"]
    # a queue that starts within its limit ends within it
    for Q in range(len(qs)):
        for r in range(3):
            lim = int(qs["limit"][Q][r])
            if lim != UNL and ld0[Q][r] <= lim:
                assert out["loads_after"][Q][r] <= lim, (Q, r)
    return out


@pytest.mark.parametrize("block", range(4))
def test_random_consequences(oracle, block):
    n_pre = n_vic = 0
    for seed in range(block * 15, block * 15 + 15):
        out = check_consequences(oracle, random_snapshot(oracle, seed))
        n_pre += int(((out["status"]["reserved0"] & T.STATUS_PREEMPTOR) != 0).sum()); n_vic += len(out["victims"])
    assert n_pre > 0 and n_vic > 0


def _same(a, b):
    for k in ("placements", "status", "scope_status", "nodes_after"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("seed", range(8))
def test_unlimited_is_the_reclaim_pass(oracle, seed):
    """no members, or only unlimited queues: grove_run_cycle_preempt's result"""
    nodes, L, (g, c, s), qs, gq, running, holdings, rq = random_snapshot(oracle, 100 + seed)
    ref = oracle.run_cycle_preempt(nodes, L, g, c, s, running, holdings)
    unl = qs.copy(); unl["limit"] = T.QUEUE_UNLIMITED
    for q2, g2 in ((unl, gq), (qs, np.full(len(g), NONE, np.uint32))):
        out = run_cycle_preempt_queues(oracle, nodes, L, g, c, s, q2, g2, running, holdings, rq)
        _same(out, ref)
        assert np.array_equal(out["victims"], ref["victims"])


@pytest.mark.parametrize("seed", range(8))
def test_nothing_evictable_is_the_queue_cycle(oracle, seed):
    nodes, L, (g, c, s), qs, gq, running, holdings, rq = random_snapshot(oracle, 200 + seed)
    running["priority"] = 100
    out = run_cycle_preempt_queues(oracle, nodes, L, g, c, s, qs, gq, running, holdings, rq)
    _same(out, run_cycle_queues(oracle, nodes, L, g, c, s, qs, gq))
    assert len(out["victims"]) == 0


def _hand(oracle, name):
    case = hand_cases()[name]()
    out = check_consequences(oracle, case)
    return case, out


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_hand_case_consequences(oracle, name):
    _hand(oracle, name)


def test_team_a(oracle):
    """the ordinary pass turns it away OVER_LIMIT; the reclaim pass evicts exactly one team-a gang, free nodes stay free"""
    (nodes, L, t, qs, gq, running, holdings, rq), out = _hand(oracle, "team_a")
    base = run_cycle_queues(oracle, nodes, L, *t, qs, gq)
    assert base["status"]["reserved0"][0] == T.STATUS_OVER_LIMIT
    assert out["status"]["state"][0] == T.GANG_ADMITTED and out["status"]["reserved0"][0] == T.STATUS_PREEMPTOR
    assert out["victims"].tolist() == [(1, 0)] and out["steps"] == [QUEUE_STEP]
    assert out["loads_after"][0][2] == 16
    placed = out["placements"]["node"].tolist()
    assert placed not in ([0], [1])   # it lands on a node that was free: node step frees nothing
    free = free_table(out["nodes_after"])[:, 2]
    assert free.tolist().count(8) == 6 - 2   # one freed node, one newly taken: four nodes free, as before


def test_sibling_victim(oracle):
    """the parent's 24 GPUs are full; the preemptor's own queue has room: the victim is the sibling queue's lower-priority gang"""
    _, out = _hand(oracle, "sibling_victim")
    assert out["status"]["reserved0"][0] == T.STATUS_PREEMPTOR
    assert out["victims"].tolist() == [(1, 0)] and out["steps"] == [QUEUE_STEP]


def test_other_queue_spared(oracle):
    """a lower-priority gang of an unrelated queue frees no room in the preemptor's queue: nothing is evicted, it stays rejected"""
    _, out = _hand(oracle, "other_queue_spared")
    assert out["status"]["state"][0] == T.GANG_REJECTED and out["status"]["reserved0"][0] == T.STATUS_OVER_LIMIT
    assert len(out["victims"]) == 0


def test_victim_order(oracle):
    """lowest priority first, then the highest index; gang 3 holds no GPU and is skipped"""
    _, out = _hand(oracle, "victim_order")
    assert out["victims"].tolist() == [(2, 0), (1, 0)] and out["steps"] == [QUEUE_STEP, QUEUE_STEP]


def test_surplus_capped(oracle):
    """12 GPUs held against a limit of 12, 8 of them evictable: room for MinReplicas and one of its three best-effort pods"""
    _, out = _hand(oracle, "surplus_capped")
    assert out["status"]["reserved0"][0] == T.STATUS_PREEMPTOR | T.STATUS_SURPLUS_CAPPED
    assert out["status"]["n_pods"][0] == 2 and out["victims"].tolist() == [(0, 0)]
    assert out["loads_after"][0][2] == 12


def test_no_queue_preemptor(oracle):
    """the node step alone: the cluster is full, one running gang is evicted for its node"""
    _, out = _hand(oracle, "no_queue_preemptor")
    assert out["status"]["reserved0"][0] == T.STATUS_PREEMPTOR
    assert out["victims"].tolist() == [(1, 0)] and out["steps"] == [NODE_STEP]


def test_runs_out(oracle):
    """one evictable gang: the first gang of the class takes it, the other two keep their OVER_LIMIT status"""
    _, out = _hand(oracle, "runs_out")
    assert out["status"]["state"].tolist() == [T.GANG_ADMITTED, T.GANG_REJECTED, T.GANG_REJECTED]
    assert out["status"]["reserved0"].tolist() == [T.STATUS_PREEMPTOR, T.STATUS_OVER_LIMIT, T.STATUS_OVER_LIMIT]
    assert out["victims"].tolist() == [(0, 0)]


def test_starts_over(oracle):
    """24 GPUs held against a limit of 12, 8 of them not handed in: the 4-GPU gang evicts both running gangs and the queue ends at
    12; the 8-GPU gang after it finds nothing left to evict"""
    _, out = _hand(oracle, "starts_over")
    assert out["status"]["state"].tolist() == [T.GANG_ADMITTED, T.GANG_REJECTED]
    assert out["victims"].tolist() == [(1, 0), (0, 0)]
    assert out["loads_after"][0][2] == 12
