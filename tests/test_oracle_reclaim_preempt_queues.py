"""Reclaim, then preempt, restated over the oracle (tests/reclaim_preempt_queue_cases.py): the cycle reduces to each pass alone
where the other has nothing to do, the guarantees of the definition on random contested clusters, and one exact hand case per
interaction of the two passes."""
import numpy as np
import pytest

from grove_b200 import tables as T
import reclaim_preempt_queue_cases as RP
from preempt_queue_cases import run_cycle_preempt_queues, usage_of
from queue_cases import NONE, REQ, UNL, chain, loads, run_cycle_queues
from reclaim_preempt_queue_cases import hand_cases, random_snapshot, run_cycle_reclaim_preempt_queues
from reclaim_queue_cases import run_cycle_reclaim_queues
from reuse_cases import free_table

R = T.GANG_REJECTED
A = T.GANG_ADMITTED
OUTPUTS = ("placements", "status", "scope_status", "nodes_after", "victims", "steps", "loads_after", "perm")


def _run(oracle, case):
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = case
    return run_cycle_reclaim_preempt_queues(oracle, nodes, L, g, c, s, qs, gq, quotas, running, holdings, rq)


def _same(a, b, keys=OUTPUTS, what=None):
    for k in keys:
        if isinstance(a[k], np.ndarray):
            assert np.array_equal(a[k], b[k]), (k, what)
        else:
            assert a[k] == b[k], (k, what)


def _gang_usage(out, cliques, g):
    pl = out["placements"][out["status"]["placement_off"][g]: out["status"]["placement_off"][g] + out["status"]["n_pods"][g]]
    return [sum(int(cliques[REQ[r]][int(e["clique"])]) for e in pl) for r in range(3)]


def check_guarantees(oracle, case):
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = case
    out = _run(oracle, case)
    base = run_cycle_queues(oracle, nodes, L, g, c, s, qs, gq)
    st, bst = out["status"], base["status"]
    use_r = usage_of(running, holdings)
    prio = running["priority"]
    flags = st["reserved0"]
    # gangs the ordinary pass did not reject keep their outcome; a rejected gang is admitted by exactly one pass, or unchanged
    keep = [f for f in T.status_dt.names if f != "placement_off"]   # (placements are merged again: offsets move)
    for x in range(len(g)):
        by_pass = flags[x] & (T.STATUS_RECLAIMER | T.STATUS_PREEMPTOR)
        assert by_pass != (T.STATUS_RECLAIMER | T.STATUS_PREEMPTOR), x   # a reclaimer is never reconsidered
        if bst["state"][x] != R or not by_pass:
            assert st[keep][x] == bst[keep][x], x
            if st["state"][x] == A:
                assert _gang_usage(out, c, x) == _gang_usage(base, c, x)
        else:
            assert st["state"][x] == A
    # every victim falls once; the reclaim pass's come first; a reclaim victim lies apart from its reclaimer's chain both ways, a
    # preempt victim ranks strictly below its preemptor
    v = out["victims"]
    assert len(set(v["running"].tolist())) == len(v)
    for i, x in enumerate(v):
        r, p = int(x["running"]), int(x["preemptor"])
        if i < out["n_reclaim"]:
            assert flags[p] & T.STATUS_RECLAIMER
            q, Q = int(rq[r]), int(gq[p])
            assert q != NONE and q not in chain(qs, Q) and Q not in chain(qs, q)
        else:
            assert flags[p] & T.STATUS_PREEMPTOR
            assert int(prio[r]) < int(g["priority"][p])
    # node resources are conserved: F_end + U(admitted) = F_0 + holdings(victims)
    lhs = free_table(out["nodes_after"]).copy()
    for x in np.nonzero(st["state"] == A)[0]:
        for e in out["placements"][st["placement_off"][x]: st["placement_off"][x] + st["n_pods"][x]]:
            q = c[int(e["clique"])]
            lhs[int(e["node"])] += [int(q["req_cpu_milli"]), int(q["req_mem_mib"]), int(q["req_gpu"]), 1]
    rhs = free_table(nodes).copy()
    for r in v["running"]:
        for h in holdings[running["holding_off"][r]: running["holding_off"][r] + running["n_holdings"][r]]:
            rhs[int(h["node"])] += [int(h["cpu_milli"]), int(h["mem_mib"]), int(h["gpu"]), int(h["pods"])]
    assert np.array_equal(lhs, rhs)
    # ... and the queue loads the same way
    ld0 = [list(x) for x in loads(qs)]
    want = [list(x) for x in ld0]
    for x in np.nonzero((st["state"] == A) & (gq != NONE))[0]:
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
def test_random_guarantees(oracle, block):
    n_rec = n_pre = 0
    for seed in range(block * 15, block * 15 + 15):
        out = check_guarantees(oracle, random_snapshot(seed, pref=seed % 2 == 1))
        n_rec += int(((out["status"]["reserved0"] & T.STATUS_RECLAIMER) != 0).sum())
        n_pre += int(((out["status"]["reserved0"] & T.STATUS_PREEMPTOR) != 0).sum())
    assert n_rec > 0 and n_pre > 0


def test_random_snapshots_run_both_passes(oracle):
    """the snapshots the GPU parity test runs at window all: 11 of the 200 cycles admit gangs in both passes"""
    both = 0
    for seed in range(200):
        f = _run(oracle, random_snapshot(seed, pref=seed % 2 == 1))["status"]["reserved0"]
        both += bool((f & T.STATUS_RECLAIMER).any() and (f & T.STATUS_PREEMPTOR).any())
    assert both >= 10


@pytest.mark.parametrize("block", range(4))
def test_each_pass_alone_is_its_entry(oracle, block):
    """the ordinary pass and then only the reclaim pass (only the preempt pass) give what the restatement of
    grove_run_cycle_reclaim_queues (grove_run_cycle_preempt_queues) gives, on every output"""
    for seed in range(block * 20, block * 20 + 20):
        nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = random_snapshot(seed, pref=seed % 2 == 1)
        st = RP.ordinary_pass(oracle, nodes, L, g, c, s, qs, gq, running, holdings)
        classes = RP.reclaim_pass(oracle, nodes, L, g, c, s, qs, gq, quotas, rq, st)
        ref = run_cycle_reclaim_queues(oracle, nodes, L, g, c, s, qs, gq, quotas, running, holdings, rq)
        _same(RP.outputs(nodes, qs, st), ref, what=("reclaim", seed))
        assert classes == ref["classes"], seed
        st = RP.ordinary_pass(oracle, nodes, L, g, c, s, qs, gq, running, holdings)
        RP.preempt_pass(oracle, nodes, L, g, c, s, qs, gq, rq, st)
        _same(RP.outputs(nodes, qs, st), run_cycle_preempt_queues(oracle, nodes, L, g, c, s, qs, gq, running, holdings, rq),
              what=("preempt", seed))


@pytest.mark.parametrize("seed", range(10))
def test_unlimited_quotas_is_preempt_queues(oracle, seed):
    """every quota unlimited: no donor, the reclaim pass does nothing"""
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = random_snapshot(100 + seed, pref=seed % 2 == 1)
    quotas = quotas.copy(); quotas["deserved"] = T.QUEUE_UNLIMITED
    out = _run(oracle, (nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq))
    _same(out, run_cycle_preempt_queues(oracle, nodes, L, g, c, s, qs, gq, running, holdings, rq), what=seed)


@pytest.mark.parametrize("seed", range(10))
def test_nothing_below_is_reclaim_queues(oracle, seed):
    """no running gang below any rejected gang's priority: E(p) is empty, the preempt pass does nothing"""
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = random_snapshot(200 + seed, pref=seed % 2 == 1)
    running = running.copy(); running["priority"] += int(g["priority"].max())
    case = (nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq)
    out = _run(oracle, case)
    ref = run_cycle_reclaim_queues(oracle, nodes, L, g, c, s, qs, gq, quotas, running, holdings, rq)
    _same(out, ref, what=seed)
    assert out["n_reclaim"] == len(out["victims"])


@pytest.mark.parametrize("seed", range(6))
def test_no_running_is_the_queue_cycle(oracle, seed):
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = random_snapshot(300 + seed)
    out = _run(oracle, (nodes, L, (g, c, s), qs, gq, quotas, running[:0], holdings[:0], rq[:0]))
    _same(out, run_cycle_queues(oracle, nodes, L, g, c, s, qs, gq), keys=("placements", "status", "scope_status", "nodes_after", "perm"))
    assert len(out["victims"]) == 0


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_hand_case_guarantees(oracle, name):
    check_guarantees(oracle, hand_cases()[name]())


def _flags(out):
    return [(int(a), int(b)) for a, b in zip(out["status"]["state"], out["status"]["reserved0"])]


def test_three_teams(oracle):
    """a-0 (gang 0) reclaims b-1 (running 1); c-high (gang 1) preempts c-low (running 2); each pass alone admits one of them"""
    case = hand_cases()["three_teams"]()
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = case
    out = _run(oracle, case)
    assert _flags(out) == [(A, T.STATUS_RECLAIMER), (A, T.STATUS_PREEMPTOR)]
    assert out["victims"].tolist() == [(1, 0), (2, 1)] and out["n_reclaim"] == 1
    assert out["placements"]["node"].tolist() == [1, 2]
    only_reclaim = run_cycle_reclaim_queues(oracle, nodes, L, g, c, s, qs, gq, quotas, running, holdings, rq)
    assert _flags(only_reclaim)[1][0] == R and only_reclaim["victims"].tolist() == [(1, 0)]
    only_preempt = run_cycle_preempt_queues(oracle, nodes, L, g, c, s, qs, gq, running, holdings, rq)
    assert _flags(only_preempt)[0][0] == R and only_preempt["victims"].tolist() == [(2, 1)]


def test_capped_then_preempted(oracle):
    """team-a's cap (its quota) turns a-new away in the reclaim pass; its unlimited limit lets it preempt its own a-old"""
    case = hand_cases()["capped_then_preempted"]()
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = case
    only_reclaim = run_cycle_reclaim_queues(oracle, nodes, L, g, c, s, qs, gq, quotas, running, holdings, rq)
    assert only_reclaim["classes"][0]["donors"] == [1] and _flags(only_reclaim) == [(R, 0)] and len(only_reclaim["victims"]) == 0
    out = _run(oracle, case)
    assert _flags(out) == [(A, T.STATUS_PREEMPTOR)] and out["victims"].tolist() == [(0, 0)] and out["n_reclaim"] == 0


def test_no_queue_gang(oracle):
    """a gang without a queue is no reclaim class's member; the preempt pass admits it"""
    out = _run(oracle, hand_cases()["no_queue_gang"]())
    assert out["classes"] == [] and _flags(out) == [(A, T.STATUS_PREEMPTOR)]
    assert len(out["victims"]) == 1 and out["n_reclaim"] == 0


def test_reclaim_empties_e(oracle):
    """the reclaim pass evicts the only running gang below priority 5: x stays rejected, as the ordinary pass left it"""
    case = hand_cases()["reclaim_empties_e"]()
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = case
    out = _run(oracle, case)
    assert _flags(out) == [(A, T.STATUS_RECLAIMER), (R, 0)] and out["victims"].tolist() == [(0, 0)] and out["n_reclaim"] == 1
    only_preempt = run_cycle_preempt_queues(oracle, nodes, L, g, c, s, qs, gq, running, holdings, rq)
    assert _flags(only_preempt)[1] == (A, T.STATUS_PREEMPTOR)   # alone, the preempt pass would have given x that gang's room


def test_skipped_class_preempts(oracle):
    """team-a's class has no donor (team-b holds exactly its quota); a-0 then preempts team-b's lower-priority gang"""
    out = _run(oracle, hand_cases()["skipped_class_preempts"]())
    assert [(cls["queue"], cls["donors"]) for cls in out["classes"]] == [(0, [])]
    assert _flags(out) == [(A, T.STATUS_PREEMPTOR)] and out["victims"].tolist() == [(0, 0)] and out["n_reclaim"] == 0
