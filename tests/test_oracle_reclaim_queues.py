"""Reclaim across queues restated over the oracle (tests/reclaim_queue_cases.py): the guarantees of the definition on random
contested clusters with random queue trees and quotas, the donor set against a direct check, the quota row against the header, the quota ingest, and one exact
hand case per rule."""
import json
import os

import numpy as np
import pytest

from grove_b200 import ingest, tables as T
from preempt_queue_cases import usage_of
from queue_cases import NONE, REQ, UNL, chain, loads, run_cycle_queues
from reclaim_queue_cases import (NODE_STEP, QUEUE_STEP, caps_of, donor_set, hand_cases, random_snapshot, run_cycle_reclaim_queues,
                                 share, share_less)
from reuse_cases import free_table

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
R = T.GANG_REJECTED
A = T.GANG_ADMITTED


def _gang_usage(out, cliques, g):
    pl = out["placements"][out["status"]["placement_off"][g]: out["status"]["placement_off"][g] + out["status"]["n_pods"][g]]
    return [sum(int(cliques[REQ[r]][int(e["clique"])]) for e in pl) for r in range(3)]


def check_guarantees(oracle, case):
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = case
    out = run_cycle_reclaim_queues(oracle, nodes, L, g, c, s, qs, gq, quotas, running, holdings, rq)
    base = run_cycle_queues(oracle, nodes, L, g, c, s, qs, gq)
    st, bst = out["status"], base["status"]
    use_r = usage_of(running, holdings)
    capq = caps_of(qs, quotas)
    # gangs the ordinary pass did not reject keep their outcome; a rejected gang is either re-admitted as a reclaimer or unchanged
    keep = [f for f in T.status_dt.names if f != "placement_off"]   # (placements are merged again: offsets move)
    for x in range(len(g)):
        if bst["state"][x] != R or not (st["reserved0"][x] & T.STATUS_RECLAIMER):
            assert st[keep][x] == bst[keep][x], x
            if st["state"][x] == A:
                assert _gang_usage(out, c, x) == _gang_usage(base, c, x)
        else:
            assert st["state"][x] == A and gq[x] != NONE
    # a victim falls once, has a queue apart from its reclaimer's chain both ways, and its reclaimer carries the flag
    v = out["victims"]
    assert len(set(v["running"].tolist())) == len(v)
    for x in v:
        q, Q = int(rq[x["running"]]), int(gq[x["preemptor"]])
        assert q != NONE and q not in chain(qs, Q) and Q not in chain(qs, q)
        assert st["reserved0"][x["preemptor"]] & T.STATUS_RECLAIMER
    # per class: donors end at or above their quota on what their victims held; the reclaimer's chain ends within its caps
    for cls in out["classes"]:
        Q, ld = cls["queue"], cls["loads_end"]
        lost = {}
        for r in cls["victims"]:
            for X in chain(qs, int(rq[r])):
                if X not in chain(qs, Q):
                    lost.setdefault(X, set()).update(k for k in range(3) if use_r[r][k] > 0)
        for X, res in lost.items():
            for k in res:
                d = int(quotas["deserved"][X][k])
                assert d == UNL or ld[X][k] >= d, (Q, X, k)
        for m in cls["members"]:
            if not (st["reserved0"][m] & T.STATUS_RECLAIMER):
                continue
            u = _gang_usage(out, c, m)
            for X in chain(qs, Q):
                for k in range(3):
                    cap = int(capq["limit"][X][k])
                    if u[k] > 0 and cap != UNL:
                        assert ld[X][k] <= cap, (Q, X, k)
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
    want = [list(x) for x in loads(qs)]
    for x in np.nonzero((st["state"] == A) & (gq != NONE))[0]:
        u = _gang_usage(out, c, x)
        for Q in chain(qs, int(gq[x])):
            for r in range(3):
                want[Q][r] += u[r]
    for r_ in v["running"]:
        for Q in chain(qs, int(rq[r_])):
            for r in range(3):
                want[Q][r] -= use_r[r_][r]
    assert want == out["loads_after"]
    # classes go by ascending share at the start of the pass, ties by index
    ld0 = [list(x) for x in loads(qs)]
    for x in np.nonzero((bst["state"] == A) & (gq != NONE))[0]:
        u = _gang_usage(base, c, x)
        for Q in chain(qs, int(gq[x])):
            for r in range(3):
                ld0[Q][r] += u[r]
    seq = [cls["queue"] for cls in out["classes"]]
    for a, b in zip(seq, seq[1:]):
        sa, sb = share(quotas[a], ld0[a]), share(quotas[b], ld0[b])
        assert share_less(sa, sb) or (not share_less(sb, sa) and a < b)
    return out


@pytest.mark.parametrize("block", range(4))
def test_random_guarantees(oracle, block):
    n_rec = n_vic = 0
    for seed in range(block * 15, block * 15 + 15):
        out = check_guarantees(oracle, random_snapshot(seed, pref=seed % 2 == 1))
        n_rec += int(((out["status"]["reserved0"] & T.STATUS_RECLAIMER) != 0).sum()); n_vic += len(out["victims"])
    assert n_rec > 0 and n_vic > 0


def _direct_donors(qs, quotas, ld, prio, use_r, rq, gone, Q):
    """E(Q) by a direct loop: walk the standing gangs in victim order and take r while, with r and every gang taken before it in
    each queue's subtree gone, every queue of D(r, Q) stays at or above its quota on what r holds, and one has a finite quota on it"""
    order = sorted(range(len(prio)), key=lambda r: (prio[r], -r))
    cq = chain(qs, Q)
    out = []
    for r in order:
        if gone[r] or rq[r] == NONE:
            continue
        cr = chain(qs, int(rq[r]))
        if int(rq[r]) in cq or Q in cr:
            continue
        good, over = True, False
        for X in (X for X in cr if X not in cq):
            before = [x for x in order[: order.index(r) + 1] if not gone[x] and rq[x] != NONE and X in chain(qs, int(rq[x]))]
            for k in range(3):
                d = int(quotas["deserved"][X][k])
                if d == UNL or use_r[r][k] == 0:
                    continue
                over = True
                good &= ld[X][k] - sum(use_r[x][k] for x in before) >= d
        if good and over:
            out.append(r)
    return sorted(out)


@pytest.mark.parametrize("seed", range(12))
def test_donor_set_direct(seed):
    nodes, L, tb, qs, gq, quotas, running, holdings, rq = random_snapshot(500 + seed)
    use_r = usage_of(running, holdings)
    prio = [int(p) for p in running["priority"]]
    ld = loads(qs)
    rng = np.random.default_rng(seed)
    gone = rng.random(len(running)) < 0.2
    for Q in range(len(qs)):
        E = donor_set(qs, quotas, ld, prio, use_r, rq, gone, Q)
        assert E == _direct_donors(qs, quotas, ld, prio, use_r, rq, gone, Q)
        # evicting E(Q) whole leaves every queue outside chain(Q) that loses a gang at or above its quota on what it lost
        after = [list(x) for x in ld]
        lost = {}
        for r in E:
            for X in chain(qs, int(rq[r])):
                for k in range(3):
                    after[X][k] -= use_r[r][k]
                if X not in chain(qs, Q):
                    lost.setdefault(X, set()).update(k for k in range(3) if use_r[r][k] > 0)
        for X, res in lost.items():
            for k in res:
                d = int(quotas["deserved"][X][k])
                assert d == UNL or after[X][k] >= d, (Q, X, k)


@pytest.mark.parametrize("seed", range(6))
def test_unlimited_or_idle_is_the_queue_cycle(oracle, seed):
    """every quota unlimited, or no running gangs: the queue cycle's result, no victims"""
    nodes, L, (g, c, s), qs, gq, quotas, running, holdings, rq = random_snapshot(100 + seed)
    ref = run_cycle_queues(oracle, nodes, L, g, c, s, qs, gq)
    unl = quotas.copy(); unl["deserved"] = UNL
    for args in ((unl, running, holdings, rq), (quotas, running[:0], holdings[:0], rq[:0])):
        out = run_cycle_reclaim_queues(oracle, nodes, L, g, c, s, qs, gq, *args)
        for k in ("placements", "status", "scope_status", "nodes_after"):
            assert np.array_equal(out[k], ref[k]), k
        assert len(out["victims"]) == 0


def test_quota_row_matches_the_header():
    import subprocess
    import tempfile
    inc = os.path.join(os.path.dirname(__file__), "..", "include")
    src = ('#include <stdio.h>\n#include <stddef.h>\n#include "grove_place.h"\nint main(void) {\n'
           'printf("%zu %zu %u\\n", sizeof(grove_queue_quota_t), offsetof(grove_queue_quota_t, deserved), GROVE_STATUS_RECLAIMER);\n'
           'return 0; }\n')
    with tempfile.TemporaryDirectory() as d:
        c_path, exe = os.path.join(d, "probe.c"), os.path.join(d, "probe")
        open(c_path, "w").write(src)
        subprocess.check_call(["cc", "-I", inc, "-o", exe, c_path])
        size, off, flag = map(int, subprocess.check_output([exe]).split())
    assert size == T.queue_quota_dt.itemsize == 24
    assert off == T.queue_quota_dt.fields["deserved"][1] == 0
    assert flag == T.STATUS_RECLAIMER


def test_quota_ingest():
    docs = [{"kind": "Queue", "metadata": {"name": "team-a"},
             "spec": {"parentQueue": "org", "resources": {"cpu": {"quota": 2.5, "limit": 4}, "gpu": {"quota": 8}}}},
            {"kind": "Queue", "metadata": {"name": "org"}, "spec": {"resources": {"gpu": {"quota": -1}, "memory": {"quota": 2048}}}}]
    qs, _, names = ingest.queues_from_manifests(docs, [], {})
    q = ingest.queue_quotas_from_manifests(docs, names)
    assert names == ["org", "team-a"]
    assert q["deserved"].tolist() == [[UNL, 2048, UNL], [2500, UNL, 8]]   # cores -> millicores; -1 or absent: unlimited
    assert qs["limit"].tolist()[1] == [4000, UNL, UNL]


def _workload(path, queue_docs):
    fx = json.load(open(os.path.join(GOLDEN, "workloads.json")))
    labels = json.load(open(os.path.join(GOLDEN, "queues.json")))["labels"][path]
    (pcs,) = fx[path]
    levels = [("zone", "topology.kubernetes.io/zone"), ("host", "kubernetes.io/hostname")]
    g, c, s, _, manifests = ingest.tables_from_pcs(pcs, levels)
    qs, gq, names = ingest.queues_from_manifests(queue_docs, manifests, ingest.podgroup_queues(manifests, labels[pcs["name"]]))
    nodes = T.make_nodes(8)
    nodes["dom"][:, 0] = np.arange(8) // 4; nodes["dom"][:, 1] = np.arange(8)
    nodes["free_cpu_milli"] = 8000; nodes["free_mem_mib"] = 1024; nodes["free_gpu"] = 0; nodes["free_pods"] = 110
    nodes["flags"] = T.NODE_SCHEDULABLE
    return nodes, 2, (g, c, s), qs, gq, ingest.queue_quotas_from_manifests(queue_docs, names)


@pytest.mark.parametrize("path", ["e2e/yaml/workload1.yaml", "e2e/yaml/workload2.yaml"])
def test_reference_workloads(oracle, path):
    """the fixture's quotas are all -1: the queue cycle's result"""
    docs = json.load(open(os.path.join(GOLDEN, "queues.json")))["queues"]
    nodes, L, tb, qs, gq, quotas = _workload(path, docs)
    assert (quotas["deserved"] == UNL).all()
    running = np.zeros(1, dtype=T.running_dt); running["n_holdings"] = 1
    holdings = np.array([(0, 1000, 100, 0, 1)], dtype=T.holding_dt)
    qs = qs.copy(); qs["used"][1] = [1000, 100, 0]
    out = run_cycle_reclaim_queues(oracle, nodes, L, *tb, qs, gq, quotas, running, holdings, np.array([1], np.uint32))
    ref = run_cycle_queues(oracle, nodes, L, *tb, qs, gq)
    for k in ("placements", "status", "scope_status", "nodes_after"):
        assert np.array_equal(out[k], ref[k]), k
    assert len(out["victims"]) == 0


# ---- one hand case per rule --------------------------------------------------------------------------------------------------------

def _hand(oracle, name):
    case = hand_cases()[name]()
    nodes, L, tb, qs, gq, quotas, running, holdings, rq = case
    out = check_guarantees(oracle, case)
    return case, out


@pytest.mark.parametrize("name", sorted(hand_cases()))
def test_hand_case_guarantees(oracle, name):
    _hand(oracle, name)


def test_starved_team(oracle):
    """team-a takes one of team-b's two gangs (the later one in victim order) and team-b ends at its quota of 8"""
    _, out = _hand(oracle, "starved_team")
    assert out["status"]["state"][0] == A and out["status"]["reserved0"][0] == T.STATUS_RECLAIMER
    assert out["victims"].tolist() == [(1, 0)] and out["steps"] == [NODE_STEP]
    assert out["loads_after"][1][2] == 8 and out["loads_after"][0][2] == 8


def test_donor_at_quota(oracle):
    _, out = _hand(oracle, "donor_at_quota")
    assert out["status"]["state"][0] == R and len(out["victims"]) == 0
    assert out["classes"][0]["donors"] == []


def test_reclaimer_at_quota(oracle):
    """team-b is over its quota, but team-a's cap (its quota) is reached: the gate turns it away, its status stays"""
    (nodes, L, tb, qs, gq, *_), out = _hand(oracle, "reclaimer_at_quota")
    assert out["classes"][0]["donors"] != []
    assert out["status"]["state"][0] == R and out["status"]["reserved0"][0] == 0 and len(out["victims"]) == 0


def test_siblings(oracle):
    """the parent is at its quota: it is not asked, and team-b's surplus gang goes"""
    _, out = _hand(oracle, "siblings")
    assert out["status"]["reserved0"][0] == T.STATUS_RECLAIMER and out["victims"].tolist() == [(1, 0)]
    assert out["loads_after"][0][2] == 16


def test_victim_outranks(oracle):
    """priority does not protect a victim: team-b's gang of priority 9 goes for team-a's gang of priority 0"""
    (nodes, L, tb, qs, gq, quotas, running, holdings, rq), out = _hand(oracle, "victim_outranks")
    assert out["victims"].tolist() == [(1, 0)]   # the first in victim order: priority 1, above the reclaimer's 0
    assert int(running["priority"][1]) > int(tb[0]["priority"][0])


def test_partial_donor(oracle):
    _, out = _hand(oracle, "partial_donor")
    assert out["classes"][0]["donors"] == [0, 1]
    assert sorted(out["victims"]["running"].tolist()) == [0, 1] and (out["status"]["state"] == A).all()
    assert out["loads_after"][1][2] == 8


def test_quota_zero(oracle):
    _, out = _hand(oracle, "quota_zero")
    assert out["classes"][0]["donors"] == [0, 1] and (out["status"]["state"] == A).all()


def test_quota_unlimited(oracle):
    _, out = _hand(oracle, "quota_unlimited")
    assert out["classes"][0]["donors"] == [] and out["status"]["state"][0] == R and len(out["victims"]) == 0


def test_no_queue_running(oracle):
    _, out = _hand(oracle, "no_queue_running")
    assert out["victims"].tolist() == [(1, 0)]
    assert out["status"]["state"].tolist() == [A, R]


def test_two_starved(oracle):
    """team-a (queue 1, share 0) goes before team-c (queue 0, share 1/2) and takes the one donor gang; team-c's class finds none"""
    _, out = _hand(oracle, "two_starved")
    assert [cls["queue"] for cls in out["classes"]] == [1, 0]
    assert out["victims"].tolist() == [(2, 1)] and out["classes"][1]["donors"] == []
    assert out["status"]["state"].tolist() == [R, A]


def test_limit_below_quota(oracle):
    _, out = _hand(oracle, "limit_below_quota")
    assert out["status"]["state"].tolist() == [A, R] and len(out["victims"]) == 1
    assert out["loads_after"][0][2] == 8


def test_over_limit_shared_parent(oracle):
    (nodes, L, tb, qs, gq, *_), out = _hand(oracle, "over_limit_shared_parent")
    base = run_cycle_queues(oracle, nodes, L, *tb, qs, gq)
    assert base["status"]["reserved0"][0] == T.STATUS_OVER_LIMIT
    assert out["status"]["reserved0"][0] == T.STATUS_RECLAIMER and out["victims"].tolist() == [(1, 0)]
    assert out["loads_after"][0][2] == 16


def test_queue_step_order(oracle):
    _, out = _hand(oracle, "queue_step_order")
    assert out["victims"].tolist() == [(2, 0), (1, 0)] and out["steps"] == [QUEUE_STEP, QUEUE_STEP]
    assert out["loads_after"][0][2] == 12

