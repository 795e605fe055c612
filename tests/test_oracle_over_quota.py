"""Over-quota weight on the CPU: the division's guarantees on random queue trees (tests/over_quota_cases.py), the ingest of
overQuotaWeight, and the two hand cases through the existing restatements fed the fair shares as the deserved quotas."""
import json
import os

import numpy as np
import pytest

from grove_b200 import ingest, tables as T
from fair_share_cases import run_fair_share
from over_quota_cases import (UNL, as_quotas, divide, fair_shares, inputs, make_weights, reclaim_beyond_quota, split_three_to_one,
                              tree_snapshot)
from reclaim_queue_cases import run_cycle_reclaim_queues

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _divisions(nodes, tables, qs, gq, quotas, w):
    """every (parent pool, children, their inputs, their fair shares, the rounds that gave something) the division makes, per
    resource"""
    NQ = len(qs)
    C, _, dem = inputs(nodes, tables[0], tables[1], qs, gq)
    kids = {q: [] for q in range(NQ + 1)}
    for q in range(NQ):
        p = int(qs["parent"][q])
        kids[NQ if p == T.NONE_U32 else p].append(q)
    fair = fair_shares(nodes, tables[0], tables[1], qs, gq, quotas, w)
    for r in range(3):
        dm = [dem[q][r] for q in range(NQ)]
        lim = [int(qs["limit"][q][r]) for q in range(NQ)]
        des = [int(quotas["deserved"][q][r]) for q in range(NQ)]
        ww = [int(w["over_quota"][q][r]) for q in range(NQ)]
        pool = {NQ: C[r]}
        for p in [NQ] + list(range(NQ)):
            if kids[p]:
                k = []
                f, pl = divide(pool[p], kids[p], dm, lim, des, ww, k)
                assert all(fair[c][r] == f[c] for c in kids[p])
                pool.update(pl)
                yield pool[p], kids[p], dm, lim, des, ww, f, pl, k[0]


@pytest.mark.parametrize("block", range(4))
def test_division_guarantees(block):
    seen = dict(need_left=0, covered=0, zero=0, pairs=0)
    for seed in range(block * 100, block * 100 + 100):
        nodes, tables, qs, gq, quotas, w = tree_snapshot(seed)
        for P, kids, dm, lim, des, ww, f, pl, k in _divisions(nodes, tables, qs, gq, quotas, w):
            fin = [c for c in kids if des[c] != UNL]
            want = {c: min(dm[c], lim[c]) for c in kids}
            base = {c: min(des[c], want[c]) for c in fin}
            took = sum(base.values()) + sum(want[c] for c in kids if des[c] == UNL)
            for c in fin:   # base <= fair <= max(base, min(demand, limit))
                assert base[c] <= f[c] <= max(base[c], want[c])
                if ww[c] == 0:   # weight 0: exactly the base
                    assert f[c] == base[c]
                    seen["zero"] += 1
            for c in kids:
                if des[c] == UNL:
                    assert f[c] == UNL and pl[c] == want[c]
            given = sum(f[c] for c in fin) + sum(want[c] for c in kids if des[c] == UNL)
            left = [c for c in fin if ww[c] > 0 and f[c] < want[c]]
            if left and P >= took:   # some weighted child still has need: the pool is used up
                assert given == P
                seen["need_left"] += 1
            if P >= took + sum(want[c] - base[c] for c in fin if ww[c] > 0):   # the pool covers every weighted child's ask
                assert all(f[c] == want[c] for c in fin if ww[c] > 0)
                seen["covered"] += 1
            for i, a in enumerate(left):   # unsaturated siblings split within rounding: under one unit per round each
                for b in left[i + 1:]:
                    xa, xb = f[a] - base[a], f[b] - base[b]
                    assert abs(xa * ww[b] - xb * ww[a]) <= max(k, 1) * (ww[a] + ww[b]), (seed, a, b)
                    seen["pairs"] += 1
    assert all(v > 0 for v in seen.values()), seen


def test_split_three_to_one(oracle):
    nodes, L, tables, qs, gq, quotas, w = split_three_to_one()
    fair = fair_shares(nodes, *tables[:2], qs, gq, quotas, w)
    assert [x[2] for x in fair] == [32, 16] and fair[0][0] == UNL
    for q, want in ((as_quotas(fair), [3, 1]), (quotas, [2, 2])):
        out = run_fair_share(oracle, nodes, L, *tables, qs, gq, q)
        adm = out["status"]["state"] == T.GANG_ADMITTED
        assert [int(adm[:4].sum()), int(adm[4:].sum())] == want


def test_reclaim_beyond_quota(oracle):
    nodes, L, tables, qs, gq, quotas, running, holdings, rq, w = reclaim_beyond_quota()
    fair = fair_shares(nodes, *tables[:2], qs, gq, quotas, w)
    assert [x[2] for x in fair] == [20, 12]
    out = run_cycle_reclaim_queues(oracle, nodes, L, *tables, qs, gq, as_quotas(fair), running, holdings, rq)
    assert ((out["status"]["reserved0"] & T.STATUS_RECLAIMER) != 0).sum() == 1 and len(out["victims"]) == 1
    assert int(rq[out["victims"]["running"][0]]) == 1
    out = run_cycle_reclaim_queues(oracle, nodes, L, *tables, qs, gq, quotas, running, holdings, rq)
    assert (out["status"]["state"] == T.GANG_ADMITTED).sum() == 0 and len(out["victims"]) == 0


def test_equal_weights_split_evenly():
    """two queues that deserve nothing and ask for everything split 16 GPUs 8 / 8 at weights 1 / 1 and 12 / 4 at 3 / 1; the odd unit
    of 17 goes to the heavier weight, then the lower index"""
    for free, wts, want in ((16, (1, 1), [8, 8]), (16, (3, 1), [12, 4]), (17, (1, 1), [9, 8]), (17, (1, 3), [4, 13])):
        P, kids = free, [0, 1]
        f, _ = divide(P, kids, [100, 100], [UNL, UNL], [0, 0], list(wts))
        assert [f[0], f[1]] == want


def test_weight_ingest():
    docs = [{"kind": "Queue", "metadata": {"name": "org"}, "spec": {"resources": {"gpu": {"overQuotaWeight": 3}}}},
            {"kind": "Queue", "metadata": {"name": "team-a"},
             "spec": {"parentQueue": "org", "resources": {"cpu": {"overQuotaWeight": 0}, "memory": {"overQuotaWeight": "2"}}}}]
    _, _, names = ingest.queues_from_manifests(docs, [], {})
    w = ingest.queue_weights_from_manifests(docs, names)
    assert w["over_quota"].tolist() == [[1, 1, 3], [0, 2, 1]]   # absent: 1
    for bad in (-1, 1.5, "x"):
        docs[1]["spec"]["resources"]["gpu"] = {"overQuotaWeight": bad}
        with pytest.raises(ValueError, match="team-a"):
            ingest.queue_weights_from_manifests(docs, names)


def test_reference_fixture_weights():
    """the reference's Queue objects set overQuotaWeight 1 on every resource"""
    docs = json.load(open(os.path.join(GOLDEN, "queues.json")))["queues"]
    _, _, names = ingest.queues_from_manifests(docs, [], {})
    w = ingest.queue_weights_from_manifests(docs, names)
    assert len(w) == len(docs) and (w["over_quota"] == 1).all()
    assert np.array_equal(w, make_weights([(1, 1, 1)] * len(docs)))
