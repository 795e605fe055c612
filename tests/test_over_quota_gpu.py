"""Over-quota weight through the C ABI (grove_set_over_quota, grove_get_fair_shares): the fair shares against their restatement
(tests/over_quota_cases.py) on random queue trees; grove_run_cycle with a fair-share set, grove_run_cycle_reclaim_queues and
grove_run_cycle_reclaim_preempt_queues with weights against their existing restatements fed those fair shares as the deserved
quotas, on every output; at (reduced) C4, the engine with weights against the engine with quotas := its own reported fair shares;
and the refusals and the set's lifecycle."""
import ctypes as C

import numpy as np
import pytest

from grove_b200 import tables as T
from fair_share_cases import run_fair_share
from over_quota_cases import (as_quotas, fair_share_snapshot, fair_shares, inputs, make_weights, reclaim_beyond_quota,
                              reclaim_snapshot, split_three_to_one, tree_snapshot)
from reclaim_preempt_queue_cases import run_cycle_reclaim_preempt_queues
from reclaim_queue_cases import run_cycle_reclaim_queues

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32
EMPTY_R, EMPTY_H, EMPTY_Q = np.zeros(0, dtype=T.running_dt), np.zeros(0, dtype=T.holding_dt), np.zeros(0, np.uint32)


def _outputs(e):
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                perm=e.debug_perm())


def _same(got, ref, keys, what=""):
    for k in keys:
        assert np.array_equal(got[k], ref[k]), (k, what)


# ---- the fair shares ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("block", range(4))
def test_fair_shares_random_trees(built_lib, block):
    from grove_b200.engine import PlacementEngine
    big = 0
    with PlacementEngine(2) as e:
        for seed in range(block * 50, block * 50 + 50):
            nodes, tables, qs, gq, quotas, w = tree_snapshot(seed)
            ref = np.array(fair_shares(nodes, *tables[:2], qs, gq, quotas, w), dtype=np.uint64).reshape(len(qs), 3)
            e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq); e.set_over_quota(w)
            e.run_cycle_reclaim_queues(quotas, EMPTY_R, EMPTY_H, EMPTY_Q)
            assert np.array_equal(e.fair_shares(len(qs)), ref), seed
            big += int(inputs(nodes, *tables[:2], qs, gq)[0][0] > 1 << 40)
    assert big > 0


# ---- the three entries against their restatements -------------------------------------------------------------------------------

def _fair_cycle(nodes, L, tables, qs, gq, quotas, w, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq); e.set_fair_share(quotas); e.set_over_quota(w)
        e.run_cycle()
        return dict(_outputs(e), order=e.turn_order(), fair=e.fair_shares(len(qs)))


def _check_fair(oracle, case, **kw):
    nodes, L, tables, qs, gq, quotas, w = case
    fair = as_quotas(fair_shares(nodes, *tables[:2], qs, gq, quotas, w))
    got = _fair_cycle(nodes, L, tables, qs, gq, quotas, w, **kw)
    assert np.array_equal(got["fair"], fair["deserved"]), kw
    _same(got, run_fair_share(oracle, nodes, L, *tables, qs, gq, fair), ("status", "placements", "scope_status", "nodes_after",
                                                                         "perm", "order"), kw)
    return got


def _reclaim(nodes, L, tables, qs, gq, quotas, running, holdings, rq, w, preempt=False, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq)
        if w is not None:
            e.set_over_quota(w)
        (e.run_cycle_reclaim_preempt_queues if preempt else e.run_cycle_reclaim_queues)(quotas, running, holdings, rq)
        return dict(_outputs(e), victims=e.victims(), fair=e.fair_shares(len(qs)) if w is not None else None)


RECLAIM_KEYS = ("status", "placements", "scope_status", "nodes_after", "victims", "perm")


def _check_reclaim(oracle, case, preempt=False, **kw):
    nodes, L, tables, qs, gq, quotas, running, holdings, rq, w = case
    fair = as_quotas(fair_shares(nodes, *tables[:2], qs, gq, quotas, w))
    got = _reclaim(nodes, L, tables, qs, gq, quotas, running, holdings, rq, w, preempt=preempt, **kw)
    assert np.array_equal(got["fair"], fair["deserved"]), kw
    restate = run_cycle_reclaim_preempt_queues if preempt else run_cycle_reclaim_queues
    _same(got, restate(oracle, nodes, L, *tables, qs, gq, fair, running, holdings, rq), RECLAIM_KEYS, kw)
    return got


ENTRIES = ["fair_share", "reclaim", "reclaim_preempt"]


def _check(oracle, entry, seed, **kw):
    pref = seed % 2 == 1
    if entry == "fair_share":
        return _check_fair(oracle, fair_share_snapshot(seed, pref=pref), **kw)
    return _check_reclaim(oracle, reclaim_snapshot(seed, pref=pref), preempt=entry == "reclaim_preempt", **kw)


@pytest.mark.parametrize("window", [0, 1])
def test_split_three_to_one(built_lib, oracle, window):
    got = _check_fair(oracle, split_three_to_one(), window=window)
    adm = got["status"]["state"] == T.GANG_ADMITTED
    assert got["fair"][:, 2].tolist() == [32, 16] and [int(adm[:4].sum()), int(adm[4:].sum())] == [3, 1]


@pytest.mark.parametrize("window", [0, 1])
@pytest.mark.parametrize("preempt", [False, True])
def test_reclaim_beyond_quota(built_lib, oracle, window, preempt):
    case = reclaim_beyond_quota()
    got = _check_reclaim(oracle, case, preempt=preempt, window=window)
    assert got["fair"][:, 2].tolist() == [20, 12]
    assert ((got["status"]["reserved0"] & T.STATUS_RECLAIMER) != 0).sum() == 1 and len(got["victims"]) == 1
    plain = _reclaim(*case[:9], None, preempt=preempt, window=window)   # without weights team-a is at its quota
    assert len(plain["victims"]) == 0 and (plain["status"]["state"] == T.GANG_ADMITTED).sum() == 0


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("block", range(4))
def test_random_window_all(built_lib, oracle, entry, block):
    for seed in range(block * 50, block * 50 + 50):
        _check(oracle, entry, seed)


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("window", [1, 7])
@pytest.mark.parametrize("block", range(2))
def test_random_narrow_windows(built_lib, oracle, entry, window, block):
    for seed in range(2000 + block * 50, 2000 + block * 50 + 50):
        _check(oracle, entry, seed, window=window)


# ---- C4: with weights = with quotas := the reported fair shares -----------------------------------------------------------------

def _leaf_weights(n):
    """C4's queues (synth.c4_queues: 0-1 the parents, 2-9 the leaves): GPU weight 1 + leaf index mod 4, cpu and memory 1"""
    return make_weights([(1, 1, 1 if q < 2 else 1 + (q - 2) % 4) for q in range(n)])


def test_reduced_c4_fair_share(built_lib):
    from test_fair_share_gpu import _c4
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, qs, gq, quotas = _c4(5040, 800)
    got = _fair_cycle(nodes, L, tables, qs, gq, quotas, _leaf_weights(len(qs)))
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq); e.set_fair_share(as_quotas(got["fair"]))
        e.run_cycle()
        plain = dict(_outputs(e), order=e.turn_order())
    _same(got, plain, ("status", "placements", "scope_status", "nodes_after", "perm", "order"))
    assert not np.array_equal(got["fair"], quotas["deserved"])


def _reclaim_c4_self(case, preempt):
    nodes, L, tables, qs, gq, quotas, running, holdings, rq = case
    got = _reclaim(nodes, L, tables, qs, gq, quotas, running, holdings, rq, _leaf_weights(len(qs)), preempt=preempt)
    plain = _reclaim(nodes, L, tables, qs, gq, as_quotas(got["fair"]), running, holdings, rq, None, preempt=preempt)
    _same(got, plain, RECLAIM_KEYS)
    assert not np.array_equal(got["fair"], quotas["deserved"])
    return got


@pytest.mark.parametrize("preempt", [False, True])
def test_reduced_c4_reclaim(built_lib, oracle, preempt):
    from test_reclaim_queues_gpu import c4_case
    _reclaim_c4_self(c4_case(oracle), preempt)


def test_full_c4_reclaim(built_lib):
    """a fresh engine per arm: the same inputs with weights and with their fair shares as the quotas"""
    from grove_b200 import synth
    from scripts.bench_reclaim_queues import layout
    L, nodes, tables, qs, gq, running, holdings, rq = layout(0.6)
    got = _reclaim_c4_self((nodes, L, tables, qs, gq, synth.c4_queue_quotas(qs, running, holdings, rq, spread=1.2), running,
                            holdings, rq), False)
    print(f"C4 reclaim with weights: {len(got['victims'])} victims, fair GPU shares {got['fair'][:, 2].tolist()}")


# ---- refusals and lifecycle -----------------------------------------------------------------------------------------------------

def test_refusals_and_lifecycle(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tables, qs, gq, quotas, running, holdings, rq, w = reclaim_beyond_quota()
    NQ = len(qs)

    def code(call):
        with pytest.raises(GroveError) as ex:
            call()
        return ex.value.code

    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        assert code(lambda: e.set_over_quota(w)) == -5                        # no queue set
        e.set_queues(qs, gq)
        assert code(lambda: e.set_over_quota(w[:1])) == -1                    # one row per queue
        assert e.lib.grove_set_over_quota(e.h, None, C.c_uint32(NQ)) == -1     # no rows
        e.set_over_quota(w)
        assert code(lambda: e.fair_shares(NQ)) == -5                          # no call with weights yet
        e.run_cycle_reclaim_queues(quotas, running, holdings, rq)
        fair = e.fair_shares(NQ)
        assert fair[:, 2].tolist() == [20, 12]
        out = np.zeros(NQ * 3, dtype=np.uint64)
        assert e.lib.grove_get_fair_shares(e.h, out.ctypes.data_as(C.c_void_p), C.c_uint32(NQ - 1)) == -4
        e.run_cycle()                                                          # takes no quotas: reads nothing, keeps the set
        assert np.array_equal(e.fair_shares(NQ), fair)
        e.update_nodes(np.arange(len(nodes), dtype=np.uint32), nodes)         # kept by an update
        e.run_cycle_reclaim_queues(quotas, running, holdings, rq)
        assert np.array_equal(e.fair_shares(NQ), fair) and len(e.victims()) == 1
        # entries that take no quotas keep the set even when their class cycles re-submit: preemption within the queue limits
        # evicts team-b's lower-priority gangs here, and the weights and shares are still in place afterwards
        low = running.copy(); low["priority"][1:] = -1
        e.update_nodes(np.arange(len(nodes), dtype=np.uint32), nodes)
        e.run_cycle_preempt_queues(low, holdings, rq)
        assert len(e.victims()) > 0 and np.array_equal(e.fair_shares(NQ), fair)
        e.update_nodes(np.arange(len(nodes), dtype=np.uint32), nodes)
        e.run_cycle_reclaim_queues(quotas, running, holdings, rq)              # still weighted
        assert np.array_equal(e.fair_shares(NQ), fair) and len(e.victims()) == 1
        e.set_queues(qs, gq)                                                   # cleared with the queue set
        assert code(lambda: e.fair_shares(NQ)) == -5
        e.run_cycle_reclaim_queues(quotas, running, holdings, rq)
        assert code(lambda: e.fair_shares(NQ)) == -5 and len(e.victims()) == 0
        for clear in (lambda: e.submit_gangs(*tables), lambda: e.load_nodes(nodes)):
            e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq); e.set_over_quota(w)
            clear()
            assert code(lambda: e.set_over_quota(w)) == -5 and code(lambda: e.fair_shares(NQ)) == -5
        # a fair-share set with weights: the shares of grove_set_fair_share's quotas
        nodes2, L2, tables2, qs2, gq2, quotas2, w2 = split_three_to_one()
        e.load_nodes(nodes2); e.submit_gangs(*tables2); e.set_queues(qs2, gq2); e.set_fair_share(quotas2); e.set_over_quota(w2)
        e.run_cycle()
        assert e.fair_shares(len(qs2))[:, 2].tolist() == [32, 16]
        after = e.nodes()
        e.run_cycle()   # the set stays; the second cycle's shares come from the table it starts from, which the first filled
        assert e.fair_shares(len(qs2)).tolist() == fair_shares(after, *tables2[:2], qs2, gq2, quotas2, w2)
