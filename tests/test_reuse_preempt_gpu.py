"""Reuse with reclaim through the C ABI (grove_run_cycle_reuse_preempt) against its gang-by-gang restatement over the sequential
oracle (tests/reuse_preempt_cases.py): statuses, placements, scope domains, the node table and the victim list.  The engine runs
each reclaim class as one cycle over a view built on the device; the restatement reconsiders the rejected gangs one at a time:
identical outputs say that the batching is exact."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from reuse_preempt_cases import half_full, one_gang as _one_gang, reclaim_rolling_cluster, run_cycle_reuse_preempt, shared_nodes

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32


def _run(nodes, L, tables, rep, running, holdings, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        st = e.run_cycle_reuse_preempt(rep, running, holdings)
        out = dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                   victims=e.victims(), stats=st)
        e.run_cycle()   # the handle is back on the caller's submission: an ordinary cycle runs on it
        assert len(e.victims()) == 0
        return out


def _check(oracle, nodes, L, tables, rep, running, holdings, **kw):
    ref = run_cycle_reuse_preempt(oracle, nodes, L, *tables, rep, running, holdings)
    got = _run(nodes, L, tables, rep, running, holdings, **kw)
    for k in ("status", "placements", "scope_status", "nodes_after", "victims"):
        assert np.array_equal(got[k], ref[k]), k
    return got, ref


def _hand_cases():
    def holds():
        b = _one_gang(4, mem=100, priority=5); _one_gang(1, mem=100, priority=5, b=b)
        return half_full([5, 0, 0, 0]), b, [0, NONE]

    def released():
        return half_full([1, 0, 2, 2]), _one_gang(4, mem=80, priority=5), [0]

    def evicted_first():
        b = _one_gang(2, mem=100, priority=9); _one_gang(1, mem=120, priority=9, b=b)
        return shared_nodes(), b, [NONE, 0]

    def outranks():
        return half_full([3, 3, 0, 3]), _one_gang(3, mem=150, priority=4), [2]

    def runs_out():
        # the first preemptor evicts the only running gang below the class: the second, which the class cycle also admits
        # on what is left, finds E(p) empty at its turn and stays REJECTED
        b = _one_gang(1, mem=100, priority=5); _one_gang(1, mem=100, priority=5, b=b)
        return half_full([0, 7]), b, [NONE, NONE]

    return dict(holds=holds, released=released, evicted_first=evicted_first, outranks=outranks, runs_out=runs_out)


@pytest.mark.parametrize("case", sorted(_hand_cases()))
def test_hand_case(built_lib, oracle, case):
    (now, running, holdings), b, rep = _hand_cases()[case]()
    got, ref = _check(oracle, now, 4, b.build(), np.array(rep, dtype=np.uint32), running, holdings)
    if case == "runs_out":
        assert list(ref["status"]["state"]) == [T.GANG_ADMITTED, T.GANG_REJECTED] and len(ref["victims"]) == 1


@pytest.mark.parametrize("seed", [61, 62, 63, 64])
def test_churned_rolling_clusters(built_lib, oracle, seed):
    nodes, L, tables, rep, running, holdings = reclaim_rolling_cluster(oracle, seed)
    got, ref = _check(oracle, nodes, L, tables, rep, running, holdings)
    assert len(ref["victims"]) > 0 and ref["released"]


@pytest.mark.parametrize("window", [1, 7, 0])
def test_windows(built_lib, oracle, window):
    nodes, L, tables, rep, running, holdings = reclaim_rolling_cluster(oracle, 65, g_pending=100)
    _check(oracle, nodes, L, tables, rep, running, holdings, window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_REFRESH", "GROVE_TUNE_HEAVY_ATT"])
def test_relaxation_knobs(built_lib, oracle, monkeypatch, knob):
    """a capacity-table rebuild every round; every gang heavy"""
    monkeypatch.setenv(knob, "1")
    nodes, L, tables, rep, running, holdings = reclaim_rolling_cluster(oracle, 66, g_pending=100)
    _check(oracle, nodes, L, tables, rep, running, holdings)


def test_reduced_c4(built_lib, oracle):
    nodes, L, tables, rep, running, holdings = reclaim_rolling_cluster(oracle, 67, n=5040, g_running=1000, g_pending=100, share=0.05)
    got, ref = _check(oracle, nodes, L, tables, rep, running, holdings)
    assert len(ref["victims"]) > 0


def test_holds_and_claims_overflow_a_claim_line(built_lib, oracle):
    """twelve new versions whose predecessors hold 20 MiB each on node 0, rejected in the ordinary pass and admitted there by
    the reclaim pass with ordinary preemptors between them, evicting some of 24 low-priority gangs of 40 MiB each: far more than
    the eight inline claim slots"""
    nodes = synth.e2e_cluster(4)
    nodes["free_mem_mib"] = 10
    k, low = 12, 24
    running = np.zeros(k + low, dtype=T.running_dt)
    running["holding_off"] = np.arange(k + low); running["n_holdings"] = 1
    running["priority"][:k] = 3   # the predecessors rank with the class: their new versions hold what they hold
    holdings = np.zeros(k + low, dtype=T.holding_dt)
    holdings["node"] = 0; holdings["mem_mib"][:k] = 20; holdings["mem_mib"][k:] = 40; holdings["pods"] = 1
    nodes["free_mem_mib"][0] = 0; nodes["free_pods"][0] -= k + low
    b = T.GangTableBuilder()
    for i in range(k):
        _one_gang(1, mem=25 + 5 * (i % 3), priority=3, b=b)   # new versions: more than they hold
        _one_gang(1, mem=15, priority=3, b=b)                 # ordinary gangs between them
    g, c, s = b.build()
    g["anchor_node"] = 0
    rep = np.full(2 * k, NONE, dtype=np.uint32)
    rep[0::2] = np.arange(k)
    got, ref = _check(oracle, nodes, 4, (g, c, s), rep, running, holdings)
    assert ((got["placements"]["node"] == 0).sum()) > 8 and len(ref["victims"]) > 1


def test_malformed_inputs_are_rejected(built_lib, oracle):
    from grove_b200.engine import GroveError, PlacementEngine
    now, running, holdings = half_full([0, 3])
    g, c, s = _one_gang(3, priority=5, b=_one_gang(3, priority=5)).build()
    bad_node = holdings.copy(); bad_node["node"][0] = 4
    big = holdings.copy(); big["pods"][0] = 0xFFFF
    cases = [
        (np.array([0], dtype=np.uint32), running, holdings, "one entry per submitted gang"),
        (np.array([2, NONE], dtype=np.uint32), running, holdings, "out of range"),
        (np.array([0, 0], dtype=np.uint32), running, holdings, "more than one gang"),
        (np.array([0, NONE], dtype=np.uint32), running, bad_node, "node out of range"),
        (np.array([0, NONE], dtype=np.uint32), running, big, "overflow"),
    ]
    with PlacementEngine(4) as e:
        e.load_nodes(now); e.submit_gangs(g, c, s)
        for rep, run, hold, why in cases:
            with pytest.raises(GroveError) as ei:
                e.run_cycle_reuse_preempt(rep, run, hold)
            assert ei.value.code == -1 and why in str(ei.value), (why, str(ei.value))
        # the handle is untouched: the well-formed call still gives the definition's result
        rep = np.array([0, NONE], dtype=np.uint32)
        e.run_cycle_reuse_preempt(rep, running, holdings)
        ref = run_cycle_reuse_preempt(oracle, now, 4, g, c, s, rep, running, holdings)
        assert np.array_equal(e.gang_status(), ref["status"]) and np.array_equal(e.nodes(), ref["nodes_after"])
        assert np.array_equal(e.victims(), ref["victims"])
