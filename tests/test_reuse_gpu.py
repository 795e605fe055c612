"""Reservation reuse through the C ABI (grove_run_cycle_reuse) against its restatement over the sequential oracle
(tests/reuse_cases.py): statuses, placements, scope domains and the node table, on hand cases, churned clusters, a full-size C4
rolling update, every relaxation knob that changes how the engine gets there, and a node whose claim line overflows."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from preempt_cases import holdings_of
from reuse_cases import rolling_cluster, run_cycle_reuse

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32


def _run(nodes, L, tables, rep, running, holdings, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        st = e.run_cycle_reuse(rep, running, holdings)
        return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(), stats=st)


def _same(got, ref):
    for k in ("status", "placements", "scope_status", "nodes_after"):
        assert np.array_equal(got[k], ref[k]), k


def _check(oracle, nodes, L, tables, rep, running, holdings, **kw):
    ref = run_cycle_reuse(oracle, nodes, L, *tables, rep, running, holdings)
    got = _run(nodes, L, tables, rep, running, holdings, **kw)
    _same(got, ref)
    return got


def _one_gang(pods, mem=80, priority=0, gated=False, base=None, b=None, anchor=None):
    b = b or T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=mem, min=pods, class_mask=synth.AGENT)])], priority=priority, gated=gated, base=base, anchor=anchor)
    return b


def _six_full(oracle):
    nodes = synth.e2e_cluster(6)
    g, c, s = _one_gang(6).build()
    ref = oracle.run_cycle(nodes, 4, g, c, s)
    running, holdings = holdings_of(ref["placements"], ref["status"], g, c)
    return ref["nodes_after"], running, holdings


def _hand_cases():
    def fits_only_there():
        b = _one_gang(1, priority=5); _one_gang(6, priority=1, b=b); _one_gang(1, priority=0, b=b)
        return b, [NONE, 0, NONE]

    def leftovers():
        b = _one_gang(3, priority=1); _one_gang(1, priority=0, b=b)
        return b, [0, NONE]

    def asks_more():
        return _one_gang(6, mem=100), [0]

    def asks_too_much():
        return _one_gang(6, mem=151), [0]

    def rejected():
        return _one_gang(7), [0]

    def gated():
        return _one_gang(6, gated=True), [0]

    def base_rejected():
        b = _one_gang(7, priority=1); _one_gang(6, priority=0, base=0, b=b)
        return b, [NONE, 0]

    return dict(fits_only_there=fits_only_there, leftovers=leftovers, asks_more=asks_more, asks_too_much=asks_too_much,
                rejected=rejected, gated=gated, base_rejected=base_rejected)


@pytest.mark.parametrize("case", sorted(_hand_cases()))
def test_hand_case(built_lib, oracle, case):
    now, running, holdings = _six_full(oracle)
    b, rep = _hand_cases()[case]()
    _check(oracle, now, 4, b.build(), np.array(rep, dtype=np.uint32), running, holdings)


@pytest.mark.parametrize("seed", [51, 52, 53, 54])
def test_churned_clusters(built_lib, oracle, seed):
    nodes, L, tables, rep, running, holdings = rolling_cluster(oracle, seed)
    got = _check(oracle, nodes, L, tables, rep, running, holdings)
    assert (got["status"]["state"][rep != NONE] == T.GANG_ADMITTED).any()


@pytest.mark.parametrize("window", [1, 7, 0])
def test_windows(built_lib, oracle, window):
    nodes, L, tables, rep, running, holdings = rolling_cluster(oracle, 55, g_pending=200)
    _check(oracle, nodes, L, tables, rep, running, holdings, window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_REFRESH", "GROVE_TUNE_HEAVY_ATT"])
def test_relaxation_knobs(built_lib, oracle, monkeypatch, knob):
    """a capacity-table rebuild every round (holds fold with their owners in between); every gang heavy"""
    monkeypatch.setenv(knob, "1")
    nodes, L, tables, rep, running, holdings = rolling_cluster(oracle, 56, g_pending=200)
    _check(oracle, nodes, L, tables, rep, running, holdings)


def test_full_size_c4_rolling_update(built_lib, oracle):
    nodes, L, tables, rep, running, holdings = rolling_cluster(oracle, 57, n=50000, g_running=10000, g_pending=2000, share=0.01)
    assert (rep != NONE).sum() >= 50
    got = _check(oracle, nodes, L, tables, rep, running, holdings)
    assert got["stats"]["gangs_admitted"] > 0


def test_holds_and_claims_overflow_a_claim_line(built_lib, oracle):
    """twelve holds on one node, and the successors and other gangs all anchored there: far more than the eight inline slots"""
    nodes = synth.e2e_cluster(4)
    nodes["free_mem_mib"] = 400
    k = 12
    running = np.zeros(k, dtype=T.running_dt)
    running["holding_off"] = np.arange(k); running["n_holdings"] = 1
    holdings = np.zeros(k, dtype=T.holding_dt)
    holdings["node"] = 0; holdings["mem_mib"] = 40; holdings["pods"] = 1
    b = T.GangTableBuilder()
    for i in range(k):
        _one_gang(1, mem=30 + 10 * (i % 3), priority=i % 2, b=b, anchor=0)   # successors: less, as much and more than they hold
        _one_gang(1, mem=25, priority=i % 2, b=b, anchor=0)                  # ordinary gangs between them
    rep = np.full(2 * k, NONE, dtype=np.uint32)
    rep[0::2] = np.arange(k)
    got = _check(oracle, nodes, 4, b.build(), rep, running, holdings)
    assert ((got["placements"]["node"] == 0).sum()) > 8


def test_without_replacements_it_is_the_ordinary_cycle(built_lib, oracle):
    nodes, L, tables, _, running, holdings = rolling_cluster(oracle, 58)
    none = np.full(len(tables[0]), NONE, dtype=np.uint32)
    got = _run(nodes, L, tables, none, running, holdings)
    _same(got, oracle.run_cycle(nodes, L, *tables))


def test_malformed_inputs_are_rejected(built_lib, oracle):
    from grove_b200.engine import GroveError, PlacementEngine
    now, running, holdings = _six_full(oracle)
    g, c, s = _one_gang(3, b=_one_gang(3)).build()
    bad_node = holdings.copy(); bad_node["node"][0] = 6
    big = holdings.copy(); big["pods"][0] = 0xFFFF
    cases = [
        (np.array([0], dtype=np.uint32), running, holdings, "one entry per submitted gang"),
        (np.array([1, NONE], dtype=np.uint32), running, holdings, "out of range"),
        (np.array([0, 0], dtype=np.uint32), running, holdings, "more than one gang"),
        (np.array([0, NONE], dtype=np.uint32), running, bad_node, "node out of range"),
        (np.array([0, NONE], dtype=np.uint32), running, big, "overflow"),
    ]
    with PlacementEngine(4) as e:
        e.load_nodes(now); e.submit_gangs(g, c, s)
        for rep, run, hold, why in cases:
            with pytest.raises(GroveError) as ei:
                e.run_cycle_reuse(rep, run, hold)
            assert ei.value.code == -1 and why in str(ei.value), (why, str(ei.value))
        # the handle is untouched: the well-formed call still gives the definition's result
        e.run_cycle_reuse(np.array([0, NONE], dtype=np.uint32), running, holdings)
        ref = run_cycle_reuse(oracle, now, 4, g, c, s, np.array([0, NONE], dtype=np.uint32), running, holdings)
        assert np.array_equal(e.gang_status(), ref["status"]) and np.array_equal(e.nodes(), ref["nodes_after"])
