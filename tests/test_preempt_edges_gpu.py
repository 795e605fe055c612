"""grove_run_cycle_preempt on the reclaim loop the other reclaim entries share, held to the oracle's one-at-a-time statement
(oracle/oracle_py.py run_cycle_preempt): the skip rule when nothing evictable is left part-way through a class, the refusals of
malformed running inputs, and narrow relaxation windows and the tuning knobs."""
import numpy as np
import pytest

from grove_b200 import tables as T
from preempt_cases import churned_cluster
from reuse_preempt_cases import half_full, one_gang

pytestmark = pytest.mark.gpu


def _same(e, ref):
    assert np.array_equal(e.gang_status(), ref["status"])
    assert np.array_equal(e.placements(), ref["placements"])
    assert np.array_equal(e.scope_domains(), ref["scope_status"])
    assert np.array_equal(e.nodes(), ref["nodes_after"])
    assert np.array_equal(e.victims(), ref["victims"])


def test_runs_out(built_lib, oracle):
    """the first preemptor evicts the only running gang below the class; the second, which the class cycle also admits on what is
    left, finds nothing evictable at its turn and stays REJECTED"""
    from grove_b200.engine import PlacementEngine
    nodes, running, holdings = half_full([0])
    g, c, s = one_gang(1, 80, 5, b=one_gang(1, 80, 5)).build()
    ref = oracle.run_cycle_preempt(nodes, 4, g, c, s, running, holdings)
    assert list(ref["status"]["state"]) == [T.GANG_ADMITTED, T.GANG_REJECTED] and len(ref["victims"]) == 1
    with PlacementEngine(4) as e:
        e.load_nodes(nodes); e.submit_gangs(g, c, s)
        e.run_cycle_preempt(running, holdings)
        _same(e, ref)


_CHURNED = {}


@pytest.mark.parametrize("window,knob", [(1, None), (7, None), (0, "GROVE_TUNE_REFRESH"), (0, "GROVE_TUNE_HEAVY_ATT")])
def test_windows_and_knobs(built_lib, oracle, monkeypatch, window, knob):
    """narrow relaxation windows; a capacity-table rebuild every round; every gang heavy"""
    from grove_b200.engine import PlacementEngine
    if knob:
        monkeypatch.setenv(knob, "1")
    if not _CHURNED:
        nodes, L, (g, c, s), running, holdings = churned_cluster(oracle, 15, g_pending=100)
        ref = oracle.run_cycle_preempt(nodes, L, g, c, s, running, holdings)
        assert ((ref["status"]["reserved0"] & T.STATUS_PREEMPTOR) != 0).any()
        _CHURNED.update(case=(nodes, L, (g, c, s), running, holdings), ref=ref)
    nodes, L, (g, c, s), running, holdings = _CHURNED["case"]
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(g, c, s)
        e.run_cycle_preempt(running, holdings)
        _same(e, _CHURNED["ref"])


def test_malformed_inputs_are_rejected(built_lib, oracle):
    from grove_b200.engine import GroveError, PlacementEngine
    now, running, holdings = half_full([0, 3])
    g, c, s = one_gang(3, priority=5, b=one_gang(3, priority=5)).build()
    bad_range = running.copy(); bad_range["n_holdings"][1] = 3
    bad_node = holdings.copy(); bad_node["node"][0] = 4
    big = holdings.copy(); big["pods"][0] = 0xFFFF
    cases = [(bad_range, holdings, "holdings out of range"), (running, bad_node, "node out of range"), (running, big, "overflow")]
    ref = oracle.run_cycle(now, 4, g, c, s)
    with PlacementEngine(4) as e:
        e.load_nodes(now); e.submit_gangs(g, c, s)
        for run, hold, why in cases:
            with pytest.raises(GroveError) as ei:
                e.run_cycle_preempt(run, hold)
            assert ei.value.code == -1 and why in str(ei.value), (why, str(ei.value))
            # the handle is untouched: an ordinary cycle gives the ordinary result
            e.run_cycle()
            assert np.array_equal(e.gang_status(), ref["status"]) and np.array_equal(e.placements(), ref["placements"])
            assert np.array_equal(e.nodes(), ref["nodes_after"])
