"""Reclaim within queue limits through the C ABI (grove_set_queues + grove_run_cycle_preempt_queues) against its restatement over
the sequential oracle (tests/preempt_queue_cases.py): statuses with their flags, placements, scope domains, victims in order, the
node table and the permutation, on the hand cases, random snapshots, knobs that change how the engine gets there, a reduced C4 in
synth.c4_queues with running gangs, one engine over several submissions, and the refusals."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from preempt_queue_cases import hand_cases, run_cycle_preempt_queues, running_layout
from test_oracle_preempt_queues import random_snapshot

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32
KEYS = ("status", "placements", "scope_status", "nodes_after", "victims", "perm")


def _run_on(e, nodes, tables, queues, gang_queue, running, holdings, running_queue):
    e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(queues, gang_queue)
    st = e.run_cycle_preempt_queues(running, holdings, running_queue)
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                victims=e.victims(), perm=e.debug_perm(), stats=st)


def _run(nodes, L, tables, queues, gang_queue, running, holdings, running_queue, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        return _run_on(e, nodes, tables, queues, gang_queue, running, holdings, running_queue)


def _same(got, ref, what=""):
    for k in KEYS:
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, case, **kw):
    nodes, L, tables, qs, gq, running, holdings, rq = case
    ref = run_cycle_preempt_queues(oracle, nodes, L, *tables, qs, gq, running, holdings, rq)
    got = _run(nodes, L, tables, qs, gq, running, holdings, rq, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    _check(oracle, hand_cases()[case](), window=window)


@pytest.mark.parametrize("block", range(8))
def test_random_snapshots_window_all(built_lib, oracle, block):
    for seed in range(block * 25, block * 25 + 25):
        _check(oracle, random_snapshot(oracle, seed))


@pytest.mark.parametrize("block", range(4))
@pytest.mark.parametrize("window", [1, 7])
def test_random_snapshots_narrow_windows(built_lib, oracle, block, window):
    for seed in range(1000 + block * 25, 1000 + block * 25 + 25):
        _check(oracle, random_snapshot(oracle, seed), window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_EVAL_CTAS=1", "GROVE_TUNE_REFRESH=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """one K3 CTA, a table rebuild every round: other rounds and evaluations, the same result"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        _check(oracle, random_snapshot(oracle, seed))


def c4_case(oracle, n=5040, g=800, seed=0):
    """reduced C4 in synth.c4_queues: the gangs a queue cycle admitted run in their queues, copies of the submission come in with
    some of them a priority higher"""
    cfg = synth.config_c4(n=n, g=g, seed=seed)
    tables = cfg["tables"]
    qs, gq = synth.c4_queues(*tables[:2])
    nodes, t2, q2, gq2, running, holdings, rq = running_layout(oracle, cfg["nodes"], cfg["n_levels"], tables, qs, gq, seed)
    return nodes, cfg["n_levels"], t2, q2, gq2, running, holdings, rq


def test_reduced_c4(built_lib, oracle):
    got, ref = _check(oracle, c4_case(oracle))
    fl = got["status"]["reserved0"]
    assert ((fl & T.STATUS_PREEMPTOR) != 0).sum() > 5 and len(got["victims"]) > 5


def test_one_engine_over_several_submissions(built_lib, oracle):
    from grove_b200.engine import PlacementEngine
    names = sorted(hand_cases())
    with PlacementEngine(2) as e:
        for k in range(2):
            for name in names:
                nodes, L, tables, qs, gq, running, holdings, rq = hand_cases()[name]()
                got = _run_on(e, nodes, tables, qs, gq, running, holdings, rq)
                _same(got, run_cycle_preempt_queues(oracle, nodes, L, *tables, qs, gq, running, holdings, rq), (k, name))
                # the queue set stays in place: the entry runs again on the same submission
                e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq)
                e.run_cycle_preempt_queues(running, holdings, rq)
                e.load_nodes(nodes)
                e.submit_gangs(*tables); e.set_queues(qs, gq)
                e.run_cycle_preempt_queues(running, holdings, rq)
                e.run_cycle_preempt_queues(running, holdings, rq)


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tables, qs, gq, running, holdings, rq = hand_cases()["sibling_victim"]()
    G = len(tables[0])

    def code(call):
        with pytest.raises(GroveError) as ex:
            call()
        return ex.value.code

    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        assert code(lambda: e.run_cycle_preempt_queues(running, holdings, rq)) == -5          # no set given
        with pytest.raises(GroveError):
            e.diagnose()
        e.set_queues(qs, np.full(G, NONE, np.uint32))                                          # a set without members counts
        e.run_cycle_preempt_queues(running, holdings, rq)
        e.run_cycle_preempt(running, holdings)                                                  # ... and refuses nothing else
        e.set_queues(qs, gq)
        assert code(lambda: e.run_cycle_preempt(running, holdings)) == -5
        assert code(lambda: e.run_cycle_preempt_queues(running, holdings, np.array([1, 2, 3], np.uint32))) == -1   # out of range
        over = rq.copy(); over[0] = 2   # queue 2's running gangs then hold 24 GPUs against its used of 16
        assert code(lambda: e.run_cycle_preempt_queues(running, holdings, over)) == -1
        bad = holdings.copy(); bad["node"][0] = len(nodes)
        assert code(lambda: e.run_cycle_preempt_queues(running, bad, rq)) == -1
        e.run_cycle_preempt_queues(running, holdings, rq)
        assert code(lambda: e.diagnose()) == -5
        e.set_fences(np.array([0], np.uint32))
        assert code(lambda: e.run_cycle_preempt_queues(running, holdings, rq)) == -5
        e.set_fences(np.zeros(0, np.uint32))
        e.update_nodes(np.array([5], np.uint32), nodes[5:6])                                   # kept across a node update
        e.run_cycle_preempt_queues(running, holdings, rq)
        e.load_nodes(nodes)                                                                     # gone with a node load
        assert code(lambda: e.run_cycle_preempt_queues(running, holdings, rq)) == -5
