"""Reclaim, then preempt, through the C ABI (grove_set_queues + grove_run_cycle_reclaim_preempt_queues) against its restatement
over the sequential oracle (tests/reclaim_preempt_queue_cases.py): statuses with their flags, placements, scope domains, victims in
order, the node table and the permutation, on the hand cases, random contested snapshots, knobs that change how the engine gets
there, a reduced C4 in synth.c4_queues with running gangs and synth.c4_queue_quotas, one engine over several submissions, and the
refusals."""
import numpy as np
import pytest

from grove_b200 import tables as T
from reclaim_preempt_queue_cases import hand_cases, random_snapshot, run_cycle_reclaim_preempt_queues
from test_reclaim_queues_gpu import c4_case

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32
KEYS = ("status", "placements", "scope_status", "nodes_after", "victims", "perm")


def _outputs(e):
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                victims=e.victims(), perm=e.debug_perm())


def _run_on(e, nodes, tables, queues, gang_queue, quotas, running, holdings, running_queue):
    e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(queues, gang_queue)
    st = e.run_cycle_reclaim_preempt_queues(quotas, running, holdings, running_queue)
    return dict(_outputs(e), stats=st)


def _run(nodes, L, tables, queues, gang_queue, quotas, running, holdings, running_queue, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        return _run_on(e, nodes, tables, queues, gang_queue, quotas, running, holdings, running_queue)


def _same(got, ref, what=""):
    for k in KEYS:
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, case, **kw):
    nodes, L, tables, qs, gq, quotas, running, holdings, rq = case
    ref = run_cycle_reclaim_preempt_queues(oracle, nodes, L, *tables, qs, gq, quotas, running, holdings, rq)
    got = _run(nodes, L, tables, qs, gq, quotas, running, holdings, rq, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    _check(oracle, hand_cases()[case](), window=window)


def test_three_teams_victims(built_lib, oracle):
    got, _ = _check(oracle, hand_cases()["three_teams"]())
    assert got["victims"].tolist() == [(1, 0), (2, 1)]
    assert got["status"]["reserved0"].tolist() == [T.STATUS_RECLAIMER, T.STATUS_PREEMPTOR]


def test_random_snapshots_window_all(built_lib, oracle):
    """200 contested snapshots; 11 of the cycles admit gangs in both passes (tests/test_oracle_reclaim_preempt_queues.py)"""
    both = 0
    for seed in range(200):
        f = _check(oracle, random_snapshot(seed, pref=seed % 2 == 1))[0]["status"]["reserved0"]
        both += bool((f & T.STATUS_RECLAIMER).any() and (f & T.STATUS_PREEMPTOR).any())
    assert both >= 10


@pytest.mark.parametrize("block", range(4))
@pytest.mark.parametrize("window", [1, 7])
def test_random_snapshots_narrow_windows(built_lib, oracle, block, window):
    for seed in range(1000 + block * 25, 1000 + block * 25 + 25):
        _check(oracle, random_snapshot(seed, pref=seed % 2 == 1), window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_EVAL_CTAS=1", "GROVE_TUNE_REFRESH=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """one K3 CTA, a table rebuild every round: other rounds and evaluations, the same result"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        _check(oracle, random_snapshot(seed, pref=seed % 2 == 1))


def test_reduced_c4(built_lib, oracle):
    got, ref = _check(oracle, c4_case(oracle))
    f = got["status"]["reserved0"]
    assert ((f & T.STATUS_RECLAIMER) != 0).sum() > 0 and len(got["victims"]) > 0
    assert ref["n_reclaim"] > 0


def test_one_engine_over_several_submissions(built_lib, oracle):
    """the hand cases one after another on one handle, and each run again on the same submission and node table"""
    from grove_b200.engine import PlacementEngine
    names = sorted(hand_cases())
    with PlacementEngine(2) as e:
        for k in range(2):
            for name in names:
                nodes, L, tables, qs, gq, quotas, running, holdings, rq = hand_cases()[name]()
                ref = run_cycle_reclaim_preempt_queues(oracle, nodes, L, *tables, qs, gq, quotas, running, holdings, rq)
                _same(_run_on(e, nodes, tables, qs, gq, quotas, running, holdings, rq), ref, (k, name))
                # the queue set stays in place: the entry runs again on the same inputs and gives the same outputs
                e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq)
                for again in range(2):
                    e.run_cycle_reclaim_preempt_queues(quotas, running, holdings, rq)
                    _same(_outputs(e), ref, (k, name, again))
                    e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq)


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tables, qs, gq, quotas, running, holdings, rq = hand_cases()["three_teams"]()
    G = len(tables[0])

    def code(call):
        with pytest.raises(GroveError) as ex:
            call()
        return ex.value.code

    with PlacementEngine(L) as e:
        run = lambda q=quotas, h=holdings, r=rq: e.run_cycle_reclaim_preempt_queues(q, running, h, r)  # noqa: E731
        e.load_nodes(nodes); e.submit_gangs(*tables)
        assert code(run) == -5                                                                         # no set given
        e.set_queues(qs, np.full(G, NONE, np.uint32))                                                  # a set without members counts
        run()
        e.set_queues(qs, gq)
        assert code(lambda: run(q=quotas[:2])) == -1                                                   # one quota row per queue
        assert code(lambda: run(r=np.array([1, 1, 7], np.uint32))) == -1                               # out of range
        over = rq.copy(); over[2] = 0   # queue 0's running gangs then hold 8 GPUs against its used of 0
        assert code(lambda: run(r=over)) == -1
        bad = holdings.copy(); bad["node"][0] = len(nodes)
        assert code(lambda: run(h=bad)) == -1
        run()
        assert code(lambda: e.diagnose()) == -5
        e.load_nodes(nodes)                                                                            # gone with a node load
        assert code(run) == -5
