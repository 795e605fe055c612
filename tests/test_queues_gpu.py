"""Queue limits through the C ABI (grove_set_queues + grove_run_cycle) against their restatement over the sequential oracle
(tests/queue_cases.py): statuses (the OVER_LIMIT and SURPLUS_CAPPED flags included), placements, scope domains, the node table
and the permutation, on the hand cases, random snapshots with queue trees, knobs that change how the engine gets there, and a
reduced C4 in eight queues under two parents; a set without a finite limit changes nothing; grove_diagnose after a queue cycle;
the refusals."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from queue_cases import assign_queues, diagnose_queue_cycle, hand_cases, make_queues, run_cycle_queues
from test_random_parity_gpu import random_case

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32


def _outputs(e):
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                perm=e.debug_perm())


def _run(nodes, L, tables, queues, gang_queue, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.set_queues(queues, gang_queue)
        st = e.run_cycle()
        out = _outputs(e)
        out["stats"] = st
        return out


def _same(got, ref, what=""):
    for k in ("status", "placements", "scope_status", "nodes_after", "perm"):
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, nodes, L, tables, queues, gang_queue, **kw):
    ref = run_cycle_queues(oracle, nodes, L, *tables, queues, gang_queue)
    got = _run(nodes, L, tables, queues, gang_queue, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    nodes, L, tables, qs, gq = hand_cases()[case]()
    _check(oracle, nodes, L, tables, qs, gq, window=window)


def test_flags_reach_the_status(built_lib, oracle):
    nodes, L, tables, qs, gq = hand_cases()["leaf_limit"]()
    got, _ = _check(oracle, nodes, L, tables, qs, gq)
    assert got["status"]["reserved0"].tolist() == [0, 0, T.STATUS_OVER_LIMIT]
    nodes, L, tables, qs, gq = hand_cases()["surplus_two_cliques"]()
    got, _ = _check(oracle, nodes, L, tables, qs, gq)
    assert got["status"]["reserved0"].tolist() == [T.STATUS_SURPLUS_CAPPED] and got["status"]["n_pods"][0] == 6


def _random(seed):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    qs, gq = assign_queues(np.random.default_rng(seed + 91), tables[0], tables[1])
    return nodes, L, tables, qs, gq


@pytest.mark.parametrize("block", range(8))
def test_random_snapshots_window_all(built_lib, oracle, block):
    for seed in range(block * 25, block * 25 + 25):
        _check(oracle, *_random(seed))


@pytest.mark.parametrize("block", range(4))
@pytest.mark.parametrize("window", [1, 7])
def test_random_snapshots_narrow_windows(built_lib, oracle, block, window):
    for seed in range(1000 + block * 25, 1000 + block * 25 + 25):
        _check(oracle, *_random(seed), window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_EVAL_CTAS=1", "GROVE_TUNE_REFRESH=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """one K3 CTA, a table rebuild every round: other rounds and evaluations, the same result"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        _check(oracle, *_random(seed))


def test_reduced_c4(built_lib, oracle):
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    qs, gq = synth.c4_queues(g, c)
    got, ref = _check(oracle, cfg["nodes"], cfg["n_levels"], (g, c, s), qs, gq)
    fl = got["status"]["reserved0"]
    assert ((fl & T.STATUS_OVER_LIMIT) != 0).sum() > 10 and (got["status"]["state"] == T.GANG_ADMITTED).sum() > 10


def test_unlimited_set_is_the_ordinary_cycle(built_lib):
    from grove_b200.engine import PlacementEngine
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    qs, gq = synth.c4_queues(g, c)
    qs["limit"] = T.QUEUE_UNLIMITED
    out = []
    for with_set in (False, True):
        with PlacementEngine(cfg["n_levels"]) as e:
            e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
            if with_set:
                e.set_queues(qs, gq)
            st = e.run_cycle()
            o = _outputs(e)
            out.append((o["status"], o["placements"], o["scope_status"], o["nodes_after"], st["rounds"], st["evaluations"]))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_one_engine_over_several_submissions(built_lib, oracle):
    """a flag never outlives membership: the set of one submission is gone with the next"""
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, qs, gq = hand_cases()["leaf_limit"]()
    n2, L2, t2, q2, g2 = hand_cases()["surplus_two_cliques"]()
    with PlacementEngine(L) as e:
        for k in range(3):   # (a cycle commits its placements: every cycle starts from the same node table)
            e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq); e.run_cycle()
            _same(_outputs(e), run_cycle_queues(oracle, nodes, L, *tables, qs, gq), k)
            e.load_nodes(nodes); e.submit_gangs(*tables); e.run_cycle()
            assert not e.gang_status()["reserved0"].any()
            assert (e.gang_status()["state"] == T.GANG_ADMITTED).all()
        e.load_nodes(n2); e.submit_gangs(*t2); e.set_queues(q2, g2); e.run_cycle()
        _same(_outputs(e), run_cycle_queues(oracle, n2, L2, *t2, q2, g2))
        e.load_nodes(n2); e.submit_gangs(*t2); e.run_cycle()
        assert not e.gang_status()["reserved0"].any()


@pytest.mark.parametrize("seed", range(500, 510))
def test_diagnose_after_a_queue_cycle(built_lib, oracle, seed):
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, qs, gq = _random(seed)
    g, c, s = tables
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(g, c, s); e.set_queues(qs, gq); e.run_cycle()
        out = _outputs(e)
        gd, qd = e.diagnose()
    rg, rq = diagnose_queue_cycle(nodes, L, g, c, s, out)
    assert np.array_equal(gd, rg) and np.array_equal(qd, rq)


def _engine_with(nodes, L, tables):
    from grove_b200.engine import PlacementEngine
    e = PlacementEngine(L)
    e.load_nodes(nodes); e.submit_gangs(*tables)
    return e


def test_validation(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tables, qs, gq = hand_cases()["cpu_and_mem"]()
    G = len(tables[0])
    deep = make_queues([(None if i == 0 else i - 1, (1, None, None), (0, 0, 0)) for i in range(5)])
    cases = [
        (qs, gq[:-1], -1, "n_gangs"),
        (make_queues([(1, (1, 1, 1), (0, 0, 0)), (None, (1, 1, 1), (0, 0, 0))]), np.zeros(G, np.uint32), -1, "parent after"),
        (make_queues([(0, (1, 1, 1), (0, 0, 0))]), np.zeros(G, np.uint32), -1, "own parent"),
        (qs, np.full(G, len(qs), np.uint32), -1, "queue out of range"),
        (make_queues([(None, (1, 1, 1), (0, 0, 0))] * (T.MAX_QUEUES + 1)), np.zeros(G, np.uint32), -4, "too many queues"),
        (deep, np.full(G, 4, np.uint32), -4, "too deep"),
    ]
    for q, g, code, why in cases:
        e = _engine_with(nodes, L, tables)
        with pytest.raises(GroveError) as ex:
            e.set_queues(q, g)
        assert ex.value.code == code, why
        e.close()
    # depth 4 is fine
    e = _engine_with(nodes, L, tables)
    e.set_queues(deep[:4], np.full(G, 3, np.uint32)); e.run_cycle(); e.close()
    # before nodes / gangs are loaded
    with PlacementEngine(L) as e:
        with pytest.raises(GroveError) as ex:
            e.set_queues(qs, gq)
        assert ex.value.code == -5


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tables, qs, gq = hand_cases()["cpu_and_mem"]()
    G = len(tables[0])
    running = np.zeros(0, dtype=T.running_dt); holdings = np.zeros(0, dtype=T.holding_dt)
    none = np.full(G, NONE, np.uint32)
    e = _engine_with(nodes, L, tables)
    e.set_queues(qs, gq)
    for call in (lambda: e.run_cycle_preempt(running, holdings), lambda: e.run_cycle_reuse(none, running, holdings),
                 lambda: e.run_cycle_reuse_preempt(none, running, holdings),
                 lambda: e.run_cycle_consolidate(np.zeros(0, np.uint32), np.zeros(0, np.uint32), running, holdings)):
        with pytest.raises(GroveError) as ex:
            call()
        assert ex.value.code == -5
    # with fences, and with spread members
    e.set_fences(np.array([1], np.uint32))
    with pytest.raises(GroveError) as ex:
        e.run_cycle()
    assert ex.value.code == -5
    e.set_fences(np.zeros(0, np.uint32))
    sp = np.zeros(1, dtype=T.spread_dt); sp["level"] = 0; sp["mode"] = T.SPREAD_HARD; sp["max_skew"] = 1
    e.set_spread(sp, np.where(tables[0]["level"] == 0, 0, NONE).astype(np.uint32))
    with pytest.raises(GroveError) as ex:
        e.run_cycle()
    assert ex.value.code == -5
    e.set_spread(sp, none)
    e.run_cycle(); e.diagnose()   # a queue cycle is diagnosed
    # grove_update_nodes keeps the set, a new submission or node load clears it
    e.update_nodes(np.array([0], np.uint32), nodes[:1])
    with pytest.raises(GroveError):
        e.run_cycle_preempt(running, holdings)
    e.submit_gangs(*tables)
    e.run_cycle_preempt(running, holdings)
    e.set_queues(qs, gq)
    e.load_nodes(nodes)
    e.run_cycle_preempt(running, holdings)
    # a set without members, or without finite limits, refuses nothing
    e.submit_gangs(*tables)
    e.set_queues(qs, none)
    e.run_cycle_preempt(running, holdings)
    e.close()
    # a wide submission
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=1, min=200, replicas=200)])], level=0)
    g, c, cnt, s = b.build_wide()
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs_wide(g, c, cnt, s)
        with pytest.raises(GroveError) as ex:
            e.set_queues(qs, np.zeros(1, np.uint32))
        assert ex.value.code == -4
