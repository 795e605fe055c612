"""Bin-packing through the C ABI (grove_set_binpack + grove_run_cycle) against its restatement over the sequential oracle
(tests/binpack_cases.py): statuses, placements, scope domains, the node table, the permutation and the picks getter, on the hand
cases, random snapshots at three window sizes, the relaxation knobs, a reduced C4 packed at block, rack and host level, a queue set
together with bin-packing, grove_diagnose and a score-matrix row after a bin-packing cycle, the fragmentation case, one engine over
several submissions, and the refusals."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from binpack_cases import Fragmentation, hand_cases, random_levels, run_cycle_binpack
from test_random_parity_gpu import random_case

pytestmark = pytest.mark.gpu


def _outputs(e, st=None, picks=True):
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                perm=e.debug_perm(), picks=e.binpack_picks() if picks else None, stats=st)


def _same(got, ref, what=""):
    for k in ("status", "placements", "scope_status", "nodes_after", "perm", "picks"):
        assert np.array_equal(got[k], ref[k]), (k, what)


def _run(nodes, L, tables, levels, window=0, queues=None):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        if queues is not None:
            e.set_queues(*queues)
        e.set_binpack(levels)
        return _outputs(e, e.run_cycle())


def _check(oracle, nodes, L, tables, levels, window=0, queues=None):
    ref = run_cycle_binpack(oracle, nodes, L, *tables, levels, *(queues or (None, None)))
    got = _run(nodes, L, tables, levels, window=window, queues=queues)
    _same(got, ref, window)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    nodes, L, tables, levels, want = hand_cases()[case]()
    got, _ = _check(oracle, nodes, L, tables, np.array(levels, np.uint8), window=window)
    assert got["picks"].tolist() == want


def _random(seed):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    return nodes, L, tables, random_levels(np.random.default_rng(seed + 77), tables[0], L)


@pytest.mark.parametrize("block,window", [(b, 0) for b in range(8)] + [(b, w) for w in (1, 7) for b in range(4)])
def test_random_snapshots(built_lib, oracle, block, window):
    for seed in range(block * 25, block * 25 + 25):
        nodes, L, tables, levels = _random(seed)
        _check(oracle, nodes, L, tables, levels, window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_REFRESH=1", "GROVE_TUNE_HEAVY_ATT=1", "GROVE_TUNE_EVAL_CTAS=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """a table rebuild every round, every gang heavy, a single K3 CTA: other rounds and evaluations, the same result"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        nodes, L, tables = random_case(seed, big=seed % 4 == 0)
        _check(oracle, nodes, L, tables, random_levels(np.random.default_rng(seed), tables[0], L))


@pytest.mark.parametrize("level", [1, 2, 3])
def test_reduced_c4(built_lib, oracle, level):
    """every gang a member: at its Required level (block), at rack level, at host level"""
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    levels = synth.binpack_levels(g, None if level == 1 else level)
    got, _ = _check(oracle, cfg["nodes"], cfg["n_levels"], (g, c, s), levels)
    assert (got["picks"] != T.NONE_U32).any()


def test_with_a_queue_set(built_lib, oracle):
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    qs, gq = synth.c4_queues(g, c)
    got, _ = _check(oracle, cfg["nodes"], cfg["n_levels"], (g, c, s), synth.binpack_levels(g, 2), queues=(qs, gq))
    assert (got["status"]["reserved0"] & T.STATUS_OVER_LIMIT).any()


def test_fragmentation(built_lib, oracle):
    from grove_b200.engine import PlacementEngine

    def cycle(nodes, L, tables, levels):
        ref = oracle.run_cycle(nodes, L, *tables) if levels is None else run_cycle_binpack(oracle, nodes, L, *tables, levels)
        with PlacementEngine(L) as e:
            e.load_nodes(nodes); e.submit_gangs(*tables)
            if levels is not None:
                e.set_binpack(levels)
            e.run_cycle()
            got = _outputs(e, picks=levels is not None)
        for k in ("status", "placements", "scope_status", "nodes_after", "perm"):
            assert np.array_equal(got[k], ref[k]), k
        return got

    f = Fragmentation()
    _, o2, used = f.run(cycle, binpack=False)
    assert used == [0, 1, 2, 3] and o2["status"]["state"][0] == T.GANG_REJECTED
    _, o2, used = f.run(cycle, binpack=True)
    assert used == [0] and o2["status"]["state"][0] == T.GANG_ADMITTED


@pytest.mark.parametrize("seed", range(600, 606))
def test_diagnose_after_a_binpack_cycle(built_lib, oracle, seed):
    from diagnose_cases import diagnose
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, levels = _random(seed)
    g, c, s = tables
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(g, c, s); e.set_binpack(levels); e.run_cycle()
        out = _outputs(e)
        gd, qd = e.diagnose()
    rg, rq = diagnose(nodes, L, g, c, s, c["min_replicas"], out)
    assert np.array_equal(gd, rg) and np.array_equal(qd, rq)


def test_score_row_uses_the_pinned_anchor(built_lib, oracle):
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, levels, want = hand_cases()["fuller_wins"]()
    pinned = tables[0].copy()
    pinned["anchor_node"][0] = want[0]
    ref = oracle.run_cycle(nodes, L, pinned, *tables[1:], want_matrices=True)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables); e.set_binpack(np.array(levels, np.uint8)); e.run_cycle()
        e.build_score_matrix()
        assert np.array_equal(e.debug_score_row(0), ref["score"][0])


def test_one_engine_over_several_submissions(built_lib, oracle):
    """a pick never outlives its set: a later cycle without one is grove_run_cycle's; update_nodes keeps the set"""
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, levels, _ = hand_cases()["fuller_wins"]()
    levels = np.array(levels, np.uint8)
    plain = dict(oracle.run_cycle(nodes, L, *tables))
    packed = run_cycle_binpack(oracle, nodes, L, *tables, levels)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables); e.set_binpack(levels)
        e.run_cycle(); _same(_outputs(e), packed, "packed")
        e.load_nodes(nodes)                                               # clears the set; the labels, and so ginfo, stay
        e.run_cycle(); got = _outputs(e); plain["picks"] = packed["picks"]   # (the getter answers for the last cycle with a set)
        _same(got, plain, "after a node reload")
        e.load_nodes(nodes); e.submit_gangs(*tables); e.run_cycle(); _same(_outputs(e), plain, "after a new submission")
        e.set_binpack(levels)
        e.update_nodes(np.arange(len(nodes), dtype=np.uint32), nodes)   # (the last cycle left its admissions in the table)
        e.run_cycle(); _same(_outputs(e), packed, "kept across update_nodes")
        e.set_binpack(np.full(len(levels), T.LEVEL_NONE, np.uint8))     # a set without members
        e.update_nodes(np.arange(len(nodes), dtype=np.uint32), nodes)
        e.run_cycle(); _same(_outputs(e), dict(plain, picks=np.full(len(levels), T.NONE_U32, np.uint32)), "no members")
    # at C4 scale: a second cycle on a handle is held to the same handle's second cycle without a set before it (a second cycle on
    # one handle at this scale is DESIGN.md section 9 open item 3, set or no set)
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    second = []
    for levels in (None, synth.binpack_levels(g, 3)):
        with PlacementEngine(cfg["n_levels"]) as e:
            e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
            if levels is not None:
                e.set_binpack(levels)
            e.run_cycle()
            e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s); e.run_cycle()
            second.append(_outputs(e, picks=False))
    for k in ("status", "placements", "scope_status", "nodes_after", "perm"):
        assert np.array_equal(second[0][k], second[1][k]), k


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    from spread_cases import spread_groups
    nodes, L, tables, levels, _ = hand_cases()["deeper_than_required"]()
    G = len(tables[0])
    levels = np.array(levels, np.uint8)

    def code(fn):
        with pytest.raises(GroveError) as ex:
            fn()
        return ex.value.code

    with PlacementEngine(L) as e:
        assert code(lambda: e.set_binpack(levels)) == -5                       # nothing loaded
        e.load_nodes(nodes)
        assert code(lambda: e.set_binpack(levels)) == -5                       # no submission
        e.submit_gangs(*tables)
        assert code(lambda: e.binpack_picks()) == -5                           # no cycle with a set yet
        assert code(lambda: e.set_binpack(levels[:1])) == -1                   # wrong n_gangs
        assert code(lambda: e.set_binpack([L, 1])) == -1                       # level out of range
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=1)])], level=1)
        e.submit_gangs(*b.build())
        assert code(lambda: e.set_binpack([0])) == -1                          # above the Required level
        e.set_binpack([1])
        e.submit_gangs(*tables); e.set_binpack(levels)
        none = np.zeros(0, T.running_dt), np.zeros(0, T.holding_dt)
        assert code(lambda: e.run_cycle_preempt(*none)) == -5
        assert code(lambda: e.run_cycle_reuse(np.full(G, T.NONE_U32, np.uint32), *none)) == -5
        assert code(lambda: e.run_cycle_reuse_preempt(np.full(G, T.NONE_U32, np.uint32), *none)) == -5
        assert code(lambda: e.run_cycle_consolidate([], np.zeros(0, np.uint32), *none)) == -5
        e.set_queues(np.zeros(0, T.queue_dt), np.full(G, T.NONE_U32, np.uint32))
        assert code(lambda: e.run_cycle_preempt_queues(*none, np.zeros(0, np.uint32))) == -5
        e.set_spread(spread_groups([0], [T.SPREAD_HARD], [1]), np.zeros(G, np.uint32))
        assert code(lambda: e.run_cycle()) == -5                               # spread members and bin-packing together
        e.set_spread(spread_groups([0], [T.SPREAD_HARD], [1]), np.full(G, T.NONE_U32, np.uint32))
        e.set_fences([0])
        assert code(lambda: e.run_cycle()) == -5                               # fences and bin-packing together
        e.set_fences([])
        e.run_cycle()
        e.diagnose()                                                           # a bin-packing cycle is diagnosed
        e.set_binpack(np.full(G, T.LEVEL_NONE, np.uint8))                      # a set without members: the entries run
        e.run_cycle_preempt(*none)
    wb = T.GangTableBuilder()
    wb.add_gang([(None, [dict(gpu=0, min=200)])], level=0)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs_wide(*wb.build_wide())
        assert code(lambda: e.set_binpack([0])) == -4                          # wide submission
