"""Topology spread through the C ABI (grove_set_spread + grove_run_cycle) against its restatement over the sequential oracle
(tests/spread_cases.py): statuses (the SPREAD_SKEWED flag included), placements, scope domains and the node table, on the hand
cases, random snapshots with groups at every level, every relaxation knob that changes how the engine gets there, and a reduced
C4 whose base gangs are grouped; a spread set without members changes nothing; the refusals."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from spread_cases import group_randomly, hand_cases, run_cycle_spread
from test_random_parity_gpu import random_case

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32


def _run(nodes, L, tables, groups, gang_group, seeds=None, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.set_spread(groups, gang_group, seeds)
        st = e.run_cycle()
        return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                    perm=e.debug_perm(), stats=st)


def _same(got, ref, what=""):
    for k in ("status", "placements", "scope_status", "nodes_after", "perm"):
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, nodes, L, tables, groups, gang_group, seeds=None, **kw):
    ref = run_cycle_spread(oracle, nodes, L, *tables, groups, gang_group, seeds)
    got = _run(nodes, L, tables, groups, gang_group, seeds, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    nodes, L, tables, groups, gg, seeds = hand_cases()[case]()
    _check(oracle, nodes, L, tables, groups, gg, seeds, window=window)


def test_soft_flag_reaches_the_status(built_lib, oracle):
    nodes, L, tables, groups, gg, seeds = hand_cases()["full_zone_soft"]()
    got, _ = _check(oracle, nodes, L, tables, groups, gg, seeds)
    assert got["status"]["reserved0"].tolist() == [0, 0, 0, T.STATUS_SPREAD_SKEWED]


@pytest.mark.parametrize("block", range(4))
@pytest.mark.parametrize("window", [0, 1, 7])
def test_random_snapshots(built_lib, oracle, block, window):
    for seed in range(block * 25, block * 25 + 25):
        nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
        rng = np.random.default_rng(seed + 77)
        groups, gg, seeds = group_randomly(rng, nodes, L, tables[0], tables[1])
        _check(oracle, nodes, L, tables, groups, gg, seeds, window=window)


@pytest.mark.parametrize("block", range(2))
def test_random_snapshots_many_gangs(built_lib, oracle, block):
    """many members relaxing at once (big snapshots: hundreds of gangs per round)"""
    for seed in range(5000 + block * 3, 5000 + block * 3 + 3):
        nodes, L, tables = random_case(seed, big=True)
        rng = np.random.default_rng(seed)
        groups, gg, seeds = group_randomly(rng, nodes, L, tables[0], tables[1], n_groups=4)
        _check(oracle, nodes, L, tables, groups, gg, seeds)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_REFRESH=1", "GROVE_TUNE_HEAVY_ATT=1", "GROVE_TUNE_EVAL_CTAS=1", "GROVE_TUNE_MAX_ATT=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """the knobs change how many rounds and evaluations the engine needs, never the result (read when an engine is created)"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        nodes, L, tables = random_case(seed, big=seed % 4 == 0)
        rng = np.random.default_rng(seed)
        groups, gg, seeds = group_randomly(rng, nodes, L, tables[0], tables[1])
        _check(oracle, nodes, L, tables, groups, gg, seeds)


@pytest.mark.parametrize("mode", [T.SPREAD_HARD, T.SPREAD_SOFT])
@pytest.mark.parametrize("level", [0, 1])
def test_reduced_c4_grouped(built_lib, oracle, mode, level):
    """C4's base gangs in groups of eight by (priority, template), spread over zones or blocks"""
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    groups, gg = synth.c4_spread_groups(g, c, level=level, mode=mode)
    assert (gg != NONE).sum() > 100
    got, ref = _check(oracle, cfg["nodes"], cfg["n_levels"], (g, c, s), groups, gg)
    plain = oracle.run_cycle(cfg["nodes"], cfg["n_levels"], g, c, s)
    assert not np.array_equal(got["status"], plain["status"])   # the spread changed where the replicas went


def test_memberless_set_is_the_ordinary_cycle(built_lib):
    from grove_b200.engine import PlacementEngine
    cfg = synth.config_c4(n=5040, g=800)
    out = []
    for with_set in (False, True):
        with PlacementEngine(cfg["n_levels"]) as e:
            e.load_nodes(cfg["nodes"]); e.submit_gangs(*cfg["tables"])
            if with_set:
                e.set_spread(_groups([0, 1]), np.full(len(cfg["tables"][0]), NONE, np.uint32))
            st = e.run_cycle()
            out.append((e.gang_status(), e.placements(), e.scope_domains(), e.nodes(), st["rounds"], st["evaluations"]))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def _groups(levels, mode=T.SPREAD_HARD, skew=1):
    out = np.zeros(len(levels), dtype=T.spread_dt)
    out["level"] = levels; out["mode"] = mode; out["max_skew"] = skew
    return out


def _engine_with(nodes, L, tables):
    from grove_b200.engine import PlacementEngine
    e = PlacementEngine(L)
    e.load_nodes(nodes); e.submit_gangs(*tables)
    return e


def test_validation(built_lib):
    from grove_b200.engine import GroveError
    nodes, L, tables, groups, gg, _ = hand_cases()["mixed"]()
    G = len(tables[0])
    bad_level = T.GangTableBuilder(); bad_level.add_gang([(None, [dict(mem=10, min=1)])], level=None)
    no_min = T.GangTableBuilder(); no_min.add_gang([(None, [dict(mem=10, min=0, replicas=1)])], level=0)
    cases = [
        (tables, _groups([0]), np.zeros(G - 1, np.uint32), None, "n_gangs"),
        (tables, _groups([0]), np.full(G, 1, np.uint32), None, "group out of range"),
        (tables, _groups([2]), np.where(gg == NONE, NONE, 0).astype(np.uint32), None, "level"),
        (tables, _groups([0], mode=3), np.where(gg == NONE, NONE, 0).astype(np.uint32), None, "mode"),
        (tables, _groups([0], skew=0), np.where(gg == NONE, NONE, 0).astype(np.uint32), None, "max_skew"),
        (bad_level.build(), _groups([0]), np.zeros(1, np.uint32), None, "Required level"),
        (no_min.build(), _groups([0]), np.zeros(1, np.uint32), None, "MinReplicas"),
        (tables, _groups([0]), np.where(gg == NONE, NONE, 0).astype(np.uint32), np.array([(1, 0)], dtype=T.spread_seed_dt), "seed group"),
        (tables, _groups([0]), np.where(gg == NONE, NONE, 0).astype(np.uint32), np.array([(0, len(nodes))], dtype=T.spread_seed_dt), "seed node"),
    ]
    for tb, grp, gang_group, seeds, why in cases:
        e = _engine_with(nodes, L, tb)
        with pytest.raises(GroveError) as ex:
            e.set_spread(grp, gang_group, seeds)
        assert ex.value.code == -1, why
        e.close()
    # a member whose gang level is broader than its group's level
    e = _engine_with(nodes, L, tables)
    with pytest.raises(GroveError) as ex:
        e.set_spread(_groups([1]), np.where(gg == NONE, NONE, 0).astype(np.uint32))
    assert ex.value.code == -1
    e.close()


def test_refusals(built_lib):
    from grove_b200.engine import GroveError
    nodes, L, tables, groups, gg, _ = hand_cases()["mixed"]()
    G = len(tables[0])
    running = np.zeros(0, dtype=T.running_dt); holdings = np.zeros(0, dtype=T.holding_dt)
    none = np.full(G, NONE, np.uint32)
    e = _engine_with(nodes, L, tables)
    e.set_spread(groups, gg)
    for call in (lambda: e.run_cycle_preempt(running, holdings), lambda: e.run_cycle_reuse(none, running, holdings),
                 lambda: e.run_cycle_reuse_preempt(none, running, holdings)):
        with pytest.raises(GroveError) as ex:
            call()
        assert ex.value.code == -5
    e.run_cycle()
    with pytest.raises(GroveError) as ex:
        e.diagnose()
    assert ex.value.code == -5
    # grove_update_nodes keeps the set, a new submission clears it
    e.update_nodes(np.array([0], np.uint32), nodes[:1])
    with pytest.raises(GroveError):
        e.run_cycle_preempt(running, holdings)
    e.submit_gangs(*tables)
    e.run_cycle_preempt(running, holdings)
    e.set_spread(groups, gg)
    e.load_nodes(nodes)
    e.run_cycle_preempt(running, holdings)
    # a memberless set does not refuse anything, and the cycle after it is diagnosed
    e.submit_gangs(*tables)
    e.set_spread(groups, none)
    e.run_cycle_preempt(running, holdings)
    e.run_cycle(); e.diagnose()
    e.close()
    # a wide submission
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=1, min=200, replicas=200)])], level=0)
    g, c, cnt, s = b.build_wide()
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L) as e:
        big = nodes.copy(); big["free_pods"] = 110
        e.load_nodes(big); e.submit_gangs_wide(g, c, cnt, s)
        with pytest.raises(GroveError) as ex:
            e.set_spread(_groups([0]), np.zeros(1, np.uint32))
        assert ex.value.code == -4


def test_flag_does_not_outlive_membership(built_lib, oracle):
    """one engine, two submissions: a SOFT member skewed in the first is a non-member of the second (whose set still has members),
    and nothing of the first cycle's flags reaches the second's statuses"""
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, groups, gg, seeds = hand_cases()["full_zone_soft"]()
    second = gg.copy(); second[3] = NONE
    ref1 = run_cycle_spread(oracle, nodes, L, *tables, groups, gg, seeds)
    ref2 = run_cycle_spread(oracle, nodes, L, *tables, groups, second, seeds)
    assert ref1["status"]["reserved0"][3] == T.STATUS_SPREAD_SKEWED and not ref2["status"]["reserved0"].any()
    with PlacementEngine(L) as e:
        for member_of, ref in ((gg, ref1), (second, ref2), (gg, ref1)):
            e.load_nodes(nodes); e.submit_gangs(*tables)
            e.set_spread(groups, member_of, seeds)
            e.run_cycle()
            assert np.array_equal(e.gang_status(), ref["status"])
            assert np.array_equal(e.placements(), ref["placements"])
        e.load_nodes(nodes); e.submit_gangs(*tables); e.run_cycle()   # no set at all
        assert not e.gang_status()["reserved0"].any()
