"""Fences through the C ABI (grove_set_fences + grove_run_cycle) against their restatement over the sequential oracle
(tests/fence_cases.py): statuses (the FENCING flag, level and domain_node included), placements, scope domains and the node table,
on the hand cases, random snapshots with fencing gangs at every level, the relaxation knobs that change how the engine gets
there, a reduced C4, the starvation case cycle by cycle and one engine over several submissions; an empty set changes nothing;
the refusals."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from fence_cases import Starvation, fence_randomly, hand_cases, run_cycle_fences
from test_random_parity_gpu import random_case

pytestmark = pytest.mark.gpu


def _outputs(e, st=None):
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                perm=e.debug_perm(), stats=st)


def _run(nodes, L, tables, fencing, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.set_fences(fencing)
        return _outputs(e, e.run_cycle())


def _same(got, ref, what=""):
    for k in ("status", "placements", "scope_status", "nodes_after", "perm"):
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, nodes, L, tables, fencing, **kw):
    ref = run_cycle_fences(oracle, nodes, L, *tables, fencing)
    got = _run(nodes, L, tables, fencing, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    nodes, L, tables, fencing = hand_cases()[case]()
    _check(oracle, nodes, L, tables, fencing, window=window)


def test_flag_reaches_the_status(built_lib, oracle):
    nodes, L, tables, fencing = hand_cases()["least_shortfall"]()
    got, _ = _check(oracle, nodes, L, tables, fencing)
    st = got["status"][0]
    assert st["reserved0"] == T.STATUS_FENCING and st["level"] == 0 and st["domain_node"] == 4


@pytest.mark.parametrize("block,window", [(b, 0) for b in range(8)] + [(b, w) for w in (1, 7) for b in range(4)])
def test_random_snapshots(built_lib, oracle, block, window):
    for seed in range(block * 25, block * 25 + 25):
        nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
        fencing = fence_randomly(np.random.default_rng(seed + 91), tables[0])
        _check(oracle, nodes, L, tables, fencing, window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_REFRESH=1", "GROVE_TUNE_HEAVY_ATT=1", "GROVE_TUNE_EVAL_CTAS=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """a table rebuild every round, every gang heavy, a single K3 CTA: other rounds and evaluations, the same result"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        nodes, L, tables = random_case(seed, big=seed % 4 == 0)
        fencing = fence_randomly(np.random.default_rng(seed), tables[0])
        _check(oracle, nodes, L, tables, fencing)


def top_rejected(oracle_out, gangs, k):
    """the k highest-ranked gangs the ordinary cycle rejected that have a gang Required level"""
    order = sorted(range(len(gangs)), key=lambda i: (-int(gangs["priority"][i]), i))
    return np.array([g for g in order if oracle_out["status"]["state"][g] == T.GANG_REJECTED
                     and gangs["level"][g] != T.LEVEL_NONE][:k], dtype=np.uint32)


def test_reduced_c4(built_lib, oracle):
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    plain = oracle.run_cycle(cfg["nodes"], cfg["n_levels"], g, c, s)
    fencing = top_rejected(plain, g, 16)
    assert len(fencing) == 16
    got, _ = _check(oracle, cfg["nodes"], cfg["n_levels"], (g, c, s), fencing)
    assert (got["status"]["reserved0"] == T.STATUS_FENCING).sum() > 0


def test_starvation_cycle_by_cycle(built_lib, oracle):
    from grove_b200.engine import PlacementEngine

    def cycle(nodes, L, tables, fencing):
        ref = run_cycle_fences(oracle, nodes, L, *tables, fencing)
        with PlacementEngine(L) as e:
            e.load_nodes(nodes); e.submit_gangs(*tables); e.set_fences(fencing)
            got = _outputs(e, e.run_cycle())
        _same(got, ref, len(fencing))
        return got

    assert Starvation().run(cycle, fence_after=None)[0] is None
    at, _ = Starvation().run(cycle, fence_after=1)
    assert at is not None and at <= 4


def test_several_submissions_on_one_engine(built_lib, oracle):
    """the set is cleared by the next submission and by a node reload; the flag never outlives it; update_nodes keeps it"""
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, fencing = hand_cases()["least_shortfall"]()
    plain = oracle.run_cycle(nodes, L, *tables)
    fenced = run_cycle_fences(oracle, nodes, L, *tables, fencing)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables); e.set_fences(fencing)
        e.run_cycle(); _same(_outputs(e), fenced, "fenced")
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.run_cycle(); _same(_outputs(e), plain, "after a new submission")
        assert not e.gang_status()["reserved0"].any()
        e.set_fences(fencing)
        e.update_nodes(np.zeros(0, np.uint32), np.zeros(0, T.node_dt))
        e.load_nodes(nodes)
        e.run_cycle(); _same(_outputs(e), plain, "after a node reload")
        e.submit_gangs(*tables); e.set_fences(fencing)
        e.update_nodes(np.arange(len(nodes), dtype=np.uint32), nodes)   # (the last cycle left its admissions in the table)
        e.run_cycle(); _same(_outputs(e), fenced, "kept across update_nodes")


def test_empty_set_is_byte_identical(built_lib):
    from grove_b200.engine import PlacementEngine
    cfg = synth.config_c4(n=5040, g=800)
    out = []
    for with_set in (False, True):
        with PlacementEngine(cfg["n_levels"]) as e:
            e.load_nodes(cfg["nodes"]); e.submit_gangs(*cfg["tables"])
            if with_set:
                e.set_fences(np.zeros(0, np.uint32))
            st = e.run_cycle()
            out.append((e.gang_status(), e.placements(), e.scope_domains(), e.nodes(), st["rounds"], st["evaluations"]))
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    from spread_cases import spread_groups
    nodes, L, tables, fencing = hand_cases()["least_shortfall"]()
    G = len(tables[0])

    def code(fn):
        with pytest.raises(GroveError) as ex:
            fn()
        return ex.value.code

    with PlacementEngine(L) as e:
        assert code(lambda: e.set_fences(fencing)) == -5                      # nothing loaded
        e.load_nodes(nodes)
        assert code(lambda: e.set_fences(fencing)) == -5                      # no submission
        e.submit_gangs(*tables)
        assert code(lambda: e.set_fences([G])) == -1                          # out of range
        assert code(lambda: e.set_fences([0, 0])) == -1                       # duplicate
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=1)])])
        for _ in range(70):
            b.add_gang([(None, [dict(gpu=1)])], level=0)
        many = b.build()
        e.submit_gangs(*many)
        assert code(lambda: e.set_fences([0])) == -1                          # no gang Required level
        assert code(lambda: e.set_fences(np.arange(1, 66))) == -4             # more than MAX_FENCES
        e.set_fences(np.arange(1, 65))                                          # exactly MAX_FENCES
        e.submit_gangs(*tables); e.set_fences(fencing)
        none = np.zeros(0, T.running_dt), np.zeros(0, T.holding_dt)
        assert code(lambda: e.run_cycle_preempt(*none)) == -5
        assert code(lambda: e.run_cycle_reuse(np.full(G, T.NONE_U32, np.uint32), *none)) == -5
        assert code(lambda: e.run_cycle_reuse_preempt(np.full(G, T.NONE_U32, np.uint32), *none)) == -5
        e.set_spread(spread_groups([0], [T.SPREAD_HARD], [1]), np.zeros(G, np.uint32))
        e.set_fences(fencing)
        assert code(lambda: e.run_cycle()) == -5                               # spread members and fences together
        e.set_spread(spread_groups([0], [T.SPREAD_HARD], [1]), np.full(G, T.NONE_U32, np.uint32))
        e.run_cycle()
        assert code(lambda: e.diagnose()) == -5                                # a fenced cycle is not diagnosed
        e.set_fences([])
        e.run_cycle()
        e.diagnose()
    wb = T.GangTableBuilder()
    wb.add_gang([(None, [dict(gpu=0, min=200)])], level=0)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs_wide(*wb.build_wide())
        assert code(lambda: e.set_fences([0])) == -4                          # wide submission
