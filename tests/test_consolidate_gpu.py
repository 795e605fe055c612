"""Consolidation through the C ABI (grove_run_cycle_consolidate + grove_get_moves) against its restatement over the sequential
oracle (tests/consolidate_cases.py): statuses (the CONSOLIDATED and MOVED flags included), placements, scope domains, the move
list and the node table, on the hand cases, random snapshots at several windows, a single K3 CTA, a reduced C4 with the gangs of an
earlier cycle running and the starvation case cycle by cycle; one engine over several calls; the refusals."""
import numpy as np
import pytest

from grove_b200 import tables as T
from consolidate_cases import Starvation, hand_cases, random_snapshot, reduced_c4, run_cycle_consolidate

pytestmark = pytest.mark.gpu

KEYS = ("status", "placements", "scope_status", "nodes_after", "moves", "perm")


def _outputs(e, st=None):
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                moves=e.moves(), perm=e.debug_perm(), stats=st)


def _run(case, window=0):
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, targets, spec_of, running, holdings = case
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        return _outputs(e, e.run_cycle_consolidate(targets, spec_of, running, holdings))


def _same(got, ref, what=""):
    for k in KEYS:
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, case, **kw):
    nodes, L, tables, targets, spec_of, running, holdings = case
    ref = run_cycle_consolidate(oracle, nodes, L, *tables, targets, spec_of, running, holdings)
    got = _run(case, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    _check(oracle, hand_cases()[case](), window=window)


@pytest.mark.parametrize("block,window", [(b, 0) for b in range(8)] + [(b, w) for w in (1, 7) for b in range(4)])
def test_random_snapshots(built_lib, oracle, block, window):
    for seed in range(block * 25, block * 25 + 25):
        _check(oracle, random_snapshot(oracle, seed), window=window)


def test_one_k3_cta(built_lib, oracle, monkeypatch):
    monkeypatch.setenv("GROVE_TUNE_EVAL_CTAS", "1")
    for seed in range(500, 516):
        _check(oracle, random_snapshot(oracle, seed))


def test_overlapping_holding_ranges(built_lib, oracle):
    """two running gangs may name overlapping holding ranges: both hold what the shared records say"""
    nodes, L, tables, targets, spec_of, running, holdings = hand_cases()["two_targets"]()
    running = running.copy()
    running["holding_off"][1] = running["holding_off"][2]
    _check(oracle, (nodes, L, tables, targets, spec_of, running, holdings))


def test_reduced_c4(built_lib, oracle):
    case = reduced_c4(oracle)
    assert len(case[3]) == T.MAX_CONSOLIDATE_TARGETS
    got, _ = _check(oracle, case)
    assert got["stats"]["gangs_admitted"] == int((got["status"]["state"] == T.GANG_ADMITTED).sum())


def test_starvation_cycle_by_cycle(built_lib, oracle):
    from grove_b200.engine import PlacementEngine

    def cycle(nodes, L, tables, targets, spec_of, running, holdings):
        ref = run_cycle_consolidate(oracle, nodes, L, *tables, targets, spec_of, running, holdings)
        with PlacementEngine(L) as e:
            e.load_nodes(nodes); e.submit_gangs(*tables)
            got = _outputs(e, e.run_cycle_consolidate(targets, spec_of, running, holdings))
        _same(got, ref, len(targets))
        return got

    at, hist = Starvation(small_per_cycle=10).run(cycle, target_after=1)
    assert at is not None and hist[at][2] > 0


def test_several_calls_on_one_engine(built_lib, oracle):
    """the moves and flags of one call never outlive it; the table it leaves is the free table; grove_diagnose refuses after it"""
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tables, targets, spec_of, running, holdings = hand_cases()["priority_bar"]()
    ref = run_cycle_consolidate(oracle, nodes, L, *tables, targets, spec_of, running, holdings)
    plain = oracle.run_cycle(nodes, L, *tables)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.run_cycle_consolidate(targets, spec_of, running, holdings)
        _same(_outputs(e), ref, "first")
        with pytest.raises(GroveError) as ex:
            e.diagnose()
        assert ex.value.code == -5
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.run_cycle_consolidate(targets, spec_of, running, holdings)
        _same(_outputs(e), ref, "again")
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.run_cycle()
        got = _outputs(e)
        for k in ("status", "placements", "scope_status", "nodes_after"):
            assert np.array_equal(got[k], plain[k]), k
        assert not len(got["moves"]) and not got["status"]["reserved0"].any()
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.run_cycle_consolidate(targets[:0], spec_of, running, holdings)   # no targets: the ordinary cycle
        got = _outputs(e)
        for k in ("status", "placements", "scope_status", "nodes_after"):
            assert np.array_equal(got[k], plain[k]), k


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    from spread_cases import spread_groups
    nodes, L, tables, targets, spec_of, running, holdings = hand_cases()["two_targets"]()
    G = len(tables[0])
    spec = int(spec_of[0])

    def code(fn):
        with pytest.raises(GroveError) as ex:
            fn()
        return ex.value.code

    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        run = lambda t=targets, s=spec_of, r=running, h=holdings: e.run_cycle_consolidate(t, s, r, h)  # noqa: E731
        assert code(lambda: run(t=np.zeros(17, np.uint32))) == -4                       # more than 16 targets
        assert code(lambda: run(t=[G])) == -1                                            # target out of range
        assert code(lambda: run(t=[0, 0])) == -1                                         # target twice
        assert code(lambda: run(s=np.array([G, T.NONE_U32, T.NONE_U32], np.uint32))) == -1    # spec row out of range
        assert code(lambda: run(s=np.array([spec, spec, T.NONE_U32], np.uint32))) == -1      # spec row twice
        assert code(lambda: run(s=np.array([0, T.NONE_U32, T.NONE_U32], np.uint32))) == -1   # spec row is a target
        assert code(lambda: run(t=[0], s=np.array([1, T.NONE_U32, T.NONE_U32], np.uint32))) == -1   # spec row not gated
        bad = holdings.copy(); bad["node"][0] = len(nodes)
        assert code(lambda: run(h=bad)) == -1                                            # holding on a node out of range
        short = running.copy(); short["n_holdings"][-1] += 1
        assert code(lambda: run(r=short)) == -1                                          # holdings out of range
        big = holdings.copy(); big["pods"][0] = 0xFFFF
        assert code(lambda: run(h=big)) == -1                                            # free + holdings overflow a field
        e.set_fences([0])
        assert code(lambda: run()) == -5                                                 # a fence set in place
        e.submit_gangs(*tables)
        e.set_spread(spread_groups([0], [T.SPREAD_HARD], [1]), np.where(np.arange(G) < 2, 0, T.NONE_U32).astype(np.uint32))
        assert code(lambda: run()) == -5                                                 # a spread set with members
        e.submit_gangs(*tables)
        run()
    wb = T.GangTableBuilder()
    wb.add_gang([(None, [dict(gpu=0, min=200)])], level=0)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs_wide(*wb.build_wide())
        assert code(lambda: e.run_cycle_consolidate([], [], np.zeros(0, T.running_dt), np.zeros(0, T.holding_dt))) == -4   # wide
