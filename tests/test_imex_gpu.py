"""ComputeDomain exclusivity through the C ABI (grove_set_compute_domains + grove_run_cycle) against its restatement over the
sequential oracle (tests/imex_cases.py): statuses, placements, scope domains, the node table, the sorted order and the owners, on
the hand cases, random snapshots with random CDs and owners, the relaxation knobs that change how the engine gets there, a reduced
C4 with one CD per PCS replica, and a replica scheduled cycle by cycle; a set without an enrolled clique changes nothing; the
refusals."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from imex_cases import NONE, enroll_randomly, hand_cases, run_cycle_imex
from test_random_parity_gpu import random_case

pytestmark = pytest.mark.gpu


def _run(nodes, L, tables, cd, owner0, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.set_compute_domains(cd, owner0)
        st = e.run_cycle()
        return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                    perm=e.debug_perm(), owners=e.compute_domain_owners(), stats=st)


def _same(got, ref, what=""):
    for k in ("status", "placements", "scope_status", "nodes_after", "perm", "owners"):
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, nodes, L, tables, cd, owner0, **kw):
    ref = run_cycle_imex(oracle, nodes, L, *tables, cd, owner0)
    got = _run(nodes, L, tables, cd, owner0, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    nodes, L, tables, cd, owner0 = hand_cases()[case]()
    _check(oracle, nodes, L, tables, cd, owner0, window=window)


def test_two_replicas_are_not_stacked(built_lib, oracle):
    """the case the plain cycle gets wrong: both replicas on node 0, whose second IMEX channel the driver refuses"""
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, cd, owner0 = hand_cases()["two_replicas"]()
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        e.run_cycle()
        assert set(e.placements()["node"].tolist()) == {0}
    got, _ = _check(oracle, nodes, L, tables, cd, owner0)
    st, pl = got["status"], got["placements"]
    assert set(pl[st["placement_off"][1]: st["placement_off"][1] + st["n_pods"][1]]["node"].tolist()) == {1}


def _case(seed):
    nodes, L, tables = random_case(seed, pref=seed % 2 == 1)
    cd, owner0 = enroll_randomly(np.random.default_rng(seed + 417), tables[0], tables[1], nodes)
    return nodes, L, tables, cd, owner0


@pytest.mark.parametrize("block,window", [(b, 0) for b in range(8)] + [(b, w) for w in (1, 7) for b in range(4)])
def test_random_snapshots(built_lib, oracle, block, window):
    for seed in range(block * 25, block * 25 + 25):
        _check(oracle, *_case(seed), window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_REFRESH=1", "GROVE_TUNE_HEAVY_ATT=1", "GROVE_TUNE_EVAL_CTAS=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """a table rebuild every round, every gang heavy, a single K3 CTA: other rounds and evaluations, the same result"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        nodes, L, tables = random_case(seed, big=seed % 4 == 0)
        cd, owner0 = enroll_randomly(np.random.default_rng(seed), tables[0], tables[1], nodes)
        _check(oracle, nodes, L, tables, cd, owner0)


def test_reduced_c4(built_lib, oracle):
    cfg = synth.config_c4(n=5040, g=800)
    g, c, s = cfg["tables"]
    cd, owner0 = synth.c4_compute_domains(cfg["nodes"], g, c)
    assert (owner0 != NONE).any() and (cd != NONE).any()
    got, _ = _check(oracle, cfg["nodes"], cfg["n_levels"], (g, c, s), cd, owner0)
    plain = oracle.run_cycle(cfg["nodes"], cfg["n_levels"], g, c, s)
    assert not np.array_equal(got["placements"], plain["placements"])   # the rule moved some pods


def test_replica_scheduled_after_a_delete(built_lib, oracle):
    """cycle by cycle, an engine per cycle, the owners fed back as the next owner0: three replicas of 4 x 1-GPU workers on two
    8-GPU nodes, the third REJECTED until replica 0 is deleted"""
    nodes, L, tables, cd, owner0 = hand_cases()["third_rejected"]()
    got, _ = _check(oracle, nodes, L, tables, cd, owner0)
    assert got["status"]["state"].tolist() == [T.GANG_ADMITTED, T.GANG_ADMITTED, T.GANG_REJECTED]
    owners, after = got["owners"].copy(), got["nodes_after"].copy()
    # replica 0 (CD 1) is deleted: its GPUs and its node's IMEX channel come back; replica 2 is submitted again
    n0 = int(got["placements"][0]["node"])
    after["free_gpu"][n0] += 4; after["free_cpu_milli"][n0] += 4000; after["free_mem_mib"][n0] += 4096; after["free_pods"][n0] += 4
    owners[n0] = NONE
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(gpu=1, cpu=1000, mem=1024, min=4)])], priority=1, anchor=0)
    t = b.build()
    got2, _ = _check(oracle, after, L, t, np.full(1, 3, np.uint32), owners)
    assert got2["status"]["state"][0] == T.GANG_ADMITTED and set(got2["placements"]["node"].tolist()) == {n0}
    assert got2["owners"][n0] == 3


def test_set_without_enrolled_clique_is_the_ordinary_cycle(built_lib):
    from grove_b200.engine import PlacementEngine
    cfg = synth.config_c4(n=5040, g=800)
    _, c, _ = cfg["tables"]
    owner0 = np.arange(len(cfg["nodes"]), dtype=np.uint32)
    out = []
    for with_set in (False, True):
        with PlacementEngine(cfg["n_levels"]) as e:
            e.load_nodes(cfg["nodes"]); e.submit_gangs(*cfg["tables"])
            if with_set:
                e.set_compute_domains(np.full(len(c), NONE, np.uint32), owner0)
            st = e.run_cycle()
            out.append((e.gang_status(), e.placements(), e.scope_domains(), e.nodes(), st["rounds"], st["evaluations"],
                        st["kernel_launches"]))
            if with_set:
                assert np.array_equal(e.compute_domain_owners(), owner0)
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    from spread_cases import spread_groups
    nodes, L, tables, cd, owner0 = hand_cases()["frontend_shares"]()
    G, Q, N = len(tables[0]), len(tables[1]), len(nodes)

    def code(fn):
        with pytest.raises(GroveError) as ex:
            fn()
        return ex.value.code

    with PlacementEngine(L) as e:
        assert code(lambda: e.set_compute_domains(cd, owner0)) == -5                   # nothing loaded
        e.load_nodes(nodes)
        assert code(lambda: e.set_compute_domains(cd, owner0)) == -5                   # no submission
        e.submit_gangs(*tables)
        assert code(lambda: e.compute_domain_owners()) == -5                           # no cycle with a set
        assert code(lambda: e.set_compute_domains(cd[:-1], owner0)) == -1              # wrong lengths
        assert code(lambda: e.set_compute_domains(cd, owner0[:-1])) == -1
        bad = cd.copy(); bad[0] = T.CD_NO_IMEX
        assert code(lambda: e.set_compute_domains(bad, owner0)) == -1                  # NO_IMEX as a clique's CD
        bad = cd.copy(); bad[1] = 5                                                     # the frontend requests no GPU
        assert code(lambda: e.set_compute_domains(bad, owner0)) == -1
        b = T.GangTableBuilder()
        b.add_gang([(None, [dict(gpu=1, min=1), dict(gpu=1, min=1)])], level=0)
        two = b.build()
        e.submit_gangs(*two)
        assert code(lambda: e.set_compute_domains(np.array([1, 2], np.uint32), owner0)) == -4   # two CDs in one gang
        e.set_compute_domains(np.array([1, 1], np.uint32), owner0)
        none = np.zeros(0, T.running_dt), np.zeros(0, T.holding_dt)
        assert code(lambda: e.run_cycle_preempt(*none)) == -5
        assert code(lambda: e.run_cycle_reuse(np.full(1, T.NONE_U32, np.uint32), *none)) == -5
        assert code(lambda: e.run_cycle_reuse_preempt(np.full(1, T.NONE_U32, np.uint32), *none)) == -5
        assert code(lambda: e.run_cycle_consolidate(np.zeros(0, np.uint32), np.zeros(0, np.uint32), *none)) == -5
        q = np.zeros(1, T.queue_dt); q["parent"] = T.NONE_U32; q["limit"] = 1 << 40
        e.set_queues(q, np.zeros(1, np.uint32))
        assert code(lambda: e.run_cycle_preempt_queues(*none, np.zeros(0, np.uint32))) == -5
        assert code(lambda: e.run_cycle()) == -5                                        # a queue set with members
        e.submit_gangs(*two); e.set_compute_domains(np.array([1, 1], np.uint32), owner0)
        e.set_fences([0])
        assert code(lambda: e.run_cycle()) == -5                                        # a fence set
        e.set_fences([])
        e.set_spread(spread_groups([0], [T.SPREAD_HARD], [1]), np.zeros(1, np.uint32))
        assert code(lambda: e.run_cycle()) == -5                                        # spread members
        e.set_spread(spread_groups([0], [T.SPREAD_HARD], [1]), np.full(1, T.NONE_U32, np.uint32))
        e.set_binpack(np.zeros(1, np.uint8))
        assert code(lambda: e.run_cycle()) == -5                                        # bin-packing members
        e.set_binpack(np.full(1, T.LEVEL_NONE, np.uint8))
        e.run_cycle()
        assert code(lambda: e.diagnose()) == -5                                         # a cycle with enrolled cliques
    with PlacementEngine(L) as e:   # a fresh engine: repeated cycles on one handle are a known defect (DESIGN.md section 9, item 3)
        e.load_nodes(nodes); e.submit_gangs(*two)
        e.set_compute_domains(np.full(2, NONE, np.uint32), owner0)                      # no enrolled clique: diagnosed
        e.run_cycle()
        e.diagnose()
    wb = T.GangTableBuilder()
    wb.add_gang([(None, [dict(gpu=1, min=200)])], level=0)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs_wide(*wb.build_wide())
        assert code(lambda: e.set_compute_domains(np.ones(1, np.uint32), owner0)) == -4   # wide submission
