"""Fair-share order through the C ABI (grove_set_queues + grove_set_fair_share + grove_run_cycle) against its restatement over the
sequential oracle (tests/fair_share_cases.py): statuses with flags, placements, scope domains, the node table, the permutation
and the turn order, on the hand cases, random contested snapshots, knobs that change how the engine gets there, a reduced C4,
one engine over several submissions, and the refusals; at full C4, the engine's outputs against a plain queue cycle in the turn
order it reports, and that order against O(R) recomputed from its outputs."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from fair_share_cases import (hand_cases, order_vec, random_snapshot, run_fair_share, use_of, with_order)

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32


def _outputs(e):
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                perm=e.debug_perm())


def _members(gq):
    return int((np.asarray(gq) != NONE).sum())


def _fair(e, nodes, tables, qs, gq, quotas):
    e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq); e.set_fair_share(quotas)
    st = e.run_cycle()
    out = _outputs(e)
    out.update(stats=st, order=e.turn_order(), fs=e.fair_share_stats())
    assert out["fs"]["iterations"] <= _members(gq) + 1
    return out


def _run(nodes, L, tables, qs, gq, quotas, window=0):
    from grove_b200.engine import PlacementEngine
    with PlacementEngine(L, window=window) as e:
        return _fair(e, nodes, tables, qs, gq, quotas)


def _same(got, ref, what=""):
    for k in ("status", "placements", "scope_status", "nodes_after", "perm", "order"):
        assert np.array_equal(got[k], ref[k]), (k, what)


def _check(oracle, nodes, L, tables, qs, gq, quotas, **kw):
    ref = run_fair_share(oracle, nodes, L, *tables, qs, gq, quotas)
    got = _run(nodes, L, tables, qs, gq, quotas, **kw)
    _same(got, ref, kw)
    return got, ref


@pytest.mark.parametrize("case", sorted(hand_cases()))
@pytest.mark.parametrize("window", [0, 1])
def test_hand_case(built_lib, oracle, case, window):
    _check(oracle, *hand_cases()[case](), window=window)


def test_many_iterations_takes_three(built_lib, oracle):
    got, _ = _check(oracle, *hand_cases()["many_iterations"]())
    assert got["fs"]["iterations"] >= 3 and got["fs"]["turns_rerun"] > 0


@pytest.mark.parametrize("block", range(8))
def test_random_snapshots_window_all(built_lib, oracle, block):
    for seed in range(block * 25, block * 25 + 25):
        _check(oracle, *random_snapshot(seed, pref=seed % 2 == 1))


@pytest.mark.parametrize("block", range(4))
@pytest.mark.parametrize("window", [1, 7])
def test_random_snapshots_narrow_windows(built_lib, oracle, block, window):
    for seed in range(1000 + block * 25, 1000 + block * 25 + 25):
        _check(oracle, *random_snapshot(seed, pref=seed % 2 == 1), window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_EVAL_CTAS=1", "GROVE_TUNE_REFRESH=1"])
def test_knobs(built_lib, oracle, monkeypatch, knob):
    """one K3 CTA, a table rebuild every round: other rounds and evaluations, the same result"""
    k, v = knob.split("=")
    monkeypatch.setenv(k, v)
    for seed in range(300, 316):
        _check(oracle, *random_snapshot(seed))


def _c4(n, g):
    """C4 in synth.c4_queues with deserved GPU quotas spread over the leaves' MinReplicas demand (0.15 to 0.5 of it), parents
    unlimited"""
    cfg = synth.config_c4(n=n, g=g)
    gg, c, s = cfg["tables"]
    qs, gq = synth.c4_queues(gg, c)
    gpu = c["min_replicas"].astype(np.int64) * c["req_gpu"].astype(np.int64)
    per_gang = np.array([gpu[int(o): int(o) + int(k)].sum() for o, k in zip(gg["clique_off"], gg["n_cliques"])], dtype=np.int64)
    need = np.bincount(gq, weights=per_gang, minlength=len(qs))
    quotas = np.zeros(len(qs), dtype=T.queue_quota_dt)
    quotas["deserved"] = T.QUEUE_UNLIMITED
    for i in range(8):
        quotas["deserved"][2 + i, 2] = int(need[2 + i] * (0.15 + 0.05 * i))
    return cfg["nodes"], cfg["n_levels"], (gg, c, s), qs, gq, quotas


def test_reduced_c4(built_lib, oracle):
    got, _ = _check(oracle, *_c4(5040, 800))
    assert (got["status"]["state"] == T.GANG_ADMITTED).sum() > 10


def test_full_c4_self_consistent(built_lib):
    """at C4 the restatement is too slow: the outputs equal a plain queue cycle on a fresh engine in the reported turn order, and
    O(R) recomputed from those outputs is that order"""
    from grove_b200.engine import PlacementEngine
    nodes, L, tables, qs, gq, quotas = _c4(50000, 10000)
    got = _run(nodes, L, tables, qs, gq, quotas)
    order = got["order"]
    assert np.array_equal(np.sort(order), np.arange(len(tables[0])))
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(with_order(tables[0], order), *tables[1:]); e.set_queues(qs, gq)
        e.run_cycle()
        plain = _outputs(e)
    for k in ("status", "placements", "scope_status", "nodes_after"):
        assert np.array_equal(got[k], plain[k]), k
    assert np.array_equal(order_vec(qs, quotas, tables[0], gq, use_of(got, tables[1])), order)
    print(f"C4 fair share: {got['fs']['iterations']} iterations, {got['fs']['turns_rerun']} turns re-run, "
          f"{int((got['status']['state'] == T.GANG_ADMITTED).sum())} admitted")


def test_one_engine_over_several_submissions(built_lib, oracle):
    """the set goes with its submission, and the cycle run again on one handle gives the same outputs"""
    from grove_b200.engine import PlacementEngine
    cases = [hand_cases()["many_iterations"](), hand_cases()["starved_team_first"](), random_snapshot(6)]   # (all on two levels)
    with PlacementEngine(2) as e:
        for k, (nodes, L, tables, qs, gq, quotas) in enumerate(cases):
            ref = run_fair_share(oracle, nodes, L, *tables, qs, gq, quotas)
            for rep in range(2):
                _same(_fair(e, nodes, tables, qs, gq, quotas), ref, (k, rep))
            e.load_nodes(nodes); e.submit_gangs(*tables); e.set_queues(qs, gq)
            e.run_cycle()
            from grove_b200.engine import GroveError
            with pytest.raises(GroveError):
                e.turn_order()


def test_second_cycle_on_one_submission(built_lib, oracle):
    """grove_run_cycle twice on one submission, no resubmission: the second cycle starts from the table the first committed, with
    the fair-share set still in place, and matches the restatement over that table on every output"""
    from grove_b200.engine import PlacementEngine
    cases = [hand_cases()["many_iterations"](), random_snapshot(6), random_snapshot(9)]
    for k, (nodes, L, tables, qs, gq, quotas) in enumerate(cases):
        with PlacementEngine(L) as e:
            first = _fair(e, nodes, tables, qs, gq, quotas)
            _same(first, run_fair_share(oracle, nodes, L, *tables, qs, gq, quotas), (k, 0))
            e.run_cycle()
            second = _outputs(e)
            second.update(order=e.turn_order())
            _same(second, run_fair_share(oracle, first["nodes_after"], L, *tables, qs, gq, quotas), (k, 1))


def test_refusals(built_lib):
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tables, qs, gq, quotas = hand_cases()["parent_before_child"]()
    empty = np.zeros(0, dtype=T.running_dt)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tables)
        with pytest.raises(GroveError, match="STATE"):    # no queue set
            e.set_fair_share(quotas)
        e.set_queues(qs, gq)
        with pytest.raises(GroveError, match="INVALID_ARG"):
            e.set_fair_share(quotas[:-1])
        with pytest.raises(GroveError, match="INVALID_ARG"):   # a member in a queue with children
            e.set_queues(qs, np.array([0, 4], np.uint32)); e.set_fair_share(quotas)
        e.set_queues(qs, gq); e.set_fair_share(quotas)
        with pytest.raises(GroveError, match="STATE"):
            e.turn_order()
        with pytest.raises(GroveError, match="STATE"):
            e.run_cycle_preempt_queues(empty, np.zeros(0, dtype=T.holding_dt), np.zeros(0, np.uint32))
        with pytest.raises(GroveError, match="STATE"):
            e.run_cycle_reclaim_queues(quotas, empty, np.zeros(0, dtype=T.holding_dt), np.zeros(0, np.uint32))
        with pytest.raises(GroveError, match="STATE"):
            e.run_cycle_reclaim_preempt_queues(quotas, empty, np.zeros(0, dtype=T.holding_dt), np.zeros(0, np.uint32))
        e.set_binpack(np.full(len(tables[0]), 0, np.uint8))
        with pytest.raises(GroveError, match="STATE"):
            e.run_cycle()
        e.submit_gangs(*tables); e.set_queues(qs, gq); e.set_fair_share(quotas)
        e.set_compute_domains(np.zeros(len(tables[1]), np.uint32), np.full(len(nodes), T.CD_NONE, np.uint32))
        with pytest.raises(GroveError, match="STATE"):
            e.run_cycle()
        e.submit_gangs(*tables); e.set_queues(qs, gq); e.set_fair_share(quotas)
        e.run_cycle()
        assert len(e.turn_order()) == len(tables[0])
        with pytest.raises(GroveError, match="STATE"):
            e.diagnose()
        e.update_nodes(np.zeros(1, np.uint32), nodes[:1])   # kept by an update
        e.run_cycle()
        assert len(e.turn_order()) == len(tables[0])
