"""-m "not gpu": reservation reuse (include/grove_place.h "reservation reuse") as its definition reads, on the CPU oracle: the
properties DESIGN.md section 1 pins, and hand cases of a new version meeting its predecessor's holdings."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T
from preempt_cases import holdings_of
from reuse_cases import free_table, hold_table, rolling_cluster, run_cycle_reuse, usage

NONE = T.NONE_U32


def _first_cycle(oracle, nodes, L, tables):
    ref = oracle.run_cycle(nodes, L, *tables)
    running, holdings = holdings_of(ref["placements"], ref["status"], *[tables[0], tables[1]])
    return ref["nodes_after"], running, holdings


def _one_gang(pods, mem=80, priority=0, gated=False, base=None, b=None):
    b = b or T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=mem, min=pods, class_mask=synth.AGENT)])], priority=priority, gated=gated, base=base)
    return b


@pytest.fixture
def six_full(oracle):
    """six e2e nodes (one 80 MiB pod each), all taken by one running gang: 70 MiB left per node"""
    nodes = synth.e2e_cluster(6)
    now, running, holdings = _first_cycle(oracle, nodes, 4, _one_gang(6).build())
    assert len(running) == 1 and (now["free_mem_mib"] == 70).all()
    return now, running, holdings


def _same(a, b):
    for k in ("placements", "status", "scope_status", "nodes_after"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("seed", [3, 4, 5])
def test_without_replacements_it_is_the_ordinary_cycle(oracle, seed):
    nodes, L, (g, c, s), _, running, holdings = rolling_cluster(oracle, seed, n=630, g_running=200, g_pending=80)
    none = np.full(len(g), NONE, dtype=np.uint32)
    _same(run_cycle_reuse(oracle, nodes, L, g, c, s, none, running, holdings), oracle.run_cycle(nodes, L, g, c, s))


@pytest.mark.parametrize("seed", [21, 22, 23, 24])
def test_pieces_equal_one_gang_per_call(oracle, seed):
    nodes, L, (g, c, s), rep, running, holdings = rolling_cluster(oracle, seed, n=630, g_running=200, g_pending=60)
    assert (rep != NONE).sum() >= 5
    a = run_cycle_reuse(oracle, nodes, L, g, c, s, rep, running, holdings)
    _same(a, run_cycle_reuse(oracle, nodes, L, g, c, s, rep, running, holdings, one_per_call=True))
    assert (a["status"]["state"][rep != NONE] == T.GANG_ADMITTED).any()


def test_successor_fits_only_on_its_predecessors_resources(oracle, six_full):
    now, running, holdings = six_full
    b = _one_gang(1, priority=5)          # ranks before the successor; would fit only on the hold
    _one_gang(6, priority=1, b=b)         # the new version
    _one_gang(1, priority=0, b=b)         # ranks after it
    g, c, s = b.build()
    out = run_cycle_reuse(oracle, now, 4, g, c, s, np.array([NONE, 0, NONE], dtype=np.uint32), running, holdings)
    assert list(out["status"]["state"]) == [T.GANG_REJECTED, T.GANG_ADMITTED, T.GANG_REJECTED]
    U = usage(out["placements"], out["status"], c, 1, 6)
    assert np.array_equal(free_table(out["nodes_after"]), free_table(now) + hold_table(6, running, holdings, 0) - U)


def test_leftovers_come_back_only_when_the_pass_ends(oracle, six_full):
    now, running, holdings = six_full
    b = _one_gang(3, priority=1)          # the new version needs half of what its predecessor holds
    _one_gang(1, priority=0, b=b)         # ranks after it: the leftovers are not free yet
    g, c, s = b.build()
    out = run_cycle_reuse(oracle, now, 4, g, c, s, np.array([0, NONE], dtype=np.uint32), running, holdings)
    assert list(out["status"]["state"]) == [T.GANG_ADMITTED, T.GANG_REJECTED]
    assert sorted(out["nodes_after"]["free_mem_mib"]) == [70, 70, 70, 150, 150, 150]


def test_successor_asking_for_more_takes_the_rest_from_the_free_table(oracle, six_full):
    now, running, holdings = six_full
    g, c, s = _one_gang(6, mem=100).build()
    out = run_cycle_reuse(oracle, now, 4, g, c, s, np.array([0], dtype=np.uint32), running, holdings)
    assert out["status"]["state"][0] == T.GANG_ADMITTED
    assert (out["nodes_after"]["free_mem_mib"] == 70 - 20).all()   # (U - H)+ = 20 MiB of the free 70 on every node
    # more than free + hold: rejected, nothing moves
    g, c, s = _one_gang(6, mem=151).build()
    out = run_cycle_reuse(oracle, now, 4, g, c, s, np.array([0], dtype=np.uint32), running, holdings)
    assert out["status"]["state"][0] == T.GANG_REJECTED


@pytest.mark.parametrize("how", ["rejected", "gated", "base_rejected"])
def test_successor_that_is_not_admitted_changes_nothing(oracle, six_full, how):
    now, running, holdings = six_full
    if how == "rejected":
        b = _one_gang(7)                               # seven nodes' worth: there are six
        rep = [0]
    elif how == "gated":
        b = _one_gang(6, gated=True)
        rep = [0]
    else:
        b = _one_gang(7, priority=1)                   # the base gang, rejected
        _one_gang(6, priority=0, base=0, b=b)          # the new version, scaled behind it
        rep = [NONE, 0]
    g, c, s = b.build()
    out = run_cycle_reuse(oracle, now, 4, g, c, s, np.array(rep, dtype=np.uint32), running, holdings)
    want = {"rejected": T.GANG_REJECTED, "gated": T.GANG_GATED_SKIP, "base_rejected": T.GANG_BASE_REJECTED}[how]
    assert out["status"]["state"][len(rep) - 1] == want
    assert np.array_equal(out["nodes_after"], now) and len(out["placements"]) == 0


@pytest.mark.parametrize("seed", [31, 32, 33])
def test_ranks_before_every_successor_get_their_ordinary_outcome(oracle, seed):
    nodes, L, (g, c, s), rep, running, holdings = rolling_cluster(oracle, seed, n=630, g_running=200, g_pending=60)
    g = g.copy()
    g["priority"][rep != NONE] = g["priority"].min() - 1   # successors rank after every other gang
    a = run_cycle_reuse(oracle, nodes, L, g, c, s, rep, running, holdings)
    b = oracle.run_cycle(nodes, L, g, c, s)
    first = rep == NONE
    assert np.array_equal(a["status"]["state"][first], b["status"]["state"][first])
    for i in np.nonzero(first & (a["status"]["state"] == T.GANG_ADMITTED))[0]:
        pa = a["placements"][a["status"]["placement_off"][i]: a["status"]["placement_off"][i] + a["status"]["n_pods"][i]]
        pb = b["placements"][b["status"]["placement_off"][i]: b["status"]["placement_off"][i] + b["status"]["n_pods"][i]]
        assert np.array_equal(pa, pb)


@pytest.mark.parametrize("seed", [41, 42, 43])
def test_resources_are_conserved(oracle, seed):
    nodes, L, (g, c, s), rep, running, holdings = rolling_cluster(oracle, seed, n=630, g_running=200, g_pending=60)
    out = run_cycle_reuse(oracle, nodes, L, g, c, s, rep, running, holdings)
    N = len(nodes)
    lhs = free_table(out["nodes_after"])
    rhs = free_table(nodes)
    for i in np.nonzero(out["status"]["state"] == T.GANG_ADMITTED)[0]:
        lhs = lhs + usage(out["placements"], out["status"], c, i, N)
        if rep[i] != NONE:
            rhs = rhs + hold_table(N, running, holdings, int(rep[i]))
    assert np.array_equal(lhs, rhs)
