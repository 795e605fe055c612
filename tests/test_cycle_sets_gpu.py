"""Which optional sets every cycle entry runs with (include/grove_place.h): the return code of grove_run_cycle, the four
running-gang entries and the three queue entries under each set alone, under the pairs grove_run_cycle decides between, under a
fair-share set over a queue set without members and for a wide submission -- and what grove_diagnose answers afterwards.  A
plain cycle runs first, so an entry that refuses leaves a cycle grove_diagnose still describes."""
import numpy as np
import pytest

from grove_b200 import tables as T
from queue_cases import make_queues, nodes_flat

pytestmark = pytest.mark.gpu
NONE = T.NONE_U32
OK, LIMIT, STATE = 0, -4, -5
G = 4

RUNNING = ("reuse", "preempt", "reuse_preempt", "consolidate")
QUEUE = ("preempt_queues", "reclaim_queues", "reclaim_preempt_queues")

# condition -> (grove_run_cycle, each running-gang entry, each queue entry), as (return code, grove_diagnose code) pairs.
# "fair_share" stands on a queue set with members; the sets are given in the order queue, fair share, then the rest.
EXPECTED = {
    "none":                    ((OK, OK), (OK, STATE), (STATE, OK)),
    "spread":                  ((OK, STATE), (STATE, OK), (STATE, OK)),
    "fence":                   ((OK, STATE), (STATE, OK), (STATE, OK)),
    "queue":                   ((OK, OK), (STATE, OK), (OK, STATE)),
    "binpack":                 ((OK, OK), (STATE, OK), (STATE, OK)),
    "imex":                    ((OK, STATE), (STATE, OK), (STATE, OK)),
    "fair_share":              ((OK, STATE), (STATE, OK), (STATE, OK)),
    "fair_share_no_members":   ((OK, STATE), (OK, STATE), (STATE, OK)),
    "spread+fence":            ((STATE, OK), (STATE, OK), (STATE, OK)),
    "spread+queue":            ((STATE, OK), (STATE, OK), (STATE, OK)),
    "spread+imex":             ((STATE, OK), (STATE, OK), (STATE, OK)),
    "fence+queue":             ((STATE, OK), (STATE, OK), (STATE, OK)),
    "fence+imex":              ((STATE, OK), (STATE, OK), (STATE, OK)),
    "queue+imex":              ((STATE, OK), (STATE, OK), (STATE, OK)),
    "binpack+spread":          ((STATE, OK), (STATE, OK), (STATE, OK)),
    "binpack+fence":           ((STATE, OK), (STATE, OK), (STATE, OK)),
    "binpack+queue":           ((OK, OK), (STATE, OK), (STATE, OK)),
    "binpack+imex":            ((STATE, OK), (STATE, OK), (STATE, OK)),
    "fair_share+spread":       ((STATE, OK), (STATE, OK), (STATE, OK)),
    "fair_share+fence":        ((STATE, OK), (STATE, OK), (STATE, OK)),
    "fair_share+binpack":      ((STATE, OK), (STATE, OK), (STATE, OK)),
    "fair_share+imex":         ((STATE, OK), (STATE, OK), (STATE, OK)),
    "wide":                    ((OK, OK), (LIMIT, STATE), (STATE, OK)),
}


def _snapshot():
    """six 8-GPU nodes in two blocks; four one-GPU gangs with a Required block level, all in a single leaf queue"""
    b = T.GangTableBuilder()
    for _ in range(G):
        b.add_gang([(None, [dict(gpu=1, min=1)])], level=0)
    return nodes_flat(6, per_block=3), b.build()


def _wide_tables():
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=1, min=200, replicas=200)])], level=0)
    return b.build_wide()


def _give(e, sets):
    if "queue" in sets or "fair_share" in sets:
        e.set_queues(make_queues([(None, (None, None, 2), (0, 0, 0))]), np.zeros(G, np.uint32))
    if "fair_share_no_members" in sets:
        e.set_queues(make_queues([(None, (None, None, 2), (0, 0, 0))]), np.full(G, NONE, np.uint32))
    if "fair_share" in sets or "fair_share_no_members" in sets:
        e.set_fair_share(np.zeros(1, dtype=T.queue_quota_dt))
    if "spread" in sets:
        sp = np.zeros(1, dtype=T.spread_dt); sp["level"] = 0; sp["mode"] = T.SPREAD_HARD; sp["max_skew"] = 1
        e.set_spread(sp, np.zeros(G, np.uint32))
    if "fence" in sets:
        e.set_fences(np.array([1], np.uint32))
    if "binpack" in sets:
        e.set_binpack(np.zeros(G, np.uint8))
    if "imex" in sets:
        e.set_compute_domains(np.array([7] + [T.CD_NONE] * (G - 1), np.uint32), np.full(e.n, T.CD_NONE, np.uint32))


def _call(e, entry, n_gangs):
    running, holdings = np.zeros(0, dtype=T.running_dt), np.zeros(0, dtype=T.holding_dt)
    none, empty = np.full(n_gangs, NONE, np.uint32), np.zeros(0, np.uint32)
    quotas = np.zeros(1, dtype=T.queue_quota_dt)
    calls = {
        "run_cycle": lambda: e.run_cycle(),
        "reuse": lambda: e.run_cycle_reuse(none, running, holdings),
        "preempt": lambda: e.run_cycle_preempt(running, holdings),
        "reuse_preempt": lambda: e.run_cycle_reuse_preempt(none, running, holdings),
        "consolidate": lambda: e.run_cycle_consolidate(empty, empty, running, holdings),
        "preempt_queues": lambda: e.run_cycle_preempt_queues(running, holdings, empty),
        "reclaim_queues": lambda: e.run_cycle_reclaim_queues(quotas, running, holdings, empty),
        "reclaim_preempt_queues": lambda: e.run_cycle_reclaim_preempt_queues(quotas, running, holdings, empty),
    }
    return _code(calls[entry])


def _code(call):
    from grove_b200.engine import GroveError
    try:
        call()
    except GroveError as ex:
        return ex.code
    return OK


def _expected(cond, entry):
    run, running, queue = EXPECTED[cond]
    return run if entry == "run_cycle" else running if entry in RUNNING else queue


@pytest.mark.parametrize("entry", ("run_cycle",) + RUNNING + QUEUE)
def test_sets_each_entry_runs_with(built_lib, entry):
    from grove_b200.engine import PlacementEngine
    nodes, tables = _snapshot()
    got = {}
    with PlacementEngine(2) as e:
        for cond in EXPECTED:
            e.load_nodes(nodes)
            if cond == "wide":
                e.submit_gangs_wide(*_wide_tables())
            else:
                e.submit_gangs(*tables)
            e.run_cycle()   # a plain cycle: grove_diagnose describes it until something changes
            assert _code(e.diagnose) == OK, cond
            if cond != "wide":
                _give(e, cond.split("+"))
            rc = _call(e, entry, e.G)
            got[cond] = (rc, _code(e.diagnose))
    want = {cond: _expected(cond, entry) for cond in EXPECTED}
    assert got == want, {c: (got[c], want[c]) for c in EXPECTED if got[c] != want[c]}
