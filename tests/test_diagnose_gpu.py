"""-m gpu: grove_diagnose equals the numpy restatement (tests/diagnose_cases.py) on every record, leaves every output of the
cycle byte for byte as it was, and refuses the states it does not describe."""
import glob
import os

import numpy as np
import pytest

from grove_b200 import synth, tables as T
from grove_b200.engine import GroveError, PlacementEngine
import diagnose_cases as D
from test_random_parity_gpu import random_case
from wide_cases import wide_case

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURES = sorted(glob.glob(os.path.join(HERE, "golden", "*.npz")))


def _outputs(e):
    return dict(placements=e.placements(), status=e.gang_status(), scope_status=e.scope_domains(), nodes_after=e.nodes())


def _check(nodes, L, tables, window=0):
    """one cycle + grove_diagnose; the records equal the restatement over the cycle's own outputs.  Returns the gang records."""
    wide = len(tables) == 4
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes)
        if wide:
            g, c, cnt, s = tables
            e.submit_gangs_wide(g, c, cnt, s)
            minr = cnt["min_replicas"]
        else:
            g, c, s = tables
            e.submit_gangs(g, c, s)
            minr = c["min_replicas"]
        e.run_cycle()
        before = _outputs(e)
        gd, qd = e.diagnose()
        after = _outputs(e)
        for k in before:
            assert before[k].tobytes() == after[k].tobytes(), k
        gd2, qd2 = e.diagnose()   # a second call gives the same records
        assert gd.tobytes() == gd2.tobytes() and qd.tobytes() == qd2.tobytes()
    rg, rq = D.diagnose(nodes, L, g, c, s, minr, before)
    assert np.array_equal(gd, rg), np.nonzero(gd != rg)[0][:8]
    assert np.array_equal(qd, rq), np.nonzero(qd != rq)[0][:8]
    return gd


@pytest.mark.parametrize("seed", range(40))
def test_random_snapshots(built_lib, seed):
    nodes, L, tables = random_case(32000 + seed, pref=seed % 2 == 1, big=seed % 10 == 9)
    _check(nodes, L, tables)


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[:-4] for p in FIXTURES])
def test_golden_fixtures(built_lib, path):
    z = np.load(path)
    _check(z["nodes"], int(z["n_levels"]), (z["gangs"], z["cliques"], z["scopes"]))


def test_reduced_c4(built_lib):
    cfg = synth.config_c4(n=5040, g=800)
    _check(cfg["nodes"], cfg["n_levels"], cfg["tables"])


def test_shrunken_c4(built_lib):
    """C4's gang mix on a node table too small for it: hundreds of gangs rejected, with every verdict"""
    cfg = synth.config_c4(n=1260, g=2400)
    gd = _check(cfg["nodes"], cfg["n_levels"], cfg["tables"])
    assert (gd["verdict"] != T.DIAG_NONE).sum() > 500
    assert set(gd["verdict"].tolist()) == {T.DIAG_NONE, T.DIAG_CLIQUE_SHORT, T.DIAG_NO_DOMAIN, T.DIAG_NO_JOINT_FIT}


@pytest.mark.parametrize("seed", range(16))
def test_wide_cases(built_lib, seed):
    nodes, L, tables = wide_case(33000 + seed, pref=seed % 2 == 1, big_nodes=seed % 4 >= 2)
    _check(nodes, L, tables)


@pytest.mark.parametrize("window", [1, 7, 0])
def test_windows(built_lib, window):
    for seed in range(34000, 34006):
        nodes, L, tables = random_case(seed, pref=seed % 2 == 0)
        _check(nodes, L, tables, window=window)


def test_refusals(built_lib):
    nodes, L, (g, c, s) = random_case(35000)
    running = np.zeros(0, dtype=T.running_dt)
    holdings = np.zeros(0, dtype=T.holding_dt)
    none = np.full(len(g), T.NONE_U32, np.uint32)

    def refused(e, code=-5):
        with pytest.raises(GroveError) as ex:
            e.diagnose()
        assert ex.value.code == code

    with PlacementEngine(L) as e:
        refused(e)                                   # no cycle
        e.load_nodes(nodes); e.submit_gangs(g, c, s)
        refused(e)
        for entry in (lambda: e.run_cycle_preempt(running, holdings), lambda: e.run_cycle_reuse(none, running, holdings),
                      lambda: e.run_cycle_reuse_preempt(none, running, holdings)):
            e.run_cycle(); e.diagnose()
            entry()
            refused(e)                               # the last cycle was a running-gang entry
        for change in (lambda: e.load_nodes(nodes), lambda: e.submit_gangs(g, c, s),
                       lambda: e.update_nodes(np.zeros(1, np.uint32), nodes[:1]),
                       lambda: e.submit_gangs_wide(g, c, np.array(list(zip(c["min_replicas"], c["replicas"])), dtype=T.clique_count_dt), s)):
            e.run_cycle(); e.diagnose()
            change()
            refused(e)                               # inputs changed since the cycle
        e.run_cycle()
        import ctypes as C
        gb = np.zeros(len(g), dtype=T.gang_diag_dt); qb = np.zeros(len(c), dtype=T.clique_diag_dt)
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        assert e.lib.grove_diagnose(e.h, p(gb), C.c_uint32(len(g) - 1), p(qb), C.c_uint32(len(c))) == -4
        assert e.lib.grove_diagnose(e.h, p(gb), C.c_uint32(len(g)), p(qb), C.c_uint32(len(c) - 1)) == -4
        assert e.lib.grove_diagnose(e.h, p(gb), C.c_uint32(len(g)), p(qb), C.c_uint32(len(c))) == 0
