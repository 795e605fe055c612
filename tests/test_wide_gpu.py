"""-m gpu: wide submissions (grove_submit_gangs_wide, PodGangs of up to 2048 pods) on the engine, held to the wide build of the
sequential oracle on every output; a non-wide submission through the wide entry; the entries that refuse a wide submission."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from grove_b200 import synth, tables as T
from grove_b200.engine import GroveError, PlacementEngine
from wide_cases import wide_case
import wide_oracle as W

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _run(nodes, L, tables, window=0):
    with PlacementEngine(L, window=window) as e:
        e.load_nodes(nodes)
        e.submit_gangs_wide(*tables)
        st = e.run_cycle()
        return dict(placements=e.placements(), status=e.gang_status(), scope_status=e.scope_domains(), nodes_after=e.nodes(), stats=st)


def _check(nodes, L, tables, **kw):
    ref = W.run_cycle_wide(nodes, L, *tables, threads=4)
    got = _run(nodes, L, tables, **kw)
    for k in ("placements", "status", "scope_status", "nodes_after"):
        assert np.array_equal(got[k], ref[k]), k
    return got


@pytest.mark.parametrize("seed", range(40))
def test_random_wide_snapshots(built_lib, seed):
    nodes, L, tables = wide_case(9000 + seed, pref=seed % 2 == 1, big_nodes=seed % 4 >= 2)
    _check(nodes, L, tables)


@pytest.mark.parametrize("window", [1, 7, 0])
def test_windows(built_lib, window):
    for seed in range(9100, 9108):
        nodes, L, tables = wide_case(seed, pref=True, big_nodes=seed % 2 == 0)
        _check(nodes, L, tables, window=window)


@pytest.mark.parametrize("knob", ["GROVE_TUNE_REFRESH", "GROVE_TUNE_HEAVY_ATT"])
def test_relaxation_knobs(built_lib, monkeypatch, knob):
    """a capacity-table rebuild every round; every gang heavy"""
    monkeypatch.setenv(knob, "1")
    for seed in range(9200, 9206):
        nodes, L, tables = wide_case(seed, pref=seed % 2 == 0, big_nodes=True)
        _check(nodes, L, tables)


def test_every_gang_heavy_on_one_cta(built_lib):
    """one k_eval CTA takes every item of every round, every gang heavy after one attempt (fresh process: the knobs are read
    when an engine is created)"""
    code = textwrap.dedent('''
        import sys, numpy as np
        sys.path.insert(0, %r)
        sys.path.insert(0, %r)
        from grove_b200.engine import PlacementEngine
        from wide_cases import wide_case
        import wide_oracle as W
        for seed in range(9300, 9310):
            nodes, L, tables = wide_case(seed, pref=seed %% 2 == 0, big_nodes=seed %% 3 == 0)
            ref = W.run_cycle_wide(nodes, L, *tables, threads=4)
            with PlacementEngine(L) as e:
                e.load_nodes(nodes); e.submit_gangs_wide(*tables); e.run_cycle()
                assert np.array_equal(e.placements(), ref["placements"]), seed
                assert np.array_equal(e.gang_status(), ref["status"]), seed
                assert np.array_equal(e.scope_domains(), ref["scope_status"]), seed
                assert np.array_equal(e.nodes(), ref["nodes_after"]), seed
        print("ok")
    ''' % (ROOT, HERE))
    env = {**os.environ, "GROVE_TUNE_EVAL_CTAS": "1", "GROVE_TUNE_MAX_ATT": "1", "GROVE_TUNE_HEAVY_ATT": "1"}
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "ok" in r.stdout, r.stderr[-1500:]


def test_synth_c4_with_large_gangs(built_lib):
    cfg = synth.config_c4_large(n=10080, g=2000, n_large=12)
    got = _check(cfg["nodes"], cfg["n_levels"], cfg["tables"])
    g, c, cnt, s = cfg["tables"]
    large = np.arange(len(g)) >= len(cfg["ordinary"][0])
    assert (got["status"]["state"][large] == T.GANG_ADMITTED).any()


def test_non_wide_submission_through_the_wide_entry(built_lib, oracle):
    """within the old limits the wide entry is the ordinary one: same outputs, rounds and evaluations"""
    from test_random_parity_gpu import random_case
    cases = [random_case(seed, pref=seed % 2 == 1) for seed in range(9400, 9410)]
    cfg = synth.config_c4(n=5040, g=800)
    cases.append((cfg["nodes"], cfg["n_levels"], cfg["tables"]))
    for nodes, L, (g, c, s) in cases:
        counts = np.zeros(len(c), dtype=T.clique_count_dt)
        counts["min_replicas"], counts["replicas"] = c["min_replicas"], c["replicas"]
        outs = []
        for wide in (False, True):
            with PlacementEngine(L) as e:
                e.load_nodes(nodes)
                e.submit_gangs_wide(g, c, counts, s) if wide else e.submit_gangs(g, c, s)
                st = e.run_cycle()
                outs.append((e.placements(), e.gang_status(), e.scope_domains(), e.nodes(), st["rounds"], st["evaluations"]))
        for a, b in zip(*outs):
            assert np.array_equal(a, b)


def test_entries_that_refuse_a_wide_submission(built_lib):
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=64, min=300)])])
    nodes = T.make_nodes(8)
    nodes["free_cpu_milli"], nodes["free_mem_mib"], nodes["free_pods"], nodes["flags"] = 64000, 524288, 110, T.NODE_SCHEDULABLE
    wide = b.build_wide()
    running = np.zeros(0, dtype=T.running_dt); holdings = np.zeros(0, dtype=T.holding_dt)
    with PlacementEngine(1) as e:
        e.load_nodes(nodes)
        e.submit_gangs_wide(*wide)
        calls = {
            "grove_run_cycle_preempt": lambda: e.run_cycle_preempt(running, holdings),
            "grove_run_cycle_reuse": lambda: e.run_cycle_reuse(np.full(1, T.NONE_U32, np.uint32), running, holdings),
            "grove_run_cycle_reuse_preempt": lambda: e.run_cycle_reuse_preempt(np.full(1, T.NONE_U32, np.uint32), running, holdings),
            "grove_run_score_pass": lambda: e.run_score_pass(),
        }
        for name, call in calls.items():
            with pytest.raises(GroveError) as ex:
                call()
            assert ex.value.code == -4 and name in str(ex.value), name
        import ctypes as C
        rc = e.lib.grove_shard_summary_device(e.h, C.c_void_p(1), C.c_uint32(1 << 20))
        assert rc == -4 and b"grove_shard_summary_device" in e.lib.grove_last_error(e.h)
        st = e.run_cycle()   # the ordinary cycle schedules it: 300 pods on 3 nodes of 110 (110, 110, 80)
        assert st["gangs_admitted"] == 1 and st["pods_bound"] == 300
    # the same submission through the wide entry within the old limits is accepted by every entry
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=64, min=100)])])
    with PlacementEngine(1) as e:
        e.load_nodes(nodes)
        e.submit_gangs_wide(*b.build_wide())
        e.run_cycle_preempt(running, holdings)
        e.run_score_pass()
