"""-m gpu: the relaxation round as one stream-ordered chain (k_eval -> k_apply -> k_detect): the k_eval work queue at its
extremes, and the launches a cycle costs."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from grove_b200 import synth

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.mark.parametrize("env", [
    # starvation: ONE k_eval CTA takes every item of every round; every gang heavy after one attempt / no gang ever heavy
    {"GROVE_TUNE_EVAL_CTAS": "1", "GROVE_TUNE_MAX_ATT": "1", "GROVE_TUNE_HEAVY_ATT": "1"},
    {"GROVE_TUNE_EVAL_CTAS": "1", "GROVE_TUNE_MAX_ATT": "0", "GROVE_TUNE_HEAVY_ATT": "200"},
    # over-provision: far more CTAs than work items (and than fit on the GPU at once), the same two extremes
    {"GROVE_TUNE_EVAL_CTAS": "4096", "GROVE_TUNE_MAX_ATT": "1", "GROVE_TUNE_HEAVY_ATT": "1"},
    {"GROVE_TUNE_EVAL_CTAS": "4096", "GROVE_TUNE_MAX_ATT": "0", "GROVE_TUNE_HEAVY_ATT": "200"},
    # more CTAs per SM than are resident at once, and the bookkeeping kernels at one CTA per SM
    {"GROVE_TUNE_HEAVY_CTAS": "3", "GROVE_TUNE_WARP_CTAS": "1"},
])
def test_eval_queue_extremes_never_change_a_result(built_lib, oracle, env):
    """every result -- placements, statuses and the committed node table -- equals the oracle's however the k_eval queue is
    served; each env in a fresh process (the knobs are read when an engine is created)"""
    code = textwrap.dedent('''
        import sys, numpy as np
        sys.path.insert(0, %r)
        sys.path.insert(0, %r)
        from grove_b200 import synth
        from grove_b200.engine import PlacementEngine
        from oracle import oracle_py as O
        from test_random_parity_gpu import random_case
        cases = [(cfg["nodes"], cfg["n_levels"], cfg["tables"], name) for name, cfg in
                 (("C3", synth.config_c3(n=2016, g=300)), ("C4", synth.config_c4(n=5040, g=800)), ("C2", synth.config_c2(n=500, g=80)))]
        cases += [(*random_case(seed, big=seed >= 4000, pref=True), seed) for seed in list(range(3000, 3030)) + [4000]]
        for nodes, L, (g, c, s), what in cases:
            ref = O.run_cycle(nodes, L, g, c, s, threads=4)
            with PlacementEngine(L) as e:
                e.load_nodes(nodes); e.submit_gangs(g, c, s); e.run_cycle()
                assert np.array_equal(e.placements(), ref["placements"]), what
                assert np.array_equal(e.gang_status(), ref["status"]), what
                assert np.array_equal(e.nodes(), ref["nodes_after"]), what
        print("ok")
    ''' % (ROOT, HERE))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env={**os.environ, **env})
    assert r.returncode == 0 and "ok" in r.stdout, (env, r.stderr[-1500:])


def _c4_cycle_stats():
    from grove_b200.engine import PlacementEngine
    cfg = synth.config_c4()
    g, c, s = cfg["tables"]
    with PlacementEngine(cfg["n_levels"]) as e:
        e.load_nodes(cfg["nodes"]); e.submit_gangs(g, c, s)
        return e.run_cycle(), len(g)


AHEAD = 3        # rounds the host keeps enqueued beyond the one that runs: at most this many return at once after the last
TABLES = 4       # k_fit, k_clear_stale, k_shape_plaus -- and a count of 4 for the capacity-table build at the cycle's start
OUTPUTS = 2 + 4  # the last k_fold + k_fold_mark; k_fin_count, k_fin_scan, k_fin_status, k_emit
REBUILD = 2 + TABLES


def test_round_is_three_launches(built_lib, monkeypatch):
    """a relaxation round is k_eval, k_apply, k_detect: three launches, no second K3 form"""
    monkeypatch.setenv("GROVE_TUNE_REFRESH", "1000000")   # no table rebuild inside the cycle: every other launch is counted exactly
    st, _ = _c4_cycle_stats()
    rounds, launches = st["rounds"], st["kernel_launches"]
    assert rounds > 1
    fixed = launches - OUTPUTS - TABLES
    assert 3 * rounds <= fixed + 1 and fixed <= 3 * (rounds + AHEAD), (rounds, launches)
    monkeypatch.delenv("GROVE_TUNE_REFRESH")
    st, G = _c4_cycle_stats()
    rebuilds = -(-G // 1536)   # the settled prefix moves at least GROVE_TUNE_REFRESH (default 1 536) ranks between two rebuilds
    assert st["kernel_launches"] <= 3 * (st["rounds"] + AHEAD) + TABLES + OUTPUTS + REBUILD * rebuilds, (st["rounds"], st["kernel_launches"])
