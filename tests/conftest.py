import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


@pytest.fixture(scope="session")
def built_lib():
    """In-tree build of libgrove_place.so (nvcc cross-compiles without a GPU)."""
    from grove_b200 import build
    return build.build()


@pytest.fixture(scope="session")
def oracle():
    from oracle import oracle_py
    oracle_py.build()
    return oracle_py


class _EnginePlacer:
    """manifests -> tables -> ENGINE (through the C ABI), every output checked against the sequential oracle on the way"""

    def __init__(self, oracle_mod):
        self.oracle = oracle_mod

    def run_cycle(self, nodes, n_levels, gangs, cliques, scopes, **kw):
        import numpy as np
        from grove_b200.engine import PlacementEngine
        ref = self.oracle.run_cycle(nodes, n_levels, gangs, cliques, scopes)
        with PlacementEngine(n_levels) as e:
            e.load_nodes(nodes); e.submit_gangs(gangs, cliques, scopes)
            stats = e.run_cycle()
            out = dict(placements=e.placements(), status=e.gang_status(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                       perm=e.debug_perm(), stats=dict(stats))
        for k in ("placements", "status", "scope_status", "nodes_after", "perm"):
            assert np.array_equal(out[k], ref[k]), k
        return out

    def topology(self, nodes, n_levels):
        return self.oracle.topology(nodes, n_levels)


@pytest.fixture(params=["oracle", pytest.param("engine", marks=pytest.mark.gpu)])
def placer(request, oracle):
    """what schedules the tables a manifest test built: the CPU oracle (everywhere), or the engine on the GPU box (-m gpu)"""
    if request.param == "oracle":
        return oracle
    request.getfixturevalue("built_lib")
    return _EnginePlacer(oracle)
