"""ctypes loader for the wide build of the sequential oracle (tests/wide_oracle.c): the same pass over clique records with
16-bit counts and up to GROVE_MAX_WIDE_GANG_PODS pods per gang.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SO = os.path.join(HERE, "libgrove_oracle_wide.so")
_DEPS = [os.path.join(HERE, "wide_oracle.c"), os.path.join(ROOT, "oracle", "grove_oracle_seq.c"),
         os.path.join(ROOT, "include", "grove_place.h")]
_LIB = None

# the clique record the wide build reads: grove_clique_t with 16-bit min_replicas / replicas
wide_clique_dt = np.dtype([
    ("req_cpu_milli", "<u4"), ("req_mem_mib", "<u4"), ("req_gpu", "<u2"), ("min_replicas", "<u2"), ("replicas", "<u2"),
    ("class_mask", "<u2"), ("level", "u1"), ("scope", "u1"),
], align=True)


def build(force: bool = False) -> str:
    stale = not os.path.exists(SO) or any(os.path.getmtime(p) > os.path.getmtime(SO) for p in _DEPS)
    if force or stale:
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-fopenmp", "-std=gnu11", "-Wall", "-Wno-unused-parameter", "-shared",
                               "-o", SO, _DEPS[0]])
    return SO


def lib():
    global _LIB
    if _LIB is None:
        from oracle import oracle_py
        _LIB = C.CDLL(build())
        _LIB.oracle_run_cycle_wide.restype = C.c_int32
        _LIB._stats = oracle_py.OracleStats
    return _LIB


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def wide_cliques(cliques, counts):
    from grove_b200 import tables as T
    cliques = np.asarray(cliques, dtype=T.clique_dt)
    w = np.zeros(len(cliques), dtype=wide_clique_dt)
    for f in ("req_cpu_milli", "req_mem_mib", "req_gpu", "class_mask", "level", "scope"):
        w[f] = cliques[f]
    w["min_replicas"], w["replicas"] = counts["min_replicas"], counts["replicas"]
    return w


def run_cycle_wide(nodes, n_levels, gangs, cliques, counts, scopes, threads=1):
    """The sequential pass of a wide submission (grove_submit_gangs_wide's inputs).  Returns dict(placements, status,
    scope_status, nodes_after, perm, stats) like oracle_py.run_cycle; raises RuntimeError(code) on a refused submission."""
    from grove_b200 import tables as T

    n, G, Q, S = len(nodes), len(gangs), len(cliques), len(scopes)
    nodes = np.ascontiguousarray(nodes, dtype=T.node_dt)
    gangs = np.ascontiguousarray(gangs, dtype=T.gang_dt)
    wq = wide_cliques(cliques, counts)
    scopes = np.ascontiguousarray(scopes, dtype=T.scope_dt)
    cap = int(counts["replicas"].astype(np.int64).sum()) if Q else 0
    pl = np.zeros(max(cap, 1), dtype=T.placement_dt)
    st = np.zeros(max(G, 1), dtype=T.status_dt)
    ss = np.zeros(max(S, 1), dtype=T.scope_status_dt)
    nodes_after = np.zeros(max(n, 1), dtype=T.node_dt)
    perm = np.zeros(max(n, 1), dtype=np.uint32)
    n_pl = C.c_uint32(0)
    L = lib()
    stats = L._stats()
    rc = L.oracle_run_cycle_wide(
        _p(nodes), C.c_uint32(n), C.c_uint32(n_levels), _p(gangs), C.c_uint32(G), _p(wq), C.c_uint32(Q),
        _p(scopes), C.c_uint32(S), C.c_int32(threads), _p(pl), C.c_uint32(len(pl)),
        C.byref(n_pl), _p(st), _p(ss), _p(nodes_after), _p(perm), None, None, C.byref(stats))
    if rc != 0:
        raise RuntimeError(rc)
    return dict(placements=pl[: n_pl.value].copy(), status=st[:G].copy(), scope_status=ss[:S].copy(),
                nodes_after=nodes_after[:n].copy(), perm=perm[:n].copy(),
                stats={k: getattr(stats, k) for k, _ in L._stats._fields_})
