"""Seeded wide submissions (grove_submit_gangs_wide): clusters that mix ordinary PodGangs with ones of more than 128 pods and
PodGroups of more than 255 replicas, optionally on nodes that take more than 255 pods.  Shared by the CPU and GPU tests."""
import numpy as np

from grove_b200 import tables as T


def wide_case(seed, pref=False, big_nodes=False, n_range=(60, 500)):
    """-> (nodes, n_levels, (gangs, cliques, counts, scopes))"""
    rng = np.random.default_rng(seed)
    L = int(rng.integers(1, 5))
    n = int(rng.integers(*n_range))
    fan = [int(rng.integers(2, 6)) for _ in range(L)]
    nodes = T.make_nodes(n)
    idx = np.arange(n)
    span = n
    for l in range(L):
        span = max(1, span // fan[l])
        nodes["dom"][:, l] = idx // span if l < L - 1 or rng.random() < 0.7 else idx
    if rng.random() < 0.3:   # ragged: labels missing from some level down
        for i in rng.choice(n, size=max(1, n // 8), replace=False):
            nodes["dom"][i, int(rng.integers(0, L)):] = T.DOM_ABSENT
    nodes["free_cpu_milli"] = rng.integers(8000, 64001, n)
    nodes["free_mem_mib"] = rng.integers(65536, 524289, n)
    nodes["free_gpu"] = rng.integers(0, 9, n)
    nodes["free_pods"] = 110
    if big_nodes:   # nodes that take more than 255 pods of a small clique: the capacity bytes saturate there
        big = rng.random(n) < 0.3
        nodes["free_pods"][big] = rng.integers(256, 1200, int(big.sum()))
        nodes["free_cpu_milli"][big] = rng.integers(400_000, 2_000_000, int(big.sum()))
        nodes["free_mem_mib"][big] = rng.integers(2_000_000, 8_000_000, int(big.sum()))
    nodes["flags"] = (rng.random(n) > 0.05) * T.NODE_SCHEDULABLE

    def lvl(lo):
        return None if rng.random() < 0.5 or lo + 1 >= L else int(rng.integers(lo + 1, L))

    def deeper(req):
        lo = 0 if req is None else req + 1
        return int(rng.integers(lo, L)) if pref and lo < L and rng.random() < 0.4 else None

    b = T.GangTableBuilder()
    G = int(rng.integers(4, 30))
    for gi in range(G):
        wide = rng.random() < 0.35
        glevel = None if rng.random() < 0.5 else int(rng.integers(0, L))
        budget = int(rng.integers(129, T.MAX_WIDE_GANG_PODS + 1)) if wide else int(rng.integers(1, T.MAX_GANG_PODS + 1))
        scopes = []
        for _ in range(int(rng.integers(1, 3))):
            slevel = lvl(-1 if glevel is None else glevel)
            cliques = []
            for _ in range(int(rng.integers(1, 3))):
                if budget <= 0:
                    break
                reps = int(rng.integers(1, budget + 1)) if wide else int(rng.integers(1, min(budget, 255) + 1))
                budget -= reps
                mn = int(rng.integers(0, reps + 1)) if rng.random() < 0.3 else reps
                small = big_nodes and rng.random() < 0.6
                cliques.append(dict(cpu=int(rng.integers(0, 4)) * (100 if small else 1000), mem=int(rng.integers(1, 8)) * (128 if small else 4096),
                                    gpu=0 if small or rng.random() < 0.6 else int(rng.integers(1, 3)), min=mn, replicas=reps,
                                    level=lvl(-1 if slevel is None else slevel) if rng.random() < 0.3 else None))
                cliques[-1]["preferred"] = deeper(cliques[-1]["level"])
            if cliques:
                scopes.append((slevel, cliques, deeper(slevel)))
        b.add_gang(scopes, level=glevel, priority=int(rng.integers(0, 3)), preferred=deeper(glevel))
    return nodes, L, b.build_wide()


def pods_per_gang(gangs, counts):
    return np.array([int(counts["replicas"][g["clique_off"]: g["clique_off"] + g["n_cliques"]].sum()) for g in gangs])
