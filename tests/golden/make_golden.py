"""Regenerates tests/golden/*.npz.

The reference (ai-dynamo/grove @ 08ad3b37) is Go and contains no scheduler, so there is no reference OUTPUT to record.  These fixtures are small
snapshots in the shapes of the reference's e2e suites and BASELINE.json configs together with the
sequential oracle's answer (oracle/grove_oracle_seq.c) at the commit that generated them; they pin (a) the oracle against silent drift and
(b) the CUDA path on the GPU, where neither the reference nor this generator needs to run.

    python tests/golden/make_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from grove_b200 import synth, tables as T  # noqa: E402
from oracle import oracle_py as O  # noqa: E402


def cases():
    A = synth.AGENT
    c = lambda mem, n, level=None, replicas=None: dict(mem=mem, min=n, replicas=n if replicas is None else replicas, level=level, class_mask=A)  # noqa: E731
    b = T.GangTableBuilder(); synth.workload1(b, pcsg_replicas=4, pcs_replicas=2)
    yield "gs_workload1_28n", synth.e2e_cluster(28, cordoned=3), 4, b.build()
    b = T.GangTableBuilder(); synth.workload2(b, pcsg_replicas=3, pcs_replicas=2)
    yield "gs_workload2_12n", synth.e2e_cluster(12, cordoned=1), 4, b.build()
    b = T.GangTableBuilder()
    b.add_gang([(2, [c(40, 2, 3), c(40, 2, 3)]), (2, [c(40, 2, 3), c(40, 2, 3)])], level=1)
    b.add_gang([(None, [c(20, 3, 2)]), (None, [c(20, 4, 1)])])
    b.add_gang([(None, [c(500, 10)])], level=2)
    yield "tas_hierarchy_mix_28n", synth.e2e_cluster(28), 4, b.build()
    nodes = synth.e2e_cluster(28); nodes["dom"][14:, 2] = T.DOM_ABSENT
    b = T.GangTableBuilder()
    for i in range(8):
        b.add_gang([(None, [c(80, 2)])], level=2, priority=i % 3)
    yield "tas17_absent_labels", nodes, 4, b.build()
    cfg = synth.config_c1(); yield "c1_simple1", cfg["nodes"], cfg["n_levels"], cfg["tables"]
    cfg = synth.config_c2(n=200, g=40); yield "c2_small", cfg["nodes"], cfg["n_levels"], cfg["tables"]
    cfg = synth.config_c3(n=756, g=120); yield "c3_small", cfg["nodes"], cfg["n_levels"], cfg["tables"]
    cfg = synth.config_c4(n=2520, g=400); yield "c4_small", cfg["nodes"], cfg["n_levels"], cfg["tables"]


def main():
    for name, nodes, L, (g, c, s) in cases():
        r = O.run_cycle(nodes, L, g, c, s, threads=4)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), nodes=nodes, n_levels=L, gangs=g, cliques=c, scopes=s,
                            placements=r["placements"], status=r["status"], scope_status=r["scope_status"],
                            nodes_after=r["nodes_after"])
        print(name, len(nodes), len(g), r["stats"]["gangs_admitted"], r["stats"]["pods_bound"])


if __name__ == "__main__":
    main()
