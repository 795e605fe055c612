"""Replay harness for the reference's multi-step gang-scheduling suites (ai-dynamo/grove
operator/e2e/tests/gang_scheduling_test.go GS2-GS12): a kwok-shaped cluster whose nodes are cordoned and
uncordoned step by step, PodCliqueSets that are scaled between scheduling passes, and a placement function
(the oracle or the CUDA engine) run once per step over everything that is pending.

What a scheduler sees between two steps, restated from the operator's side of the contract:
  * a PodGang that is not scheduled yet is pending as a whole (MinReplicas all-or-nothing, surplus best effort);
  * a scaled PodGang is only visible once its base PodGang is scheduled (pod/syncflow.go:319-358) -- the
    base_gang column when both are in one pass;
  * pods of a scheduled PodGang that found no node stay Pending and are retried: they come back as a
    remainder gang (MinReplicas 0: the gang guarantee is already met), after every PodGang that still has
    to get its minimum.
The suites assert pod COUNTS per step (testctx WaitForPodPhases(running, pending)); so do the tests.
"""
import numpy as np

from grove_b200 import synth, tables as T

A = synth.AGENT


def clq(mn, replicas=None, mem=80):
    return dict(mem=mem, min=mn, replicas=mn if replicas is None else replicas, class_mask=A)


class Gang:
    def __init__(self, name, scopes, base=None):
        self.name, self.scopes, self.base = name, scopes, base
        self.scheduled = False
        self.bound = [[0] * len(cl) for _, cl in scopes]

    def total(self):
        return sum(c["replicas"] for _, cl in self.scopes for c in cl)

    def n_bound(self):
        return sum(sum(b) for b in self.bound)


class E2ESim:
    def __init__(self, n_nodes, cordoned, split_surplus=False, same_pass_unlock=True):
        # same_pass_unlock: a scaled PodGang rides in the same pass as its unscheduled base, gated by base_gang (the
        # engine unlocks it the round after the base is admitted).  False: it only shows up in the pass AFTER its base
        # was scheduled -- the operator removes the pods' gates in a later reconcile (pod/syncflow.go:255-312) -- and a
        # step repeats passes until nothing changes, as the suites wait for the cluster to settle.
        self.split_surplus, self.same_pass_unlock = split_surplus, same_pass_unlock
        self.nodes = synth.e2e_cluster(n_nodes)
        self.cordoned = list(range(n_nodes - cordoned, n_nodes))
        synth.cordon(self.nodes, self.cordoned)
        self.gangs = []

    # ---- workload shapes (e2e/yaml/workload1.yaml, workload2.yaml) ----
    def deploy(self, wl, pcs_replicas=1, pcsg_replicas=2):
        """returns the PCS replica indices deployed"""
        self.wl = wl
        self.pcsg = {}
        for r in range(pcs_replicas):
            self._add_pcs_replica(r, pcsg_replicas)
        return list(range(pcs_replicas))

    def _sg(self):   # one sg-x replica: pc-b x1 + pc-c x3
        return [clq(1), clq(3)] if self.wl == 1 else [clq(1, 1), clq(1, 3)]

    def _add_pcs_replica(self, r, pcsg_replicas):
        min_avail = 2 if self.wl == 1 else 1            # sg-x minAvailable
        scopes = [(None, [clq(2) if self.wl == 1 else clq(1, 2)])]   # pc-a
        scopes += [(None, self._sg()) for _ in range(min_avail)]
        base = Gang(f"pcs-{r}", scopes)
        self.gangs.append(base)
        self.pcsg[r] = (base, min_avail)
        self.scale_pcsg(r, pcsg_replicas)

    def scale_pcs(self, replicas, pcsg_replicas=2):
        for r in range(len(self.pcsg), replicas):
            self._add_pcs_replica(r, pcsg_replicas)

    def scale_pcsg(self, r, replicas):
        base, have = self.pcsg[r]
        for i in range(have, replicas):
            self.gangs.append(Gang(f"pcs-{r}-sg-x-{i}", [(None, self._sg())], base=base))
        self.pcsg[r] = (base, max(have, replicas))

    # ---- cluster steps ----
    def uncordon(self, k):
        idx, self.cordoned = self.cordoned[:k], self.cordoned[k:]
        self.nodes["flags"][idx] |= np.uint32(T.NODE_SCHEDULABLE)

    def pods(self):
        return sum(g.total() for g in self.gangs)

    def running(self):
        return sum(g.n_bound() for g in self.gangs)

    def tables(self):
        """(gangs, cliques, scopes), rows = [(gang, [(scope index, clique index) per table clique], remainder?)]

        split_surplus (the encoding GpuBackend::Encode uses for PodGangs without pack constraints): a PodGang that is
        not scheduled yet goes in as its minimum only; its best-effort pods follow as a remainder row gated behind it
        (base_gang), after every minimum row -- "minimums of every gang before anybody's surplus", what the step
        descriptions of GS8 / GS10 / GS12 say happens (which pods, not only how many)."""
        b, rows, row_of = T.GangTableBuilder(), [], {}
        for g in self.gangs:            # PodGangs that still have to get their minimum, in creation order
            if g.scheduled:
                continue
            base = None
            if g.base is not None and not g.base.scheduled:
                if not self.same_pass_unlock:
                    continue
                base = row_of[id(g.base)]
            scopes = g.scopes
            if self.split_surplus:
                scopes = [(lvl, [dict(c, replicas=c["min"]) for c in cl]) for lvl, cl in g.scopes]
            row_of[id(g)] = b.add_gang(scopes, base=base)
            rows.append((g, [(si, ci) for si, (_, cl) in enumerate(g.scopes) for ci in range(len(cl))], False))
        for g in self.gangs:            # then the pods beyond the minimum: Pending pods of scheduled PodGangs, surplus of the others
            if g.n_bound() == g.total() or (not g.scheduled and (not self.split_surplus or id(g) not in row_of)):
                continue
            scopes, index = [], []
            for si, (lvl, cl) in enumerate(g.scopes):
                have = [g.bound[si][ci] if g.scheduled else c["min"] for ci, c in enumerate(cl)]
                rem = [(ci, dict(c, min=0, replicas=c["replicas"] - have[ci])) for ci, c in enumerate(cl) if c["replicas"] > have[ci]]
                if rem:
                    scopes.append((lvl, [c for _, c in rem])); index += [(si, ci) for ci, _ in rem]
            if scopes:
                b.add_gang(scopes, base=None if g.scheduled else row_of[id(g)])
                rows.append((g, index, True))
        return b.build(), rows

    def step(self, place):
        """scheduling passes until the cluster settles (one pass when scaled gangs unlock inside the pass)"""
        while True:
            before = (self.running(), sum(g.scheduled for g in self.gangs))
            self.one_pass(place)
            if self.same_pass_unlock or (self.running(), sum(g.scheduled for g in self.gangs)) == before:
                return

    def one_pass(self, place):
        """place(nodes, gangs, cliques, scopes) -> dict(status, placements, nodes_after)"""
        (g, c, s), rows = self.tables()
        if len(g) == 0:
            return None
        r = place(self.nodes, g, c, s)
        for row, (gang, index, remainder) in enumerate(rows):
            st = r["status"][row]
            if st["state"] != T.GANG_ADMITTED:
                continue
            if not remainder:
                gang.scheduled = True
            pl = r["placements"][st["placement_off"]: st["placement_off"] + st["n_pods"]]
            for q in pl["clique"]:
                si, ci = index[int(q) - int(g["clique_off"][row])]
                gang.bound[si][ci] += 1
        self.nodes = r["nodes_after"]
        return r
