"""Kubernetes manifests -> packed tables (the data formats either side of the hot path).

* Node manifests in the shape the reference's KWOK generator emits
  (ai-dynamo/grove operator/hack/infra_manager/kwok.py:74-117): allocatable {cpu, memory, pods[, nvidia.com/gpu]},
  topology labels, NoSchedule taints, spec.unschedulable.
* PodGang manifests in the CRD's shape (scheduler/api/core/v1alpha1/podgang.go:51-131,
  crds/scheduler.grove.io_podgangs.yaml): podgroups[].{name, podReferences, minReplicas,
  topologyConstraint.packConstraint.required}, topologyConstraint, topologyConstraintGroupConfigs,
  priorityClassName.  What a PodGroup's pods request is not in the CRD (a scheduler reads the Pods); it is
  passed alongside as {podGroupName: {"cpu": "...", "memory": "...", "nvidia.com/gpu": n}}.

The C++ host mirror (grove_b200/csrc/host) does the same from structs; this module is the file-format
counterpart used by tools and tests.
"""
from __future__ import annotations


import numpy as np

from . import tables as T

from fractions import Fraction

# resource.Quantity suffixes (k8s.io/apimachinery/pkg/api/resource): binary SI, decimal SI, milli
_BIN = {"Ki": 2 ** 10, "Mi": 2 ** 20, "Gi": 2 ** 30, "Ti": 2 ** 40, "Pi": 2 ** 50, "Ei": 2 ** 60}
_DEC = {"m": Fraction(1, 1000), "k": 10 ** 3, "M": 10 ** 6, "G": 10 ** 9, "T": 10 ** 12, "P": 10 ** 15, "E": 10 ** 18}


def _quantity(q) -> Fraction:
    """a Kubernetes quantity as an exact number of base units ("1500m" -> 3/2, "1Gi" -> 2**30, "1e3" -> 1000)"""
    s = str(q).strip()
    for suf, mul in _BIN.items():
        if s.endswith(suf):
            return Fraction(s[: -len(suf)]) * mul
    for suf, mul in _DEC.items():
        if s.endswith(suf) and not s[: -len(suf)].endswith(("e", "E")):
            return Fraction(s[: -len(suf)]) * mul
    return Fraction(s)


def _ceil(x: Fraction) -> int:
    return -((-x.numerator) // x.denominator)


def parse_cpu_milli(q, request: bool = False) -> int:
    """Kubernetes CPU quantity -> millicores ("64" -> 64000, "500m" -> 500, 0.5 -> 500, "2k" -> 2000000).  A pod's request is
    rounded UP, what a node offers DOWN (Kubernetes rounds requests up: under-counting them would over-commit nodes)."""
    x = _quantity(q) * 1000
    return _ceil(x) if request else x.numerator // x.denominator


def parse_mem_mib(q, request: bool = False) -> int:
    """Kubernetes memory quantity -> MiB ("512Gi" -> 524288, "150Mi" -> 150, "100M" -> 95 offered / 96 requested,
    "500Ki" -> 0 offered / 1 requested)."""
    x = _quantity(q) / 2 ** 20
    return _ceil(x) if request else x.numerator // x.denominator


def nodes_from_manifests(manifests, level_keys, class_key=None, used=None):
    """Node manifests -> (node table, node names, per-level label interning, class values).

    level_keys: ordered label keys, broadest first (ClusterTopology.spec.levels[].key).
    class_key:  label whose value partitions nodes into selector classes (class 0 = label absent).
    used:       optional {node name: {"cpu": q, "memory": q, "nvidia.com/gpu": n, "pods": n}} already requested.
    """
    if len(level_keys) > T.MAX_LEVELS:
        raise ValueError("at most %d topology levels" % T.MAX_LEVELS)
    nodes = T.make_nodes(len(manifests))
    names, intern, classes = [], [dict() for _ in level_keys], {}
    for i, m in enumerate(manifests):
        meta, spec, status = m.get("metadata", {}), m.get("spec", {}) or {}, m.get("status", {}) or {}
        names.append(meta.get("name", f"node-{i}"))
        alloc = status.get("allocatable") or status.get("capacity") or {}
        u = (used or {}).get(names[-1], {})
        nodes["free_cpu_milli"][i] = max(0, parse_cpu_milli(alloc.get("cpu", 0)) - parse_cpu_milli(u.get("cpu", 0), request=True))
        nodes["free_mem_mib"][i] = max(0, parse_mem_mib(alloc.get("memory", 0)) - parse_mem_mib(u.get("memory", 0), request=True))
        nodes["free_gpu"][i] = max(0, int(alloc.get("nvidia.com/gpu", 0)) - int(u.get("nvidia.com/gpu", 0)))
        nodes["free_pods"][i] = max(0, int(alloc.get("pods", 110)) - int(u.get("pods", 0)))
        labels = meta.get("labels", {}) or {}
        cls = 0
        if class_key is not None and class_key in labels:
            cls = classes.setdefault(labels[class_key], len(classes) + 1)
            if cls > 15:
                raise ValueError("more than 15 selector classes")
        sched = not spec.get("unschedulable", False)
        nodes["flags"][i] = (T.NODE_SCHEDULABLE if sched else 0) | (cls << T.NODE_CLASS_SHIFT)
        for l, key in enumerate(level_keys):
            if key in labels:
                nodes["dom"][i, l] = intern[l].setdefault(labels[key], len(intern[l]))
    return nodes, names, intern, classes


def _level(tc, level_keys, which="required"):
    key = (((tc or {}).get("packConstraint") or {}).get(which))
    if key is None:
        return None
    if key not in level_keys:
        raise ValueError(f"{which} topology key {key!r} is not a level of the cluster topology")
    return level_keys.index(key)


def _preferred(tc, level_keys):
    """packConstraint.preferred (podgang.go:110-117) as a level index; one that is not deeper than the
    required level adds nothing (best effort) and is dropped"""
    req, pref = _level(tc, level_keys), _level(tc, level_keys, "preferred")
    return None if pref is None or (req is not None and pref <= req) else pref


def podgangs_from_manifests(podgangs, requests, level_keys, priority_classes=None, class_mask=0xFFFF, base_of=None, placed_on=None):
    """PodGang manifests -> (gangs, cliques, scopes, clique_names) with clique_names[row] = (gang name, PodGroup name).

    Cliques of one TopologyConstraintGroupConfig are made adjacent (one scope each); PodGroups in no group form
    the implicit first scope.  base_of: optional {scaled gang name: base gang name} (gating, syncflow.go:319-358).
    placed_on: optional {PodGang name: node index} of earlier placements; spec.reuseReservationRef (podgang.go:66-71,
    a locality hint) resolves through it to the gang's anchor node.
    """
    b = T.GangTableBuilder()
    names, row_of = [], {pg["metadata"]["name"]: i for i, pg in enumerate(podgangs)}
    for pg in podgangs:
        spec = pg["spec"]
        groups = {g["name"]: g for g in spec["podgroups"]}
        grouped = [n for gc in spec.get("topologyConstraintGroupConfigs") or [] for n in gc["podGroupNames"]]
        scopes = []

        def clique(g):
            rq = requests.get(g["name"], {})
            names.append((pg["metadata"]["name"], g["name"]))
            return dict(cpu=parse_cpu_milli(rq.get("cpu", 0), request=True), mem=parse_mem_mib(rq.get("memory", 0), request=True),
                        gpu=int(rq.get("nvidia.com/gpu", 0)), min=int(g["minReplicas"]), replicas=len(g["podReferences"]),
                        level=_level(g.get("topologyConstraint"), level_keys),
                        preferred=_preferred(g.get("topologyConstraint"), level_keys), class_mask=class_mask)

        loose = [g for g in spec["podgroups"] if g["name"] not in grouped]
        if loose:
            scopes.append((None, [clique(g) for g in loose]))
        for gc in spec.get("topologyConstraintGroupConfigs") or []:
            scopes.append((_level(gc.get("topologyConstraint"), level_keys), [clique(groups[n]) for n in gc["podGroupNames"]],
                           _preferred(gc.get("topologyConstraint"), level_keys)))
        base = (base_of or {}).get(pg["metadata"]["name"])
        anchor = (placed_on or {}).get((spec.get("reuseReservationRef") or {}).get("name"))
        b.add_gang(scopes, level=_level(spec.get("topologyConstraint"), level_keys), anchor=anchor,
                   preferred=_preferred(spec.get("topologyConstraint"), level_keys),
                   priority=(priority_classes or {}).get(spec.get("priorityClassName", ""), 0),
                   base=row_of[base] if base in row_of else None)
    g, c, s = b.build()
    return g, c, s, names


# ------------------------------------------------------------------------------------------------
# The producer: PodCliqueSet -> PodGang manifests (the Python counterpart of ComputeExpectedPodGangs in
# grove_b200/csrc/host; ai-dynamo/grove operator/internal/controller/podcliqueset/components/podgang/syncflow.go:145-371,
# names from operator/api/common/namegen.go:70-117, PodGroups from .../podgang/podgang.go:165-186).
# ------------------------------------------------------------------------------------------------
def podgangs_from_pcs(pcs: dict, topology_levels, tas_enabled: bool = True):
    """PodCliqueSet (the compact dict of tests/golden/workloads.json: name, replicas, packDomain, cliques[],
    podCliqueScalingGroups[]) -> (PodGang manifests, requests by PodGroup name, {scaled gang: base gang}).

    topology_levels: ordered [(domain, node label key)], broadest first (ClusterTopology.spec.levels).
    Base PodGang per PCS replica = standalone cliques + PCSG replicas [0, minAvailable) (one
    TopologyConstraintGroupConfig per such replica when the PCSG has a constraint); a scaled PodGang per PCSG
    replica >= minAvailable, carrying the PCSG's constraint or else the PCS's.  Defaults as the webhooks set them:
    clique minAvailable = replicas, PCSG replicas = minAvailable = 1.
    """
    key_of = dict(topology_levels)

    def constraint(domain):  # createTopologyPackConstraint: unknown domain or TAS off -> no constraint; Required only
        if not tas_enabled or domain is None or domain not in key_of:
            return None
        return {"packConstraint": {"required": key_of[domain]}}

    ns = pcs.get("namespace", "default")
    cliques = {c["name"]: c for c in pcs["cliques"]}
    groups = pcs.get("podCliqueScalingGroups") or []
    grouped = {n for g in groups for n in g["cliqueNames"]}
    requests, base_of, gangs = {}, {}, []

    def podgroup(fqn, tmpl):
        c = cliques[tmpl]
        replicas = int(c.get("replicas") or 1)
        mn = c.get("minAvailable")
        requests[fqn] = dict(c.get("requests") or {})
        pg = dict(name=fqn, minReplicas=int(replicas if mn is None else mn),
                  podReferences=sorted(({"namespace": ns, "name": f"{fqn}-{i}"} for i in range(replicas)), key=lambda r: r["name"]))
        tc = constraint(c.get("packDomain"))
        if tc:
            pg["topologyConstraint"] = tc
        return pg

    def manifest(name, podgroups, tc, configs=()):
        spec = {"podgroups": podgroups}
        if tc:
            spec["topologyConstraint"] = tc
        if configs:
            spec["topologyConstraintGroupConfigs"] = list(configs)
        if pcs.get("priorityClassName"):
            spec["priorityClassName"] = pcs["priorityClassName"]
        return {"apiVersion": "scheduler.grove.io/v1alpha1", "kind": "PodGang", "metadata": {"name": name, "namespace": ns}, "spec": spec}

    for r in range(int(pcs.get("replicas") or 0)):
        pgs = [podgroup(f"{pcs['name']}-{r}-{c['name']}", c["name"]) for c in pcs["cliques"] if c["name"] not in grouped]
        configs = []
        for g in groups:
            fqn = f"{pcs['name']}-{r}-{g['name']}"
            for ri in range(int(g.get("minAvailable") or 1)):
                names = []
                for cn in g["cliqueNames"]:
                    if cn not in cliques:
                        raise ValueError(f"PodCliqueScalingGroup {g['name']!r} references a PodClique {cn!r} that does not exist in the PodCliqueSet")
                    pgs.append(podgroup(f"{fqn}-{ri}-{cn}", cn)); names.append(f"{fqn}-{ri}-{cn}")
                tc = constraint(g.get("packDomain"))
                if tas_enabled and g.get("packDomain") is not None:   # the config is emitted even when the domain went stale
                    configs.append({"name": f"{fqn}-{ri}", "podGroupNames": names, **({"topologyConstraint": tc} if tc else {})})
        gangs.append(manifest(f"{pcs['name']}-{r}", pgs, constraint(pcs.get("packDomain")), configs))
    for r in range(int(pcs.get("replicas") or 0)):
        for g in groups:
            fqn = f"{pcs['name']}-{r}-{g['name']}"
            replicas, mn = int(g.get("replicas") or 1), int(g.get("minAvailable") or 1)
            for idx, pr in enumerate(range(mn, replicas)):
                pgs = [podgroup(f"{fqn}-{pr}-{cn}", cn) for cn in g["cliqueNames"]]
                tc = constraint(g["packDomain"] if g.get("packDomain") is not None else pcs.get("packDomain"))
                name = f"{fqn}-{idx}"
                gangs.append(manifest(name, pgs, tc)); base_of[name] = f"{pcs['name']}-{r}"
    return gangs, requests, base_of


# ------------------------------------------------------------------------------------------------
# KAI queues (scheduling.run.ai/v2 Queue) -> the queue table of grove_set_queues (DESIGN.md section 1 "Queue limits").
# ------------------------------------------------------------------------------------------------
QUEUE_LABEL = "kai.scheduler/queue"


def podgroup_queues(podgangs, template_queue):
    """PodGroup name -> queue name (or None): the kai.scheduler/queue label of the PodClique template each PodGroup was stamped
    from.  template_queue: template name -> label value or None.  A PodGroup's name ends in "-<template name>"
    (namegen.go:70-117); the longest template name that matches wins."""
    names = sorted(template_queue, key=len, reverse=True)
    out = {}
    for pg in podgangs:
        for grp in pg["spec"]["podgroups"]:
            t = next((n for n in names if grp["name"].endswith("-" + n)), None)
            out[grp["name"]] = template_queue[t] if t is not None else None
    return out


MNNVL_CLAIM = "mnnvl-claim"   # the resource claim auto-MNNVL injects into an enrolled pod (operator/internal/mnnvl)


def compute_domains(podgangs, template_pod_spec, intern=None):
    """PodGroup name -> ComputeDomain id for grove_set_compute_domains (tables.CD_NONE when not enrolled): the
    resourceClaimTemplateName of the `mnnvl-claim` entry of the pod spec's resourceClaims, in the PodClique template each PodGroup
    was stamped from (matched as podgroup_queues does).  template_pod_spec: template name -> pod spec dict.  Names are interned in
    `intern` (name -> id, extended in place, new ids from len(intern)), so that a caller keeps ids stable across cycles."""
    intern = {} if intern is None else intern
    names = sorted(template_pod_spec, key=len, reverse=True)
    out = {}
    for pg in podgangs:
        for grp in pg["spec"]["podgroups"]:
            t = next((n for n in names if grp["name"].endswith("-" + n)), None)
            spec = template_pod_spec[t] if t is not None else None
            claims = (spec or {}).get("resourceClaims") or []
            tmpl = next((c.get("resourceClaimTemplateName") for c in claims if c.get("name") == MNNVL_CLAIM), None)
            if tmpl is None:
                out[grp["name"]] = T.CD_NONE
                continue
            out[grp["name"]] = intern.setdefault(tmpl, len(intern))
    return out


def _queue_limit(res, key, scale, field="limit"):
    lim = ((res or {}).get(key) or {}).get(field, -1)
    if lim is None or float(lim) < 0:
        return T.QUEUE_UNLIMITED
    return int(_quantity(lim) * scale)


def queues_from_manifests(queue_docs, podgangs, podgroup_queue, used=None):
    """Queue manifests + PodGang manifests -> (tables.queue_dt[n], gang_queue[G] uint32, queue names in table order).

    A Queue's spec.parentQueue names its parent; spec.resources.{cpu,memory,gpu}.limit is its hard limit, -1 (or absent) none.
    KAI's source is not part of the reference, so the units are this repository's assumption (INTEGRATION.md): cpu in cores
    (x 1000 -> millicores), memory in MiB, gpu in whole GPUs.  A PodGang's queue is the queue its PodGroups name
    (podgroup_queue: PodGroup name -> queue or None); PodGroups of one PodGang that name different queues are an error, a queue
    that is not among queue_docs makes the PodGang a non-member.  used: queue name -> (cpu milli, mem MiB, gpu) that its running
    PodGangs hold.  Parents come before their children in the table."""
    docs = {d["metadata"]["name"]: d for d in queue_docs if d and d.get("kind", "Queue") == "Queue"}
    parent = {n: (d.get("spec") or {}).get("parentQueue") or None for n, d in docs.items()}
    for n, p in parent.items():
        if p is not None and p not in docs:
            raise ValueError(f"Queue {n!r}: parent queue {p!r} does not exist")

    def depth(n, seen=()):
        if n in seen:
            raise ValueError(f"Queue {n!r} is its own ancestor")
        return 0 if parent[n] is None else 1 + depth(parent[n], seen + (n,))

    names = sorted(docs, key=lambda n: (depth(n), n))
    idx = {n: i for i, n in enumerate(names)}
    q = np.zeros(len(names), dtype=T.queue_dt)
    for n, i in idx.items():
        res = (docs[n].get("spec") or {}).get("resources")
        q["parent"][i] = T.NONE_U32 if parent[n] is None else idx[parent[n]]
        q["limit"][i] = [_queue_limit(res, "cpu", 1000), _queue_limit(res, "memory", 1), _queue_limit(res, "gpu", 1)]
        q["used"][i] = (used or {}).get(n, (0, 0, 0))
    gq = np.full(len(podgangs), T.NONE_U32, dtype=np.uint32)
    for g, pg in enumerate(podgangs):
        named = {podgroup_queue.get(grp["name"]) for grp in pg["spec"]["podgroups"]} - {None}
        if len(named) > 1:
            raise ValueError(f"PodGang {pg['metadata']['name']!r}: its PodGroups name different queues {sorted(named)}")
        if named and next(iter(named)) in idx:
            gq[g] = idx[next(iter(named))]
    return q, gq, names


def queue_quotas_from_manifests(queue_docs, names):
    """Queue manifests + the queue names in table order (as queues_from_manifests returns them) -> tables.queue_quota_dt[n] for
    grove_run_cycle_reclaim_queues.  spec.resources.{cpu,memory,gpu}.quota is the queue's deserved quota, -1 (or absent) none; the
    units are those of the limits (cpu in cores x 1000, memory in MiB, gpu in whole GPUs)."""
    docs = {d["metadata"]["name"]: d for d in queue_docs if d and d.get("kind", "Queue") == "Queue"}
    out = np.zeros(len(names), dtype=T.queue_quota_dt)
    for i, n in enumerate(names):
        res = (docs[n].get("spec") or {}).get("resources")
        out["deserved"][i] = [_queue_limit(res, "cpu", 1000, "quota"), _queue_limit(res, "memory", 1, "quota"),
                              _queue_limit(res, "gpu", 1, "quota")]
    return out


def queue_weights_from_manifests(queue_docs, names):
    """Queue manifests + the queue names in table order (as queues_from_manifests returns them) -> tables.queue_weight_dt[n] for
    grove_set_over_quota.  spec.resources.{cpu,memory,gpu}.overQuotaWeight is the queue's share of the capacity nobody deserves
    relative to its siblings; absent means 1, KAI's default.  A negative or fractional weight raises ValueError naming the queue."""
    docs = {d["metadata"]["name"]: d for d in queue_docs if d and d.get("kind", "Queue") == "Queue"}
    out = np.zeros(len(names), dtype=T.queue_weight_dt)
    for i, n in enumerate(names):
        res = (docs[n].get("spec") or {}).get("resources") or {}
        for r, key in enumerate(("cpu", "memory", "gpu")):
            w = (res.get(key) or {}).get("overQuotaWeight")
            if w is None:
                out["over_quota"][i, r] = 1
                continue
            try:
                x = _quantity(w)
            except (ValueError, ZeroDivisionError):
                x = Fraction(-1)
            if x < 0 or x.denominator != 1 or x >= 1 << 32:
                raise ValueError(f"Queue {n!r}: {key} overQuotaWeight {w!r} is not a whole number from 0 to 2^32 - 1")
            out["over_quota"][i, r] = int(x)
    return out


def tables_from_pcs(pcs: dict, topology_levels, tas_enabled: bool = True, class_mask=0xFFFF):
    """PodCliqueSet -> (gangs, cliques, scopes, clique_names, PodGang manifests): the producer, then the encoder."""
    gangs, requests, base_of = podgangs_from_pcs(pcs, topology_levels, tas_enabled)
    g, c, s, names = podgangs_from_manifests(gangs, requests, [k for _, k in topology_levels], class_mask=class_mask, base_of=base_of)
    return g, c, s, names, gangs


# ------------------------------------------------------------------------------------------------
# The way back: a cycle's outputs in the shapes the API objects carry them.
# ------------------------------------------------------------------------------------------------
def bindings(placements, podgangs, clique_names, node_names):
    """placement entries -> [(pod namespace, pod name, node name)]: the r-th entry of a clique binds the r-th
    PodReference of its PodGroup (podgang.go:75-91; sorted by name by the operator, podgang.go:175-177)."""
    refs = {(pg["metadata"]["name"], g["name"]): g["podReferences"] for pg in podgangs for g in pg["spec"]["podgroups"]}
    seen, out = {}, []
    for q, n in zip(placements["clique"].tolist(), placements["node"].tolist()):
        r = seen.get(q, 0); seen[q] = r + 1
        ref = refs[clique_names[q]][r]
        out.append((ref.get("namespace", "default"), ref["name"], node_names[n]))
    return out


def podgang_status(row) -> dict:
    """one grove_gang_status_t -> PodGang.status (podgang.go:141-190): phase, placementScore (1.0 = best), and the
    Scheduled condition with the reason a user sees on an unschedulable gang"""
    state = int(row["state"])
    reason = {T.GANG_ADMITTED: "Scheduled", T.GANG_REJECTED: "Unschedulable", T.GANG_BASE_REJECTED: "BaseNotScheduled",
              T.GANG_GATED_SKIP: "Gated"}.get(state, "Pending")
    st = {"phase": "Starting" if state == T.GANG_ADMITTED else "Pending",
          "conditions": [{"type": "Scheduled", "status": "True" if state == T.GANG_ADMITTED else "False", "reason": reason}]}
    if state == T.GANG_ADMITTED and int(row["score_den"]):
        st["placementScore"] = int(row["score_num"]) / int(row["score_den"])
    return st
