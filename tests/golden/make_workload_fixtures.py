"""Extract the PodCliqueSets of the reference's e2e / sample workloads into a small JSON fixture.

    GROVE_REFERENCE=<checkout of ai-dynamo/grove @ 08ad3b37> python tests/golden/make_workload_fixtures.py

Only the fields a scheduler's input depends on are kept: per clique name / replicas / minAvailable / resource
requests / node selector + tolerations (as a flag) / packDomain; per PodCliqueScalingGroup name / cliqueNames /
replicas / minAvailable / packDomain; the PodCliqueSet's replicas and packDomain.  The output
(tests/golden/workloads.json) pins the synthetic workload shapes (grove_b200/synth.py) and drives
tests/test_workload_fixtures.py; the YAML itself is not copied.
"""
import glob
import json
import os

import yaml

REF = os.path.join(os.environ["GROVE_REFERENCE"], "operator")
HERE = os.path.dirname(os.path.abspath(__file__))


def domain(tc):
    return (tc or {}).get("packDomain")


def extract(path):
    out = []
    for doc in yaml.safe_load_all(open(path)):
        if not doc or doc.get("kind") != "PodCliqueSet":
            continue
        t = doc["spec"]["template"]
        cliques = []
        for c in t["cliques"]:
            sp = c["spec"]
            pod = sp["podSpec"]
            req = {}
            for cont in pod.get("containers", []):
                for k, v in ((cont.get("resources") or {}).get("requests") or {}).items():
                    req[k] = str(v)
            cliques.append(dict(name=c["name"], replicas=sp.get("replicas"), minAvailable=sp.get("minAvailable"), requests=req,
                                agentOnly=bool(pod.get("affinity") or pod.get("nodeSelector")), tolerations=len(pod.get("tolerations") or []),
                                schedulerName=pod.get("schedulerName"), packDomain=domain(c.get("topologyConstraint"))))
        groups = [dict(name=g["name"], cliqueNames=g["cliqueNames"], replicas=g.get("replicas"), minAvailable=g.get("minAvailable"),
                       packDomain=domain(g.get("topologyConstraint"))) for g in (t.get("podCliqueScalingGroups") or [])]
        out.append(dict(name=doc["metadata"]["name"], replicas=doc["spec"].get("replicas", 1), packDomain=domain(t.get("topologyConstraint")),
                        priorityClassName=t.get("priorityClassName"), cliques=cliques, podCliqueScalingGroups=groups))
    return out


def main():
    files = sorted(glob.glob(os.path.join(REF, "e2e/yaml/workload[0-9].yaml")) + glob.glob(os.path.join(REF, "e2e/yaml/tas-*.yaml"))
                   + [os.path.join(REF, "samples/simple/simple1.yaml")])
    fx = {}
    for f in files:
        pcs = extract(f)
        if pcs:
            fx[os.path.relpath(f, REF)] = pcs
    with open(os.path.join(HERE, "workloads.json"), "w") as fh:
        json.dump(fx, fh, indent=1, sort_keys=True)
    print(len(fx), "files,", sum(len(v) for v in fx.values()), "PodCliqueSets")


if __name__ == "__main__":
    main()
