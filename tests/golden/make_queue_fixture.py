"""Extract the reference's KAI queues and the queue label of each PodClique template into a small JSON fixture.

    GROVE_REFERENCE=<checkout of ai-dynamo/grove @ 08ad3b37> python tests/golden/make_queue_fixture.py

tests/golden/queues.json holds `queues` (the Queue objects of operator/e2e/yaml/queues.yaml, as parsed) and `labels` (per
workload file of tests/golden/workloads.json, per PodCliqueSet, per PodClique template: its kai.scheduler/queue label or null).
workloads.json was extracted without labels; the YAML itself is not copied.
"""
import json
import os

import yaml

REF = os.path.join(os.environ["GROVE_REFERENCE"], "operator")
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    queues = [d for d in yaml.safe_load_all(open(os.path.join(REF, "e2e/yaml/queues.yaml"))) if d and d.get("kind") == "Queue"]
    labels = {}
    for f in sorted(json.load(open(os.path.join(HERE, "workloads.json")))):
        per = {}
        for doc in yaml.safe_load_all(open(os.path.join(REF, f))):
            if not doc or doc.get("kind") != "PodCliqueSet":
                continue
            per[doc["metadata"]["name"]] = {c["name"]: ((c.get("labels") or {}).get("kai.scheduler/queue"))
                                            for c in doc["spec"]["template"]["cliques"]}
        labels[f] = per
    with open(os.path.join(HERE, "queues.json"), "w") as fh:
        json.dump(dict(queues=queues, labels=labels), fh, indent=1, sort_keys=True)
    print(len(queues), "queues,", sum(len(v) for v in labels.values()), "PodCliqueSets")


if __name__ == "__main__":
    main()
