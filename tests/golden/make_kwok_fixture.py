"""Generates tests/golden/kwok_nodes_60.json by RUNNING the reference's own KWOK node generator
(ai-dynamo/grove operator/hack/infra_manager/kwok.py: topology_labels :55-71, node_manifest :74-117).  The reference package imports `sh` (a CLI helper, not installed and not needed by
the two pure functions used here); it is stubbed for the import only -- nothing of the reference
is modified or copied.  The tests read the fixture; they never need the reference.

    GROVE_REFERENCE=<checkout of ai-dynamo/grove @ 08ad3b37> python tests/golden/make_kwok_fixture.py
"""
import json
import os
import sys
import types

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.environ["GROVE_REFERENCE"], "operator", "hack")


def main():
    sys.modules.setdefault("sh", types.ModuleType("sh"))
    sys.path.insert(0, REF)
    from infra_manager import constants, kwok  # noqa: E402
    from infra_manager.config import KwokConfig  # noqa: E402

    cfg = KwokConfig(nodes=60)  # reference defaults: cpu 64, memory 512Gi, pods 110 (constants.py:195-197)
    out = {
        "generator": "infra_manager.kwok.node_manifest @ ai-dynamo/grove 08ad3b37",
        "nodes_per": {"zone": constants.NODES_PER_ZONE, "block": constants.NODES_PER_BLOCK, "rack": constants.NODES_PER_RACK},
        "label_keys": {"zone": constants.LABEL_ZONE, "block": constants.LABEL_BLOCK, "rack": constants.LABEL_RACK,
                       "host": constants.LABEL_HOSTNAME},
        "e2e_preset": {"node_cpu": "4", "node_memory": "150Mi"},  # hack/e2e.yaml
        "manifests": [kwok.node_manifest(i, cfg) for i in range(60)],
        "manifests_e2e": [kwok.node_manifest(i, KwokConfig(nodes=30, node_cpu="4", node_memory="150Mi")) for i in range(30)],
    }
    with open(os.path.join(HERE, "kwok_nodes_60.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print("wrote", len(out["manifests"]), "+", len(out["manifests_e2e"]), "manifests; first labels:", out["manifests"][0]["metadata"]["labels"])


if __name__ == "__main__":
    main()
