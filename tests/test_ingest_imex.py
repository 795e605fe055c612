"""-m "not gpu": the ComputeDomain of each PodGroup, read from the `mnnvl-claim` entry auto-MNNVL puts into its PodClique
template's pod spec."""
from grove_b200 import ingest, tables as T


def _pg(name, groups):
    return {"metadata": {"name": name}, "spec": {"podgroups": [{"name": g} for g in groups]}}


def test_compute_domains_interns_the_claim_template():
    worker = {"containers": [{"name": "w"}], "resourceClaims": [{"name": "mnnvl-claim", "resourceClaimTemplateName": "pcs-0"}]}
    worker1 = {"containers": [{"name": "w"}], "resourceClaims": [{"name": "mnnvl-claim", "resourceClaimTemplateName": "pcs-1"}]}
    frontend = {"containers": [{"name": "f"}], "resourceClaims": [{"name": "other", "resourceClaimTemplateName": "x"}]}
    gangs = [_pg("pcs-0", ["pcs-0-frontend", "pcs-0-worker"]), _pg("pcs-1", ["pcs-1-worker1"])]
    intern = {"older": 0}
    got = ingest.compute_domains(gangs, {"frontend": frontend, "worker": worker, "worker1": worker1}, intern)
    assert got == {"pcs-0-frontend": T.CD_NONE, "pcs-0-worker": 1, "pcs-1-worker1": 2}
    assert intern == {"older": 0, "pcs-0": 1, "pcs-1": 2}
    # ids stay put across cycles
    again = ingest.compute_domains(gangs, {"frontend": frontend, "worker": worker, "worker1": worker1}, intern)
    assert again == got


def test_podgroup_without_a_template_is_not_enrolled():
    assert ingest.compute_domains([_pg("a", ["a-x"])], {}) == {"a-x": T.CD_NONE}
