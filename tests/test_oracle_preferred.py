"""Preferred pack levels (ai-dynamo/grove scheduler/api/core/v1alpha1/podgang.go:110-117): "best-effort
topology constraint ... not binding on the scheduler ... Scheduler can fall back to higher topology levels
(upto Required constraint) if preferred cannot be satisfied."  The operator never populates the field
(syncflow.go:366-368 sets Required only) and no reference test exercises it, so these properties restate
the API comment on the e2e cluster shape (150 MiB nodes, 7 hosts per rack, 14 per block, 28 per zone)."""
import numpy as np
import pytest

from grove_b200 import synth, tables as T

A = synth.AGENT
ZONE, BLOCK, RACK, HOST = 0, 1, 2, 3


def run(oracle, nodes, b, **kw):
    g, c, s = b.build()
    return oracle.run_cycle(nodes, synth.E2E_LEVELS, g, c, s, **kw), (g, c, s)


def clq(n, mem=40, **kw):
    return dict(mem=mem, min=n, class_mask=A, **kw)


def doms(nodes, pl, level):
    return set(int(nodes["dom"][int(n), level]) for n in pl["node"])


def test_preferred_level_is_honoured_when_it_fits(oracle):
    nodes = synth.e2e_cluster(56)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(10), clq(8)])], preferred=RACK)   # 18 pods, a rack holds 21
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and len(r["placements"]) == 18
    assert len(doms(nodes, r["placements"], RACK)) == 1


def test_preferred_falls_back_one_level_at_a_time(oracle):
    nodes = synth.e2e_cluster(56)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(15), clq(15)])], preferred=RACK)  # 30 pods: no rack (21), a block (42)
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    assert len(doms(nodes, r["placements"], RACK)) == 2 and len(doms(nodes, r["placements"], BLOCK)) == 1
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(25), clq(25)])], preferred=RACK)  # 50 pods: no block (42), a zone (84)
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    assert len(doms(nodes, r["placements"], BLOCK)) == 2 and len(doms(nodes, r["placements"], ZONE)) == 1
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(50), clq(50)])], preferred=RACK)  # 100 pods: not even a zone
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and len(r["placements"]) == 100
    assert len(doms(nodes, r["placements"], ZONE)) == 2


def test_required_bounds_the_fallback(oracle):
    nodes = synth.e2e_cluster(56)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(15), clq(15)])], level=BLOCK, preferred=RACK)
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED and len(doms(nodes, r["placements"], BLOCK)) == 1
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(25), clq(25)])], level=BLOCK, preferred=RACK)  # 50 pods > a block
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_REJECTED and len(r["placements"]) == 0
    assert np.array_equal(r["nodes_after"], nodes)


def test_another_domain_of_the_preferred_level_beats_widening(oracle):
    """The anchor's rack is nearly full; a farther rack that fits the gang is taken before any block."""
    nodes = synth.e2e_cluster(28)
    nodes["free_mem_mib"][0:7] = 30   # rack 0: nothing of 40 MiB fits
    nodes["free_mem_mib"][7:12] = 30  # rack 1: 2 hosts left = 6 pods
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(10)])], preferred=RACK, anchor=0)
    r, _ = run(oracle, nodes, b)
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    assert doms(nodes, r["placements"], RACK) == {int(nodes["dom"][14, RACK])}


def test_clique_and_scope_preferred_levels(oracle):
    nodes = synth.e2e_cluster(28)
    b = T.GangTableBuilder()
    b.add_gang([(None, [clq(3, preferred=HOST), clq(4, preferred=HOST)]),     # 3 fit one host, 4 do not
                (None, [clq(6), clq(6)], RACK),                                # scope prefers a rack: 12 <= 21
                (BLOCK, [clq(12), clq(12)], RACK)])                            # 24 > 21: widen to the Required block
    r, tabs = run(oracle, nodes, b)
    g = tabs[0]
    assert r["status"]["state"][0] == T.GANG_ADMITTED
    pl = r["placements"]
    by = lambda c: pl[pl["clique"] == g["clique_off"][0] + c]
    assert len(set(by(0)["node"])) == 1
    assert len(set(by(1)["node"])) == 2
    s1 = np.concatenate([by(2), by(3)]); s2 = np.concatenate([by(4), by(5)])
    assert len(doms(nodes, s1, RACK)) == 1
    assert len(doms(nodes, s2, RACK)) == 2 and len(doms(nodes, s2, BLOCK)) == 1


def test_preferred_never_costs_admission(oracle):
    """Best effort: whatever is admitted without the Preferred level is admitted with it."""
    rng = np.random.default_rng(7)
    for _ in range(20):
        nodes = synth.e2e_cluster(56)
        nodes["free_mem_mib"] = rng.integers(0, 151, size=56)
        n1, n2 = int(rng.integers(1, 30)), int(rng.integers(1, 30))
        req = [None, ZONE, BLOCK][int(rng.integers(0, 3))]
        states = []
        for pref in (None, RACK, HOST):
            b = T.GangTableBuilder(); b.add_gang([(None, [clq(n1), clq(n2)])], level=req, preferred=pref, anchor=3)
            r, _ = run(oracle, nodes, b)
            states.append(int(r["status"]["state"][0]))
        assert states[0] == states[1] == states[2]


def test_preferred_must_be_deeper_than_required(oracle):
    nodes = synth.e2e_cluster(14)
    for kw in (dict(level=RACK, preferred=RACK), dict(level=RACK, preferred=BLOCK), dict(preferred=7)):
        b = T.GangTableBuilder(); b.add_gang([(None, [clq(1)])], **kw)
        with pytest.raises(Exception):
            run(oracle, nodes, b)
    b = T.GangTableBuilder(); b.add_gang([(RACK, [clq(1)], BLOCK)])
    with pytest.raises(Exception):
        run(oracle, nodes, b)
    b = T.GangTableBuilder(); b.add_gang([(None, [clq(1, level=RACK, preferred=RACK)])])
    with pytest.raises(Exception):
        run(oracle, nodes, b)
