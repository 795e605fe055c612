"""The diagnosis of rejected gangs (DESIGN.md section 1 "Diagnosis"), on the CPU: the state V_g each gang is judged against is
the table the sequential pass evaluated it against (re-running the unchanged oracle on V_g reproduces the gang's fate), the
restatement's counts agree with the oracle's K1 fit rows and with their own definition, and a hand case per failure predicate
and per verdict."""
import numpy as np
import pytest

from grove_b200 import tables as T
from oracle import oracle_py
import diagnose_cases as D
from test_random_parity_gpu import random_case


def one_gang(view, L, gangs, cliques, scopes, g, perm, want_matrices=False):
    """gang g alone on the node table `view`, with the anchor the cycle derived for it and no base gang"""
    sg = gangs[g: g + 1].copy()
    co, so = int(sg["clique_off"][0]), int(sg["scope_off"][0])
    sq = cliques[co: co + int(sg["n_cliques"][0])].copy()
    ss = scopes[so: so + int(sg["n_scopes"][0])].copy()
    if sg["anchor_node"][0] == T.NONE_U32:
        sg["anchor_node"][0] = perm[oracle_py._fmix32(g) % len(view)]
    sg["base_gang"][0] = T.NONE_U32
    sg["clique_off"][0] = 0
    sg["scope_off"][0] = 0
    return oracle_py.run_cycle(view, L, sg, sq, ss, want_matrices=want_matrices), co


def _popcount(words):
    return int(np.unpackbits(np.ascontiguousarray(words).view(np.uint8)).sum())


def _cases():
    for seed in range(48):
        nodes, L, tables = random_case(31000 + seed, pref=seed % 2 == 1)
        yield seed, nodes, L, tables


@pytest.mark.parametrize("seed,nodes,L,tables", list(_cases()), ids=lambda x: str(x) if isinstance(x, int) else "")
def test_view_reproduces_each_gang(seed, nodes, L, tables):
    g_, c_, s_ = tables
    out = oracle_py.run_cycle(nodes, L, g_, c_, s_)
    gd, qd = D.diagnose(nodes, L, g_, c_, s_, c_["min_replicas"], out)
    n = len(nodes)
    for g, view in D.views(nodes, g_, c_, out):
        one, co = one_gang(view, L, g_, c_, s_, g, out["perm"], want_matrices=True)
        st = out["status"][g]
        assert one["status"]["state"][0] == st["state"], g
        if st["state"] == T.GANG_ADMITTED:
            mine = out["placements"][int(st["placement_off"]): int(st["placement_off"]) + int(st["n_pods"])].copy()
            got = one["placements"].copy()
            got["clique"] += co
            assert np.array_equal(got, mine), g
            assert gd[g]["verdict"] == T.DIAG_NONE and not qd[co: co + int(g_["n_cliques"][g])]["nodes_fit"].any()
            continue
        recs = qd[co: co + int(g_["n_cliques"][g])]
        for c, rec in enumerate(recs):
            assert int(rec["nodes_fit"]) == _popcount(one["fit"][c]), (g, c)   # K1 of the oracle on V_g
            assert int(rec["nodes_fit"]) + sum(int(rec[f]) for f in T.DIAG_FAILURES) == n
            assert rec["pods_fit"] >= rec["nodes_fit"]
        short = [c for c in range(len(recs)) if int(recs["pods_fit"][c]) < int(c_["min_replicas"][co + c])]
        assert (gd[g]["verdict"] == T.DIAG_CLIQUE_SHORT) == bool(short)
        if short:
            assert gd[g]["clique"] == short[0]
        if gd[g]["verdict"] == T.DIAG_NO_DOMAIN:
            assert g_["level"][g] != T.LEVEL_NONE and gd[g]["domains_ok"] == 0
        assert gd[g]["domains_ok"] <= gd[g]["domains"]
    for g in range(len(g_)):
        if out["status"]["state"][g] != T.GANG_REJECTED:
            assert gd[g].tobytes() == bytes(T.gang_diag_dt.itemsize)


# ---- hand cases ------------------------------------------------------------------------------------------------------
def _nodes(n, blocks=1, gpu=4, pods=110):
    nodes = T.make_nodes(n)
    nodes["free_cpu_milli"], nodes["free_mem_mib"], nodes["free_gpu"], nodes["free_pods"] = 8000, 65536, gpu, pods
    nodes["flags"] = T.NODE_SCHEDULABLE
    nodes["dom"][:, 0] = np.arange(n) * blocks // n
    nodes["dom"][:, 1] = np.arange(n)
    return nodes


def _diag(nodes, b, L=2):
    g, c, s = b.build()
    out = oracle_py.run_cycle(nodes, L, g, c, s)
    gd, qd = D.diagnose(nodes, L, g, c, s, c["min_replicas"], out)
    return out, gd, qd


def _spoil(nodes, i, what):
    if what == "unschedulable":
        nodes["flags"][i] = 0
        nodes["free_cpu_milli"][i] = 0   # fails cpu too: counted under the first predicate only
    elif what == "selector":
        nodes["flags"][i] |= 2 << T.NODE_CLASS_SHIFT
    elif what == "labels":
        nodes["dom"][i, 1] = T.DOM_ABSENT
    elif what == "cpu":
        nodes["free_cpu_milli"][i] = 999
    elif what == "mem":
        nodes["free_mem_mib"][i] = 100
    elif what == "gpu":
        nodes["free_gpu"][i] = 0
    elif what == "pods":
        nodes["free_pods"][i] = 0


@pytest.mark.parametrize("what", T.DIAG_FAILURES)
def test_each_failure_predicate(what):
    nodes = _nodes(6)
    for i in (1, 4):
        _spoil(nodes, i, what)
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(cpu=1000, mem=1024, gpu=1, min=20, class_mask=0b1, level=1)])])
    out, gd, qd = _diag(nodes, b)
    assert out["status"]["state"][0] == T.GANG_REJECTED
    assert qd[0]["nodes_fit"] == 4 and qd[0][what] == 2
    assert sum(int(qd[0][f]) for f in T.DIAG_FAILURES) == 2
    assert qd[0]["pods_fit"] == 16   # 4 gpus on each of the 4 nodes that fit
    assert gd[0]["verdict"] == T.DIAG_CLIQUE_SHORT and gd[0]["clique"] == 0 and gd[0]["level"] == T.LEVEL_NONE
    assert gd[0]["domains"] == 1 and gd[0]["domains_ok"] == 0


def test_no_domain():
    """8 gpus in the cluster, 4 per block: a gang that wants 6 in one block"""
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(gpu=1, min=6)])], level=0)
    out, gd, qd = _diag(_nodes(4, blocks=2, gpu=2), b)
    assert out["status"]["state"][0] == T.GANG_REJECTED
    assert qd[0]["pods_fit"] == 8 and qd[0]["nodes_fit"] == 4
    assert (gd[0]["verdict"], gd[0]["level"], gd[0]["domains"], gd[0]["domains_ok"]) == (T.DIAG_NO_DOMAIN, 0, 2, 0)


def test_no_joint_fit():
    """two PodGroups of 3 gpus each, blocks of 4: each fits a block alone, both together fit none"""
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(gpu=1, min=3), dict(gpu=1, min=3)])], level=0)
    out, gd, qd = _diag(_nodes(4, blocks=2, gpu=2), b)
    assert out["status"]["state"][0] == T.GANG_REJECTED
    assert (gd[0]["verdict"], gd[0]["domains"], gd[0]["domains_ok"]) == (T.DIAG_NO_JOINT_FIT, 2, 2)
    assert list(qd["pods_fit"]) == [8, 8]


def test_no_joint_fit_without_a_required_level():
    """a scope's Required level the gang itself does not have: every PodGroup fits the cluster, no rack holds the scope"""
    b = T.GangTableBuilder()
    b.add_gang([(1, [dict(gpu=1, min=2), dict(gpu=1, min=2)])])
    out, gd, qd = _diag(_nodes(4, blocks=2, gpu=2), b)
    assert out["status"]["state"][0] == T.GANG_REJECTED
    assert (gd[0]["verdict"], gd[0]["level"], gd[0]["domains"], gd[0]["domains_ok"]) == (T.DIAG_NO_JOINT_FIT, T.LEVEL_NONE, 1, 1)


def test_view_gives_back_what_later_gangs_took():
    """A (first) takes 3 of block 0's 4 gpus, B (second) wants 6 in one block, C (last) takes block 1: at B's turn block 1 was
    still free, so 1 + 4 gpus fit -- not the 1 the final table shows, nor the 8 of the snapshot"""
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(gpu=1, min=3)])], level=0, priority=2, anchor=0)
    b.add_gang([(None, [dict(gpu=1, min=6)])], level=0, priority=1)
    b.add_gang([(None, [dict(gpu=1, min=4)])], level=0, priority=0, anchor=3)
    out, gd, qd = _diag(_nodes(4, blocks=2, gpu=2), b)
    assert list(out["status"]["state"]) == [T.GANG_ADMITTED, T.GANG_REJECTED, T.GANG_ADMITTED]
    assert qd[1]["pods_fit"] == 5 and qd[1]["nodes_fit"] == 3
    assert gd[1]["verdict"] == T.DIAG_CLIQUE_SHORT and gd[1]["domains_ok"] == 0
    assert gd[0].tobytes() == gd[2].tobytes() == bytes(16) and not qd[[0, 2]].tobytes().strip(b"\0")


def test_wide_submission():
    """16-bit MinReplicas: 300 pods on blocks of 2 x 110 pod slots; the whole cluster holds 440"""
    import wide_oracle as W
    b = T.GangTableBuilder()
    b.add_gang([(None, [dict(mem=64, min=300)])], level=0)
    b.add_gang([(None, [dict(mem=64, min=500)])])
    g, c, cnt, s = b.build_wide()
    nodes = _nodes(4, blocks=2)
    out = W.run_cycle_wide(nodes, 2, g, c, cnt, s)
    assert list(out["status"]["state"]) == [T.GANG_REJECTED, T.GANG_REJECTED]
    gd, qd = D.diagnose(nodes, 2, g, c, s, cnt["min_replicas"], out)
    assert list(qd["pods_fit"]) == [440, 440]
    assert (gd[0]["verdict"], gd[0]["domains"], gd[0]["domains_ok"]) == (T.DIAG_NO_DOMAIN, 2, 0)
    assert (gd[1]["verdict"], gd[1]["clique"]) == (T.DIAG_CLIQUE_SHORT, 0)


def test_record_layouts_match_header(tmp_path):
    """sizeof / offsetof of grove_gang_diag_t and grove_clique_diag_t against the numpy dtypes"""
    import subprocess
    from test_abi import HEADER
    fields = {"grove_gang_diag_t": T.gang_diag_dt, "grove_clique_diag_t": T.clique_diag_dt}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void){"]
    for name, dt in fields.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f in dt.names]
    lines.append("return 0;}")
    (tmp_path / "probe.c").write_text("\n".join(lines))
    subprocess.check_call(["gcc", "-std=c11", "-o", str(tmp_path / "probe"), str(tmp_path / "probe.c")])
    got = dict(l.split() for l in subprocess.check_output([str(tmp_path / "probe")], text=True).splitlines())
    for name, dt in fields.items():
        assert int(got[name]) == dt.itemsize, name
        for f in dt.names:
            assert int(got[f"{name}.{f}"]) == dt.fields[f][1], f"{name}.{f}"
