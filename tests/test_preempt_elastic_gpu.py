"""grove_run_cycle_preempt_elastic held to its one-at-a-time statement (tests/elastic_cases.py run_cycle_preempt_elastic) on every
output, flags included: the hand cases, random churned clusters whose running gangs carry surplus pods, narrow relaxation windows
and the tuning knobs; the degenerate case against grove_run_cycle_preempt; both skip rules; and the refusals."""
import os
import subprocess

import numpy as np
import pytest

from elastic_cases import elastic_cluster, hand_case, run_cycle_preempt_elastic
from grove_b200 import tables as T
from preempt_cases import churned_cluster

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_KEYS = ("status", "placements", "scope_status", "nodes_after", "victims", "surplus_victims")


def _run(e, nodes, tabs, running, holdings, surplus):
    e.load_nodes(nodes); e.submit_gangs(*tabs)
    e.run_cycle_preempt_elastic(running, holdings, surplus)
    return dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                victims=e.victims(), surplus_victims=e.surplus_victims())


def _same(got, ref, keys=_KEYS):
    for k in keys:
        assert np.array_equal(got[k], ref[k]), k


@pytest.mark.parametrize("p_gpu,b_priority", [(4, 0), (8, 0), (4, 3)])
def test_hand_cases(built_lib, oracle, p_gpu, b_priority):
    from grove_b200.engine import PlacementEngine
    nodes, L, tabs, running, holdings, surplus = hand_case(p_gpu, b_priority)
    ref = run_cycle_preempt_elastic(oracle, nodes, L, *tabs, running, holdings, surplus)
    with PlacementEngine(L) as e:
        got = _run(e, nodes, tabs, running, holdings, surplus)
        _same(got, ref)
        if p_gpu == 4:
            assert got["status"]["reserved0"][0] == T.STATUS_PREEMPTOR | T.STATUS_SURPLUS_ONLY
            assert len(got["victims"]) == 0 and [tuple(v) for v in got["surplus_victims"]] == [(0, 0)]
        else:
            e.load_nodes(nodes); e.submit_gangs(*tabs)
            e.run_cycle_preempt(running, holdings)
            assert np.array_equal(e.victims(), got["victims"]) and len(got["victims"]) == 1
            assert np.array_equal(e.gang_status(), got["status"]) and len(got["surplus_victims"]) == 0


def test_random_churned_clusters(built_lib, oracle):
    """100 churned clusters whose running worker cliques carry 1-3 surplus pods each"""
    from grove_b200.engine import PlacementEngine
    seen = np.zeros(3, dtype=np.int64)   # surplus preemptors, whole victims, surplus victims
    for seed in range(100):
        nodes, L, tabs, running, holdings, surplus = elastic_cluster(oracle, 1000 + seed, n=504, g_running=160, g_pending=60,
                                                                     share=0.8)
        ref = run_cycle_preempt_elastic(oracle, nodes, L, *tabs, running, holdings, surplus)
        with PlacementEngine(L) as e:
            _same(_run(e, nodes, tabs, running, holdings, surplus), ref)
        seen += [int(((ref["status"]["reserved0"] & T.STATUS_SURPLUS_ONLY) != 0).sum()), len(ref["victims"]),
                 len(ref["surplus_victims"])]
    assert (seen > 0).all(), seen


_CHURNED = {}


@pytest.mark.parametrize("window,knob", [(1, None), (7, None), (0, "GROVE_TUNE_REFRESH"), (0, "GROVE_TUNE_EVAL_CTAS")])
def test_windows_and_knobs(built_lib, oracle, monkeypatch, window, knob):
    """narrow relaxation windows; a capacity-table rebuild every round; one K3 CTA"""
    from grove_b200.engine import PlacementEngine
    if knob:
        monkeypatch.setenv(knob, "1")
    if not _CHURNED:
        case = elastic_cluster(oracle, 11, g_pending=100)
        ref = run_cycle_preempt_elastic(oracle, *case[:2], *case[2], *case[3:])
        assert (ref["status"]["reserved0"] & T.STATUS_SURPLUS_ONLY).any() and len(ref["surplus_victims"])
        _CHURNED.update(case=case, ref=ref)
    nodes, L, tabs, running, holdings, surplus = _CHURNED["case"]
    with PlacementEngine(L, window=window) as e:
        _same(_run(e, nodes, tabs, running, holdings, surplus), _CHURNED["ref"])


@pytest.mark.parametrize("seed", [15, 23, 31])
def test_no_surplus_is_the_reclaim_pass(built_lib, oracle, seed):
    """n_surplus == 0: every output equals grove_run_cycle_preempt's, the victims included"""
    from grove_b200.engine import PlacementEngine
    nodes, L, tabs, running, holdings = churned_cluster(oracle, seed, g_pending=100)
    none = np.zeros(0, dtype=T.surplus_pod_dt)
    with PlacementEngine(L) as e:
        got = _run(e, nodes, tabs, running, holdings, none)
        e.load_nodes(nodes); e.submit_gangs(*tabs)
        e.run_cycle_preempt(running, holdings)
        ref = dict(status=e.gang_status(), placements=e.placements(), scope_status=e.scope_domains(), nodes_after=e.nodes(),
                   victims=e.victims(), surplus_victims=e.surplus_victims())
    assert len(ref["victims"]) > 0
    _same(got, ref)


def _full(n, spread=False):
    """n 8-GPU nodes, nothing free.  Running gangs of priority 0 hold two 4-GPU pods on each node, MinReplicas 1 per node: one gang
    per node, or with spread one gang over all of them.  The second pod on every node is surplus; with spread only the last one."""
    from grove_b200 import synth
    nodes = synth.kwok_nodes(n, [n, n, 1, 1], gpu=8)
    nodes["free_gpu"] = 0; nodes["free_pods"] = 108
    k = 1 if spread else n
    running = np.zeros(k, dtype=T.running_dt)
    running["holding_off"] = np.arange(k) * (n // k); running["n_holdings"] = n // k
    holdings = np.zeros(n, dtype=T.holding_dt)
    holdings["node"] = np.arange(n); holdings["gpu"] = 8; holdings["pods"] = 2
    surplus = np.zeros(1 if spread else n, dtype=T.surplus_pod_dt)
    surplus["running"] = 0 if spread else np.arange(n); surplus["node"] = np.arange(n)[-len(surplus):]; surplus["gpu"] = 4
    return nodes, running, holdings, surplus


def _gangs(*gpus, priority=5):
    b = T.GangTableBuilder()
    for x in gpus:
        b.add_gang([(None, [dict(gpu=x, min=1)])], priority=priority)
    return b.build()


def test_surplus_runs_out(built_lib, oracle):
    """ten 2-GPU preemptors over four 4-GPU surplus pods: the pass-1 class cycle admits eight; the last of them meets no untaken
    surplus pod at its turn (2 GPUs are still free where a pod was taken), gives its room back and goes on to pass 2 with the two
    the class cycle rejected"""
    from grove_b200.engine import PlacementEngine
    nodes, running, holdings, surplus = _full(4)
    tabs = _gangs(*[2] * 10)
    ref = run_cycle_preempt_elastic(oracle, nodes, 4, *tabs, running, holdings, surplus)
    only = (ref["status"]["reserved0"] & T.STATUS_SURPLUS_ONLY) != 0
    assert only.sum() == 7 and not only[7:].any() and len(ref["surplus_victims"]) == 4
    assert (ref["status"]["state"] == T.GANG_ADMITTED).all()
    with PlacementEngine(4) as e:
        _same(_run(e, nodes, tabs, running, holdings, surplus), ref)


def test_gangs_run_out(built_lib, oracle):
    """two 8-GPU preemptors against one running gang over two nodes: pass 1 admits neither; the pass-2 class cycle admits both,
    but the first evicts the gang whole, and the second meets E(p) empty at its turn and stays REJECTED"""
    from grove_b200.engine import PlacementEngine
    nodes, running, holdings, surplus = _full(2, spread=True)
    tabs = _gangs(8, 8)
    ref = run_cycle_preempt_elastic(oracle, nodes, 4, *tabs, running, holdings, surplus)
    assert list(ref["status"]["state"]) == [T.GANG_ADMITTED, T.GANG_REJECTED]
    assert len(ref["victims"]) == 1 and len(ref["surplus_victims"]) == 0
    with PlacementEngine(4) as e:
        _same(_run(e, nodes, tabs, running, holdings, surplus), ref)


def test_refusals(built_lib, oracle):
    from grove_b200.engine import GroveError, PlacementEngine
    nodes, L, tabs, running, holdings, surplus = hand_case(4)
    bad_run = surplus.copy(); bad_run["running"] = 2
    bad_node = surplus.copy(); bad_node["node"] = 2
    not_held = surplus.copy(); not_held["node"] = 0   # B holds nothing on n0
    too_many = np.concatenate([surplus, surplus, surplus])   # 3 pods where B holds 2
    too_big = surplus.copy(); too_big["gpu"] = 9
    too_much_mem = surplus.copy(); too_much_mem["mem_mib"] = 1
    cases = [(bad_run, "out of range"), (bad_node, "out of range"), (not_held, "exceed"), (too_many, "exceed"),
             (too_big, "exceed"), (too_much_mem, "exceed")]
    ref = oracle.run_cycle(nodes, L, *tabs)
    with PlacementEngine(L) as e:
        e.load_nodes(nodes); e.submit_gangs(*tabs)
        with pytest.raises(GroveError) as ei:
            e.surplus_victims()
        assert ei.value.code == -5   # no cycle yet
        for sp, why in cases:
            with pytest.raises(GroveError) as ei:
                e.run_cycle_preempt_elastic(running, holdings, sp)
            assert ei.value.code == -1 and why in str(ei.value), (why, str(ei.value))
            e.run_cycle()   # the handle is untouched
            assert np.array_equal(e.gang_status(), ref["status"]) and np.array_equal(e.nodes(), ref["nodes_after"])
            assert len(e.surplus_victims()) == 0
        # malformed running inputs, as grove_run_cycle_preempt refuses them
        bad = running.copy(); bad["n_holdings"][1] = 3
        with pytest.raises(GroveError) as ei:
            e.run_cycle_preempt_elastic(bad, holdings, surplus)
        assert ei.value.code == -1
        # the cycle that follows cannot be diagnosed; another entry's cycle reports no surplus victims
        e.run_cycle_preempt_elastic(running, holdings, surplus)
        assert len(e.surplus_victims()) == 1
        with pytest.raises(GroveError) as ei:
            e.diagnose()
        assert ei.value.code == -5
        e.run_cycle_preempt(running, holdings)
        assert len(e.surplus_victims()) == 0


def test_refused_sets_and_wide(built_lib):
    """under every set and pair of sets, and for a wide submission, the return code and what grove_diagnose answers afterwards are
    grove_run_cycle_preempt's"""
    from grove_b200.engine import PlacementEngine
    from test_cycle_sets_gpu import EXPECTED, _code, _give, _snapshot, _wide_tables
    nodes, tables = _snapshot()
    running, holdings = np.zeros(0, dtype=T.running_dt), np.zeros(0, dtype=T.holding_dt)
    surplus = np.zeros(0, dtype=T.surplus_pod_dt)
    got = {}
    with PlacementEngine(2) as e:
        for cond in EXPECTED:
            for entry in ("preempt", "elastic"):
                e.load_nodes(nodes)
                if cond == "wide":
                    e.submit_gangs_wide(*_wide_tables())
                else:
                    e.submit_gangs(*tables)
                e.run_cycle()
                if cond != "wide":
                    _give(e, cond.split("+"))
                call = ((lambda: e.run_cycle_preempt(running, holdings)) if entry == "preempt"
                        else (lambda: e.run_cycle_preempt_elastic(running, holdings, surplus)))
                got[cond, entry] = (_code(call), _code(e.diagnose))
    assert got[("wide", "elastic")][0] == -4 and got[("spread", "elastic")][0] == -5
    bad = {c: (got[c, "preempt"], got[c, "elastic"]) for c in EXPECTED if got[c, "preempt"] != got[c, "elastic"]}
    assert not bad, bad


def test_struct_layouts_match_dtypes(tmp_path):
    """sizeof / offsetof of the two new structs against their numpy dtypes"""
    header = os.path.join(ROOT, "include", "grove_place.h")
    fields = {"grove_surplus_pod_t": T.surplus_pod_dt, "grove_surplus_victim_t": T.surplus_victim_dt}
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{header}"', "int main(void){"]
    for name, dt in fields.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for f in dt.names:
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    lines.append("return 0;}")
    probe = tmp_path / "probe.c"
    probe.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-std=c11", "-o", str(exe), str(probe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for name, dt in fields.items():
        assert int(got[name]) == dt.itemsize, name
        for f in dt.names:
            assert int(got[f"{name}.{f}"]) == dt.fields[f][1], f"{name}.{f}"
