"""-m "not gpu": the C-ABI library builds, loads and exports every symbol include/grove_place.h
declares; packed-table layouts match the header; there is no CPU fallback behind the ABI."""
import ctypes as C
import os
import re
import subprocess

import pytest

from grove_b200 import tables as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "grove_place.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(grove_[a-z_0-9]+)\s*\(", src)))


def test_header_declares_what_python_binds():
    from grove_b200 import engine
    assert declared_symbols() == sorted(engine.SYMBOLS)


def test_library_exports_every_declared_symbol(built_lib):
    lib = C.CDLL(built_lib)
    for s in declared_symbols():
        assert hasattr(lib, s), s
    lib.grove_abi_version.restype = C.c_uint32
    assert lib.grove_abi_version() == 2


def test_library_is_sm90a_only(built_lib):
    out = subprocess.run(["cuobjdump", "-lelf", built_lib], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_\d+a?", out))
    assert archs == {"sm_90a"}, archs


def test_struct_layouts_match_header(tmp_path):
    """compile a C probe against the header and compare sizeof/offsetof with the numpy dtypes"""
    probe = tmp_path / "probe.c"
    fields = {
        "grove_node_t": T.node_dt, "grove_clique_t": T.clique_dt, "grove_scope_t": T.scope_dt,
        "grove_gang_t": T.gang_dt, "grove_placement_t": T.placement_dt, "grove_gang_status_t": T.status_dt,
        "grove_scope_status_t": T.scope_status_dt,
        "grove_config_t": T.config_dt, "grove_cycle_stats_t": T.stats_dt,
        "grove_holding_t": T.holding_dt, "grove_running_gang_t": T.running_dt, "grove_victim_t": T.victim_dt,
    }
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{HEADER}"', "int main(void){"]
    for name, dt in fields.items():
        lines.append(f'printf("{name} %zu\\n", sizeof({name}));')
        for f in dt.names:
            lines.append(f'printf("{name}.{f} %zu\\n", offsetof({name}, {f}));')
    lines.append("return 0;}")
    probe.write_text("\n".join(lines))
    exe = tmp_path / "probe"
    subprocess.check_call(["gcc", "-std=c11", "-o", str(exe), str(probe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for name, dt in fields.items():
        assert int(got[name]) == dt.itemsize, name
        for f in dt.names:
            assert int(got[f"{name}.{f}"]) == dt.fields[f][1], f"{name}.{f}"


def test_no_cpu_fallback(built_lib):
    """Without a CUDA device the engine cannot be created (and says so); it never routes to a CPU path."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from grove_b200.engine import GroveError, PlacementEngine
    with pytest.raises(GroveError) as ei:
        PlacementEngine(4)
    assert ei.value.code == -2  # GROVE_ERR_NO_DEVICE


def test_product_never_touches_the_oracle():
    """grove_b200/ (the shipped path) must not import, load or link anything under oracle/."""
    pkg = os.path.join(ROOT, "grove_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dp, f)).read()
                for needle in ("oracle_py", "libgrove_oracle", "from oracle", "import oracle", "oracle/grove_oracle"):
                    assert needle not in txt, (f, needle)
    ldd = subprocess.run(["ldd", os.path.join(pkg, "libgrove_place.so")], capture_output=True, text=True).stdout
    assert "oracle" not in ldd


def test_oracle_rejects_malformed_tables(oracle):
    from grove_b200 import synth
    nodes = synth.e2e_cluster(4)
    b = T.GangTableBuilder(); b.add_gang([(None, [dict(mem=1, min=2, replicas=1)])])  # replicas < min
    g, c, s = b.build()
    with pytest.raises(RuntimeError):
        oracle.run_cycle(nodes, 4, g, c, s)
    b = T.GangTableBuilder(); b.add_gang([(None, [dict(mem=1, min=1)])], level=7)  # level out of range
    g, c, s = b.build()
    with pytest.raises(RuntimeError):
        oracle.run_cycle(nodes, 4, g, c, s)
    b = T.GangTableBuilder(); b.add_gang([(None, [dict(mem=1, min=100), dict(mem=1, min=100)])])  # > 128 pods
    g, c, s = b.build()
    with pytest.raises(RuntimeError):
        oracle.run_cycle(nodes, 4, g, c, s)
