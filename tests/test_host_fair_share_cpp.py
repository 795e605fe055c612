"""GpuBackend with the fair-share order on and off (tests/cpp/test_host_fair_share.cpp), through the C ABI on the GPU."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
def test_host_fair_share(built_lib, tmp_path):
    out = str(tmp_path / "test_host_fair_share.bin")
    srcs = [os.path.join(ROOT, "tests", "cpp", "test_host_fair_share.cpp"), os.path.join(ROOT, "grove_b200", "csrc", "host", "grove_host.cpp")]
    libdir = os.path.join(ROOT, "grove_b200")
    env = dict(os.environ); env.pop("CC", None); env.pop("CXX", None)
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-pthread", "-o", out, *srcs, f"-L{libdir}", "-lgrove_place",
                           f"-Wl,-rpath,{libdir}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"], env=env)
    r = subprocess.run([out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "host fair share tests ok" in r.stdout
