"""CPU checks of the drop-in boundary: libserfsim.so builds, loads, exports exactly the symbols
include/serfsim.h declares, and refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import pytest

from serf_b200 import build as sb
from serf_b200 import sim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "serfsim.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(serfsim_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_every_declared_symbol():
    so = sb.build()
    out = subprocess.check_output(["nm", "-D", "--defined-only", so]).decode()
    exported = sorted(l.split()[-1] for l in out.splitlines() if " T " in l)
    declared = _declared()
    assert declared, "header parse failed"
    assert exported == declared, (set(declared) ^ set(exported))


def test_library_is_sm90a_with_red_and_no_oracle_dependency():
    so = sb.build()
    sass = subprocess.check_output(["cuobjdump", "-sass", so]).decode()
    assert "sm_90a" in sass
    assert "RED.E.MAX" in sass or "REDG.E.MAX" in sass or "RED.MAX" in sass or ".MAX" in sass      # inbox reduction is a hardware RED.MAX
    needed = subprocess.check_output(["readelf", "-d", so]).decode()
    assert "oracle" not in needed.lower()


def test_struct_layouts_match_header():
    assert C.sizeof(sim.Config) == 12 * 4 + 8 + 4 * 4 + 4 * 4
    assert C.sizeof(sim.Stats) == 12 * 8 and C.sizeof(sim.TickRow) == 8 * 8
    assert sim.RECORD_DTYPE.itemsize == 32


def test_create_fails_loudly_without_gpu():
    lib = sim.load_library()
    assert lib.serfsim_abi_version() == sim.ABI_VERSION == 4
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present: covered by the gpu tests")
    with pytest.raises(sim.SerfsimError) as e:
        sim.GossipSim(100, 1)
    assert e.value.code == -2 and "no CPU" in str(e.value)


def test_cpp_host_layer_compiles_links_and_fails_loudly_without_gpu(tmp_path):
    """include/serfsim.hpp (the C++ host layer with the reference's names) builds against libserfsim.so; without a GPU
    creating a cluster throws SERFSIM_E_NO_DEVICE (exit code 10 of the check program), with one it runs configs[0]."""
    so = sb.build()
    exe = str(tmp_path / "host_layer_check")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "cpp", "host_layer_check.cpp"),
                           "-o", exe, so, "-Wl,-rpath," + os.path.dirname(so)])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    import torch
    if torch.cuda.is_available():
        assert r.returncode == 0, r.stdout + r.stderr
    else:
        assert r.returncode == 10 and "no CPU execution path" in r.stdout, r.stdout + r.stderr


def test_product_loader_refuses_the_host_compiled_test_build():
    """SERFSIM_LIB may point at another nvcc build of the library (A/B runs) but never at tests/emu's host build."""
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import emu_lib
    env = dict(os.environ, SERFSIM_LIB=emu_lib.build())
    r = subprocess.run([sys.executable, "-c", "from serf_b200 import sim; sim.load_library()"], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode != 0 and "refusing to use it as the product" in r.stderr


def test_bind_thread_near_gpu_without_a_gpu_changes_nothing():
    """The NUMA helper of the Python driver: without a GPU / NVML it returns None and leaves the thread's affinity alone."""
    import os
    from serf_b200 import bind_thread_near_gpu
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: covered by bench.py")
    before = os.sched_getaffinity(0)
    assert bind_thread_near_gpu(0) is None
    assert os.sched_getaffinity(0) == before
