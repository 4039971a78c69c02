"""CPU checks of the drop-in boundary: the C-ABI library builds, loads, and exports every function declared in
include/vinsb200/*.h; the C++ host shims with the reference's class names compile and link against it; creating a
handle without a GPU fails loudly (no CPU fallback)."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_functions():
    names = []
    inc = os.path.join(ROOT, "include", "vinsb200")
    for f in sorted(os.listdir(inc)):
        src = open(os.path.join(inc, f)).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names += re.findall(r"\b(v[terp]_[a-z0-9_]+)\s*\(", src)
    return sorted(set(names))


@pytest.fixture(scope="module")
def lib():
    from vins_mono_b200 import build, load_library
    build.build()
    return load_library()


def test_every_declared_symbol_is_exported(lib):
    names = declared_functions()
    assert len(names) >= 36 and "vr_advance" in names
    missing = [n for n in names if not hasattr(lib, n)]
    assert not missing, missing


def test_create_fails_loudly_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from vins_mono_b200 import FeatureTracker, Estimator
    with pytest.raises(RuntimeError):
        FeatureTracker()
    with pytest.raises(RuntimeError):
        Estimator()


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "vins_mono_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".h", ".cuh")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src and "import orc" not in src, os.path.join(dirpath, f)


def test_host_shims_compile_and_link(lib, tmp_path):
    from vins_mono_b200 import LIB_PATH
    exe = tmp_path / "shim_check"
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "vins_mono_b200", "host"),
           os.path.join(ROOT, "vins_mono_b200", "host", "shim_check.cpp"), LIB_PATH, "-Wl,-rpath," + os.path.dirname(LIB_PATH),
           "-o", str(exe)]
    subprocess.check_call(cmd)
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stderr
    assert "no device" in out.stdout or "tracked" in out.stdout


def test_offline_replay_example_builds(lib, tmp_path):
    """examples/offline_replay.cpp: a ROS-free C++ client of the three headers (tracker, estimator, replay)."""
    from vins_mono_b200 import LIB_PATH
    exe = tmp_path / "offline_replay"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "examples", "offline_replay.cpp"), "-L", os.path.dirname(LIB_PATH), "-lvinsb200",
                           f"-Wl,-rpath,{os.path.dirname(LIB_PATH)}", "-lpthread", "-o", str(exe)])
    out = subprocess.run([str(exe)], capture_output=True, text=True)
    assert out.returncode == 2 and "usage" in out.stderr
