"""Host and device builds of vins_mono_b200/csrc/rotation.h agree: tests/hostlib/rotation_ops.cpp runs every operation
in a kernel compiled with --fmad=false and on the host compiled with g++ -ffp-contract=off.  The operations built from
+, -, *, / and sqrt are IEEE-exact on both sides and must give the same bits.  R2ypr, ypr2R and rodrigues call atan2,
sin or cos, where CUDA's math library and glibc differ in the last bits: they must agree within 2 ulp at full scale
(180 degrees for angles, 1 for rotation entries)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from test_rotation_cpu import OPS, SRC, evaluate, load, rotations, unit_quats, within_ulp
from vins_mono_b200 import build as vb_build

FULL_SCALE = {"R2ypr": 180.0, "ypr2R": 1.0, "rodrigues": 1.0}
N = 4096


def compile_lib(out):
    subprocess.check_call(["nvcc", *vb_build.NVCC_FLAGS, "--fmad=false", "-shared", "-x", "cu", "-o", str(out), SRC],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def test_library_compiles(tmp_path):
    """Cross-compiles the test library for sm_90a (no GPU needed), so it cannot rot on machines without one."""
    out = tmp_path / "librotdev.so"
    compile_lib(out)
    assert out.stat().st_size > 0


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("rotdev") / "librotdev.so"
    compile_lib(out)
    lib = load(out)
    lib.rot_eval_device.argtypes = lib.rot_eval.argtypes
    return lib


def inputs(name, width, rng):
    if name in ("R2ypr", "FromR"):
        return rotations(rng, N).reshape(-1, 9)
    if name == "ypr2R":
        return np.column_stack([rng.uniform(-180, 180, N), rng.uniform(-90, 90, N), rng.uniform(-180, 180, N)])
    if name == "normalize_angle":
        a = rng.uniform(-540.0, 540.0, N)
        return np.concatenate([a, [180.0, -180.0, np.nextafter(180.0, 200.0), np.nextafter(-180.0, -200.0), -0.0]])
    if name == "rodrigues":  # rotation angles from 1e-14 (the small-angle branch) to pi
        return unit_quats(rng, N)[:, 1:] * 10.0 ** rng.uniform(-14, np.log10(np.pi), (N, 1))
    return rng.normal(size=(N, width))


@pytest.mark.gpu
@pytest.mark.parametrize("name", OPS)
def test_host_and_device_agree(lib, name):
    x = inputs(name, lib.rot_op_width(OPS.index(name), 0), np.random.default_rng(OPS.index(name)))
    host = evaluate(lib, name, x)
    dev = evaluate(lib, name, x, fn="rot_eval_device")
    if name in FULL_SCALE:
        assert within_ulp(dev, host, FULL_SCALE[name]).all(), np.max(np.abs(dev - host)) / np.spacing(FULL_SCALE[name])
    else:
        assert np.array_equal(dev.view(np.uint64), host.view(np.uint64))
