"""The rotation utilities of vins_mono_b200/csrc/rotation.h, compiled with g++ alone as the build compiles host code
(-ffp-contract=off), against the numpy restatements of oracle/pose_graph.py.  Quaternion <-> matrix and normalize_angle
use numpy's term order and must match exactly.  R2ypr and ypr2R call atan2, sin and cos and must agree within 2 ulp at
full scale (180 degrees for angles, 1 for rotation entries): R2ypr's roll comes out of a difference of products that can
cancel, so a bound relative to each result would not hold.  R2ypr gets 2 ulp more for its degree conversion: numpy,
like the reference, divides by pi and then multiplies by 180, where the library multiplies once by 1 / pi * 180."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pose_graph as pg  # noqa: E402

SRC = os.path.join(ROOT, "tests", "hostlib", "rotation_ops.cpp")
CSRC = os.path.join(ROOT, "vins_mono_b200", "csrc")
P_D = ctypes.POINTER(ctypes.c_double)
# the op numbers of rotation_ops.cpp
OPS = ["R2ypr", "ypr2R", "qR", "FromR", "normalize_angle", "qmul", "qrot", "mmul", "mv", "normalized", "skew", "cross",
       "dot", "qinv", "deltaQ", "mT", "rodrigues"]


def load(path):
    lib = ctypes.CDLL(str(path))
    lib.rot_eval.argtypes = [ctypes.c_int, ctypes.c_int, P_D, P_D]
    assert lib.rot_op_count() == len(OPS)
    return lib


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    out = tmp_path_factory.mktemp("rotation") / "librothost.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", "-Wall", "-Werror",
                           "-I", CSRC, SRC, "-o", str(out)])
    return load(out)


def evaluate(lib, name, x, fn="rot_eval"):
    op = OPS.index(name)
    x = np.ascontiguousarray(x, dtype=np.float64).reshape(len(x), -1)
    assert x.shape[1] == lib.rot_op_width(op, 0)
    out = np.zeros((len(x), lib.rot_op_width(op, 1)))
    rc = getattr(lib, fn)(op, len(x), x.ctypes.data_as(P_D), out.ctypes.data_as(P_D))
    assert not rc
    return out


def within_ulp(a, b, scale, n=2):
    return np.abs(a - b) <= n * np.spacing(scale)


def unit_quats(rng, n):
    q = rng.normal(size=(n, 4))
    return q / np.linalg.norm(q, axis=1, keepdims=True)


def rotations(rng, n):
    """Rotations from random unit quaternions, plus the identity and the half turns about each axis (the three arms of
    FromR's trace <= 0 branch)."""
    R = np.array([pg.quat_to_R(q) for q in unit_quats(rng, n)])
    special = [np.eye(3), np.diag([1.0, -1, -1]), np.diag([-1.0, 1, -1]), np.diag([-1.0, -1, 1])]
    return np.concatenate([R, np.array(special)])


def test_quaternion_to_matrix(host):
    q = unit_quats(np.random.default_rng(1), 20000)
    q = np.concatenate([q, 3.0 * q[:100]])  # not unit: R() does not normalise
    ref = np.array([pg.quat_to_R(x).ravel() for x in q])
    assert np.array_equal(evaluate(host, "qR", q).view(np.uint64), ref.view(np.uint64))


def test_matrix_to_quaternion(host):
    R = rotations(np.random.default_rng(2), 20000)
    ref = np.array([pg.R_to_quat(r) for r in R])
    assert np.array_equal(evaluate(host, "FromR", R).view(np.uint64), ref.view(np.uint64))


def test_normalize_angle(host):
    a = np.random.default_rng(3).uniform(-540.0, 540.0, 20000)
    a = np.concatenate([a, [180.0, -180.0, np.nextafter(180.0, 200.0), np.nextafter(-180.0, -200.0), 0.0, -0.0, 540.0]])
    ref = np.array([pg.normalize_angle(x) for x in a])
    assert np.array_equal(evaluate(host, "normalize_angle", a)[:, 0].view(np.uint64), ref.view(np.uint64))


def test_R2ypr(host):
    R = rotations(np.random.default_rng(4), 50000)
    ref = np.array([pg.R2ypr(r) for r in R])
    assert within_ulp(evaluate(host, "R2ypr", R), ref, 180.0, n=4).all()


def test_ypr2R(host):
    rng = np.random.default_rng(5)
    n = 50000
    ypr = np.column_stack([rng.uniform(-180, 180, n), rng.uniform(-90, 90, n), rng.uniform(-180, 180, n)])
    ref = np.array([pg.ypr2R(x).ravel() for x in ypr])
    assert within_ulp(evaluate(host, "ypr2R", ypr), ref, 1.0).all()
