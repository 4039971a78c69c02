"""CPU checks of the pose graph: the oracle's FourDOFError / FourDOFWeightError against finite differences (also across
yaw +-180), the oracle's LM run to convergence against scipy's minimum on graphs with Huber-active loops, its bookkeeping
(recovering an injected yaw + translation drift from noise-free loops, the cross-sequence shift), the vp_ C ABI exported
by the library and refusing to run without a GPU, the buffer layouts (pg_layout.h, with g++), and the cross-compile of
the pose-graph kernels for sm_90a."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import pose_graph as opg  # noqa: E402


@pytest.mark.parametrize("weighted,robust", [(False, False), (True, False), (True, True)])
def test_oracle_factor_jacobian_matches_finite_differences(weighted, robust):
    rng = np.random.default_rng(1)
    for trial in range(30):
        xi = np.r_[rng.uniform(-180, 180), rng.normal(0, 2, 3)]
        xj = np.r_[rng.uniform(-180, 180), rng.normal(0, 2, 3)]
        if trial % 3 == 0:
            xi[0], xj[0] = 179.95, -179.9
        meas, pr = np.r_[rng.normal(0, 2, 3), rng.uniform(-20, 20)], rng.uniform(-20, 20, 2)
        if trial % 2:
            xj[1:] = xi[1:] + 0.01 * (xj[1:] - xi[1:])
            meas[:3] = 0.01 * meas[:3]
        r, J, c = opg.four_dof(xi, xj, pr[0], pr[1], meas, weighted, robust)
        x = np.r_[xi, xj]
        h = 1e-6
        for col in range(8):
            xp, xm = x.copy(), x.copy()
            xp[col] += h
            xm[col] -= h
            rp = opg.four_dof(xp[:4], xp[4:], pr[0], pr[1], meas, weighted, False)[0]
            rm = opg.four_dof(xm[:4], xm[4:], pr[0], pr[1], meas, weighted, False)[0]
            if robust:  # the corrector's rho'' <= 0 branch: sqrt(rho') times the plain Jacobian
                r0 = opg.four_dof(xi, xj, pr[0], pr[1], meas, weighted, False)[0]
                s = float(r0 @ r0)
                sc = 1.0 if s <= 0.01 else np.sqrt(0.1 / np.sqrt(s))
                fd = sc * (rp - rm) / (2 * h)
            else:
                fd = (rp - rm) / (2 * h)
            assert np.abs(fd - J[:, col]).max() < 1e-6, (trial, col)


def _graph(n, loops, seed):
    rng = np.random.default_rng(seed)
    P = np.cumsum(rng.normal(0, 0.3, (n, 3)), axis=0)
    R = [opg.ypr2R([y, p, r]) for y, p, r in zip(np.cumsum(rng.normal(0, 5, n)), rng.normal(0, 3, n), rng.normal(0, 3, n))]
    ye, pe = np.cumsum(rng.normal(0, 0.5, n)), np.cumsum(rng.normal(0, 0.05, (n, 3)), axis=0)
    vio_P = [opg.ypr2R([ye[k], 0, 0]) @ P[k] + pe[k] for k in range(n)]
    vio_R = [opg.ypr2R([ye[k], 0, 0]) @ R[k] for k in range(n)]
    lp = [None] * n
    for k, (j, noise) in loops.items():
        t = R[j].T @ (P[k] - P[j]) + noise * rng.normal(0, 1, 3)
        yaw = opg.R2ypr(R[k])[0] - opg.R2ypr(R[j])[0] + noise * 30 * rng.normal()
        lp[k] = (j, np.r_[t, opg.normalize_angle(yaw)])
    return opg.Problem(vio_P, vio_R, [1] * n, lp)


def test_oracle_reaches_scipy_minimum_with_huber_active_loops():
    from scipy.optimize import least_squares
    pb = _graph(40, {20: (0, 0.01), 25: (3, 0.5), 30: (7, 0.02), 35: (3, 0.8), 39: (11, 0.01)}, seed=3)
    x, info = pb.solve(max_iterations=200, function_tolerance=1e-15)
    assert info["converged"]
    active = [lp for (a, b, m, lp) in pb.edges if lp]
    assert len(active) == 5
    ls = least_squares(pb.robust_residuals, pb.x0[1:].ravel(), loss="linear", xtol=1e-15, ftol=1e-15, gtol=1e-15)
    r = pb.robust_residuals(x[1:].ravel())
    # at least one loop edge sits in the Huber region (|r|^2 > 0.1^2) at the minimum
    s = [float(np.sum(opg.four_dof(x[a], x[b], pb.ypr[a, 1], pb.ypr[a, 2], m, True, False)[0] ** 2)) for (a, b, m, lp) in pb.edges if lp]
    assert max(s) > 0.01
    assert abs(0.5 * r @ r - ls.cost) <= 1e-9 * ls.cost, (0.5 * r @ r, ls.cost)
    assert abs(info["cost"] - ls.cost) <= 1e-9 * ls.cost


def test_oracle_bookkeeping_recovers_injected_drift():
    """Key frames 30.. form a second sequence whose VIO frame carries a pure yaw + translation offset; noise-free loops
    back onto the first sequence: the cross-sequence shift removes the offset, and the optimised poses are the ground
    truth."""
    n = 60
    rng = np.random.default_rng(5)
    P = np.cumsum(rng.normal(0, 0.3, (n, 3)), axis=0)
    R = [opg.ypr2R([y, p, r]) for y, p, r in zip(np.cumsum(rng.normal(0, 5, n)), rng.normal(0, 3, n), rng.normal(0, 3, n))]
    Rd, td = opg.ypr2R([7.0, 0, 0]), np.array([0.4, -0.3, 0.2])
    g = opg.OraclePoseGraph()
    for k in range(n):
        if k == 30:
            g.new_sequence()
        vP, vR = (Rd @ P[k] + td, Rd @ R[k]) if k >= 30 else (P[k], R[k])
        l, li = -1, None
        if k >= 40 and k % 5 == 0:
            l = k - 35
            li = np.r_[R[l].T @ (P[k] - P[l]), opg.R_to_quat(R[l].T @ R[k]), opg.R2ypr(R[k])[0] - opg.R2ypr(R[l])[0]]
        g.add_keyframe(0.1 * k, vP, opg.R_to_quat(vR), l, li)
    assert abs(opg.R2ypr(g.w_r_vio)[0] + 7.0) < 1e-9
    g.optimize(max_iterations=100, function_tolerance=1e-15)
    _, Po, _, _ = g.path()
    assert np.abs(Po - P).max() < 1e-6
    assert abs(g.yaw_drift) < 1e-6


def test_oracle_cross_sequence_shift():
    g = opg.OraclePoseGraph()
    q = opg.R_to_quat(opg.ypr2R([10, 2, 1]))
    for k in range(5):
        g.add_keyframe(k, [k, 0, 0], q)
    g.new_sequence()
    q2 = opg.R_to_quat(opg.ypr2R([40, 2, 1]))
    g.add_keyframe(10, [0, 5, 0], q2)
    rel = np.r_[0.5, 0, 0, opg.R_to_quat(np.eye(3)), 0.0]
    g.add_keyframe(11, [0, 6, 0], q2, 2, rel)
    # the whole second sequence moved so that key frame 6 sits at key frame 2's pose + rel
    assert np.allclose(g.kfs[6]["vio_P"], g.kfs[2]["vio_R"] @ rel[:3] + g.kfs[2]["vio_P"])
    assert abs(opg.R2ypr(g.kfs[6]["vio_R"])[0] - 10.0) < 1e-9
    assert np.allclose(g.kfs[5]["vio_P"] - g.kfs[6]["vio_P"], opg.ypr2R([-30, 0, 0]) @ np.array([0, -1.0, 0]))
    assert g.pending == 6 and g.sequence_loop[2] == 1


def _declared():
    src = open(os.path.join(ROOT, "include", "vinsb200", "pose_graph.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(vp_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib():
    from vins_mono_b200 import build, load_library
    build.build()
    return load_library()


def test_every_vp_symbol_is_exported(lib):
    names = _declared()
    assert len(names) >= 23 and "vp_batch_optimize" in names
    assert not [n for n in names if not hasattr(lib, n)]


def test_vp_create_fails_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from vins_mono_b200 import PoseGraph, PoseGraphBatch
    with pytest.raises(RuntimeError):
        PoseGraph()
    with pytest.raises(RuntimeError):
        PoseGraphBatch(2)


def test_pg_layouts(tmp_path):
    out = tmp_path / "libpglayout.so"
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wall", "-Werror", "-I",
                           os.path.join(ROOT, "vins_mono_b200", "csrc"), os.path.join(ROOT, "tests", "hostlib", "pg_layout_host.cpp"),
                           "-o", str(out)])
    l = ctypes.CDLL(str(out))
    l.check_pg_layouts.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_long), ctypes.c_char_p, ctypes.c_int]
    l.check_pg_layouts.restype = ctypes.c_long
    for cap in (8, 500, 2048):
        n = ctypes.c_long(0)
        msg = ctypes.create_string_buffer(256)
        assert l.check_pg_layouts(cap, ctypes.byref(n), msg, len(msg)) == 0, msg.value.decode()
        assert n.value > 4


def test_pg_kernels_cross_compile_for_sm90a(tmp_path):
    from vins_mono_b200 import build
    csrc = os.path.join(ROOT, "vins_mono_b200", "csrc")
    for src in ("pg_kernels.cu", "ba_kernels.cu"):
        subprocess.check_call(["nvcc", *build.ARCH, "-O3", "-std=c++17", "--fmad=true", "-I", csrc, "-I", os.path.join(ROOT, "include"),
                               "-c", os.path.join(csrc, src), "-o", str(tmp_path / (src + ".o"))])
