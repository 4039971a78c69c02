"""Loop verification on the device (include/vinsb200/loop_verify.h) against the cv2 / numpy twin of findConnection
(oracle/loop_verify.py): blur, FAST corners, BRIEF descriptors and matches bit-identical; accept / reject agreeing on
revisits, non-overlapping pairs and pairs with too few matches; the PnP pose against cv2.solvePnPRansac and the ground
truth; batch members bit-identical to stand-alone runs; errors leaving the arena unchanged."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import loop_verify as olv  # noqa: E402
from harness import synth  # noqa: E402

pytestmark = pytest.mark.gpu

ROWS, COLS = 480, 752
INTR = np.array([460.0, 460.0, 376.0, 240.0, 0, 0, 0, 0])
RIC, TIC = np.eye(3), np.zeros(3)
SHIFT = 3  # the old view is the current one moved 3 pixels to the right: a small rotation about the camera's y axis


@pytest.fixture(scope="module")
def pattern():
    return olv.load_pattern()


def _scene(seed, n_win, pattern, sub=0.25):
    """Current image, window points (3-D at random depths along the rays of FAST corners) and the old image."""
    img = synth.value_noise_image(ROWS, COLS, seed)
    kp, _ = olv.fast(img)
    inner = kp[(kp[:, 0] > 40) & (kp[:, 0] < COLS - 40) & (kp[:, 1] > 40) & (kp[:, 1] < ROWS - 40)]
    sel = inner[np.linspace(0, len(inner) - 1, n_win).astype(int)]
    uv = sel.astype(np.float32) + np.float32(sub)
    norm = olv.lift_pinhole(INTR, uv).astype(np.float32)
    depth = np.random.default_rng(seed).uniform(3, 8, n_win)
    p3d = (np.c_[norm.astype(np.float64), np.ones(n_win)] * depth[:, None]).astype(np.float32)
    old = np.roll(img, SHIFT, axis=1)
    return img, uv, norm, p3d, old


def _kf(img, uv, norm, p3d, pattern, P=np.zeros(3), R=np.eye(3)):
    return olv.KeyFrame(img, P, R, p3d, uv, norm, np.arange(len(uv)) + 1000.0, pattern, INTR)


def _graph(pattern, max_window=256, max_corners=16384):
    from vins_mono_b200.pose_graph import PoseGraph, loop_config
    g = PoseGraph(max_keyframes=8)
    g.enable_loop(loop_config(ROWS, COLS, INTR, RIC, TIC, pattern, max_window, max_corners))
    return g


def _attach(g, index, img, uv=None, norm=None, p3d=None, P=np.zeros(3), Q=(1.0, 0, 0, 0)):
    n = 0 if uv is None else len(uv)
    z2, z3 = np.zeros((n, 2), np.float32), np.zeros((n, 3), np.float32)
    return g.attach_keyframe(index, P, Q, img, z3 if p3d is None else p3d, z2 if uv is None else uv,
                             z2 if norm is None else norm, np.arange(n) + 1000.0)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_blur_fast_brief_match_bit_identical(seed, pattern):
    from vins_mono_b200 import pose_graph as pg
    img, uv, norm, p3d, old = _scene(seed, 150, pattern)
    assert np.array_equal(pg.debug_brief_blur(img), olv.gaussian_blur(img))
    for im in (img, old):
        kp = pg.debug_fast(im)
        assert np.array_equal(kp, olv.fast(im)[0])
    ref_old = _kf(old, uv, norm, p3d, pattern)
    assert np.array_equal(pg.debug_brief(img, pattern, uv), olv.brief(img, uv, pattern))
    kd = pg.debug_brief(old, pattern, ref_old.kp[:1024].astype(np.float32))
    assert np.array_equal(kd, ref_old.kp_desc[:1024])
    wd = olv.brief(img, uv, pattern)
    assert np.array_equal(pg.debug_match(wd, ref_old.kp_desc), olv.match(wd, ref_old.kp_desc)[0])
    # ties: duplicated old descriptors must resolve to the first index
    dup = np.r_[ref_old.kp_desc[:50], ref_old.kp_desc[:50]]
    assert np.array_equal(pg.debug_match(wd, dup), olv.match(wd, dup)[0])


@pytest.mark.parametrize("shape", [(17, 2048), (9, 33), (8, 8), (18, 34), (480, 752)])
def test_blur_and_fast_at_tile_overhang_sizes(shape):
    import cv2
    from vins_mono_b200 import pose_graph as pg
    img = np.random.default_rng(shape[0] * 7 + shape[1]).integers(0, 256, shape).astype(np.uint8)
    assert np.array_equal(pg.debug_brief_blur(img), cv2.GaussianBlur(img, (9, 9), 2, 2))
    assert np.array_equal(pg.debug_fast(img), olv.fast(img)[0])


def _verify_pair(g, pattern, cur_img, uv, norm, p3d, old_img, P=np.zeros(3), Q=(1.0, 0, 0, 0)):
    _attach(g, 0, old_img)
    _attach(g, 1, cur_img, uv, norm, p3d, P, Q)
    return g.find_connection(1, 0)


GATE_YAW = 40.0  # degrees: the current VIO frame turned about z, so the relative yaw fails |yaw| < 30
GATE_T = np.array([25.0, 0.0, 0.0])  # metres: the current VIO frame moved, so the relative t fails |t| < 20


@pytest.mark.parametrize("case", ["revisit", "revisit_b", "disjoint", "too_few", "few_inliers", "yaw_gate", "t_gate", "yaw_29"])
def test_accept_reject_agrees_with_twin(case, pattern):
    seed = {"revisit": 0, "revisit_b": 1, "disjoint": 2, "too_few": 3, "few_inliers": 4, "yaw_gate": 5, "t_gate": 6, "yaw_29": 7}[case]
    img, uv, norm, p3d, old = _scene(seed, {"too_few": 25, "few_inliers": 40}.get(case, 150), pattern)
    if case == "disjoint":
        old = synth.value_noise_image(ROWS, COLS, 77)
    if case == "few_inliers":  # every window point matches, but only 23 carry their true 3-D point
        rng = np.random.default_rng(9)
        p3d = p3d.copy()
        p3d[23:] = rng.permutation(p3d[23:]) * np.float32(1.7)
    P, R = np.zeros(3), np.eye(3)
    # the current key frame's VIO pose turned about z (29 degrees: just inside the gate) or moved, while its window
    # points stay where they are: PnP still succeeds, the relative yaw or t is off by that much
    if case in ("yaw_gate", "yaw_29"):
        R =olv.quat_to_R([np.cos(np.radians(GATE_YAW if case == "yaw_gate" else 29.0) / 2), 0, 0,
                           np.sin(np.radians(GATE_YAW if case == "yaw_gate" else 29.0) / 2)])
    if case == "t_gate":
        P = GATE_T.copy()
    cur_kf = _kf(img, uv, norm, p3d, pattern, P, R)
    old_kf = _kf(old, uv[:0], norm[:0], p3d[:0], pattern)
    twin = olv.find_connection(cur_kf, old_kf, RIC, TIC)
    g = _graph(pattern)
    r = _verify_pair(g, pattern, img, uv, norm, p3d, old, P, olv.R_to_quat(R))
    print(case, "matches", r["n_matches"], twin["n_matches"], "inliers", r["n_inliers"], twin["n_inliers"],
          "accepted", r["accepted"], twin["accepted"], "t", r["loop_info"][:3], twin.get("rel_t"), "yaw", r["loop_info"][7], twin.get("rel_yaw"))
    assert r["n_matches"] == twin["n_matches"]
    assert r["accepted"] == twin["accepted"]
    if case.startswith("revisit"):
        assert r["accepted"]
        # the consensus sets of two different samplers: within 10 % of cv2's
        assert abs(r["n_inliers"] - twin["n_inliers"]) <= 0.1 * twin["n_inliers"]
        assert np.abs(r["loop_info"][:3] - twin["rel_t"]).max() < 0.05
        assert abs(r["loop_info"][7] - twin["rel_yaw"]) < 0.1
        assert np.abs(r["loop_info"][3:7] - twin["rel_q"]).max() < 1e-4
        # ground truth: the old camera sees each window point at its corner moved SHIFT pixels right (integer corner, so
        # within the 0.25 px sub-pixel offset plus the fit's residual), with no real translation
        Xc = (p3d.astype(np.float64) - r["old_T"]) @ r["old_R"]
        px = INTR[0] * Xc[:, :2] / Xc[:, 2:] + INTR[2:4]
        assert np.abs(px - (np.floor(uv) + [SHIFT, 0])).max() < 1.0
        assert np.abs(r["loop_info"][:3]).max() < 0.05
        pts = r["points"]
        assert len(pts) == r["n_inliers"] and np.all(np.diff(pts[:, 2]) > 0)
    if case == "too_few":
        assert r["n_matches"] <= olv.MIN_LOOP_NUM and not r["accepted"]
    if case == "few_inliers":
        assert r["n_matches"] > olv.MIN_LOOP_NUM and 0 < r["n_inliers"] <= olv.MIN_LOOP_NUM and not r["accepted"]
        assert abs(r["n_inliers"] - twin["n_inliers"]) <= 2
    if case in ("yaw_gate", "t_gate", "yaw_29"):  # PnP succeeds; only the gate decides
        assert r["n_inliers"] > olv.MIN_LOOP_NUM and abs(r["n_inliers"] - twin["n_inliers"]) <= 0.1 * twin["n_inliers"]
        assert abs(r["loop_info"][7] - twin["rel_yaw"]) < 0.1 and np.abs(r["loop_info"][:3] - twin["rel_t"]).max() < 0.05
        assert r["accepted"] == (case == "yaw_29")


def test_batch_members_equal_standalone_and_repeat_runs(pattern):
    from vins_mono_b200.pose_graph import PoseGraphBatch, loop_config
    scenes = [_scene(s, 150, pattern) for s in (0, 1, 4)]
    solo = []
    g = _graph(pattern)
    for img, uv, norm, p3d, old in scenes:
        solo.append(_verify_pair(g, pattern, img, uv, norm, p3d, old))
        again = g.find_connection(1, 0)
        for k in solo[-1]:
            assert np.array_equal(np.asarray(solo[-1][k]), np.asarray(again[k])), k
    b = PoseGraphBatch(4, max_keyframes=8)
    b.enable_loop(loop_config(ROWS, COLS, INTR, RIC, TIC, pattern, 256, 16384))
    for k, (img, uv, norm, p3d, old) in enumerate(scenes):
        _attach(b[k], 0, old)
        _attach(b[k], 1, img, uv, norm, p3d)
    res = b.find_connection([1, 1, 1, -1], [0, 0, 0, 0])
    assert res[3] is None
    for k in range(3):
        for key in solo[k]:
            assert np.array_equal(np.asarray(solo[k][key]), np.asarray(res[k][key])), (k, key)
    ms = b.loop_timing()
    assert np.all(ms[3:] > 0)


def test_errors_leave_the_arena_unchanged(pattern):
    from vins_mono_b200.pose_graph import PoseGraphError
    img, uv, norm, p3d, old = _scene(0, 150, pattern)
    g = _graph(pattern, max_window=150, max_corners=16384)
    for k in range(3):  # the pose graph's own state must not move either
        g.add_keyframe(k, [k, 0, 0], [1, 0, 0, 0])
    path0, info0 = g.path(), g.info()
    ref = _verify_pair(g, pattern, img, uv, norm, p3d, old)
    with pytest.raises(PoseGraphError) as e:  # more window points than max_window
        _attach(g, 1, img, np.r_[uv, uv[:1]], np.r_[norm, norm[:1]], np.r_[p3d, p3d[:1]])
    assert e.value.status == -4
    with pytest.raises(PoseGraphError) as e:  # a slot index outside the graph's capacity
        _attach(g, 8, img)
    assert e.value.status == -1
    with pytest.raises(PoseGraphError) as e:  # a slot that was never attached
        g.find_connection(1, 5)
    assert e.value.status == -1
    again = g.find_connection(1, 0)
    for k in ref:
        assert np.array_equal(np.asarray(ref[k]), np.asarray(again[k])), k
    small = _graph(pattern, max_window=150, max_corners=1000)  # a textured image has more corners than that
    with pytest.raises(PoseGraphError) as e:
        _attach(small, 0, old)
    assert e.value.status == -4
    with pytest.raises(PoseGraphError):
        small.find_connection(1, 0)
    for a, b in zip(path0, g.path()):
        assert np.array_equal(a, b)
    assert g.info() == info0


def test_debug_pnp_recovers_a_pose_with_outliers():
    from vins_mono_b200 import pose_graph as pg
    rng = np.random.default_rng(5)
    n = 120
    X = rng.uniform([-3, -2, 4], [3, 2, 9], (n, 3))
    R = olv.quat_to_R([0.99, 0.05, -0.08, 0.03])
    t = np.array([0.3, -0.2, 0.5])
    Xc = X @ R.T + t
    u = Xc[:, :2] / Xc[:, 2:] + rng.normal(0, 0.5 / 460, (n, 2))
    out = rng.random(n) < 0.3
    u[out] += rng.uniform(-0.3, 0.3, (out.sum(), 2))
    Rd, td, n_in, mask = pg.debug_pnp(X, u)
    assert np.abs(Rd - R).max() < 5e-3 and np.abs(td - t).max() < 2e-2
    assert n_in == mask.sum() and n_in >= (~out).sum() * 0.95
