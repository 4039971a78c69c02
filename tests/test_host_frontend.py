"""The product's host-side front-end pieces (vins_mono_b200/csrc/{fm_ransac.cpp,tracker.cu}) checked on a box without
a GPU through handle-free debug entries: the F-matrix RANSAC of rejectWithF (inlier masks bit-identical to
cv2.findFundamentalMat on the golden problems of tests/golden/frontend_ops.npz, plus degenerate inputs), the disc table of
setMask (reproduces cv2's filled circles) and PinholeCamera::liftProjective."""
import ctypes as C
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ransac():
    from vins_mono_b200 import build, load_library
    build.build()
    lib = load_library()

    def run(p1, p2, thr=1.0, conf=0.99):
        p1, p2 = np.ascontiguousarray(p1, np.float32), np.ascontiguousarray(p2, np.float32)
        mask = np.zeros(len(p1), np.uint8)
        ok = lib.vt_debug_fundamental_ransac(p1.ctypes.data, p2.ctypes.data, len(p1), thr, conf, mask.ctypes.data)
        return ok, mask
    return run


def test_masks_equal_cv2_golden(ransac):
    ops = np.load(os.path.join(ROOT, "tests", "golden", "frontend_ops.npz"))
    n = int(ops["fm_count"])
    assert n >= 10
    for t in range(n):
        ok, mask = ransac(ops[f"fm{t}_p1"], ops[f"fm{t}_p2"])
        assert ok == 1 and np.array_equal(mask, ops[f"fm{t}_mask"]), f"trial {t}"


def test_degenerate_inputs(ransac):
    rng = np.random.default_rng(0)
    p = rng.uniform(0, 400, (6, 2)).astype(np.float32)
    ok, mask = ransac(p, p + 1)
    assert ok == 0 and mask.sum() == 0                    # < 7 points: no model
    p = rng.uniform(0, 400, (40, 2)).astype(np.float32)
    q = p.copy()
    q[:, 0] = 5.0                                          # collinear in image 2: no valid subset
    ok, mask = ransac(p, q)
    assert ok == 0 and mask.sum() == 0
    ok, mask = ransac(np.zeros((0, 2), np.float32), np.zeros((0, 2), np.float32))
    assert ok == 0


def _sha(a):
    import hashlib
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_disc_table_reproduces_cv2_circle_masks():
    """The half-width table the mask kernel rasterises from, applied on the host to the golden centres, gives cv2's filled
    circles bit for bit (clipping at the image border included)."""
    from vins_mono_b200 import load_library
    lib = load_library()
    ops = np.load(os.path.join(ROOT, "tests", "golden", "frontend_ops.npz"))
    r = 30
    hw = np.zeros(r + 1, np.int32)
    assert lib.vt_debug_disc_half_widths(r, hw.ctypes.data_as(C.c_void_p)) == 0
    assert hw[0] == r and hw[r] >= 0 and (np.diff(hw) <= 0).all()
    for k in (0, 1):
        rows, cols = (int(v) for v in ops[f"img{k}_shape"])
        mask = np.full((rows, cols), 255, np.uint8)
        for cx, cy in ops[f"mask{k}_centres"]:
            for dy in range(-r, r + 1):
                y = int(cy) + dy
                if 0 <= y < rows:
                    w = int(hw[abs(dy)])
                    mask[y, max(int(cx) - w, 0):min(int(cx) + w, cols - 1) + 1] = 0
        assert _sha(mask) == str(ops[f"mask{k}_sha"])


def test_lift_projective_equals_oracle_and_inverts_the_distortion():
    import orc
    from harness import synth
    from vins_mono_b200 import load_library
    lib = load_library()
    cfg = synth.tracker_config_dict()
    K = np.array([cfg[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")], np.float64)
    rng = np.random.default_rng(5)
    px = np.ascontiguousarray(np.c_[rng.uniform(0, 752, 500), rng.uniform(0, 480, 500)])
    out = np.zeros_like(px)
    assert lib.vt_debug_lift_projective(K.ctypes.data_as(C.c_void_p), px.ctypes.data_as(C.c_void_p), len(px),
                                        out.ctypes.data_as(C.c_void_p)) == 0
    assert np.array_equal(out, orc.lift_projective(cfg, px))          # same operation sequence as the CPU oracle
    x, y = out[:, 0], out[:, 1]
    r2 = x * x + y * y
    rad = cfg["k1"] * r2 + cfg["k2"] * r2 * r2
    xd = x + x * rad + 2 * cfg["p1"] * x * y + cfg["p2"] * (r2 + 2 * x * x)
    yd = y + y * rad + 2 * cfg["p2"] * x * y + cfg["p1"] * (r2 + 2 * y * y)
    back = np.c_[cfg["fx"] * xd + cfg["cx"], cfg["fy"] * yd + cfg["cy"]]
    centre = np.hypot(px[:, 0] - cfg["cx"], px[:, 1] - cfg["cy"]) < 150
    assert np.abs(back - px)[centre].max() < 1e-3                     # 8 fixed-point iterations: exact near the centre
    assert np.abs(back - px).max() < 0.3                              # and to a fraction of a pixel in the corners


# camera parameter sets of the reference's own configurations (config/3dm, config/black_box, config/tum, config/cla), plus one
# Kannala-Brandt set with an interior zero coefficient: the reference then lowers the polynomial degree and DROPS k5
# (EquidistantCamera.cc:733-770), which the product and the oracle reproduce.
MEI_SETS = {
    "3dm": dict(xi=2.057, k1=7.145e-02, k2=5.059e-01, p1=4.727e-05, p2=-5.492e-04, fx=1.115e+03, fy=1.114e+03, cx=3.672e+02, cy=2.385e+02,
                size=(752, 480)),
    "black_box": dict(xi=2.2134257311108083, k1=1.4213768437132895e-01, k2=9.1226950620748259e-01, p1=1.2056297779277966e-03,
                      p2=2.0300076091651340e-03, fx=1.1659242643040975e+03, fy=1.1656143723709608e+03, cx=3.9238492754088008e+02,
                      cy=2.4392485271819217e+02, size=(752, 480)),
    "xi_one": dict(xi=1.0, k1=-0.05, k2=0.02, p1=1e-4, p2=-2e-4, fx=600.0, fy=601.0, cx=370.0, cy=240.0, size=(752, 480)),
}
KB_SETS = {
    "tum": dict(k1=0.0034823894022493434, k2=0.0007150348452162257, p1=-0.0020532361418706202, p2=0.00020293673591811182,
                fx=190.97847715128717, fy=190.9733070521226, cx=254.93170605935475, cy=256.8974428996504, size=(512, 512)),
    "cla": dict(k1=-0.005740195474458931, k2=0.02878252863739417, p1=-0.04010621197185408, p2=0.02008469575876223,
                fx=472.2863830700696, fy=470.83759684346785, cx=368.8316828103749, cy=232.23688706965652, size=(752, 480)),
    "interior_zero": dict(k1=-0.01, k2=0.0, p1=0.004, p2=-0.002, fx=300.0, fy=300.0, cx=376.0, cy=240.0, size=(752, 480)),
    "equidistant": dict(k1=0.0, k2=0.0, p1=0.0, p2=0.0, fx=300.0, fy=300.0, cx=376.0, cy=240.0, size=(752, 480)),
}


def _lift_all(model, prm, px):
    import sys
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import camera_models as cm
    import orc
    from harness import synth
    from vins_mono_b200 import load_library
    lib = load_library()
    K = np.array([prm[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")], np.float64)
    out = np.zeros_like(px)
    assert lib.vt_debug_lift_projective_model(model, K.ctypes.data, float(prm.get("xi", 0.0)), px.ctypes.data, len(px), out.ctypes.data) == 0
    cfg = synth.tracker_config_dict()
    cfg.update({k: prm[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")}, camera_model=model, xi=float(prm.get("xi", 0.0)))
    oracle = orc.lift_projective(cfg, px)
    if model == 1:
        rays = np.array([cm.mei_lift(u, v, prm["xi"], prm["k1"], prm["k2"], prm["p1"], prm["p2"], prm["fx"], prm["fy"], prm["cx"], prm["cy"])
                         for u, v in px])
    else:
        rays = np.array([cm.kb_lift(u, v, prm["k1"], prm["k2"], prm["p1"], prm["p2"], prm["fx"], prm["fy"], prm["cx"], prm["cy"])
                         for u, v in px])
    return out, oracle, rays, cm


def _pixel_grid(size, prm):
    w, h = size
    gx, gy = np.meshgrid(np.linspace(1, w - 2, 17), np.linspace(1, h - 2, 13))
    return np.ascontiguousarray(np.r_[np.c_[gx.ravel(), gy.ravel()], [[prm["cx"], prm["cy"]]]])  # incl. the principal point itself


@pytest.mark.parametrize("name", sorted(MEI_SETS))
def test_mei_lift_projective(name):
    """CataCamera::liftProjective (CataCamera.cc:556-625) / z: product host code and CPU oracle against the numpy restatement;
    spaceToPlane (:632-658) inverts it up to the 8-step recursive undistortion."""
    prm = MEI_SETS[name]
    px = _pixel_grid(prm["size"], prm)
    out, oracle, rays, cm = _lift_all(1, prm, px)
    twin = rays[:, :2] / rays[:, 2:3]
    assert np.abs(out - twin).max() < 1e-13 * max(1.0, np.abs(twin).max()) and np.abs(oracle - twin).max() < 1e-13 * max(1.0, np.abs(twin).max())
    assert np.array_equal(out, oracle)  # identical operation sequence in the product and the oracle
    back = np.array([cm.mei_space_to_plane(np.r_[xy, 1.0], prm["xi"], prm["k1"], prm["k2"], prm["p1"], prm["p2"], prm["fx"], prm["fy"],
                                           prm["cx"], prm["cy"]) for xy in out])
    assert np.abs(back - px).max() < 0.05


@pytest.mark.parametrize("name", sorted(KB_SETS))
def test_kannala_brandt_lift_projective(name):
    """EquidistantCamera::liftProjective (EquidistantCamera.cc:428-442) / z.  The reference reads theta off the companion-matrix
    eigenvalues (numpy.roots does the same); the product brackets + Newton-polishes the same root, the oracle uses false position."""
    prm = KB_SETS[name]
    px = _pixel_grid(prm["size"], prm)
    out, oracle, rays, cm = _lift_all(2, prm, px)
    twin = rays[:, :2] / rays[:, 2:3]
    scale = max(1.0, np.abs(twin).max())
    assert np.abs(out - twin).max() < 1e-10 * scale and np.abs(oracle - twin).max() < 1e-10 * scale
    assert np.abs(out - oracle).max() < 1e-13 * scale
    if name != "interior_zero":  # there the reference's own lift is not the inverse of its projection (dropped k5)
        # rays beyond 90 degrees (the 512 x 512 TUM lens in its corners) flip sign on the z = 1 plane: project the 3-D ray with the
        # sign of its z restored
        back = np.array([cm.kb_space_to_plane(np.r_[xy, 1.0] * np.sign(ray[2]), prm["k1"], prm["k2"], prm["p1"], prm["p2"], prm["fx"],
                                              prm["fy"], prm["cx"], prm["cy"]) for xy, ray in zip(out, rays)])
        assert np.abs(back - px).max() < 1e-8
