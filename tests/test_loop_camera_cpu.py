"""CPU checks of loop verification under MEI and KANNALA_BRANDT cameras: the twin's corner lift against
oracle/camera_models.py and the library's host lift, loop_kwargs against tracker_kwargs / estimator_kwargs on the reference's
configuration files, the fisheye revisit sequence's project(lift(pixel)) round trip, the new symbols exported and creation
failing without a GPU.  The fisheye twin is tests/loop_camera_twin.py."""
import glob
import os
import re
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from harness import loop_revisit, synth  # noqa: E402
from loop_camera_twin import lift_corners  # noqa: E402
from oracle import camera_models as cm  # noqa: E402
from oracle import loop_verify as olv  # noqa: E402
from vins_mono_b200 import config  # noqa: E402

CONFIG = os.path.join(ROOT, "tests", "golden", "config")
# (name, camera_model, intrinsics in the tracker's order, xi, (cols, rows)): the reference's MEI and KANNALA_BRANDT files, and
# synthetic sets for MEI xi = 1, a KANNALA_BRANDT interior zero coefficient (the degree-lowering quirk) and all coefficients zero
FILES = ["3dm/3dm_config", "black_box/black_box_config", "cla/cla_config", "tum/tum_config", "realsense/realsense_fisheye_config"]


def camera_sets():
    out = []
    for f in FILES:
        kw = config.loop_kwargs(config.load(os.path.join(CONFIG, f + ".yaml")))
        out.append((f.split("/")[0] if "realsense" not in f else "realsense_fisheye", kw["camera_model"], kw["intrinsics"], kw["xi"],
                    (kw["cols"], kw["rows"])))
    out += [("xi_one", 1, [600.0, 601.0, 370.0, 240.0, -0.05, 0.02, 1e-4, -2e-4], 1.0, (752, 480)),
            ("interior_zero", 2, [300.0, 300.0, 376.0, 240.0, -0.01, 0.0, 0.004, -0.002], 0.0, (752, 480)),
            ("equidistant", 2, [300.0, 300.0, 376.0, 240.0, 0.0, 0.0, 0.0, 0.0], 0.0, (752, 480))]
    return out


SETS = {s[0]: s for s in camera_sets()}


def host_lift(model, intr, xi, px):
    from vins_mono_b200 import load_library
    lib = load_library()
    K, px = np.ascontiguousarray(intr, np.float64), np.ascontiguousarray(px, np.float64)
    out = np.zeros_like(px)
    assert lib.vt_debug_lift_projective_model(model, K.ctypes.data, float(xi), px.ctypes.data, len(px), out.ctypes.data) == 0
    return out


def ulps(a, b):
    """Distance in float32 units in the last place (same-sign finite values)."""
    ia, ib = np.asarray(a, np.float32).view(np.int32).astype(np.int64), np.asarray(b, np.float32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


@pytest.mark.parametrize("name", sorted(SETS))
def test_twin_corner_lift_equals_camera_models_and_host_lift(name):
    _, model, intr, xi, (w, h) = SETS[name]
    gx, gy = np.meshgrid(np.arange(3, w - 3, 9), np.arange(3, h - 3, 7))  # FAST corners are integer pixels 3 inside
    px = np.r_[np.c_[gx.ravel(), gy.ravel()], [[round(intr[2]), round(intr[3])]]].astype(np.float64)
    twin = lift_corners(model, intr, xi, px).astype(np.float32)
    a, b, c, d, e, f, g, hh = intr
    rays = np.array([cm.mei_lift(u, v, xi, e, f, g, hh, a, b, c, d) if model == 1 else cm.kb_lift(u, v, e, f, g, hh, a, b, c, d)
                     for u, v in px])
    assert np.array_equal(twin, (rays[:, :2] / rays[:, 2:3]).astype(np.float32))
    host = host_lift(model, intr, xi, px).astype(np.float32)
    if model == 1:  # the same operation sequence as the host code
        assert np.array_equal(twin, host)
    else:  # np.roots against bracketing + Newton: the same root to rounding, so at most one float ulp apart
        d = ulps(twin, host)
        print(name, "corners whose float lift differs from the host's:", int((d.max(1) > 0).sum()), "of", len(px))
        assert d.max() <= 1


def test_twin_pinhole_default_is_unchanged():
    intr = [synth.FX, synth.FY, synth.CX, synth.CY, synth.K1, synth.K2, synth.P1, synth.P2]
    px = np.random.default_rng(3).uniform(0, 700, (200, 2))
    assert np.array_equal(lift_corners(0, intr, 0.0, px), olv.lift_pinhole(intr, px))


def test_loop_kwargs_read_what_the_tracker_and_estimator_read():
    files = [f for f in sorted(glob.glob(os.path.join(CONFIG, "*", "*.yaml"))) if int(config.load(f).get("loop_closure", 0))]
    assert len(files) == 6
    for f in files:
        cfg = config.load(f)
        kw, trk, est = config.loop_kwargs(cfg), config.tracker_kwargs(cfg), config.estimator_kwargs(cfg)
        assert (kw["rows"], kw["cols"], kw["camera_model"], kw["xi"]) == (trk["rows"], trk["cols"], trk["camera_model"], trk["xi"]), f
        assert kw["intrinsics"] == [trk[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")], f
        assert np.array_equal(kw["ric"], est["ric"]) and np.array_equal(kw["tic"], est["tic"]), f
        if int(cfg["estimate_extrinsic"]) != 2:
            assert np.abs(kw["ric"] - np.asarray(cfg["extrinsicRotation"], float)).max() < 1e-6, f
            assert np.array_equal(kw["tic"], np.asarray(cfg["extrinsicTranslation"], float).reshape(3)), f
        # a calibrated extrinsic replaces the file's (estimate_extrinsic = 2)
        kw2 = config.loop_kwargs(cfg, ric=synth.RIC, tic=synth.TIC)
        assert np.array_equal(kw2["ric"], synth.RIC) and np.array_equal(kw2["tic"], synth.TIC)
    models = {os.path.basename(f): config.loop_kwargs(config.load(f))["camera_model"] for f in files}
    assert models["black_box_config.yaml"] == 1 and models["cla_config.yaml"] == 2 and models["realsense_fisheye_config.yaml"] == 2


@pytest.mark.parametrize("name", sorted(SETS))
def test_fisheye_sequence_project_inverts_lift(name):
    _, model, intr, xi, (w, h) = SETS[name]
    seq = loop_revisit.CameraSequence(model, intr, xi, seed=0, duration=2.0, rows=h, cols=w)
    gx, gy = np.meshgrid(np.arange(0, w, 4.0), np.arange(0, h, 4.0))
    px = np.r_[np.c_[gx.ravel(), gy.ravel()], [[w - 1.0, h - 1.0], intr[2:4]]]
    rays = seq.lift(px)
    assert np.isfinite(rays).all()
    assert np.abs(seq.space_to_plane(rays) - px).max() < 1e-6
    # through loop_revisit.project: world points 4 m along the rays of the camera at t, in front of it
    t = 0.7
    p, R, *_ = seq.pose(t)
    R_wc, o = R @ synth.RIC, p + R @ synth.TIC
    sel = rays[:, 2] > 0.2
    world = o + (4.0 * rays[sel]) @ R_wc.T
    uv, norm, vis = loop_revisit.project(seq, t, world)
    inner = (px[sel, 0] > 5) & (px[sel, 0] < w - 5) & (px[sel, 1] > 5) & (px[sel, 1] < h - 5)
    assert np.array_equal(vis, inner & (4.0 * rays[sel, 2] > 0.3))
    assert np.abs(uv - px[sel]).max() < 1e-6
    assert np.abs(norm - rays[sel, :2] / rays[sel, 2:3]).max() < 1e-9


def test_camera_symbols_exported_and_no_gpu_fails_loudly():
    import torch
    from vins_mono_b200 import build, load_library
    build.build()
    lib = load_library()
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "vinsb200", "loop_camera.h")).read(), flags=re.S)
    names = sorted(set(re.findall(r"\b(vp_[a-z0-9_]+)\s*\(", src)))
    assert names == ["vp_batch_loop_enable_camera", "vp_debug_lift", "vp_loop_enable_camera"]
    assert all(hasattr(lib, n) for n in names)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from vins_mono_b200 import pose_graph as pg
    with pytest.raises(RuntimeError):
        pg.debug_lift(1, SETS["3dm"][2], SETS["3dm"][3], np.zeros((4, 2)))
    with pytest.raises(RuntimeError):
        pg.PoseGraph()
