"""The reference's YAML configuration files (config/*/*.yaml, OpenCV FileStorage format) -> the two C-ABI configurations.

Mirrors feature_tracker/src/parameters.cpp:37-74, vins_estimator/src/parameters.cpp:42-137 and the camera part read by
camodocal's CameraFactory (camera_model/src/camera_models/{Pinhole,Cata,Equidistant}Camera.cc readFromYamlFile): the same keys, the same
defaults (FOCAL_LENGTH = 460, WINDOW_SIZE = 10, INIT_DEPTH = 5, FREQ 0 -> 100, TR only with rolling_shutter, the extrinsic rotation
normalised through a quaternion, identity / zero extrinsics when estimate_extrinsic = 2).  `max_solver_time` is read and reported
but not applied: the library has no wall-clock cap (DESIGN.md 5).

    cfg = load("config/euroc/euroc_config.yaml")
    trk = FeatureTracker(**tracker_kwargs(cfg));  est = Estimator(**estimator_kwargs(cfg))
"""
from __future__ import annotations

import numpy as np
import yaml

CAMERA_MODELS = {"PINHOLE": 0, "MEI": 1, "KANNALA_BRANDT": 2}


class _Loader(yaml.SafeLoader):
    pass


def _opencv_matrix(loader, node):
    m = loader.construct_mapping(node, deep=True)
    data = np.asarray(m["data"], np.float64 if m.get("dt", "d") in ("d", "f") else np.int64)
    return data.reshape(int(m["rows"]), int(m["cols"]))


_Loader.add_constructor("tag:yaml.org,2002:opencv-matrix", _opencv_matrix)


def loads(text: str) -> dict:
    """Parses the text of an OpenCV FileStorage YAML file (the "%YAML:1.0" directive and !!opencv-matrix nodes included)."""
    lines = text.splitlines()
    if lines and lines[0].startswith("%YAML"):
        lines = lines[1:]
    if lines and lines[0].strip() == "---":
        lines = lines[1:]
    return yaml.load("\n".join(lines), Loader=_Loader) or {}


def load(path: str) -> dict:
    with open(path) as f:
        return loads(f.read())


def _normalised_rotation(R):
    """Eigen::Quaterniond Q(R); R = Q.normalized()  (vins_estimator/src/parameters.cpp:100-101)."""
    from scipy.spatial.transform import Rotation
    q = Rotation.from_matrix(np.asarray(R, float)).as_quat()
    return Rotation.from_quat(q / np.linalg.norm(q)).as_matrix()


def tracker_kwargs(cfg: dict, fisheye_mask=None) -> dict:
    """Keyword arguments of vins_mono_b200.FeatureTracker / TrackerBatch.  fisheye_mask (uint8 image, 255 = usable) must be given when
    the file says fisheye: 1 (the reference loads config/fisheye_mask.jpg)."""
    model = str(cfg.get("model_type", "PINHOLE")).strip()
    if model not in CAMERA_MODELS:
        raise ValueError(f"camera model {model!r} is not supported (PINHOLE, MEI, KANNALA_BRANDT)")
    proj, dist = cfg.get("projection_parameters", {}), cfg.get("distortion_parameters", {}) or {}
    kw = dict(rows=int(cfg["image_height"]), cols=int(cfg["image_width"]), max_cnt=int(cfg["max_cnt"]), min_dist=int(cfg["min_dist"]),
              freq=int(cfg["freq"]) or 100, equalize=int(cfg["equalize"]), fisheye=int(cfg.get("fisheye", 0)), focal_length=460,
              f_threshold=float(cfg["F_threshold"]), camera_model=CAMERA_MODELS[model], xi=0.0)
    if model == "PINHOLE":
        kw.update(fx=proj["fx"], fy=proj["fy"], cx=proj["cx"], cy=proj["cy"], k1=dist.get("k1", 0.0), k2=dist.get("k2", 0.0),
                  p1=dist.get("p1", 0.0), p2=dist.get("p2", 0.0))
    elif model == "MEI":
        kw.update(fx=proj["gamma1"], fy=proj["gamma2"], cx=proj["u0"], cy=proj["v0"], k1=dist.get("k1", 0.0), k2=dist.get("k2", 0.0),
                  p1=dist.get("p1", 0.0), p2=dist.get("p2", 0.0), xi=float(cfg["mirror_parameters"]["xi"]))
    else:
        kw.update(fx=proj["mu"], fy=proj["mv"], cx=proj["u0"], cy=proj["v0"], k1=proj["k2"], k2=proj["k3"], p1=proj["k4"], p2=proj["k5"])
    for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2"):
        kw[k] = float(kw[k])
    if kw["fisheye"]:
        if fisheye_mask is None:
            raise ValueError("fisheye: 1 needs the mask image (config/fisheye_mask.jpg in the reference)")
        kw["fisheye_mask"] = fisheye_mask
    return kw


def estimator_kwargs(cfg: dict, max_features: int = 1000) -> dict:
    """Keyword arguments of vins_mono_b200.Estimator / EstimatorBatch."""
    ee = int(cfg["estimate_extrinsic"])
    if ee == 2:
        ric, tic = np.eye(3), np.zeros(3)
    else:
        ric = _normalised_rotation(cfg["extrinsicRotation"])
        tic = np.asarray(cfg["extrinsicTranslation"], float).reshape(3)
    return dict(window_size=10, max_features=max_features, num_iterations=int(cfg["max_num_iterations"]), estimate_extrinsic=ee,
                estimate_td=int(cfg.get("estimate_td", 0)), focal_length=460.0, keyframe_parallax=float(cfg["keyframe_parallax"]),
                acc_n=float(cfg["acc_n"]), gyr_n=float(cfg["gyr_n"]), acc_w=float(cfg["acc_w"]), gyr_w=float(cfg["gyr_w"]),
                g_norm=float(cfg["g_norm"]), init_depth=5.0, td=float(cfg.get("td", 0.0)),
                tr=float(cfg.get("rolling_shutter_tr", 0.0)) if int(cfg.get("rolling_shutter", 0)) else 0.0, row=float(cfg.get("image_height", 0)),  # absent keys read as 0 (cv::FileStorage), e.g. config/simulation
                tic=tic, ric=ric)


def loop_kwargs(cfg: dict, ric=None, tic=None) -> dict:
    """What loop verification needs from the file (pose_graph_node.cpp reads the same YAML as the tracker): the image size, the
    camera model, its intrinsics (in vt_config's order for that model) and xi as tracker_kwargs reads them, and qic / tic as
    estimator_kwargs normalises them.  ric / tic replace the file's extrinsic, e.g. with the estimator's calibration when
    estimate_extrinsic = 2.

        kw = loop_kwargs(cfg)
        g.enable_loop(loop_config(kw["rows"], kw["cols"], kw["intrinsics"], kw["ric"], kw["tic"], pattern), kw["camera_model"], kw["xi"])
    """
    trk = tracker_kwargs(dict(cfg, fisheye=0))  # the fisheye mask only concerns the tracker
    est = estimator_kwargs(cfg)
    return dict(rows=trk["rows"], cols=trk["cols"], camera_model=trk["camera_model"], xi=trk["xi"],
                intrinsics=[trk[k] for k in ("fx", "fy", "cx", "cy", "k1", "k2", "p1", "p2")],
                ric=np.asarray(est["ric"] if ric is None else ric, float).reshape(3, 3),
                tic=np.asarray(est["tic"] if tic is None else tic, float).reshape(3))


def ignored(cfg: dict) -> dict:
    """Keys of the file that have no effect here (reported so that nothing is dropped silently)."""
    return {k: cfg[k] for k in ("max_solver_time", "show_track", "loop_closure", "fast_relocalization", "load_previous_pose_graph",
                                "pose_graph_save_path", "save_image", "visualize_imu_forward", "visualize_camera_size",
                                "image_topic", "imu_topic", "output_path") if k in cfg}
