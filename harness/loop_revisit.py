"""Rendered revisits for loop verification (test / bench input; not product code).

The synthetic room of harness/synth.py is textured value noise, which FAST and BRIEF see as texture: about 9000 corners per
752x480 frame.  Its trajectory passes the same places again, so two key frames seconds apart can look at the same wall.
This module makes the landmarks of the feature stream FAST corners of rendered frames, back-projected onto the walls, so
that what the estimator tracks is what findConnection describes and matches:
  corner_landmarks   world points of the strongest FAST corners of frames at the given times
  revisit_candidate  the old key frame a ground-truth place recognition would propose
  window_points      a key frame's window points (point_3d in the VIO frame, uv, normalised, ids) from its visible landmarks
"""
from __future__ import annotations

import numpy as np

from . import synth


def _cast(seq, o, d):
    """Ray / room-box intersection: the wall points o + t d."""
    lo, hi = seq.room_lo, seq.room_hi
    with np.errstate(divide="ignore", invalid="ignore"):
        tt = np.where(d > 0, (hi - o) / d, (lo - o) / d)
    tt = np.where(np.isfinite(tt), tt, 1e9)
    return o + d * tt.min(1)[:, None]


def corner_landmarks(seq: synth.Sequence, times, per_frame=400, margin=12):
    """World points of the per_frame strongest FAST (20, non-max suppression) corners of the frames rendered at `times`."""
    import cv2
    rays = seq._pixel_rays().astype(np.float64)
    pts = []
    for t in times:
        img = seq.render(t)
        kp = cv2.FastFeatureDetector_create(20, True).detect(img)
        kp = [k for k in kp if margin < k.pt[0] < seq.cols - margin and margin < k.pt[1] < seq.rows - margin]
        kp.sort(key=lambda k: -k.response)
        px = np.array([[int(k.pt[0]), int(k.pt[1])] for k in kp[:per_frame]])
        p, R, *_ = seq.pose(t)
        R_wc, o = R @ synth.RIC, p + R @ synth.TIC
        d = rays[px[:, 1] * seq.cols + px[:, 0]] @ R_wc.T
        pts.append(_cast(seq, o[None, :], d))
    return np.concatenate(pts)


def project(seq: synth.Sequence, t, pts):
    """Pixel (radtan-distorted) and normalised coordinates of pts in the camera at t, and which are visible."""
    p, R, *_ = seq.pose(t)
    Pc = (pts - (p + R @ synth.TIC)) @ (R @ synth.RIC)
    z = Pc[:, 2]
    x, y = Pc[:, 0] / z, Pc[:, 1] / z
    r2 = x * x + y * y
    rad = synth.K1 * r2 + synth.K2 * r2 * r2
    xd = x + x * rad + 2 * synth.P1 * x * y + synth.P2 * (r2 + 2 * x * x)
    yd = y + y * rad + 2 * synth.P2 * x * y + synth.P1 * (r2 + 2 * y * y)
    u, v = synth.FX * xd + synth.CX, synth.FY * yd + synth.CY
    vis = (z > 0.3) & (u > 5) & (u < seq.cols - 5) & (v > 5) & (v < seq.rows - 5) & (r2 < 1.2)
    return np.c_[u, v], np.c_[x, y], vis


def window_points(seq: synth.Sequence, t, ids, pts, vio_P, vio_R):
    """point_3d (in the key frame's VIO frame: the body-frame point carried by the VIO pose), point_2d_uv, point_2d_norm and
    point_id of the landmarks `ids` visible at t."""
    ids = np.asarray(ids, np.int64)
    uv, norm, vis = project(seq, t, pts[ids])
    ids, uv, norm = ids[vis], uv[vis], norm[vis]
    p, R, *_ = seq.pose(t)
    body = (pts[ids] - p) @ R
    p3d = body @ np.asarray(vio_R).T + np.asarray(vio_P)
    return p3d.astype(np.float32), uv.astype(np.float32), norm.astype(np.float32), ids.astype(np.float64)


def revisit_candidate(seq: synth.Sequence, stamps, t_cur, min_age=3.0, max_dist=1.0, max_yaw=15.0):
    """Index of the closest earlier key frame at least min_age older, within max_dist and max_yaw of the current pose
    (ground truth), or None."""
    from oracle import pose_graph as opg
    p1, R1, *_ = seq.pose(t_cur)
    best = None
    for idx, t in enumerate(stamps):
        if t > t_cur - min_age:
            break
        p0, R0, *_ = seq.pose(t)
        dyaw = opg.normalize_angle(opg.R2ypr(R1)[0] - opg.R2ypr(R0)[0])
        dist = np.linalg.norm(p1 - p0)
        if abs(dyaw) < max_yaw and dist < max_dist and (best is None or dist < best[1]):
            best = (idx, dist)
    return None if best is None else best[0]
