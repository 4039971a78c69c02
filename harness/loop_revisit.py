"""Rendered revisits for loop verification (test / bench input; not product code).

The synthetic room of harness/synth.py is textured value noise, which FAST and BRIEF see as texture: about 9000 corners per
752x480 frame.  Its trajectory passes the same places again, so two key frames seconds apart can look at the same wall.
This module makes the landmarks of the feature stream FAST corners of rendered frames, back-projected onto the walls, so
that what the estimator tracks is what findConnection describes and matches:
  corner_landmarks   world points of the strongest FAST corners of frames at the given times
  revisit_candidate  the old key frame a ground-truth place recognition would propose
  window_points      a key frame's window points (point_3d in the VIO frame, uv, normalised, ids) from its visible landmarks
  CameraSequence     the same sequence seen through a MEI or KANNALA_BRANDT camera
"""
from __future__ import annotations

import numpy as np

from . import synth


class CameraSequence(synth.Sequence):
    """synth.Sequence (trajectory, room, textures, IMU unchanged) rendered through a MEI (camera_model 1) or KANNALA_BRANDT (2)
    camera of rows x cols pixels; intrinsics in the tracker's order for the model (MEI gamma1 gamma2 u0 v0 k1 k2 p1 p2 plus xi,
    KANNALA_BRANDT mu mv u0 v0 k2 k3 k4 k5).  The pixel rays invert oracle/camera_models.py's spaceToPlane to rounding, so
    that project(lift(pixel)) returns the pixel; the library's own lift is the reference's (8 undistortion steps for MEI)."""

    def __init__(self, camera_model, intrinsics, xi=0.0, **kw):
        super().__init__(**kw)
        self.camera_model, self.intrinsics, self.xi = int(camera_model), [float(v) for v in intrinsics], float(xi)
        assert self.camera_model in (1, 2)

    def lift(self, px):
        """Unit rays (n, 3) of the pixels px (n, 2), vectorised."""
        g1, g2, u0, v0, a, b, c, d = self.intrinsics
        px = np.asarray(px, np.float64).reshape(-1, 2)
        xd, yd = (px[:, 0] - u0) / g1, (px[:, 1] - v0) / g2
        if self.camera_model == 1:  # undistort by fixed-point iteration to convergence, then the unit sphere
            x, y = xd.copy(), yd.copy()
            for _ in range(100):
                r2 = x * x + y * y
                rad = a * r2 + b * r2 * r2
                x = xd - (x * rad + 2.0 * c * x * y + d * (r2 + 2.0 * x * x))
                y = yd - (y * rad + 2.0 * d * x * y + c * (r2 + 2.0 * y * y))
            rho2, xi = x * x + y * y, self.xi
            z = (1.0 - rho2) / 2.0 if xi == 1.0 else 1.0 - xi * (rho2 + 1.0) / (xi + np.sqrt(1.0 + (1.0 - xi * xi) * rho2))
            P = np.stack([x, y, z], 1)
        else:  # theta (1 + k2 t^2 + k3 t^4 + k4 t^6 + k5 t^8) = r: bisection on the increasing part, then Newton
            r, phi = np.hypot(xd, yd), np.arctan2(yd, xd)

            def f(t):
                t2 = t * t
                return t * (1 + t2 * (a + t2 * (b + t2 * (c + t2 * d))))

            grid = np.linspace(0.0, np.pi, 4097)
            fg = f(grid)
            top = int(np.argmax(fg >= r.max())) if (fg >= r.max()).any() else len(grid) - 1
            assert (np.diff(fg[:top + 1]) > 0).all(), "the lens polynomial must increase over the image"
            lo, hi = np.zeros_like(r), np.full_like(r, grid[top])
            for _ in range(60):
                mid = 0.5 * (lo + hi)
                below = f(mid) < r
                lo, hi = np.where(below, mid, lo), np.where(below, hi, mid)
            t = 0.5 * (lo + hi)
            for _ in range(3):
                t2 = t * t
                t = t - (f(t) - r) / (1 + t2 * (3 * a + t2 * (5 * b + t2 * (7 * c + t2 * 9 * d))))
            P = np.stack([np.sin(t) * np.cos(phi), np.sin(t) * np.sin(phi), np.cos(t)], 1)
        return P / np.linalg.norm(P, axis=1)[:, None]

    def space_to_plane(self, Pc):
        """Pixels (n, 2) of the camera-frame points Pc (n, 3): camera_models' spaceToPlane, point by point."""
        from oracle import camera_models as cm
        g1, g2, u0, v0, a, b, c, d = self.intrinsics
        if self.camera_model == 1:
            return np.array([cm.mei_space_to_plane(P, self.xi, a, b, c, d, g1, g2, u0, v0) for P in Pc]).reshape(-1, 2)
        return np.array([cm.kb_space_to_plane(P, a, b, c, d, g1, g2, u0, v0) for P in Pc]).reshape(-1, 2)

    def _pixel_rays(self):
        if self._rays is None:
            u, v = np.meshgrid(np.arange(self.cols, dtype=np.float64), np.arange(self.rows, dtype=np.float64))
            self._rays = self.lift(np.c_[u.ravel(), v.ravel()]).astype(np.float32)
        return self._rays


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
    """Pixel (radtan-distorted, or the CameraSequence's model) and normalised coordinates of pts in the camera at t, and which
    are visible."""
    p, R, *_ = seq.pose(t)
    Pc = (pts - (p + R @ synth.TIC)) @ (R @ synth.RIC)
    z = Pc[:, 2]
    x, y = Pc[:, 0] / z, Pc[:, 1] / z
    if isinstance(seq, CameraSequence):
        uv = np.full((len(Pc), 2), -1.0)
        front = z > 0.3
        if front.any():
            uv[front] = seq.space_to_plane(Pc[front])
        u, v = uv[:, 0], uv[:, 1]
        vis = front & (u > 5) & (u < seq.cols - 5) & (v > 5) & (v < seq.rows - 5)
        return uv, np.c_[x, y], vis
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


def revisit_pair(seq: synth.Sequence, pts, t_old, t_cur, n_win=150):
    """An old key frame (image, P, Q wxyz) at t_old with no window points, and a current one at t_cur (image, P, Q, point_3d,
    uv, norm, ids) with n_win of its visible landmarks, both at their true poses."""
    from oracle import loop_verify as olv
    p, R, *_ = seq.pose(t_cur)
    _, _, vis = project(seq, t_cur, pts)
    ids = np.nonzero(vis)[0]
    ids = ids[np.linspace(0, len(ids) - 1, min(n_win, len(ids))).astype(int)]
    p3d, uv, norm, pid = window_points(seq, t_cur, ids, pts, p, R)
    p0, R0, *_ = seq.pose(t_old)
    return (seq.render(t_old), p0, olv.R_to_quat(R0)), (seq.render(t_cur), p, olv.R_to_quat(R), p3d, uv, norm, pid)
