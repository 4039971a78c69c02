"""cv2 / numpy twin of KeyFrame::findConnection (pose_graph/src/keyframe.cpp) and what it needs.

Stages, restated from the reference:
  * computeBRIEFPoint (keyframe.cpp:87-113): cv::FAST(image, 20, nonmax = true), then BRIEF on those corners and
    liftProjective of each corner, stored as float (cv::Point2f).
  * computeWindowBRIEFPoint (:75-85): BRIEF on the window points point_2d_uv.
  * DVision BRIEF::compute (BRIEF.cpp:39-106): GaussianBlur(9 x 9, sigma 2) of the image, then for each of the 256 pairs
    (x1, y1, x2, y2) of the pattern bit i = blurred(y1, x1) < blurred(y2, x2), where x1 = (int)(pt.x + x1_i) in float
    arithmetic (truncation toward zero); a test with either end outside the image leaves the bit 0.
  * searchInAera (:121-150): brute-force Hamming distance; best = the first index of the smallest distance, starting from
    128 with a strict <; accepted when best < 80.
  * findConnection (:259-520): more than MIN_LOOP_NUM = 25 matches, then PnPRANSAC (:200-256): solvePnPRansac(3-D window
    points, old normalised points, K = I, no distortion, extrinsic guess from the current VIO pose, 100 iterations,
    10 / 460, 0.99); more than 25 inliers; relative_t = R_old^T (T_cur - T_old), relative_q = R_old^T R_cur,
    relative_yaw = normalizeAngle(yaw(R_cur) - yaw(R_old)); accepted when |yaw| < 30 and |t| < 20.

Every integer stage (blur, FAST, BRIEF, matching) is restated in numpy and checked against cv2 where cv2 has the stage.
"""
from __future__ import annotations

import math
import os

import numpy as np

FAST_THRESHOLD = 20
BRIEF_KSIZE, BRIEF_SIGMA = 9, 2.0
MATCH_INIT, MATCH_ACCEPT = 128, 80
MIN_LOOP_NUM = 25
PNP_ITERATIONS, PNP_THRESHOLD, PNP_CONFIDENCE = 100, 10.0 / 460.0, 0.99

# the 16-pixel Bresenham circle of radius 3 in cyclic order, (dx, dy)
CIRCLE = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3),
          (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3)]


def load_pattern(path=None):
    """(256, 4) int32: x1 y1 x2 y2."""
    if path is None:
        path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "brief_pattern_256.txt")
    return np.loadtxt(path, dtype=np.int32, comments="#").reshape(256, 4)


# ---- Gaussian blur as OpenCV does it for 8-bit images: a fixed-point kernel with 8 fraction bits, a row pass kept
#      exact in 16 bits, a column pass in 32 bits, rounded half up; border reflect-101.

def gaussian_kernel_q8(n=BRIEF_KSIZE, sigma=BRIEF_SIGMA):
    scale2 = -0.125 / (sigma * sigma)  # x runs over twice the tap offset: 1 - n, 3 - n, ..
    half = (n - 1) // 2
    vals = [math.exp(float(x * x) * scale2) for x in range(1 - n, 0, 2)][:half]
    s = 2.0 * sum(vals) + 1.0
    mul = 1.0 / s
    k = [v * mul for v in vals]
    out, err, acc = [0] * n, 0.0, 0
    for i in range(half):
        adj = k[i] * 256.0 + err
        v = int(np.rint(adj))
        err = adj - v
        out[i] = out[n - 1 - i] = v
        acc += v
    out[half] = 256 - 2 * acc
    return np.array(out, np.int64)


def _reflect101(idx, n):
    idx = np.abs(idx)
    return np.where(idx >= n, 2 * (n - 1) - idx, idx)


def gaussian_blur(img):
    img = np.asarray(img, np.uint8)
    k = gaussian_kernel_q8()
    r = len(k) // 2
    H, W = img.shape
    xs, ys = np.arange(W), np.arange(H)
    rows = sum(k[i] * img[:, _reflect101(xs + i - r, W)].astype(np.int64) for i in range(len(k)))
    cols = sum(k[j] * rows[_reflect101(ys + j - r, H), :] for j in range(len(k)))
    return ((cols + 32768) >> 16).astype(np.uint8)


# ---- FAST-9 with non-maximum suppression (cv::FAST, TYPE_9_16)

def fast_scores(img, threshold=FAST_THRESHOLD):
    """Score map (int32, 0 where no corner): a pixel at least 3 from every border is a corner when 9 contiguous circle
    pixels are all brighter than v + t or all darker than v - t; its score is the largest such margin minus 1:
    max(t, max over 9-arcs of min(v - p), max over 9-arcs of min(p - v)) - 1."""
    img = np.asarray(img, np.int32)
    H, W = img.shape
    v = img[3:H - 3, 3:W - 3]
    d = np.stack([v - img[3 + dy:H - 3 + dy, 3 + dx:W - 3 + dx] for dx, dy in CIRCLE])  # v - p
    dd = np.concatenate([d, d[:8]])
    arc_min_dark = np.stack([dd[s:s + 9].min(0) for s in range(16)]).max(0)      # darker ring: v - p > t
    arc_min_bright = np.stack([(-dd[s:s + 9]).min(0) for s in range(16)]).max(0)  # brighter ring: p - v > t
    corner = (arc_min_dark > threshold) | (arc_min_bright > threshold)
    score = np.maximum(threshold, np.maximum(arc_min_dark, arc_min_bright)) - 1
    out = np.zeros((H, W), np.int32)
    out[3:H - 3, 3:W - 3] = np.where(corner, score, 0)
    return out


def fast(img, threshold=FAST_THRESHOLD):
    """Corners (n, 2) int32 (x, y) in row-major order and their scores; a corner survives when its score is strictly
    greater than each of its 8 neighbours' (0 for a non-corner)."""
    s = fast_scores(img, threshold)
    H, W = s.shape
    p = np.pad(s, 1)
    keep = s > 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            if dx or dy:
                keep &= s > p[1 + dy:1 + dy + H, 1 + dx:1 + dx + W]
    ys, xs = np.nonzero(keep)
    return np.stack([xs, ys], 1).astype(np.int32), s[ys, xs]


# ---- BRIEF

def brief(img, pts, pattern):
    """Descriptors (n, 4) uint64, bit i in word i // 64 at position i % 64, of the float32 points pts (n, 2)."""
    im = gaussian_blur(img)
    H, W = im.shape
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    pat = np.asarray(pattern, np.float32)
    x1 = np.trunc(pts[:, :1] + pat[None, :, 0]).astype(np.int64)
    y1 = np.trunc(pts[:, 1:] + pat[None, :, 1]).astype(np.int64)
    x2 = np.trunc(pts[:, :1] + pat[None, :, 2]).astype(np.int64)
    y2 = np.trunc(pts[:, 1:] + pat[None, :, 3]).astype(np.int64)
    ok = (x1 >= 0) & (x1 < W) & (y1 >= 0) & (y1 < H) & (x2 >= 0) & (x2 < W) & (y2 >= 0) & (y2 < H)
    a = im[np.clip(y1, 0, H - 1), np.clip(x1, 0, W - 1)]
    b = im[np.clip(y2, 0, H - 1), np.clip(x2, 0, W - 1)]
    bits = (ok & (a < b)).astype(np.uint64)
    words = np.zeros((len(pts), 4), np.uint64)
    for w in range(4):
        words[:, w] = (bits[:, 64 * w:64 * w + 64] << np.arange(64, dtype=np.uint64)[None, :]).sum(1, dtype=np.uint64)
    return words


def hamming(a, b):
    """(na, nb) int32 Hamming distances between descriptor sets."""
    x = np.bitwise_xor(np.asarray(a, np.uint64)[:, None, :], np.asarray(b, np.uint64)[None, :, :])
    by = x.view(np.uint8).reshape(x.shape[0], x.shape[1], 32)
    return np.unpackbits(by, axis=2).sum(2).astype(np.int32)


def match(desc_cur, desc_old):
    """searchByBRIEFDes: per current descriptor the matched old index (-1 none) and its distance."""
    n = len(desc_cur)
    idx, dist = np.full(n, -1, np.int32), np.full(n, MATCH_INIT, np.int32)
    if n == 0 or len(desc_old) == 0:
        return idx, dist
    D = hamming(desc_cur, desc_old)
    best = D.argmin(1)  # the first index of the smallest distance
    bd = D[np.arange(n), best]
    hit = (bd < MATCH_INIT) & (bd < MATCH_ACCEPT)
    idx[hit] = best[hit]
    dist[hit] = bd[hit]
    return idx, dist


# ---- camera and poses

def lift_pinhole(intr, px):
    """PinholeCamera::liftProjective with the recursive distortion model (8 iterations), then the division by z."""
    fx, fy, cx, cy, k1, k2, p1, p2 = [float(v) for v in intr]
    px = np.asarray(px, np.float64).reshape(-1, 2)
    mx = (1.0 / fx) * px[:, 0] + (-cx / fx)
    my = (1.0 / fy) * px[:, 1] + (-cy / fy)
    ux, uy = mx.copy(), my.copy()
    if not (k1 == 0 and k2 == 0 and p1 == 0 and p2 == 0):
        for _ in range(8):
            x2, y2, xy = ux * ux, uy * uy, ux * uy
            rho2 = x2 + y2
            rad = k1 * rho2 + k2 * rho2 * rho2
            dx = ux * rad + 2.0 * p1 * xy + p2 * (rho2 + 2.0 * x2)
            dy = uy * rad + 2.0 * p2 * xy + p1 * (rho2 + 2.0 * y2)
            ux, uy = mx - dx, my - dy
    return np.stack([ux, uy], 1)


def quat_to_R(q):
    w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def R_to_quat(R):
    from scipy.spatial.transform import Rotation
    x, y, z, w = Rotation.from_matrix(R).as_quat()
    q = np.array([w, x, y, z])
    return q if q[0] >= 0 else -q


def R2ypr_deg(R):
    n, o, a = R[:, 0], R[:, 1], R[:, 2]
    y = math.atan2(n[1], n[0])
    p = math.atan2(-n[2], n[0] * math.cos(y) + n[1] * math.sin(y))
    r = math.atan2(a[0] * math.sin(y) - a[1] * math.cos(y), -o[0] * math.sin(y) + o[1] * math.cos(y))
    return np.degrees([y, p, r])


def normalize_angle(a):
    if a > 180.0:
        return a - 360.0
    if a < -180.0:
        return a + 360.0
    return a


def relative_pose(R_pnp, T_pnp, vio_R_cur, vio_T_cur, ric, tic):
    """From the world-to-old-camera PnP pose to the old body pose in the current VIO frame (PnPRANSAC's tail), then the
    loop measurement of findConnection: (relative_t, relative_q wxyz, relative_yaw)."""
    R_w_c_old = R_pnp.T
    T_w_c_old = R_w_c_old @ (-T_pnp)
    R_old = R_w_c_old @ ric.T
    T_old = T_w_c_old - R_old @ tic
    rel_t = R_old.T @ (vio_T_cur - T_old)
    rel_q = R_to_quat(R_old.T @ vio_R_cur)
    rel_yaw = normalize_angle(R2ypr_deg(vio_R_cur)[0] - R2ypr_deg(R_old)[0])
    return rel_t, rel_q, rel_yaw, R_old, T_old


class KeyFrame:
    """A key frame as the reference constructs it: the window points and their descriptors, the FAST corners, their
    descriptors and normalised coordinates."""

    def __init__(self, image, vio_T, vio_R, p3d, uv, norm, ids, pattern, intr):
        self.image = np.asarray(image, np.uint8)
        self.vio_T, self.vio_R = np.asarray(vio_T, np.float64), np.asarray(vio_R, np.float64)
        self.p3d = np.asarray(p3d, np.float32).reshape(-1, 3)
        self.uv = np.asarray(uv, np.float32).reshape(-1, 2)
        self.norm = np.asarray(norm, np.float32).reshape(-1, 2)
        self.ids = np.asarray(ids, np.float64).reshape(-1)
        self.win_desc = brief(self.image, self.uv, pattern)
        self.kp, self.kp_score = fast(self.image)
        self.kp_desc = brief(self.image, self.kp.astype(np.float32), pattern)
        self.kp_norm = lift_pinhole(intr, self.kp.astype(np.float64)).astype(np.float32)


def find_connection(cur: KeyFrame, old: KeyFrame, ric, tic):
    """Returns a dict: matches (window index -> old corner index), n_matches, and when PnP ran its cv2 result
    (inlier count, relative pose, accepted)."""
    import cv2
    idx, _ = match(cur.win_desc, old.kp_desc)
    sel = np.nonzero(idx >= 0)[0]
    out = dict(match_idx=idx, n_matches=len(sel), n_inliers=0, accepted=False)
    if len(sel) <= MIN_LOOP_NUM:
        return out
    p3 = cur.p3d[sel]
    p2 = old.kp_norm[idx[sel]]
    R_w_c = cur.vio_R @ ric
    T_w_c = cur.vio_T + cur.vio_R @ tic
    R_init = R_w_c.T
    rvec0, _ = cv2.Rodrigues(R_init)
    tvec0 = (-(R_init @ T_w_c)).reshape(3, 1)
    ok, rvec, tvec, inl = cv2.solvePnPRansac(p3, p2, np.eye(3), None, rvec0.copy(), tvec0.copy(), True, PNP_ITERATIONS,
                                             PNP_THRESHOLD, PNP_CONFIDENCE)
    inl = np.zeros(0, np.int64) if inl is None else inl.reshape(-1)
    R_pnp, _ = cv2.Rodrigues(rvec)
    rel_t, rel_q, rel_yaw, R_old, T_old = relative_pose(R_pnp, tvec.reshape(3), cur.vio_R, cur.vio_T, ric, tic)
    out.update(n_inliers=len(inl), inliers=sel[inl], rel_t=rel_t, rel_q=rel_q, rel_yaw=rel_yaw, R_old=R_old, T_old=T_old)
    out["accepted"] = bool(len(inl) > MIN_LOOP_NUM and abs(rel_yaw) < 30.0 and np.linalg.norm(rel_t) < 20.0)
    return out
