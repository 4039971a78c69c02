"""EuRoC-shaped synthetic visual-inertial sequences (test/bench input generator; not product code).

One sequence = a camera (752x480 mono8 @ 20 Hz) and an IMU (200 Hz) rigidly mounted on a MAV-like
body flying a smooth analytic trajectory inside a textured box room.  Calibration (PINHOLE + radtan,
imu-camera extrinsics, IMU noise densities, gravity) is the reference's EuRoC configuration
(config/euroc/euroc_config.yaml:9-42,59-63).  The trajectory is analytic (sums of sinusoids with
EuRoC-like extents/speeds) so position, velocity, acceleration and body rates are exact; SURVEY.md
proposed replaying the EuRoC ground-truth CSVs, which do not travel to the GPU box (harness/euroc_format.py reads and writes the
dataset's ASL directory layout, so a downloaded sequence or an exported synthetic one feeds the same replay driver).

IMU model (the one Estimator::processIMU inverts, vins_estimator/src/estimator.cpp:107-114):
    acc = R_wb^T (a_w + g) + b_a + n_a,   gyr = w_b + b_g + n_g,   g = (0, 0, 9.81007).
"""
from __future__ import annotations

import os

import numpy as np

G_NORM = 9.81007
ROWS, COLS = 480, 752
FX, FY, CX, CY = 461.6, 460.3, 363.0, 248.1
K1, K2, P1, P2 = -0.2917, 0.08228, 5.333e-05, -1.578e-04
RIC = np.array([[0.0148655429818, -0.999880929698, 0.00414029679422],
                [0.999557249008, 0.0149672133247, 0.025715529948],
                [-0.0257744366974, 0.00375618835797, 0.999660727178]])
TIC = np.array([-0.0216401454975, -0.064676986768, 0.00981073058949])
ACC_N, GYR_N, ACC_W, GYR_W = 0.08, 0.004, 0.00004, 2.0e-6

# body axes in the world at zero attitude: body x up, body z forward (EuRoC IMU mounting)
R_WB0 = np.array([[0.0, 0.0, 1.0], [0.0, -1.0, 0.0], [1.0, 0.0, 0.0]])


def _rz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def _ry(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1.0, 0], [-s, 0, c]])


def _rx(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1.0, 0, 0], [0, c, -s], [0, s, c]])


def rot_to_quat_wxyz(R):
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0) * 2
        q = np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    else:
        i = int(np.argmax(np.diag(R)))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k]) * 2
        q = np.zeros(4)
        q[0] = (R[k, j] - R[j, k]) / s
        q[1 + i] = 0.25 * s
        q[1 + j] = (R[j, i] + R[i, j]) / s
        q[1 + k] = (R[k, i] + R[i, k]) / s
    return q / np.linalg.norm(q)


class _Harmonics:
    """sum_k a_k sin(w_k t + p_k) with exact derivatives."""

    def __init__(self, amps, freqs, phases):
        self.a, self.w, self.p = map(np.asarray, (amps, freqs, phases))

    def val(self, t):
        return float(np.sum(self.a * np.sin(self.w * t + self.p)))

    def d1(self, t):
        return float(np.sum(self.a * self.w * np.cos(self.w * t + self.p)))

    def d2(self, t):
        return float(np.sum(-self.a * self.w ** 2 * np.sin(self.w * t + self.p)))


class Sequence:
    def __init__(self, seed=0, duration=30.0, cam_hz=20.0, imu_hz=200.0, rows=ROWS, cols=COLS,
                 pixel_noise=2.0, imu_noise=True, t0=0.0, rot_gain=1.0):
        self.seed, self.duration, self.cam_hz, self.imu_hz = seed, duration, cam_hz, imu_hz
        self.rows, self.cols, self.pixel_noise, self.imu_noise, self.t0 = rows, cols, pixel_noise, imu_noise, t0
        rng = np.random.default_rng(1000 + seed)
        two_pi = 2 * np.pi

        def harm(a1, a2, f1, f2):
            return _Harmonics([a1, a2], [two_pi * f1 * rng.uniform(0.8, 1.2), two_pi * f2 * rng.uniform(0.8, 1.2)],
                              rng.uniform(0, two_pi, 2))

        # extents ~ +-2.5 m horizontally, +-0.6 m vertically, peak speed ~1.5 m/s (EuRoC MH_01-like)
        self.px, self.py, self.pz = harm(2.2, 0.5, 0.05, 0.17), harm(1.8, 0.4, 0.07, 0.21), harm(0.5, 0.15, 0.09, 0.3)
        # rot_gain > 1 speeds the attitude harmonics up ("rotation movement is needed": the online extrinsic calibration,
        # ESTIMATE_EXTRINSIC = 2, only converges under rotational excitation); 1.0 leaves every existing sequence unchanged
        g_ = float(rot_gain)
        self.yaw = harm(1.2, 0.3, 0.04 * g_, 0.13 * g_)
        self.pitch, self.roll = harm(0.18, 0.05, 0.11 * g_, 0.37 * g_), harm(0.15, 0.05, 0.09 * g_, 0.41 * g_)
        self.ba = np.array([0.02, -0.015, 0.03]) + 0 * rng.normal(0, 1, 3)
        self.bg = np.array([0.003, -0.002, 0.001])
        ext = np.array([2.7, 2.2, 0.65])
        self.room_lo, self.room_hi = -ext - 3.0, ext + 3.0
        self._tex = None
        self._rays = None

    # ---- ground truth -------------------------------------------------------------------------
    def pose(self, t):
        """returns p_wb(3), R_wb(3x3), v_w(3), a_w(3), w_b(3) at time t."""
        p = np.array([self.px.val(t), self.py.val(t), self.pz.val(t)])
        v = np.array([self.px.d1(t), self.py.d1(t), self.pz.d1(t)])
        a = np.array([self.px.d2(t), self.py.d2(t), self.pz.d2(t)])
        psi, th, ph = self.yaw.val(t), self.pitch.val(t), self.roll.val(t)
        dpsi, dth, dph = self.yaw.d1(t), self.pitch.d1(t), self.roll.d1(t)
        Rz, Ry, Rx = _rz(psi), _ry(th), _rx(ph)
        R = Rz @ Ry @ Rx @ R_WB0
        w_world = dpsi * np.array([0, 0, 1.0]) + Rz @ (dth * np.array([0, 1.0, 0]) + Ry @ (dph * np.array([1.0, 0, 0])))
        return p, R, v, a, R.T @ w_world

    def imu(self):
        """t[n], acc[n,3], gyr[n,3] at imu_hz over [t0, t0+duration]."""
        n = int(round(self.duration * self.imu_hz)) + 1
        t = self.t0 + np.arange(n) / self.imu_hz
        acc, gyr = np.zeros((n, 3)), np.zeros((n, 3))
        g = np.array([0, 0, G_NORM])
        for i, ti in enumerate(t):
            _, R, _, a, w = self.pose(ti)
            acc[i] = R.T @ (a + g) + self.ba
            gyr[i] = w + self.bg
        if self.imu_noise:
            rng = np.random.default_rng(3000 + self.seed)
            # the reference treats acc_n / gyr_n as the per-sample discrete sigma (integration_base.h:21-27)
            acc += rng.normal(0, ACC_N * 0.1, acc.shape)
            gyr += rng.normal(0, GYR_N * 0.1, gyr.shape)
        return t, acc, gyr

    def image_times(self):
        n = int(round(self.duration * self.cam_hz)) + 1
        return self.t0 + np.arange(n) / self.cam_hz

    # ---- rendering ----------------------------------------------------------------------------
    def _textures(self):
        if self._tex is None:
            rng = np.random.default_rng(2000 + self.seed)
            size, tex = 2048, []
            for _ in range(6):
                img = np.zeros((size, size), np.float32)
                for o, lat in enumerate([8, 16, 32, 64, 128]):
                    g = rng.random((size // lat + 3, size // lat + 3)).astype(np.float32)
                    # bilinear upsample of the lattice (value noise)
                    idx = np.arange(size, dtype=np.float32) / lat
                    i0 = idx.astype(np.int32)
                    f = idx - i0
                    f = f * f * (3 - 2 * f)
                    rows0 = g[i0][:, i0] * (1 - f)[None, :] + g[i0][:, i0 + 1] * f[None, :]
                    rows1 = g[i0 + 1][:, i0] * (1 - f)[None, :] + g[i0 + 1][:, i0 + 1] * f[None, :]
                    img += (rows0 * (1 - f)[:, None] + rows1 * f[:, None]) / (o + 1)
                img = (img - img.min()) / (img.max() - img.min())
                tex.append((30.0 + 195.0 * img).astype(np.float32))
            self._tex = tex
            self._tex_ppm = 110.0  # texture pixels per metre
        return self._tex

    def _pixel_rays(self):
        if self._rays is None:
            u, v = np.meshgrid(np.arange(self.cols, dtype=np.float64), np.arange(self.rows, dtype=np.float64))
            xd, yd = (u - CX) / FX, (v - CY) / FY
            x, y = xd.copy(), yd.copy()
            for _ in range(20):  # invert radtan distortion
                r2 = x * x + y * y
                rad = K1 * r2 + K2 * r2 * r2
                dx = x * rad + 2 * P1 * x * y + P2 * (r2 + 2 * x * x)
                dy = y * rad + 2 * P2 * x * y + P1 * (r2 + 2 * y * y)
                x, y = xd - dx, yd - dy
            self._rays = np.stack([x, y, np.ones_like(x)], -1).reshape(-1, 3).astype(np.float32)
        return self._rays

    def render(self, t, frame_index=0):
        tex = self._textures()
        rays = self._pixel_rays()
        p, R, *_ = self.pose(t)
        R_wc = (R @ RIC).astype(np.float32)
        o = (p + R @ TIC).astype(np.float32)
        d = rays @ R_wc.T
        lo, hi = self.room_lo.astype(np.float32), self.room_hi.astype(np.float32)
        with np.errstate(divide="ignore", invalid="ignore"):
            tt = np.where(d > 0, (hi - o) / d, (lo - o) / d)
        tt = np.where(np.isfinite(tt), tt, np.float32(1e9))
        ax = np.argmin(tt, axis=1)
        th = np.take_along_axis(tt, ax[:, None], 1)[:, 0]
        hit = o + d * th[:, None]
        side = (np.take_along_axis(d, ax[:, None], 1)[:, 0] > 0).astype(np.int32)
        wall = ax * 2 + side
        a1, a2 = (ax + 1) % 3, (ax + 2) % 3
        uu = (np.take_along_axis(hit, a1[:, None], 1)[:, 0] + 8.0) * self._tex_ppm
        vv = (np.take_along_axis(hit, a2[:, None], 1)[:, 0] + 8.0) * self._tex_ppm
        uu = np.clip(uu, 0, 2046.0)
        vv = np.clip(vv, 0, 2046.0)
        u0, v0 = uu.astype(np.int32), vv.astype(np.int32)
        fu, fv = uu - u0, vv - v0
        out = np.zeros(len(uu), np.float32)
        for w in range(6):
            m = wall == w
            if not m.any():
                continue
            T = tex[w]
            a, b, c, e = T[v0[m], u0[m]], T[v0[m], u0[m] + 1], T[v0[m] + 1, u0[m]], T[v0[m] + 1, u0[m] + 1]
            out[m] = (a * (1 - fu[m]) + b * fu[m]) * (1 - fv[m]) + (c * (1 - fu[m]) + e * fu[m]) * fv[m]
        if self.pixel_noise > 0:
            rng = np.random.default_rng((4000 + self.seed) * 100003 + frame_index)
            out = out + rng.normal(0, self.pixel_noise, out.shape).astype(np.float32)
        return np.clip(np.rint(out), 0, 255).astype(np.uint8).reshape(self.rows, self.cols)

    def images(self, n=None, start=0, workers=None):
        """Frames start .. start+n-1.  Long runs are rendered by a fork pool (textures and rays are built first and
        shared copy-on-write); call before any CUDA context exists in the process."""
        ts = self.image_times()
        if n is None:
            n = len(ts) - start
        idx = list(range(start, start + n))
        if workers is None:
            workers = min(32, os.cpu_count() or 1) if n >= 24 else 1
        if workers <= 1:
            return ts[start:start + n], np.stack([self.render(ts[i], i) for i in idx])
        import multiprocessing as mp
        self._textures()
        self._pixel_rays()
        global _RENDER_SEQ
        _RENDER_SEQ = self
        with mp.get_context("fork").Pool(workers) as pool:
            frames = pool.map(_render_one, idx, chunksize=max(1, n // (4 * workers)))
        return ts[start:start + n], np.stack(frames)


_RENDER_SEQ = None


def _render_one(i):
    return _RENDER_SEQ.render(_RENDER_SEQ.image_times()[i], i)


def tracker_config_dict(rows=ROWS, cols=COLS, max_cnt=150, min_dist=30, freq=10, equalize=1):
    return dict(rows=rows, cols=cols, max_cnt=max_cnt, min_dist=min_dist, equalize=equalize, freq=freq,
                focal_length=460, fisheye=0, f_threshold=1.0, fx=FX, fy=FY, cx=CX, cy=CY, k1=K1, k2=K2, p1=P1, p2=P2)


def value_noise_image(rows, cols, seed):
    """Stand-alone textured test image (no geometry)."""
    rng = np.random.default_rng(seed)
    img = np.zeros((rows, cols), np.float32)
    for o, lat in enumerate([4, 8, 16, 32, 64]):
        g = rng.random((rows // lat + 3, cols // lat + 3)).astype(np.float32)
        yi, xi = np.arange(rows, dtype=np.float32) / lat, np.arange(cols, dtype=np.float32) / lat
        y0, x0 = yi.astype(np.int32), xi.astype(np.int32)
        fy, fx = yi - y0, xi - x0
        fy, fx = fy * fy * (3 - 2 * fy), fx * fx * (3 - 2 * fx)
        top = g[y0][:, x0] * (1 - fx)[None, :] + g[y0][:, x0 + 1] * fx[None, :]
        bot = g[y0 + 1][:, x0] * (1 - fx)[None, :] + g[y0 + 1][:, x0 + 1] * fx[None, :]
        img += (top * (1 - fy)[:, None] + bot * fy[:, None]) / (o + 1)
    img = (img - img.min()) / (img.max() - img.min())
    img = 30 + 195 * img + rng.normal(0, 2, (rows, cols))
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def scene_landmarks(seq: Sequence, n_points: int = 2500):
    """The random wall landmarks track_messages observes (feature id = index + start_id) and the generator state after drawing them."""
    rng = np.random.default_rng(5000 + seq.seed)
    lo, hi = seq.room_lo, seq.room_hi
    pts = []
    for _ in range(n_points):
        ax = int(rng.integers(0, 3))
        p = rng.uniform(lo, hi)
        p[ax] = lo[ax] if rng.random() < 0.5 else hi[ax]
        pts.append(p)
    return np.array(pts), rng


def loop_frame_matches(seq: Sequence, t_loop: float, ids, n_points: int = 2500, pixel_sigma: float = 0.0, seed: int = 0):
    """What pose_graph sends on /pose_graph/match_points for a loop between an old key frame at t_loop and a window frame whose
    features are `ids`: the normalised coordinates of those landmarks in the OLD frame (those in front of it), as rows (x, y, id)
    sorted by id (keyframe.cpp:485-520), plus the old frame's true pose (p_wb, R_wb)."""
    pts, _ = scene_landmarks(seq, n_points)
    p, R, *_ = seq.pose(t_loop)
    rng = np.random.default_rng(7000 + seed)
    rows = []
    for i in sorted(int(k) for k in ids):
        Pc = (R @ RIC).T @ (pts[i] - (p + R @ TIC))
        if Pc[2] > 0.3 and abs(Pc[0] / Pc[2]) < 1.0 and abs(Pc[1] / Pc[2]) < 0.7:
            e = rng.normal(0, pixel_sigma, 2) / 460.0 if pixel_sigma > 0 else np.zeros(2)
            rows.append([Pc[0] / Pc[2] + e[0], Pc[1] / Pc[2] + e[1], float(i)])
    return np.array(rows).reshape(-1, 3), p, R


def track_messages(seq: Sequence, n_pub: int, n_points: int = 2500, max_feats: int = 150, pub_hz: float = 10.0, pixel_sigma: float = 0.3,
                   start_id: int = 0, landmarks=None):
    """Feature messages (stamp, ids, xyz_uv_vel[n,7]) made directly from the scene geometry (no images), in the
    spirit of the reference's data_generator (data_generator/src/data_generator.cpp:11-59): random landmarks on
    the room walls, projected through the EuRoC pinhole+radtan model, at most `max_feats` per frame with stable
    ids, pixel noise sigma `pixel_sigma`.  Back-end tests/benchmarks use this to avoid rendering.  `landmarks` (world points)
    replaces the random wall points, e.g. with harness/loop_revisit.py's texture corners."""
    pts, rng = scene_landmarks(seq, n_points)
    if landmarks is not None:
        pts = np.asarray(landmarks, np.float64)

    def project(t):
        p, R, *_ = seq.pose(t)
        Pc = ((pts - (p + R @ TIC)) @ (R @ RIC))  # rows: R_wc^T (X - o)
        z = Pc[:, 2]
        x, y = Pc[:, 0] / z, Pc[:, 1] / z
        r2 = x * x + y * y
        rad = K1 * r2 + K2 * r2 * r2
        xd = x + x * rad + 2 * P1 * x * y + P2 * (r2 + 2 * x * x)
        yd = y + y * rad + 2 * P2 * x * y + P1 * (r2 + 2 * y * y)
        u, v = FX * xd + CX, FY * yd + CY
        vis = (z > 0.3) & (u > 5) & (u < COLS - 5) & (v > 5) & (v < ROWS - 5) & (r2 < 1.2)
        return np.c_[x, y], np.c_[u, v], vis

    active = []
    msgs = []
    noise = {}
    for k in range(n_pub):
        t = seq.t0 + (k + 2) / pub_hz
        un, uv, vis = project(t)
        un_prev, _, _ = project(t - 0.05)
        active = [i for i in active if vis[i]]
        if len(active) < max_feats:
            cand = [i for i in np.nonzero(vis)[0] if i not in active]
            rng.shuffle(cand)
            active += cand[: max_feats - len(active)]
        ids = np.array(sorted(active), np.int32)
        d = np.zeros((len(ids), 7))
        for r, i in enumerate(ids):
            e = rng.normal(0, pixel_sigma, 2)
            d[r, 0:2] = un[i] + e / 460.0
            d[r, 2] = 1.0
            d[r, 3:5] = uv[i] + e
            d[r, 5:7] = (un[i] - un_prev[i]) / 0.05
        msgs.append((float(t), ids + start_id, d))
    return msgs
