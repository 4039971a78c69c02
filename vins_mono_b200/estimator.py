"""ctypes mirror of include/vinsb200/estimator.h; method names follow the reference's Estimator
(vins_estimator/src/estimator.h:25-139)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import Batch, EstimatorConfig, Handle, check, f64, load_library, ptr


def _make_config(window_size=10, max_features=1000, num_iterations=8, estimate_extrinsic=0, estimate_td=0,
                 focal_length=460.0, keyframe_parallax=10.0, acc_n=0.08, gyr_n=0.004, acc_w=0.00004, gyr_w=2.0e-6,
                 g_norm=9.81007, init_depth=5.0, td=0.0, tr=0.0, row=480.0, tic=(0, 0, 0), ric=np.eye(3), device=0):
    cfg = EstimatorConfig(window_size=window_size, max_features=max_features, num_iterations=num_iterations,
                          estimate_extrinsic=estimate_extrinsic, estimate_td=estimate_td, focal_length=focal_length,
                          keyframe_parallax=keyframe_parallax, acc_n=acc_n, gyr_n=gyr_n, acc_w=acc_w, gyr_w=gyr_w,
                          g_norm=g_norm, init_depth=init_depth, td=td, tr=tr, row=row, device=device)
    cfg.tic[:] = list(np.asarray(tic, float))
    cfg.ric[:] = list(np.asarray(ric, float).ravel())
    return cfg


class Estimator(Handle):
    """Drop-in for the reference Estimator: processIMU / processImage, then read Ps, Rs, Vs, Bas, Bgs."""
    _destroy, _last_error = "ve_destroy", "ve_last_error"

    def __init__(self, **kw):
        cfg = _make_config(**kw)
        self.cfg, self.W = cfg, cfg.window_size
        self._open("ve_create", C.byref(cfg))

    @classmethod
    def _member(cls, batch, k):
        """Borrowed handle of a batch member (driven and destroyed through its EstimatorBatch)."""
        self = cls._borrow(batch, batch.lib.ve_batch_member(batch.h, k))
        self.cfg, self.W = batch.cfg, batch.cfg.window_size
        return self

    def setReloFrame(self, frame_stamp, frame_index, match_points, relo_t, relo_r):
        """Estimator::setReloFrame (estimator.h:36): match_points = n x (x, y, feature id).  True when the stamp is in the window."""
        mp = f64(match_points).reshape(-1, 3)
        return bool(self._check(self.lib.ve_set_relo_frame(self.h, float(frame_stamp), int(frame_index), len(mp), ptr(mp), ptr(f64(relo_t)),
                                                           ptr(f64(relo_r).reshape(9)))))

    def headers(self):
        """Stamps of the window frames (Headers[0 .. WINDOW_SIZE])."""
        h = np.zeros(self.W + 1)
        self._check(self.lib.ve_get_headers(self.h, ptr(h)))
        return h

    def relo(self):
        o = np.zeros(24)
        self._check(self.lib.ve_get_relocalization(self.h, ptr(o)))
        return dict(drift_correct_r=o[0:9].reshape(3, 3).copy(), drift_correct_t=o[9:12].copy(), relo_relative_t=o[12:15].copy(),
                    relo_relative_q=o[15:19].copy(), relo_relative_yaw=float(o[19]), pending=bool(o[20]), local_index=int(o[21]),
                    factors=int(o[22]), solves=int(o[23]))

    def init_info(self):
        """How the window was initialised: own initialStructure (self_initialised) or a caller-supplied seed."""
        r = np.zeros(8)
        rc = self._check(self.lib.ve_init_info(self.h, ptr(r)))
        return dict(self_initialised=bool(rc), l=int(r[0]), scale=float(r[1]), g=r[2:5].copy(), bundle_iterations=int(r[5]),
                    bundle_cost=float(r[6]), failed_attempts=int(r[7]))

    def clearState(self):
        self._check(self.lib.ve_clear_state(self.h))

    def set_seed(self, rows, ba, bg):
        rows, ba, bg = f64(rows), f64(ba), f64(bg)
        self._check(self.lib.ve_set_seed(self.h, len(rows), ptr(rows), ptr(ba), ptr(bg)))

    def processIMU(self, dt, linear_acceleration, angular_velocity):
        a, g = f64(linear_acceleration), f64(angular_velocity)
        self._check(self.lib.ve_process_imu(self.h, float(dt), ptr(a), ptr(g)))

    def processImage(self, ids, xyz_uv_vel, stamp):
        ids = np.ascontiguousarray(ids, np.int32)
        d = f64(xyz_uv_vel)
        self._check(self.lib.ve_process_image(self.h, len(ids), ptr(ids), ptr(d), float(stamp)))

    def states(self):
        out, td = np.zeros((self.W + 1, 16)), C.c_double(0)
        self._check(self.lib.ve_get_states(self.h, ptr(out), C.byref(td)))
        return out, td.value

    def info(self):
        o, c = np.zeros(10, np.int32), np.zeros(2)
        self._check(self.lib.ve_info(self.h, ptr(o), ptr(c)))
        keys = ["solver_flag", "frame_count", "marginalization_flag", "n_solves", "n_reboots", "landmarks", "visual",
                "iterations", "successful_steps", "termination"]
        d = {k: int(v) for k, v in zip(keys, o)}
        d["initial_cost"], d["final_cost"] = float(c[0]), float(c[1])
        return d

    def prior(self, cap=256):
        A, b = np.zeros(cap * cap), np.zeros(cap)
        nb, blk = C.c_int(0), np.zeros(4 * 64, np.int32)
        n = self._check(self.lib.ve_get_prior(self.h, cap, ptr(A), ptr(b), C.byref(nb), ptr(blk)))
        return A[: n * n].reshape(n, n).copy(), b[:n].copy(), [tuple(int(v) for v in blk[4 * k:4 * k + 4]) for k in range(nb.value)]

    KERNELS = ["ba_eval", "ba_reduce", "ba_step", "unused", "marg_build", "marg_solve", "preint_jobs", "ba_finish"]

    def processIMU_batch(self, dt, acc, gyr):
        dt, acc, gyr = f64(dt), f64(acc), f64(gyr)
        self._check(self.lib.ve_process_imu_batch(self.h, len(dt), ptr(dt), ptr(acc), ptr(gyr)))

    def set_profile(self, on):
        self._check(self.lib.ve_set_profile(self.h, int(on)))

    def kernel_times(self):
        ms, cnt = np.zeros(8), np.zeros(8, np.int32)
        self._check(self.lib.ve_kernel_times(self.h, ptr(ms), ptr(cnt)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(self.KERNELS)}

    def traffic(self):
        a, b = C.c_double(0), C.c_double(0)
        self._check(self.lib.ve_last_traffic(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def solver_debug(self):
        out = np.zeros(18)
        self._check(self.lib.ve_solver_debug(self.h, ptr(out)))
        return dict(retries=int(out[0]), mu=out[1], radius=out[2], clk=out[3:].astype(np.int64).tolist(), floor_pairs=int(out[12]))

    def launch_count(self):
        """Kernel launches of the last processImage (does not wait for a pending marginalisation)."""
        k = C.c_int(0)
        self._check(self.lib.ve_last_timing(self.h, None, C.byref(k)))
        return k.value

    def timing(self):
        ms, k = np.zeros(4, np.float32), C.c_int(0)
        self._check(self.lib.ve_last_timing(self.h, ptr(ms), C.byref(k)))
        return dict(preint_ms=float(ms[0]), solve_ms=float(ms[1]), marg_ms=float(ms[2]), total_ms=float(ms[3]), launches=k.value)

    def extrinsic(self):
        t, r = np.zeros(3), np.zeros(9)
        self._check(self.lib.ve_get_extrinsic(self.h, ptr(t), ptr(r)))
        return t, r.reshape(3, 3)


class EstimatorBatch(Batch):
    """n independent estimators advancing together (include/vinsb200/estimator.h, ve_batch_*): one launch chain per frame
    for the whole batch.  members[k] is an Estimator mirror for the per-sequence calls (set_seed, processIMU, states ...)."""
    _destroy, _last_error = "ve_batch_destroy", "ve_batch_last_error"

    def __init__(self, n, **kw):
        self.cfg, self.n = _make_config(**kw), n
        self._open("ve_batch_create", C.byref(self.cfg), n)
        self.members = [Estimator._member(self, k) for k in range(n)]

    def processImage(self, msgs):
        """msgs[k] = (ids, xyz_uv_vel, stamp) or None (member k idles this frame).  Returns the per-member status list."""
        n = self.n
        active = np.zeros(n, np.int32)
        cnt = np.zeros(n, np.int32)
        stamps = np.zeros(n)
        idp, obp, keep = (C.c_void_p * n)(), (C.c_void_p * n)(), []
        for k, m in enumerate(msgs):
            if m is None:
                continue
            ids, d = np.ascontiguousarray(m[0], np.int32), f64(m[1])
            keep += [ids, d]
            active[k], cnt[k], stamps[k] = 1, len(ids), float(m[2])
            idp[k], obp[k] = ids.ctypes.data, d.ctypes.data
        status = np.zeros(n, np.int32)
        self._check(self.lib.ve_batch_process_image(self.h, ptr(active), ptr(cnt), idp, obp, ptr(stamps), ptr(status)))
        return status

    def timing(self):
        ms, k = np.zeros(4, np.float32), C.c_int(0)
        self._check(self.lib.ve_batch_last_timing(self.h, ptr(ms), C.byref(k)))
        return dict(preint_ms=float(ms[0]), solve_ms=float(ms[1]), marg_ms=float(ms[2]), total_ms=float(ms[3]), launches=k.value)

    def launch_count(self):
        k = C.c_int(0)
        self._check(self.lib.ve_batch_last_timing(self.h, None, C.byref(k)))
        return k.value

    def groups(self):
        return self._check(self.lib.ve_batch_groups(self.h))

    def set_profile(self, on):
        self._check(self.lib.ve_batch_set_profile(self.h, int(on)))

    def kernel_times(self):
        ms, cnt = np.zeros(8), np.zeros(8, np.int32)
        self._check(self.lib.ve_batch_kernel_times(self.h, ptr(ms), ptr(cnt)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(Estimator.KERNELS)}

    def sync(self):
        self._check(self.lib.ve_batch_sync(self.h))


def debug_projection_factor(params23, data12, use_td=False, focal_length=460.0, tr=0.0, row=480.0, robust=False):
    """Residual (2), Jacobian (2 x 20: pose_i 6, pose_j 6, ex 6, depth, td) and rho/2 of one visual factor, evaluated by the
    device code of the solve."""
    lib = load_library()
    prm, dat, out = f64(params23), f64(data12), np.zeros(43)
    assert prm.size == 23 and dat.size == 12
    check(lib.ve_debug_projection_factor(ptr(prm), ptr(dat), int(use_td), float(focal_length), float(tr), float(row), int(robust),
                                         ptr(out)), "ve_debug_projection_factor")
    return out[0:2].copy(), out[2:42].reshape(2, 20).copy(), float(out[42])


def debug_imu_factor(ba, bg, dt, acc, gyr, params32=None, noise=(0.08, 0.004, 0.00004, 2.0e-6), g_norm=9.81007):
    """Device pre-integration of the samples (sample 0 seeds acc_0 / gyr_0) and, with params32, the whitened IMU factor."""
    lib = load_library()
    dt, acc, gyr = f64(dt), f64(acc), f64(gyr)
    pre, fac = np.zeros(686), np.zeros(465)
    prm = f64(params32) if params32 is not None else None
    noise = f64(noise)
    check(lib.ve_debug_imu_factor(ptr(noise), float(g_norm), ptr(f64(ba)), ptr(f64(bg)), len(dt), ptr(dt), ptr(acc), ptr(gyr), ptr(prm),
                                  ptr(pre), ptr(fac) if prm is not None else None), "ve_debug_imu_factor")
    out = dict(sum_dt=pre[0], dp=pre[1:4].copy(), dq=pre[4:8].copy(), dv=pre[8:11].copy(), jacobian=pre[11:236].reshape(15, 15).copy(),
               covariance=pre[236:461].reshape(15, 15).copy(), sqrt_info=pre[461:686].reshape(15, 15).copy())
    if prm is not None:
        out["residual"], out["jacobian_w"] = fac[:15].copy(), fac[15:].reshape(15, 30).copy()
    return out


# ---- initialisation stages (host code, no device needed; include/vinsb200/estimator.h "Initialisation") -------------------
def _tracks_flat(tracks):
    ids = np.array([t[0] for t in tracks], np.int32)
    start = np.array([t[1] for t in tracks], np.int32)
    nobs = np.array([len(np.asarray(t[2]).reshape(-1, 2)) for t in tracks], np.int32)
    xy = f64(np.concatenate([np.asarray(t[2], float).reshape(-1, 2) for t in tracks])) if len(tracks) else np.zeros((0, 2))
    return ids, start, nobs, xy


def debug_relative_rt(corres):
    """MotionEstimator::solveRelativeRT on n x (x0 y0 x1 y1): (ok, Rotation, Translation, inlier_cnt)."""
    lib = load_library()
    c = f64(corres).reshape(-1, 4)
    R, T, cnt = np.zeros(9), np.zeros(3), C.c_int()
    rc = check(lib.ve_debug_relative_rt(ptr(c), len(c), ptr(R), ptr(T), C.byref(cnt)), "ve_debug_relative_rt")
    return bool(rc), R.reshape(3, 3), T, cnt.value


def debug_solve_pnp(pts3, pts2, R_initial, P_initial):
    """cv::solvePnP(..., useExtrinsicGuess=true) from (R_initial, P_initial) (world -> camera): (ok, R, t)."""
    lib = load_library()
    p3, p2 = f64(pts3).reshape(-1, 3), f64(pts2).reshape(-1, 2)
    R, t = f64(R_initial).reshape(9).copy(), f64(P_initial).reshape(3).copy()
    rc = check(lib.ve_debug_solve_pnp(ptr(p3), ptr(p2), len(p2), ptr(R), ptr(t)), "ve_debug_solve_pnp")
    return bool(rc), R.reshape(3, 3), t


def debug_sfm_construct(frame_num, l, relative_R, relative_T, tracks, function_tolerance=0.0):
    """GlobalSFM::construct; tracks = [(id, start_frame, xy[nobs, 2])].  Returns dict(ok, q[F,4] wxyz, T[F,3], points{id: xyz},
    iterations, cost)."""
    lib = load_library()
    ids, start, nobs, xy = _tracks_flat(tracks)
    q, T = np.zeros((frame_num, 4)), np.zeros((frame_num, 3))
    n_pts, it, cost = C.c_int(), C.c_int(), C.c_double()
    pid, pts = np.zeros(max(len(ids), 1), np.int32), np.zeros((max(len(ids), 1), 3))
    rR, rT = f64(relative_R).reshape(9), f64(relative_T).reshape(3)
    rc = check(lib.ve_debug_sfm_construct(frame_num, l, ptr(rR), ptr(rT), len(ids), ptr(ids), ptr(start), ptr(nobs), ptr(xy),
                                          float(function_tolerance), ptr(q), ptr(T), C.byref(n_pts), ptr(pid), ptr(pts), C.byref(it),
                                          C.byref(cost)), "ve_debug_sfm_construct")
    return dict(ok=bool(rc), q=q, T=T, points={int(pid[k]): pts[k].copy() for k in range(n_pts.value)}, iterations=it.value,
                cost=cost.value)


def debug_initial_structure(headers, frames, tracks, ric, tic, g_norm=9.81007, function_tolerance=0.0):
    """Estimator::initialStructure up to VisualIMUAlignment.  frames = [dict(t, ids, xy[n,2], imu[m,7] (dt acc gyr), lin[6])] for every
    image (imu / lin of frame 0 unused); tracks = [(id, start_frame, xy[nobs,2])].  Returns dict(code, l, R[n,3,3], T[n,3], x, g,
    delta_bg, bundle_iterations, bundle_cost, key_frames)."""
    lib = load_library()
    hd = f64(headers)
    na = len(frames)
    stamps = f64([f["t"] for f in frames])
    pts_off = np.zeros(na + 1, np.int32)
    pts_off[1:] = np.cumsum([len(f["ids"]) for f in frames])
    pt_ids = np.ascontiguousarray(np.concatenate([np.asarray(f["ids"], np.int32) for f in frames]), np.int32)
    pt_xy = f64(np.concatenate([np.asarray(f["xy"], float).reshape(-1, 2) for f in frames]))
    imu_off = np.zeros(na + 1, np.int32)
    imu_off[1:] = np.cumsum([0 if k == 0 else len(f["imu"]) for k, f in enumerate(frames)])
    rows = [np.asarray(f["imu"], float).reshape(-1, 7) for k, f in enumerate(frames) if k > 0]
    imu7 = f64(np.concatenate(rows)) if rows else np.zeros((0, 7))
    lin6 = f64([np.zeros(6) if k == 0 else np.asarray(f["lin"], float) for k, f in enumerate(frames)])
    ids, start, nobs, xy = _tracks_flat(tracks)
    fR, fT, x = np.zeros((na, 9)), np.zeros((na, 3)), np.zeros(3 * na + 3)
    g3, dbg, info, cost = np.zeros(3), np.zeros(3), np.zeros(4, np.int32), C.c_double()
    rc = check(lib.ve_debug_initial_structure(len(hd), ptr(hd), na, ptr(stamps), ptr(pts_off), ptr(pt_ids), ptr(pt_xy), ptr(imu_off),
                                              ptr(imu7), ptr(lin6), len(ids), ptr(ids), ptr(start), ptr(nobs), ptr(xy), ptr(f64(ric).reshape(9)),
                                              ptr(f64(tic).reshape(3)), float(g_norm), float(function_tolerance), ptr(fR), ptr(fT), ptr(x),
                                              ptr(g3), ptr(dbg), ptr(info), C.byref(cost)), "ve_debug_initial_structure")
    return dict(code=rc, l=int(info[0]), R=fR.reshape(na, 3, 3), T=fT, x=x, g=g3, delta_bg=dbg, bundle_iterations=int(info[1]),
                bundle_cost=cost.value, key_frames=int(info[2]))


def debug_ex_rotation(corres_list, dq_list, window_size=10, rc_given=None):
    """InitialEXRotation::CalibrationExRotation called once per (corres[n,4], delta_q wxyz) pair: (ric[k,3,3], ok[k], cov[k], Rc[k,3,3] = the camera rotations solveRelativeR found)."""
    lib = load_library()
    n = len(corres_list)
    off = np.zeros(n + 1, np.int32)
    off[1:] = np.cumsum([len(np.asarray(c).reshape(-1, 4)) for c in corres_list])
    c4 = f64(np.concatenate([np.asarray(c, float).reshape(-1, 4) for c in corres_list])) if n else np.zeros((0, 4))
    dq = f64(dq_list).reshape(-1, 4)
    ric, ok, cov, rcam = np.zeros((n, 9)), np.zeros(n, np.int32), np.zeros(n), np.zeros((n, 9))
    check(lib.ve_debug_ex_rotation(n, ptr(off), ptr(c4), ptr(dq), int(window_size), ptr(ric), ptr(ok), ptr(cov), ptr(rcam),
                                   ptr(f64(rc_given).reshape(-1, 9)) if rc_given is not None else None), "ve_debug_ex_rotation")
    return ric.reshape(n, 3, 3), ok.astype(bool), cov, rcam.reshape(n, 3, 3)
