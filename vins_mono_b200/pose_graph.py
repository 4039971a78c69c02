"""ctypes mirror of include/vinsb200/pose_graph.h; method names follow the reference's PoseGraph
(pose_graph/src/pose_graph.h)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import Batch, Handle, LoopConfig, LoopResult, PoseGraphConfig, VinsError, check, f64, load_library, ptr

PoseGraphError = VinsError
VP_ERR_CAPACITY = -4


class PoseGraph(Handle):
    """The reference's PoseGraph with the loop already found: addKeyFrame / updateKeyFrameLoop / optimize4DoF.
    max_anchors: free loop anchors an optimised range may hold (0 = 88, at most 1024); the workspace grows with it."""
    _destroy, _last_error = "vp_destroy", "vp_last_error"

    def __init__(self, max_keyframes=2000, fast_relocalization=False, device=0, max_anchors=0):
        self.cfg = PoseGraphConfig(max_keyframes=max_keyframes, fast_relocalization=int(fast_relocalization), device=device,
                                   max_anchors=max_anchors)
        self._open("vp_create", C.byref(self.cfg))

    def new_sequence(self):
        self._check(self.lib.vp_new_sequence(self.h))

    def add_keyframe(self, stamp, P, Q_wxyz, loop_index=-1, loop_info=None):
        """Returns (index, stored P, stored Q wxyz)."""
        idx, P_out, Q_out = C.c_int(), np.zeros(3), np.zeros(4)
        li = f64(loop_info) if loop_info is not None else None
        self._check(self.lib.vp_add_keyframe(self.h, float(stamp), ptr(f64(P)), ptr(f64(Q_wxyz)), int(loop_index), ptr(li), C.byref(idx),
                                             ptr(P_out), ptr(Q_out)))
        return idx.value, P_out, Q_out

    def update_loop(self, index, loop_info):
        self._check(self.lib.vp_update_loop(self.h, int(index), ptr(f64(loop_info))))

    def optimize(self):
        return self._check(self.lib.vp_optimize(self.h))

    def sync(self):
        self._check(self.lib.vp_sync(self.h))

    def correct_pose(self, P, Q_wxyz):
        P_out, Q_out = np.zeros(3), np.zeros(4)
        self._check(self.lib.vp_correct_pose(self.h, ptr(f64(P)), ptr(f64(Q_wxyz)), ptr(P_out), ptr(Q_out)))
        return P_out, Q_out

    def drift(self):
        r, t, y = np.zeros(9), np.zeros(3), np.zeros(1)
        self._check(self.lib.vp_get_drift(self.h, ptr(r), ptr(t), ptr(y)))
        return r.reshape(3, 3), t, float(y[0])

    def keyframe(self, index):
        v, li, lidx = np.zeros(14), np.zeros(8), C.c_int()
        self._check(self.lib.vp_get_keyframe(self.h, int(index), ptr(v), C.byref(lidx), ptr(li)))
        return dict(vio_P=v[:3], vio_Q=v[3:7], P=v[7:10], Q=v[10:14], loop_index=lidx.value, loop_info=li)

    def path(self):
        n = self._check(self.lib.vp_get_path(self.h, 0, None, None, None, None))
        st, P, Q, sq = np.zeros(n), np.zeros((n, 3)), np.zeros((n, 4)), np.zeros(n, np.int32)
        if n:
            self._check(self.lib.vp_get_path(self.h, n, ptr(st), ptr(P), ptr(Q), ptr(sq)))
        return st, P, Q, sq

    def info(self):
        o, c = np.zeros(8, np.int32), np.zeros(2)
        self._check(self.lib.vp_info(self.h, ptr(o), ptr(c)))
        keys = ["keyframes", "loops", "earliest_loop_index", "optimizations", "last_n", "last_border", "iterations", "successful"]
        d = dict(zip(keys, (int(v) for v in o)))
        d["initial_cost"], d["final_cost"] = float(c[0]), float(c[1])
        return d

    def save(self, prefix):
        """savePoseGraph into prefix + "pose_graph.txt", prefix + <i> + "_keypoints.txt", prefix + <i> + "_briefdes.dat".
        Returns the number of key frames written."""
        return self._check(self.lib.vp_save(self.h, str(prefix).encode()))

    def load(self, prefix):
        """loadPoseGraph into a graph with no key frame: the saved key frames become sequence 0, constant in every
        optimisation.  Returns the number of key frames loaded."""
        return self._check(self.lib.vp_load(self.h, str(prefix).encode()))

    def timing(self):
        ms, n = C.c_float(), C.c_int()
        self._check(self.lib.vp_last_timing(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    # ---- loop verification (include/vinsb200/loop_verify.h, loop_camera.h)
    def enable_loop(self, cfg, camera_model=0, xi=0.0):
        """camera_model: 0 PINHOLE, 1 MEI (xi = mirror_parameters.xi), 2 KANNALA_BRANDT; cfg.intrinsics in the model's order
        (config.loop_kwargs reads both from a YAML file)."""
        self._loop_cap = cfg.max_window
        self._check(self.lib.vp_loop_enable_camera(self.h, C.byref(cfg), int(camera_model), float(xi)))

    def attach_keyframe(self, index, vio_P, vio_Q_wxyz, image, point_3d, point_uv, point_norm, point_id):
        """KeyFrame's constructor: descriptors of the window points and of the FAST corners.  Returns the corner count."""
        img = np.ascontiguousarray(image, np.uint8)
        p3, uv = np.ascontiguousarray(point_3d, np.float32).reshape(-1, 3), np.ascontiguousarray(point_uv, np.float32).reshape(-1, 2)
        nm, ids = np.ascontiguousarray(point_norm, np.float32).reshape(-1, 2), np.ascontiguousarray(point_id, np.float64).reshape(-1)
        nc = C.c_int()
        self._check(self.lib.vp_attach_keyframe(self.h, int(index), ptr(f64(vio_P)), ptr(f64(vio_Q_wxyz)), ptr(img), img.strides[0],
                                                len(p3), ptr(p3), ptr(uv), ptr(nm), ptr(ids), C.byref(nc)))
        return nc.value

    def find_connection(self, cur, old):
        """findConnection: dict(accepted, n_matches, n_inliers, loop_info 8, old_R, old_T, points = inliers' (x, y, id))."""
        r, lst = LoopResult(), np.zeros((self._loop_cap, 3))
        self._check(self.lib.vp_find_connection(self.h, int(cur), int(old), C.byref(r), self._loop_cap, ptr(lst)))
        return _result(r, lst)

    def loop_timing(self):
        ms = np.zeros(6, np.float32)
        self._check(self.lib.vp_loop_last_timing(self.h, ptr(ms)))
        return ms


class PoseGraphBatch(Batch):
    """n independent pose graphs whose pending optimisations run in one launch chain."""
    _destroy, _last_error = "vp_batch_destroy", "vp_batch_last_error"

    def __init__(self, n, max_keyframes=2000, fast_relocalization=False, device=0, max_anchors=0):
        self.cfg = PoseGraphConfig(max_keyframes=max_keyframes, fast_relocalization=int(fast_relocalization), device=device,
                                   max_anchors=max_anchors)
        self.n = n
        self._open("vp_batch_create", C.byref(self.cfg), int(n))
        self.members = [PoseGraph._borrow(self, self.lib.vp_batch_member(self.h, k)) for k in range(n)]

    def __getitem__(self, k):
        return self.members[k]

    def optimize(self, active=None):
        """Returns the per-member status (1 enqueued, 0 nothing pending, VP_ERR_CAPACITY = -4 for a member whose range does
        not fit; the other members still run).  Any other error (the launch itself failed) raises."""
        st = np.zeros(self.n, np.int32)
        act = None if active is None else np.ascontiguousarray(active, np.int32)
        rc = self.lib.vp_batch_optimize(self.h, ptr(act), ptr(st))
        failed = [int(v) for v in st if v < 0 and v != VP_ERR_CAPACITY]
        self._check(failed[0] if failed else 0 if rc == VP_ERR_CAPACITY else rc)
        return st

    def sync(self):
        self._check(self.lib.vp_batch_sync(self.h))

    def timing(self):
        ms, n = np.zeros(2, np.float32), C.c_int()
        self._check(self.lib.vp_batch_last_timing(self.h, ptr(ms), C.byref(n)))
        return float(ms[0]), float(ms[1]), n.value

    def enable_loop(self, cfg, camera_model=0, xi=0.0):
        self._loop_cap = cfg.max_window
        for m in self.members:
            m._loop_cap = cfg.max_window
        self._check(self.lib.vp_batch_loop_enable_camera(self.h, C.byref(cfg), int(camera_model), float(xi)))

    def find_connection(self, cur, old):
        """One launch chain for every member k with cur[k] >= 0; returns a list (None for skipped members)."""
        res = (LoopResult * self.n)()
        lst = np.zeros((self.n, self._loop_cap, 3))
        st = np.zeros(self.n, np.int32)
        c, o = np.ascontiguousarray(cur, np.int32), np.ascontiguousarray(old, np.int32)
        self._check(self.lib.vp_batch_find_connection(self.h, ptr(c), ptr(o), res, self._loop_cap, ptr(lst), ptr(st)))
        return [_result(res[k], lst[k]) if st[k] == 1 else None for k in range(self.n)]

    def loop_timing(self):
        ms = np.zeros(6, np.float32)
        self._check(self.lib.vp_batch_loop_last_timing(self.h, ptr(ms)))
        return ms


def debug_four_dof_error(params8, meas6, weighted=False, robust=False):
    """Device FourDOFError / FourDOFWeightError: returns (r 4, J 4x8, cost)."""
    out = np.zeros(37)
    check(load_library().vp_debug_four_dof_error(ptr(f64(params8)), ptr(f64(meas6)), int(weighted), int(robust), ptr(out)),
          "vp_debug_four_dof_error")
    return out[:4], out[4:36].reshape(4, 8), out[36]


def loop_config(rows, cols, intrinsics, ric, tic, pattern, max_window=256, max_corners=4096):
    pat = np.ascontiguousarray(pattern, np.int32).reshape(256, 4)
    cfg = LoopConfig(rows=rows, cols=cols, max_window=max_window, max_corners=max_corners)
    cfg.intrinsics[:] = [float(v) for v in intrinsics]
    cfg.ric9[:] = [float(v) for v in np.asarray(ric, np.float64).reshape(9)]
    cfg.tic3[:] = [float(v) for v in np.asarray(tic, np.float64).reshape(3)]
    cfg.brief_pattern = pat.ctypes.data
    cfg._pattern = pat  # kept alive until the enable call has copied it
    return cfg


def _result(r, lst):
    return dict(accepted=bool(r.accepted), n_matches=r.n_matches, n_inliers=r.n_inliers, loop_info=np.array(r.loop_info[:]),
                old_R=np.array(r.old_R9[:]).reshape(3, 3), old_T=np.array(r.old_T3[:]), points=lst[:r.n_points].copy())


def debug_brief_blur(image):
    img = np.ascontiguousarray(image, np.uint8)
    out = np.zeros_like(img)
    check(load_library().vp_debug_brief_blur(ptr(img), img.shape[0], img.shape[1], ptr(out)), "vp_debug_brief_blur")
    return out


def debug_fast(image, cap=65536):
    img = np.ascontiguousarray(image, np.uint8)
    xy = np.zeros((cap, 2), np.float32)
    n = check(load_library().vp_debug_fast(ptr(img), img.shape[0], img.shape[1], cap, ptr(xy)), "vp_debug_fast")
    return xy[:n].astype(np.int32)


def debug_brief(image, pattern, uv):
    img = np.ascontiguousarray(image, np.uint8)
    pat = np.ascontiguousarray(pattern, np.int32)
    pts = np.ascontiguousarray(uv, np.float32).reshape(-1, 2)
    desc = np.zeros((len(pts), 4), np.uint64)
    check(load_library().vp_debug_brief(ptr(img), img.shape[0], img.shape[1], ptr(pat), len(pts), ptr(pts), ptr(desc)), "vp_debug_brief")
    return desc


def debug_match(desc_a, desc_b):
    a, b = np.ascontiguousarray(desc_a, np.uint64), np.ascontiguousarray(desc_b, np.uint64)
    idx = np.zeros(len(a), np.int32)
    check(load_library().vp_debug_match(len(a), ptr(a), len(b), ptr(b) if len(b) else None, ptr(idx)), "vp_debug_match")
    return idx


def debug_pnp(point_3d, norm):
    p3, nm = np.ascontiguousarray(point_3d, np.float32).reshape(-1, 3), np.ascontiguousarray(norm, np.float32).reshape(-1, 2)
    Rt, n_in, mask = np.zeros(12), C.c_int(), np.zeros(len(p3), np.uint8)
    check(load_library().vp_debug_pnp(len(p3), ptr(p3), ptr(nm), ptr(Rt), C.byref(n_in), ptr(mask)), "vp_debug_pnp")
    return Rt[:9].reshape(3, 3), Rt[9:], n_in.value, mask.astype(bool)


def debug_lift(camera_model, intrinsics, xi, uv):
    """The device lift of the key-frame corners (liftProjective / z) of float pixel positions uv (n, 2): (n, 2) float32."""
    K = f64(intrinsics).reshape(8)
    pts = np.ascontiguousarray(uv, np.float32).reshape(-1, 2)
    xy = np.zeros_like(pts)
    check(load_library().vp_debug_lift(int(camera_model), ptr(K), float(xi), len(pts), ptr(pts), ptr(xy)), "vp_debug_lift")
    return xy
