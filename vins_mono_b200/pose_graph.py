"""ctypes mirror of include/vinsb200/pose_graph.h; method names follow the reference's PoseGraph
(pose_graph/src/pose_graph.h)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .tracker import load_library


class PoseGraphConfig(C.Structure):
    _fields_ = [("max_keyframes", C.c_int), ("fast_relocalization", C.c_int), ("device", C.c_int), ("max_anchors", C.c_int)]


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _d(a):
    return np.ascontiguousarray(a, np.float64)


_bound = False


def _bind(lib):
    global _bound
    if _bound:
        return
    V = C.c_void_p
    lib.vp_last_error.restype = C.c_char_p
    lib.vp_last_error.argtypes = [V]
    lib.vp_create.argtypes = [C.POINTER(PoseGraphConfig), C.POINTER(V)]
    lib.vp_destroy.argtypes = [V]
    lib.vp_new_sequence.argtypes = [V]
    lib.vp_add_keyframe.argtypes = [V, C.c_double, V, V, C.c_int, V, C.POINTER(C.c_int), V, V]
    lib.vp_update_loop.argtypes = [V, C.c_int, V]
    lib.vp_optimize.argtypes = [V]
    lib.vp_sync.argtypes = [V]
    lib.vp_correct_pose.argtypes = [V, V, V, V, V]
    lib.vp_get_drift.argtypes = [V, V, V, V]
    lib.vp_get_keyframe.argtypes = [V, C.c_int, V, C.POINTER(C.c_int), V]
    lib.vp_get_path.argtypes = [V, C.c_int, V, V, V, V]
    lib.vp_info.argtypes = [V, V, V]
    lib.vp_last_timing.argtypes = [V, C.POINTER(C.c_float), C.POINTER(C.c_int)]
    lib.vp_batch_create.argtypes = [C.POINTER(PoseGraphConfig), C.c_int, C.POINTER(V)]
    lib.vp_batch_destroy.argtypes = [V]
    lib.vp_batch_size.argtypes = [V]
    lib.vp_batch_member.argtypes = [V, C.c_int]
    lib.vp_batch_member.restype = V
    lib.vp_batch_last_error.argtypes = [V]
    lib.vp_batch_last_error.restype = C.c_char_p
    lib.vp_batch_optimize.argtypes = [V, V, V]
    lib.vp_batch_sync.argtypes = [V]
    lib.vp_batch_last_timing.argtypes = [V, V, C.POINTER(C.c_int)]
    lib.vp_debug_four_dof_error.argtypes = [V, V, C.c_int, C.c_int, V]
    _bound = True


class PoseGraphError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"vinsb200 pose graph error {status}: {msg}")
        self.status = status


class PoseGraph:
    """The reference's PoseGraph with the loop already found: addKeyFrame / updateKeyFrameLoop / optimize4DoF.
    max_anchors: free loop anchors an optimised range may hold (0 = 88, at most 1024); the workspace grows with it."""

    def __init__(self, max_keyframes=2000, fast_relocalization=False, device=0, max_anchors=0):
        self.lib = load_library()
        _bind(self.lib)
        self.cfg = PoseGraphConfig(max_keyframes=max_keyframes, fast_relocalization=int(fast_relocalization), device=device,
                                   max_anchors=max_anchors)
        h = C.c_void_p()
        rc = self.lib.vp_create(C.byref(self.cfg), C.byref(h))
        if rc != 0:
            raise RuntimeError(f"vp_create failed with status {rc} (-1 = invalid configuration, -2 = no CUDA device; this library "
                               "has no CPU path)")
        self.h, self._borrowed = h, False

    @classmethod
    def _member(cls, lib, handle):
        self = cls.__new__(cls)
        self.lib, self.h, self._borrowed = lib, C.c_void_p(handle), True
        return self

    def close(self):
        if getattr(self, "h", None):
            if not self._borrowed:
                self.lib.vp_destroy(self.h)
            self.h = None

    __del__ = close

    def _check(self, rc):
        if rc < 0:
            raise PoseGraphError(rc, self.lib.vp_last_error(self.h).decode())
        return rc

    def new_sequence(self):
        self._check(self.lib.vp_new_sequence(self.h))

    def add_keyframe(self, stamp, P, Q_wxyz, loop_index=-1, loop_info=None):
        """Returns (index, stored P, stored Q wxyz)."""
        idx, P_out, Q_out = C.c_int(), np.zeros(3), np.zeros(4)
        li = _d(loop_info) if loop_info is not None else None
        self._check(self.lib.vp_add_keyframe(self.h, float(stamp), _p(_d(P)), _p(_d(Q_wxyz)), int(loop_index), _p(li), C.byref(idx),
                                             _p(P_out), _p(Q_out)))
        return idx.value, P_out, Q_out

    def update_loop(self, index, loop_info):
        self._check(self.lib.vp_update_loop(self.h, int(index), _p(_d(loop_info))))

    def optimize(self):
        return self._check(self.lib.vp_optimize(self.h))

    def sync(self):
        self._check(self.lib.vp_sync(self.h))

    def correct_pose(self, P, Q_wxyz):
        P_out, Q_out = np.zeros(3), np.zeros(4)
        self._check(self.lib.vp_correct_pose(self.h, _p(_d(P)), _p(_d(Q_wxyz)), _p(P_out), _p(Q_out)))
        return P_out, Q_out

    def drift(self):
        r, t, y = np.zeros(9), np.zeros(3), np.zeros(1)
        self._check(self.lib.vp_get_drift(self.h, _p(r), _p(t), _p(y)))
        return r.reshape(3, 3), t, float(y[0])

    def keyframe(self, index):
        v, li, lidx = np.zeros(14), np.zeros(8), C.c_int()
        self._check(self.lib.vp_get_keyframe(self.h, int(index), _p(v), C.byref(lidx), _p(li)))
        return dict(vio_P=v[:3], vio_Q=v[3:7], P=v[7:10], Q=v[10:14], loop_index=lidx.value, loop_info=li)

    def path(self):
        n = self._check(self.lib.vp_get_path(self.h, 0, None, None, None, None))
        st, P, Q, sq = np.zeros(n), np.zeros((n, 3)), np.zeros((n, 4)), np.zeros(n, np.int32)
        if n:
            self._check(self.lib.vp_get_path(self.h, n, _p(st), _p(P), _p(Q), _p(sq)))
        return st, P, Q, sq

    def info(self):
        o, c = np.zeros(8, np.int32), np.zeros(2)
        self._check(self.lib.vp_info(self.h, _p(o), _p(c)))
        keys = ["keyframes", "loops", "earliest_loop_index", "optimizations", "last_n", "last_border", "iterations", "successful"]
        d = dict(zip(keys, (int(v) for v in o)))
        d["initial_cost"], d["final_cost"] = float(c[0]), float(c[1])
        return d

    def timing(self):
        ms, n = C.c_float(), C.c_int()
        self._check(self.lib.vp_last_timing(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value


class PoseGraphBatch:
    """n independent pose graphs whose pending optimisations run in one launch chain."""

    def __init__(self, n, max_keyframes=2000, fast_relocalization=False, device=0, max_anchors=0):
        self.lib = load_library()
        _bind(self.lib)
        self.cfg = PoseGraphConfig(max_keyframes=max_keyframes, fast_relocalization=int(fast_relocalization), device=device,
                                   max_anchors=max_anchors)
        h = C.c_void_p()
        rc = self.lib.vp_batch_create(C.byref(self.cfg), int(n), C.byref(h))
        if rc != 0:
            raise RuntimeError(f"vp_batch_create failed with status {rc} (-2 = no CUDA device; this library has no CPU path)")
        self.h, self.n = h, n
        self.members = [PoseGraph._member(self.lib, self.lib.vp_batch_member(h, k)) for k in range(n)]

    def close(self):
        if getattr(self, "h", None):
            self.lib.vp_batch_destroy(self.h)
            self.h = None

    __del__ = close

    def __getitem__(self, k):
        return self.members[k]

    def optimize(self, active=None):
        """Returns the per-member status (1 enqueued, 0 nothing pending, VP_ERR_CAPACITY = -4 for a member whose range does
        not fit; the other members still run).  Any other error (the launch itself failed) raises."""
        st = np.zeros(self.n, np.int32)
        act = None if active is None else np.ascontiguousarray(active, np.int32)
        rc = self.lib.vp_batch_optimize(self.h, _p(act), _p(st))
        failed = [int(v) for v in st if v < 0 and v != -4]
        if failed or (rc < 0 and rc != -4):
            raise PoseGraphError(failed[0] if failed else rc, self.lib.vp_batch_last_error(self.h).decode())
        return st

    def sync(self):
        rc = self.lib.vp_batch_sync(self.h)
        if rc < 0:
            raise PoseGraphError(rc, self.lib.vp_batch_last_error(self.h).decode())

    def timing(self):
        ms, n = np.zeros(2, np.float32), C.c_int()
        rc = self.lib.vp_batch_last_timing(self.h, _p(ms), C.byref(n))
        if rc < 0:
            raise PoseGraphError(rc, self.lib.vp_batch_last_error(self.h).decode())
        return float(ms[0]), float(ms[1]), n.value


def debug_four_dof_error(params8, meas6, weighted=False, robust=False):
    """Device FourDOFError / FourDOFWeightError: returns (r 4, J 4x8, cost)."""
    lib = load_library()
    _bind(lib)
    out = np.zeros(37)
    rc = lib.vp_debug_four_dof_error(_p(_d(params8)), _p(_d(meas6)), int(weighted), int(robust), _p(out))
    if rc != 0:
        raise RuntimeError(f"vp_debug_four_dof_error failed with status {rc}")
    return out[:4], out[4:36].reshape(4, 8), out[36]


# ---- loop verification (include/vinsb200/loop_verify.h)

class LoopConfig(C.Structure):
    _fields_ = [("rows", C.c_int), ("cols", C.c_int), ("intrinsics", C.c_double * 8), ("ric9", C.c_double * 9), ("tic3", C.c_double * 3),
                ("brief_pattern", C.c_void_p), ("max_window", C.c_int), ("max_corners", C.c_int)]


class LoopResult(C.Structure):
    _fields_ = [("accepted", C.c_int), ("n_matches", C.c_int), ("n_inliers", C.c_int), ("n_points", C.c_int),
                ("loop_info", C.c_double * 8), ("old_R9", C.c_double * 9), ("old_T3", C.c_double * 3)]


def _bind_loop(lib):
    V = C.c_void_p
    lib.vp_loop_enable.argtypes = [V, C.POINTER(LoopConfig)]
    lib.vp_batch_loop_enable.argtypes = [V, C.POINTER(LoopConfig)]
    lib.vp_attach_keyframe.argtypes = [V, C.c_int, V, V, V, C.c_size_t, C.c_int, V, V, V, V, C.POINTER(C.c_int)]
    lib.vp_find_connection.argtypes = [V, C.c_int, C.c_int, C.POINTER(LoopResult), C.c_int, V]
    lib.vp_batch_find_connection.argtypes = [V, V, V, V, C.c_int, V, V]
    lib.vp_loop_last_timing.argtypes = [V, V]
    lib.vp_batch_loop_last_timing.argtypes = [V, V]
    lib.vp_debug_brief_blur.argtypes = [V, C.c_int, C.c_int, V]
    lib.vp_debug_fast.argtypes = [V, C.c_int, C.c_int, C.c_int, V]
    lib.vp_debug_brief.argtypes = [V, C.c_int, C.c_int, V, C.c_int, V, V]
    lib.vp_debug_match.argtypes = [C.c_int, V, C.c_int, V, V]
    lib.vp_debug_pnp.argtypes = [C.c_int, V, V, V, C.POINTER(C.c_int), V]


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


def _enable_loop(self, cfg):
    _bind_loop(self.lib)
    self._loop_cap = cfg.max_window
    self._check(self.lib.vp_loop_enable(self.h, C.byref(cfg)))


def _attach_keyframe(self, index, vio_P, vio_Q_wxyz, image, point_3d, point_uv, point_norm, point_id):
    """KeyFrame's constructor: descriptors of the window points and of the FAST corners.  Returns the corner count."""
    img = np.ascontiguousarray(image, np.uint8)
    p3, uv = np.ascontiguousarray(point_3d, np.float32).reshape(-1, 3), np.ascontiguousarray(point_uv, np.float32).reshape(-1, 2)
    nm, ids = np.ascontiguousarray(point_norm, np.float32).reshape(-1, 2), np.ascontiguousarray(point_id, np.float64).reshape(-1)
    nc = C.c_int()
    self._check(self.lib.vp_attach_keyframe(self.h, int(index), _p(_d(vio_P)), _p(_d(vio_Q_wxyz)), _p(img), img.strides[0], len(p3),
                                            _p(p3), _p(uv), _p(nm), _p(ids), C.byref(nc)))
    return nc.value


def _find_connection(self, cur, old):
    """findConnection: dict(accepted, n_matches, n_inliers, loop_info 8, old_R, old_T, points = inliers' (x, y, id))."""
    r, lst = LoopResult(), np.zeros((self._loop_cap, 3))
    self._check(self.lib.vp_find_connection(self.h, int(cur), int(old), C.byref(r), self._loop_cap, _p(lst)))
    return _result(r, lst)


def _loop_timing(self):
    ms = np.zeros(6, np.float32)
    self._check(self.lib.vp_loop_last_timing(self.h, _p(ms)))
    return ms


PoseGraph.enable_loop = _enable_loop
PoseGraph.attach_keyframe = _attach_keyframe
PoseGraph.find_connection = _find_connection
PoseGraph.loop_timing = _loop_timing


def _batch_enable_loop(self, cfg):
    _bind_loop(self.lib)
    self._loop_cap = cfg.max_window
    for m in self.members:
        m._loop_cap = cfg.max_window
    rc = self.lib.vp_batch_loop_enable(self.h, C.byref(cfg))
    if rc < 0:
        raise PoseGraphError(rc, self.lib.vp_batch_last_error(self.h).decode())


def _batch_find_connection(self, cur, old):
    """One launch chain for every member k with cur[k] >= 0; returns a list (None for skipped members)."""
    res = (LoopResult * self.n)()
    lst = np.zeros((self.n, self._loop_cap, 3))
    st = np.zeros(self.n, np.int32)
    c, o = np.ascontiguousarray(cur, np.int32), np.ascontiguousarray(old, np.int32)
    rc = self.lib.vp_batch_find_connection(self.h, _p(c), _p(o), res, self._loop_cap, _p(lst), _p(st))
    if rc < 0:
        raise PoseGraphError(rc, self.lib.vp_batch_last_error(self.h).decode())
    return [_result(res[k], lst[k]) if st[k] == 1 else None for k in range(self.n)]


def _batch_loop_timing(self):
    ms = np.zeros(6, np.float32)
    self.lib.vp_batch_loop_last_timing(self.h, _p(ms))
    return ms


PoseGraphBatch.enable_loop = _batch_enable_loop
PoseGraphBatch.find_connection = _batch_find_connection
PoseGraphBatch.loop_timing = _batch_loop_timing


def _lib():
    lib = load_library()
    _bind_loop(lib)
    return lib


def debug_brief_blur(image):
    img = np.ascontiguousarray(image, np.uint8)
    out = np.zeros_like(img)
    rc = _lib().vp_debug_brief_blur(_p(img), img.shape[0], img.shape[1], _p(out))
    if rc:
        raise RuntimeError(f"vp_debug_brief_blur failed with status {rc}")
    return out


def debug_fast(image, cap=65536):
    img = np.ascontiguousarray(image, np.uint8)
    xy = np.zeros((cap, 2), np.float32)
    n = _lib().vp_debug_fast(_p(img), img.shape[0], img.shape[1], cap, _p(xy))
    if n < 0:
        raise RuntimeError(f"vp_debug_fast failed with status {n}")
    return xy[:n].astype(np.int32)


def debug_brief(image, pattern, uv):
    img = np.ascontiguousarray(image, np.uint8)
    pat = np.ascontiguousarray(pattern, np.int32)
    pts = np.ascontiguousarray(uv, np.float32).reshape(-1, 2)
    desc = np.zeros((len(pts), 4), np.uint64)
    rc = _lib().vp_debug_brief(_p(img), img.shape[0], img.shape[1], _p(pat), len(pts), _p(pts), _p(desc))
    if rc:
        raise RuntimeError(f"vp_debug_brief failed with status {rc}")
    return desc


def debug_match(desc_a, desc_b):
    a, b = np.ascontiguousarray(desc_a, np.uint64), np.ascontiguousarray(desc_b, np.uint64)
    idx = np.zeros(len(a), np.int32)
    rc = _lib().vp_debug_match(len(a), _p(a), len(b), _p(b) if len(b) else None, _p(idx))
    if rc:
        raise RuntimeError(f"vp_debug_match failed with status {rc}")
    return idx


def debug_pnp(point_3d, norm):
    p3, nm = np.ascontiguousarray(point_3d, np.float32).reshape(-1, 3), np.ascontiguousarray(norm, np.float32).reshape(-1, 2)
    Rt, n_in, mask = np.zeros(12), C.c_int(), np.zeros(len(p3), np.uint8)
    rc = _lib().vp_debug_pnp(len(p3), _p(p3), _p(nm), _p(Rt), C.byref(n_in), _p(mask))
    if rc:
        raise RuntimeError(f"vp_debug_pnp failed with status {rc}")
    return Rt[:9].reshape(3, 3), Rt[9:], n_in.value, mask.astype(bool)
