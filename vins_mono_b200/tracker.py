"""ctypes mirror of include/vinsb200/tracker.h; class/method names follow the reference's
FeatureTracker (feature_tracker/src/feature_tracker.h:28-64)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import LIB_PATH, Batch, Handle, TrackerConfig, load_library, ptr  # noqa: F401


def _make_tracker_config(rows=480, cols=752, max_cnt=150, min_dist=30, freq=10, equalize=1, focal_length=460,
                         f_threshold=1.0, fx=461.6, fy=460.3, cx=363.0, cy=248.1, k1=-0.2917, k2=0.08228, p1=5.333e-05,
                         p2=-1.578e-04, fisheye=0, fisheye_mask=None, device=0, camera_model=0, xi=0.0, **_ignored):
    """camera_model 0 PINHOLE (fx fy cx cy k1 k2 p1 p2), 1 MEI (the same slots hold gamma1 gamma2 u0 v0 k1 k2 p1 p2, plus xi),
    2 KANNALA_BRANDT (mu mv u0 v0 k2 k3 k4 k5)."""
    cfg = TrackerConfig(rows=rows, cols=cols, max_cnt=max_cnt, min_dist=min_dist, freq=freq, equalize=equalize,
                        fisheye=fisheye, focal_length=focal_length, f_threshold=f_threshold, camera_model=int(camera_model),
                        device=device, xi=float(xi))
    cfg.intrinsics[:] = [fx, fy, cx, cy, k1, k2, p1, p2]
    mask = np.ascontiguousarray(fisheye_mask, np.uint8) if fisheye_mask is not None else None
    cfg.fisheye_mask = mask.ctypes.data if mask is not None else None
    return cfg, mask


class FeatureTracker(Handle):
    """Drop-in for the reference FeatureTracker: readImage(img, t) then read the public result arrays."""
    _destroy, _last_error = "vt_destroy", "vt_last_error"

    def __init__(self, **kw):
        cfg, self._mask = _make_tracker_config(**kw)
        self.cfg, self.rows, self.cols, self.max_cnt = cfg, cfg.rows, cfg.cols, cfg.max_cnt
        self.PUB_THIS_FRAME = False
        self._open("vt_create", C.byref(cfg))

    @classmethod
    def _member(cls, batch, k):
        self = cls._borrow(batch, batch.lib.vt_batch_member(batch.h, k))
        self.cfg, self.rows, self.cols, self.max_cnt = batch.cfg, batch.cfg.rows, batch.cfg.cols, batch.cfg.max_cnt
        self.PUB_THIS_FRAME, self._mask = False, None
        return self

    # FeatureTracker::readImage(const cv::Mat&, double) + updateID loop; PUB_THIS_FRAME is the reference's global
    def readImage(self, img, cur_time, pub_this_frame=None):
        img = np.ascontiguousarray(img, np.uint8)
        assert img.shape == (self.rows, self.cols)
        pub = self.PUB_THIS_FRAME if pub_this_frame is None else pub_this_frame
        self._check(self.lib.vt_read_image(self.h, ptr(img), img.strides[0], float(cur_time), int(bool(pub))))
        return self.result()

    def read_image_device(self, dptr, stride, cur_time, pub):
        self._check(self.lib.vt_read_image_device(self.h, C.c_void_p(dptr), stride, float(cur_time), int(bool(pub))))

    def node_image(self, img, stamp):
        """img_callback: returns (ret, restart) with ret 0/1/2 as in vt_node_image."""
        img = np.ascontiguousarray(img, np.uint8)
        restart = C.c_int(0)
        r = self._check(self.lib.vt_node_image(self.h, ptr(img), img.strides[0], float(stamp), C.byref(restart)))
        return r, restart.value

    def node_image_device(self, dptr, stride, stamp):
        restart = C.c_int(0)
        return self._check(self.lib.vt_node_image_device(self.h, C.c_void_p(dptr), stride, float(stamp), C.byref(restart)))

    def result(self):
        n = self._check(self.lib.vt_count(self.h))
        ids, tc = np.zeros(n, np.int32), np.zeros(n, np.int32)
        cur, un, vel = (np.zeros((n, 2), np.float32) for _ in range(3))
        self._check(self.lib.vt_get(self.h, ptr(ids), ptr(tc), ptr(cur), ptr(un), ptr(vel)))
        self.ids, self.track_cnt, self.cur_pts, self.cur_un_pts, self.pts_velocity = ids, tc, cur, un, vel
        return dict(ids=ids, track_cnt=tc, cur_pts=cur, un_pts=un, velocity=vel)

    def feature_message(self):
        """PointCloud payload of the last published frame: dict id -> (x, y, z, u, v, vx, vy)."""
        cap = self.max_cnt
        xy = np.zeros((cap, 2), np.float32)
        ch = [np.zeros(cap, np.float32) for _ in range(5)]
        n = self._check(self.lib.vt_node_pack(self.h, cap, ptr(xy), *[ptr(c) for c in ch]))
        return {int(ch[0][i]): (float(xy[i, 0]), float(xy[i, 1]), 1.0, float(ch[1][i]), float(ch[2][i]),
                                float(ch[3][i]), float(ch[4][i])) for i in range(n)}

    KERNEL_GROUPS = ["clahe", "pyrdown", "lk_track", "mask_discs", "min_eig", "gftt_tail"]

    def set_profile(self, on):
        self._check(self.lib.vt_set_profile(self.h, int(on)))

    def kernel_times(self):
        ms, cnt = np.zeros(6), np.zeros(6, np.int32)
        self._check(self.lib.vt_kernel_times(self.h, ptr(ms), ptr(cnt)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(self.KERNEL_GROUPS)}

    def traffic(self):
        a, b = C.c_double(0), C.c_double(0)
        self._check(self.lib.vt_last_traffic(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def timing(self):
        ms, k = C.c_float(0), C.c_int(0)
        self._check(self.lib.vt_last_timing(self.h, C.byref(ms), C.byref(k)))
        return ms.value, k.value

    # --- single-stage access for parity tests ---
    def debug_level(self, level):
        out = np.zeros((self.rows, self.cols), np.uint8)
        r, c = C.c_int(0), C.c_int(0)
        self._check(self.lib.vt_debug_equalized(self.h, level, ptr(out), C.byref(r), C.byref(c)))
        return out.ravel()[: r.value * c.value].reshape(r.value, c.value).copy()

    def debug_gftt(self, img, mask, max_corners, want_eig=False):
        img = np.ascontiguousarray(img, np.uint8)
        mask = np.ascontiguousarray(mask, np.uint8) if mask is not None else None
        out = np.zeros((max_corners, 2), np.float32)
        nc = C.c_int(0)
        eig = np.zeros((self.rows, self.cols), np.float32) if want_eig else None
        n = self._check(self.lib.vt_debug_gftt(self.h, ptr(img), img.strides[0], ptr(mask), max_corners, ptr(out),
                                               C.byref(nc), ptr(eig)))
        return out[:n].copy(), nc.value, eig

    def debug_lk(self, prev, nxt, pts):
        prev, nxt = np.ascontiguousarray(prev, np.uint8), np.ascontiguousarray(nxt, np.uint8)
        pts = np.ascontiguousarray(pts, np.float32)
        n = len(pts)
        out, st = np.zeros((n, 2), np.float32), np.zeros(n, np.uint8)
        self._check(self.lib.vt_debug_lk(self.h, ptr(prev), ptr(nxt), prev.strides[0], ptr(pts), n, ptr(out), ptr(st)))
        return out, st


class TrackerBatch(Batch):
    """n trackers advancing image by image together (include/vinsb200/tracker.h, vt_batch_*): one launch per kernel stage
    for the whole batch.  members[k] is a FeatureTracker mirror for result() / feature_message()."""
    _destroy, _last_error = "vt_batch_destroy", "vt_batch_last_error"

    def __init__(self, n, **kw):
        self.cfg, self._mask = _make_tracker_config(**kw)
        self.n, self.rows, self.cols = n, self.cfg.rows, self.cfg.cols
        self._open("vt_batch_create", C.byref(self.cfg), n)
        self.members = [FeatureTracker._member(self, k) for k in range(n)]

    def _pointers(self, imgs):
        n = self.n
        active = np.zeros(n, np.int32)
        ptrs, keep, stride, dev = (C.c_void_p * n)(), [], self.cols, 0
        for k, im in enumerate(imgs):
            if im is None:
                continue
            active[k] = 1
            if isinstance(im, np.ndarray):
                im = np.ascontiguousarray(im, np.uint8)
                assert im.shape == (self.rows, self.cols)
                keep.append(im)
                ptrs[k] = im.ctypes.data
            else:  # device pointer (int), rows x cols contiguous
                ptrs[k], dev = int(im), 1
        return active, ptrs, keep, stride, dev

    def readImage(self, imgs, cur_times, pubs):
        """imgs[k]: numpy frame, device pointer or None (member idles)."""
        active, ptrs, keep, stride, dev = self._pointers(imgs)
        t = np.ascontiguousarray(cur_times, np.float64)
        p = np.ascontiguousarray(pubs, np.int32)
        self._check(self.lib.vt_batch_read_image(self.h, ptr(active), ptrs, stride, ptr(t), ptr(p), dev))

    def node_image(self, imgs, stamps):
        """img_callback for every member with a frame; returns (results, restarts) arrays (0 / 1 / 2 per member)."""
        active, ptrs, keep, stride, dev = self._pointers(imgs)
        t = np.ascontiguousarray(stamps, np.float64)
        res, rst = np.zeros(self.n, np.int32), np.zeros(self.n, np.int32)
        self._check(self.lib.vt_batch_node_image(self.h, ptr(active), ptrs, stride, ptr(t), dev, ptr(res), ptr(rst)))
        return res, rst

    def timing(self):
        ms, k = C.c_float(0), C.c_int(0)
        self._check(self.lib.vt_batch_last_timing(self.h, C.byref(ms), C.byref(k)))
        return ms.value, k.value

    def set_profile(self, on):
        self._check(self.lib.vt_batch_set_profile(self.h, int(on)))

    def kernel_times(self):
        ms, cnt = np.zeros(6), np.zeros(6, np.int32)
        self._check(self.lib.vt_batch_kernel_times(self.h, ptr(ms), ptr(cnt)))
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(FeatureTracker.KERNEL_GROUPS)}
