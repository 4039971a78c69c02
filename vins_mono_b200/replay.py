"""ctypes mirror of include/vinsb200/replay.h: the reference's two node loops (feature_tracker_node.cpp img_callback,
estimator_node.cpp process) around the CUDA handles, for sequences already in memory; any number of sequences
concurrently on one GPU."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._abi import Handle, ReplaySequence, f64, ptr


class ReplaySession(Handle):
    """sequences: list of dicts(images=<numpy u8 [n,h,w] | int device pointer>, shape=(n,h,w) when a pointer is given,
    stamps, imu_t, acc, gyr).  trackers / estimators: the Python mirrors (their .h handles are borrowed)."""
    _destroy, _last_error = "vr_close", "vr_last_error"

    def __init__(self, trackers, estimators, sequences):
        """trackers / estimators: lists of FeatureTracker / Estimator mirrors (one thread pair per sequence), or a TrackerBatch
        and an EstimatorBatch (batch mode: one tracker loop and one estimator loop, one launch chain per step for all)."""
        batch_mode = not isinstance(trackers, (list, tuple))
        n = len(sequences)
        assert (trackers.n == n and estimators.n == n) if batch_mode else (len(trackers) == n and len(estimators) == n)
        self._keep = [trackers, estimators]  # the handles and arrays the session borrows
        arr = (ReplaySequence * n)()
        for k, sq in enumerate(sequences):
            img = sq["images"]
            if isinstance(img, np.ndarray):
                img = np.ascontiguousarray(img, np.uint8)
                self._keep.append(img)
                nimg, h, w = img.shape
                arr[k].images, arr[k].images_on_device = img.ctypes.data, 0
            else:
                nimg, h, w = sq["shape"]
                arr[k].images, arr[k].images_on_device = int(img), 1
            arr[k].row_stride, arr[k].frame_stride, arr[k].n_images = w, h * w, nimg
            for name in ("stamps", "imu_t", "acc", "gyr"):
                a = f64(sq[name])
                self._keep.append(a)
                setattr(arr[k], name, a.ctypes.data)
            arr[k].n_imu = len(sq["imu_t"])
        self._arr, self.n = arr, n
        if batch_mode:
            self._open("vr_open_batch", trackers.h, estimators.h, arr)
        else:
            self._open("vr_open", n, (C.c_void_p * n)(*[t.h for t in trackers]), (C.c_void_p * n)(*[e.h for e in estimators]), arr)

    def advance(self, n_pub: int) -> int:
        return self._check(self.lib.vr_advance(self.h, n_pub))

    def queue_relo(self, seq: int, arrival_stamp, frame_stamp, frame_index, match_points, relo_t, relo_r):
        """A /pose_graph/match_points message for sequence seq (vr_queue_relo): applied before the first image at or after
        arrival_stamp, like process() drains relo_buf (estimator_node.cpp:266-291).  Not concurrently with advance()."""
        mp, t3, r9 = f64(match_points).reshape(-1, 3), f64(relo_t).reshape(3), f64(relo_r).reshape(9)
        self._check(self.lib.vr_queue_relo(self.h, seq, float(arrival_stamp), float(frame_stamp), int(frame_index), len(mp), ptr(mp),
                                           ptr(t3), ptr(r9)))

    def stats(self, seq: int):
        f, l, a, b = C.c_int(0), C.c_longlong(0), C.c_double(0), C.c_double(0)
        self._check(self.lib.vr_stats(self.h, seq, C.byref(f), C.byref(l), C.byref(a), C.byref(b)))
        return dict(frames=f.value, launches=l.value, h2d=a.value, d2h=b.value)

    def trajectory(self, seq: int):
        n = self._check(self.lib.vr_trajectory(self.h, seq, 0, None, None))
        t, p = np.zeros(n), np.zeros((n, 3))
        if n:
            self._check(self.lib.vr_trajectory(self.h, seq, n, ptr(t), ptr(p)))
        return t, p
