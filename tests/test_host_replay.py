"""The IMU side of the native node loop (vins_mono_b200/csrc/replay.cpp) against the Python feeder the parity tests use
(harness/pipeline.py ImuFeeder: estimator_node.cpp:98-136, 225-265) — no device needed."""
import ctypes as C

import numpy as np

from harness import synth, pipeline


class _Rec:
    def __init__(self):
        self.rows = []

    def processIMU(self, dt, a, g):
        self.rows.append(np.r_[dt, a, g])


def test_imu_batches_equal_python_feeder():
    from vins_mono_b200 import build, load_library
    build.build()
    lib = load_library()
    seq = synth.Sequence(seed=6, duration=3.0)
    t_imu, acc, gyr = seq.imu()
    t_imu, acc, gyr = (np.ascontiguousarray(v, np.float64) for v in (t_imu, acc, gyr))
    # image stamps: regular 10 Hz, one that coincides with an IMU sample, one just after the previous, one beyond the data
    stamps = np.array(sorted(list(0.3 + 0.1 * np.arange(20)) + [float(t_imu[137]), 1.0000001, float(t_imu[-1]) + 0.02]))
    feeder, want, counts_want = pipeline.ImuFeeder(t_imu, acc, gyr), [], []
    for s in stamps:
        rec = _Rec()
        feeder.feed(rec, float(s))
        counts_want.append(len(rec.rows))
        want += rec.rows
    want = np.array(want)
    cap = len(want) + 8
    counts = np.zeros(len(stamps), np.int32)
    dt, a, g = np.zeros(cap), np.zeros((cap, 3)), np.zeros((cap, 3))
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    n = lib.vr_debug_imu_batches(len(t_imu), p(t_imu), p(acc), p(gyr), len(stamps), p(stamps), cap, p(counts), p(dt), p(a), p(g))
    assert n == len(want) and counts.tolist() == counts_want
    got = np.c_[dt[:n], a[:n], g[:n]]
    assert np.array_equal(got, want)                      # same operations in the same order: bit-identical
    assert counts[0] > 20 and (dt[:n] >= 0).all()
