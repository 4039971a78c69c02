"""CPU tests of the node-shell remainder in the replay library (include/vinsb200/replay.h, SURVEY.md 8f next-3): the
high-rate predict()/update() of estimator_node.cpp:42-96, the result-file row of visualization.cpp:156-172 and the
PointCloud decoding of estimator_node.cpp:275-302.  Host only: no device is needed."""
import ctypes as C

import numpy as np

from vins_mono_b200 import load_library


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] + a[2] * b[0] + a[3] * b[1] - a[1] * b[3], a[0] * b[3] + a[3] * b[0] + a[1] * b[2] - a[2] * b[1]])


def qrot(q, v):
    u = q[1:]
    uv = 2 * np.cross(u, v)
    return v + q[0] * uv + np.cross(u, uv)


def test_predict_and_update_follow_the_node():
    lib = load_library()
    rng = np.random.default_rng(1)
    n = 40
    t = 10.0 + 0.005 * np.arange(n)
    acc = rng.normal(0, 1, (n, 3)) + [0, 0, 9.8]
    gyr = rng.normal(0, 0.3, (n, 3))
    P0, V0 = np.array([1.0, -2.0, 0.5]), np.array([0.3, 0.1, -0.2])
    Q0 = np.array([0.9, 0.1, -0.3, 0.2])
    Q0 /= np.linalg.norm(Q0)
    Ba, Bg = np.array([0.02, -0.01, 0.03]), np.array([0.003, -0.002, 0.001])
    a0, g0, G = acc[0] * 0.9, gyr[0] * 1.1, np.array([0, 0, 9.81007])
    h = lib.vr_prop_create()
    # update(): state at current_time, then the queued messages are re-applied
    assert lib.vr_prop_update(h, 9.999, _p(P0), _p(Q0), _p(V0), _p(Ba), _p(Bg), _p(a0), _p(g0), _p(G), 10, _p(t[:10].copy()),
                              _p(acc[:10].copy()), _p(gyr[:10].copy())) == 0
    out = np.zeros(10)
    for k in range(10, n):
        assert lib.vr_prop_predict(h, float(t[k]), _p(acc[k].copy()), _p(gyr[k].copy()), _p(out)) == 0
    # numpy restatement of predict() (estimator_node.cpp:42-78); init_imu: the very first message only latches its stamp
    P, Q, V, la, lg, lt = P0.copy(), Q0.copy(), V0.copy(), a0.copy(), g0.copy(), 9.999
    first = True
    for k in range(n):
        if first:
            lt, first = t[k], False
            continue
        dt = t[k] - lt
        lt = t[k]
        un_acc_0 = qrot(Q, la - Ba) - G
        un_gyr = 0.5 * (lg + gyr[k]) - Bg
        Q = qmul(Q, np.r_[1.0, un_gyr * dt / 2])
        un_acc_1 = qrot(Q, acc[k] - Ba) - G
        un_acc = 0.5 * (un_acc_0 + un_acc_1)
        P = P + dt * V + 0.5 * dt * dt * un_acc
        V = V + dt * un_acc
        la, lg = acc[k], gyr[k]
    assert np.allclose(out[0:3], P, rtol=0, atol=1e-12) and np.allclose(out[3:7], Q, rtol=0, atol=1e-12)
    assert np.allclose(out[7:10], V, rtol=0, atol=1e-12)
    lib.vr_prop_destroy(h)


def test_result_row_format():
    lib = load_library()
    buf = C.create_string_buffer(256)
    P, Q, V = np.array([1.234567, -0.000004, 12.5]), np.array([0.7071068, 0.0, -0.7071068, 1e-7]), np.array([0.1, -2.25, 3.999996])
    n = lib.vr_format_result_row(1403636579.763555527, _p(P), _p(Q), _p(V), buf, 256)
    # ofstream, ios::fixed: stamp * 1e9 with precision 0, the other fields with precision 5, a comma after every field
    expect = "%.0f," % (1403636579.763555527 * 1e9) + "".join("%.5f," % v for v in list(P) + list(Q) + list(V)) + "\n"
    assert n == len(expect) and buf.value.decode() == expect
    assert expect.startswith("1403636579763555") and expect.count(",") == 11
    assert lib.vr_format_result_row(1.0, _p(P), _p(Q), _p(V), buf, 8) < 0   # too small a buffer is reported, never overrun


def test_pointcloud_decoding():
    lib = load_library()
    n = 5
    xyz = np.array([[0.1, -0.2, 1], [0.3, 0.4, 1], [0, 0, 1], [-0.5, 0.25, 1], [0.01, 0.02, 1]], np.float32)
    idp = np.array([7, 123456, 0, 16777216, 42], np.float32)   # ids travel as float32 channel values (exact up to 2^24)
    u, v = np.arange(n, dtype=np.float32) * 10, np.arange(n, dtype=np.float32) * 7 + 1
    vx, vy = np.linspace(-1, 1, n).astype(np.float32), np.linspace(2, 3, n).astype(np.float32)
    ids, cams, obs = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros((n, 7))
    assert lib.vr_decode_pointcloud(n, _p(xyz), _p(idp), _p(u), _p(v), _p(vx), _p(vy), _p(ids), _p(cams), _p(obs)) == n
    assert list(ids) == [7, 123456, 0, 16777216, 42] and not cams.any()
    assert np.array_equal(obs[:, 0:3], xyz.astype(np.float64)) and np.array_equal(obs[:, 3], u) and np.array_equal(obs[:, 6], vy)
    xyz[2, 2] = 0.5   # the node asserts z == 1
    assert lib.vr_decode_pointcloud(n, _p(xyz), _p(idp), _p(u), _p(v), _p(vx), _p(vy), _p(ids), _p(cams), _p(obs)) == -1


def test_relo_message_decoding():
    """estimator_node.cpp:273-291: match_points PointCloud -> (match_points, relo_t, relo_r, frame_index)."""
    lib = load_library()
    rng = np.random.default_rng(2)
    n = 17
    xyz = np.c_[rng.uniform(-0.5, 0.5, (n, 2)), np.sort(rng.integers(0, 4000, n))].astype(np.float32)
    q = rng.normal(0, 1, 4)
    q /= np.linalg.norm(q)
    ch = np.r_[rng.normal(0, 2, 3), q, 41.0].astype(np.float32)
    mp, t3, r9, idx = np.zeros((n, 3)), np.zeros(3), np.zeros(9), C.c_int()
    assert lib.vr_decode_relo_message(n, _p(xyz), _p(ch), _p(mp), _p(t3), _p(r9), C.byref(idx)) == n
    assert np.array_equal(mp, xyz.astype(np.float64)) and np.array_equal(t3, ch[:3].astype(np.float64)) and idx.value == 41
    w, x, y, z = ch[3:7].astype(np.float64)
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                  [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    assert np.abs(r9.reshape(3, 3) - R).max() < 1e-15
    assert lib.vr_decode_relo_message(n, None, _p(ch), _p(mp), _p(t3), _p(r9), None) == -1
