"""The batched key-frame attach (vp_batch_attach_keyframes, include/vinsb200/loop_attach.h) on the device: one call over
several members and slots, host and device images and different window sizes, is bit-identical to the same key frames
attached one call at a time on stand-alone graphs (corner counts, saved keypoints and descriptors, verification
results); a call with an invalid job changes no slot; a job whose corners overflow is reported alone."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import loop_verify as olv  # noqa: E402
from harness import synth  # noqa: E402

pytestmark = pytest.mark.gpu

ROWS, COLS = 480, 752
INTR = np.array([460.0, 460.0, 376.0, 240.0, 0, 0, 0, 0])
RIC, TIC = np.eye(3), np.zeros(3)
MEMBERS, SLOTS = 8, 3
INVALID, CAPACITY = -1, -4


@pytest.fixture(scope="module")
def pattern():
    return olv.load_pattern()


def _window(img, n, seed):
    """n window points on FAST corners of img (sub-pixel offset), lifted, at random depths."""
    kp, _ = olv.fast(img)
    inner = kp[(kp[:, 0] > 40) & (kp[:, 0] < COLS - 40) & (kp[:, 1] > 40) & (kp[:, 1] < ROWS - 40)]
    sel = inner[np.linspace(0, len(inner) - 1, n).astype(int)] if n else inner[:0]
    uv = sel.astype(np.float32) + np.float32(0.25)
    norm = olv.lift_pinhole(INTR, uv).astype(np.float32)
    depth = np.random.default_rng(seed).uniform(3, 8, n)
    p3d = (np.c_[norm.astype(np.float64), np.ones(n)] * depth[:, None]).astype(np.float32)
    return p3d, uv, norm, np.arange(n) + 1000.0 * seed


def _keyframes():
    """Per member 3 key frames: slot 0 an old view without window points, slots 1 and 2 two current views (the old one
    moved 3 and 5 pixels) with window points of different sizes."""
    out = {}
    for m in range(MEMBERS):
        base = synth.value_noise_image(ROWS, COLS, 100 + m)
        P = np.array([0.1 * m, 0.0, 0.0])
        Q = olv.R_to_quat(olv.quat_to_R([np.cos(0.01 * m), 0, 0, np.sin(0.01 * m)]))
        out[(m, 0)] = (P, Q, np.roll(base, 3, axis=1), _window(base, 0, 0))
        out[(m, 1)] = (P, Q, base, _window(base, 60 + 20 * m, 10 * m + 1))
        out[(m, 2)] = (P + 0.5, Q, np.roll(base, -2, axis=1), _window(np.roll(base, -2, axis=1), 256 - 10 * m, 10 * m + 2))
    return out


def _cfg(pattern, max_corners=16384):
    from vins_mono_b200.pose_graph import loop_config
    return loop_config(ROWS, COLS, INTR, RIC, TIC, pattern, 256, max_corners)


def _on_device(img, pad):
    """img as a CUDA tensor whose rows are pad bytes longer than the image (a pitched device image)."""
    import torch
    t = torch.zeros((ROWS, COLS + pad), dtype=torch.uint8, device="cuda")
    t[:, :COLS] = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    return t[:, :COLS]


def _files(g, d):
    import pose_graph_map_twin as tw
    pre = tw.scratch_prefix(str(d))
    n = g.save(pre)
    return {f: open(pre + f, "rb").read() for f in sorted(os.listdir(os.path.dirname(pre)))}, n


def _graphs_with_keyframes(b_or_graphs):
    for g in b_or_graphs:
        for k in range(SLOTS):
            g.add_keyframe(float(k), [float(k), 0, 0], [1.0, 0, 0, 0])


def test_batched_attach_equals_single_attaches(pattern, tmp_path):
    from vins_mono_b200.pose_graph import PoseGraph, PoseGraphBatch
    kfs = _keyframes()
    # stand-alone graphs, one attach call per key frame
    solo, solo_nc = [], {}
    for m in range(MEMBERS):
        g = PoseGraph(max_keyframes=8)
        g.enable_loop(_cfg(pattern))
        for k in range(SLOTS):
            P, Q, img, win = kfs[(m, k)]
            solo_nc[(m, k)] = g.attach_keyframe(k, P, Q, img, *win)
        solo.append(g)
    _graphs_with_keyframes(solo)
    # one batch, one call: jobs in a shuffled order, every other member's images on the device (two of them pitched)
    b = PoseGraphBatch(MEMBERS, max_keyframes=8)
    b.enable_loop(_cfg(pattern))
    order = list(np.random.default_rng(3).permutation([(m, k) for m in range(MEMBERS) for k in range(SLOTS)]))
    jobs = []
    for m, k in order:
        P, Q, img, win = kfs[(m, k)]
        if m % 2:
            img = _on_device(img, 64 * (m % 4 == 1))
        jobs.append((m, k, P, Q, img, *win))
    nc, st = b.attach_keyframes(jobs)
    assert (st == 0).all()
    for j, (m, k) in enumerate(order):
        assert nc[j] == solo_nc[(m, k)] > 0, (m, k)
    _graphs_with_keyframes(b.members)
    for m in range(MEMBERS):
        fs, n = _files(solo[m], tmp_path / f"solo{m}")
        fb, nb = _files(b[m], tmp_path / f"batch{m}")
        assert n == nb == SLOTS and fs == fb, m
    results = {cur: b.find_connection([cur] * MEMBERS, [0] * MEMBERS) for cur in (1, 2)}
    accepted = 0
    for m in range(MEMBERS):
        for cur in (1, 2):
            r, rb = solo[m].find_connection(cur, 0), results[cur][m]
            for key in r:
                assert np.array_equal(np.asarray(r[key]), np.asarray(rb[key])), (m, cur, key)
            accepted += r["accepted"]
    assert accepted > 0  # the comparison covers accepted loops and their point lists
    ms = b.loop_timing()
    assert np.all(ms[:3] > 0)


def _raw_jobs(specs):
    """ctypes jobs from (member, index, P, Q, img or None, window[, row stride]) tuples (host images, stride COLS by
    default); returns the array and what keeps it alive."""
    from vins_mono_b200._abi import AttachJob
    arr, keep = (AttachJob * len(specs))(), []
    for j, (m, k, P, Q, img, (p3d, uv, norm, ids), *stride) in enumerate(specs):
        P, Q = np.ascontiguousarray(P, np.float64), np.ascontiguousarray(Q, np.float64)
        arrays = [np.ascontiguousarray(p3d, np.float32), np.ascontiguousarray(uv, np.float32), np.ascontiguousarray(norm, np.float32),
                  np.ascontiguousarray(ids, np.float64)]
        a = arr[j]
        a.member, a.index, a.vio_P3, a.vio_Qwxyz = m, k, P.ctypes.data, Q.ctypes.data
        a.img, a.row_stride, a.img_on_device = (img.ctypes.data if img is not None else None), stride[0] if stride else COLS, 0
        a.n = len(arrays[0])
        a.point_3d, a.point_uv, a.point_norm, a.point_id = (v.ctypes.data for v in arrays)
        keep += [P, Q, img, *arrays]
    return arr, keep


def test_invalid_jobs_change_no_slot(pattern, tmp_path):
    from vins_mono_b200.pose_graph import PoseGraphBatch
    kfs = _keyframes()
    b = PoseGraphBatch(2, max_keyframes=8)
    b.enable_loop(_cfg(pattern))
    nc, st = b.attach_keyframes([(m, k, *kfs[(m, k)][:3], *kfs[(m, k)][3]) for m in range(2) for k in range(SLOTS)])
    assert (st == 0).all()
    _graphs_with_keyframes(b.members)
    before = [_files(b[m], tmp_path / f"before{m}") for m in range(2)]
    ref = [b[m].find_connection(1, 0) for m in range(2)]
    # every job writes a different key frame over an attached slot: a slot that changed would show
    other = {(m, k): kfs[((m + 1) % 2, (k + 1) % SLOTS)] for m in range(2) for k in range(SLOTS)}
    too_many = _window(kfs[(0, 1)][2], 257, 5)  # max_window is 256
    cases = [  # (what, slots, change to the last job, expected text)
        ("duplicate slot", [(0, 1), (1, 2), (0, 1)], None, "member 0 slot 1 appears twice"),
        ("bad member", [(0, 1), (2, 0)], None, "invalid argument"),
        ("null image", [(1, 1), (0, 2)], lambda j: j[:4] + (None,) + j[5:], "invalid argument"),
        ("row stride below cols", [(1, 1), (0, 2)], lambda j: j + (COLS - 1,), "invalid argument"),
        # VP_ERR_INVALID in a batch call, where vp_attach_keyframe reports VP_ERR_CAPACITY
        ("window above max_window", [(1, 1), (0, 2)], lambda j: j[:5] + (too_many,), "257 window points, at most max_window = 256"),
    ]
    for what, slots, change, text in cases:
        specs = [(m, k, *other[(m % 2, k)][:2], other[(m % 2, k)][2], other[(m % 2, k)][3]) for m, k in slots]
        if change:
            specs[-1] = change(specs[-1])
        arr, keep = _raw_jobs(specs)
        st = np.full(len(specs), 7, np.int32)
        rc = b.lib.vp_batch_attach_keyframes(b.h, len(specs), arr, None, st.ctypes.data)
        assert rc == INVALID, what
        bad = len(specs) - 1
        assert list(st) == [0] * bad + [INVALID], what
        msg = b.lib.vp_batch_last_error(b.h).decode()
        assert msg == f"vp_batch_attach_keyframes: job {bad}: {text}", (what, msg)
    for m in range(2):
        assert _files(b[m], tmp_path / f"after{m}") == before[m]
        again = b[m].find_connection(1, 0)
        for key in ref[m]:
            assert np.array_equal(np.asarray(ref[m][key]), np.asarray(again[key])), (m, key)


def test_corner_overflow_reports_that_job_alone(pattern, tmp_path):
    from vins_mono_b200.pose_graph import PoseGraph, PoseGraphBatch
    kfs = _keyframes()
    # a mostly flat image: a textured patch gives far fewer corners than a full textured frame
    sparse = np.full((ROWS, COLS), 128, np.uint8)
    sparse[100:260, 200:420] = synth.value_noise_image(ROWS, COLS, 7)[100:260, 200:420]
    n_sparse, n_full = len(olv.fast(sparse)[0]), len(olv.fast(kfs[(0, 1)][2])[0])
    cap = (n_sparse + n_full) // 2
    assert n_sparse < cap < n_full
    b = PoseGraphBatch(2, max_keyframes=8)
    b.enable_loop(_cfg(pattern, max_corners=cap))
    P, Q = np.zeros(3), np.array([1.0, 0, 0, 0])
    empty = _window(sparse, 0, 0)
    nc, st = b.attach_keyframes([(0, 0, P, Q, sparse, *empty), (1, 0, P, Q, sparse, *empty)])
    assert (st == 0).all()
    _graphs_with_keyframes(b.members)
    before = _files(b[1], tmp_path / "before")
    # job 1 overflows into member 1's attached slot 0; jobs 0 and 2 fit
    other = np.roll(sparse, 5, axis=0)
    nc, st = b.attach_keyframes([(0, 1, P, Q, other, *empty), (1, 0, P, Q, kfs[(0, 1)][2], *empty), (0, 2, P, Q, sparse, *empty)])
    assert list(st) == [0, CAPACITY, 0] and nc[1] == n_full and nc[0] == nc[2] == n_sparse
    assert f"job 1: {n_full} FAST corners, at most max_corners = {cap}" in b.lib.vp_batch_last_error(b.h).decode()
    assert _files(b[1], tmp_path / "after") == before
    g = PoseGraph(max_keyframes=8)  # the written jobs equal stand-alone attaches
    g.enable_loop(_cfg(pattern, max_corners=cap))
    for k, img in enumerate((sparse, other, sparse)):
        assert g.attach_keyframe(k, P, Q, img, *empty) == n_sparse
    _graphs_with_keyframes([g])
    assert _files(g, tmp_path / "solo") == _files(b[0], tmp_path / "batch")
