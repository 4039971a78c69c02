"""GPU checks of pose-graph reuse (vp_save / vp_load, include/vinsb200/pose_graph.h) and of the device solve with a fixed
base map, against the numpy twin tests/pose_graph_map_twin.py.  Inputs are seeded and synthetic."""
import os

import numpy as np
import pytest

import oracle.pose_graph as opg
import pose_graph_map_twin as tw
from harness import loop_revisit, pose_graph_synth as pgs, synth
from oracle import loop_verify as olv

pytestmark = pytest.mark.gpu

INTR = [synth.FX, synth.FY, synth.CX, synth.CY, synth.K1, synth.K2, synth.P1, synth.P2]
TOL = 1e-12


def _loop_cfg(seq, max_corners=16384):
    from vins_mono_b200.pose_graph import loop_config
    return loop_config(seq.rows, seq.cols, INTR, synth.RIC, synth.TIC, olv.load_pattern(), 256, max_corners)


def _rows(prefix):
    return np.array([[float(x) for x in l.split()] for l in open(prefix + "pose_graph.txt") if l.strip()])


@pytest.fixture(scope="module")
def revisit(tmp_path_factory):
    """A graph of rendered key frames with a verified loop, optimised and saved.  Returns what the tests compare."""
    from vins_mono_b200 import PoseGraph
    seq = synth.Sequence(seed=0, duration=12.0)
    pts = loop_revisit.corner_landmarks(seq, np.arange(0.2, 12.0, 0.5))
    stamps = [0.2 + 0.6 * k for k in range(15)]  # 1.4 is key frame 2; 8.9 revisits it (2.3 m apart)
    g = PoseGraph(max_keyframes=64)
    g.enable_loop(_loop_cfg(seq))
    for idx, t in enumerate(stamps):
        p, R, *_ = seq.pose(t)
        g.attach_keyframe(idx, p, opg.R_to_quat(R), seq.render(t), np.zeros((0, 3)), np.zeros((0, 2)), np.zeros((0, 2)), np.zeros(0))
        g.add_keyframe(t, p, opg.R_to_quat(R))
    _, (img, P, Q, *win) = loop_revisit.revisit_pair(seq, pts, 1.4, 8.9)
    idx = len(stamps)
    g.attach_keyframe(idx, P, Q, img, *win)
    res = g.find_connection(idx, 2)
    loops = [(idx, 2, res, (P, Q, img, win))] if res["accepted"] else []
    g.add_keyframe(8.9, P, Q, 2 if loops else -1, res["loop_info"] if loops else None)
    stamps.append(8.9)
    g.optimize()
    g.sync()
    assert loops, "no loop was accepted"
    pre = tw.scratch_prefix(str(tmp_path_factory.mktemp("rt")))
    assert g.save(pre) == len(stamps)
    return dict(seq=seq, g=g, prefix=pre, loops=loops, n=len(stamps))


def test_save_load_round_trip(revisit, tmp_path):
    from vins_mono_b200 import PoseGraph
    r = revisit
    g2 = PoseGraph(max_keyframes=64)
    g2.enable_loop(_loop_cfg(r["seq"]))
    assert g2.load(r["prefix"]) == r["n"]
    rows = _rows(r["prefix"])
    _, P, Q, sq = g2.path()
    assert (sq == 0).all() and np.abs(P - rows[:, 5:8]).max() == 0
    _, P1, Q1, _ = r["g"].path()
    assert np.abs(P - P1).max() <= 5e-7
    for i in range(r["n"]):
        kf = g2.keyframe(i)
        assert np.array_equal(kf["P"], rows[i, 5:8]) and np.array_equal(kf["vio_P"], rows[i, 5:8])
        assert np.abs(opg.quat_to_R(kf["Q"]) - opg.quat_to_R(Q1[i])).max() < 5e-6
        assert kf["loop_index"] == int(rows[i, 16])
    assert g2.info()["earliest_loop_index"] == r["g"].info()["earliest_loop_index"]
    # saving the loaded graph reproduces the points byte for byte and the rows to the sixth decimal
    pre2 = tw.scratch_prefix(str(tmp_path))
    assert g2.save(pre2) == r["n"]
    for i in range(r["n"]):
        for s in ("keypoints.txt", "briefdes.dat"):
            assert open(r["prefix"] + f"{i}_{s}", "rb").read() == open(pre2 + f"{i}_{s}", "rb").read()
    rows2 = _rows(pre2)
    cols = [0, 1, 5, 6, 7, 12, 13, 14, 15] + list(range(16, 26))
    assert np.abs(rows2[:, cols] - rows[:, cols]).max() <= 1.000001e-6
    assert np.array_equal(rows2[:, 2:5], rows2[:, 5:8]) and np.array_equal(rows2[:, 8:12], rows2[:, 12:16])
    assert rows[:, 25].min() >= 0 and rows[:, 25].sum() > 0
    # a loaded key frame as the old one of a verification
    cur, old, res, (P, Q, img, win) = r["loops"][0]
    idx, _, _ = g2.add_keyframe(100.0, P, Q)
    g2.attach_keyframe(idx, P, Q, img, *win)
    res2 = g2.find_connection(idx, old)
    assert res2["n_matches"] == res["n_matches"] and res2["n_inliers"] == res["n_inliers"]
    assert np.array_equal(res2["points"][:, 2], res["points"][:, 2])
    # t and q within 1e-5; the relative yaw is in degrees, compared in radians
    assert np.abs(res2["loop_info"][:7] - res["loop_info"][:7]).max() < 1e-5
    assert abs(np.deg2rad(res2["loop_info"][7] - res["loop_info"][7])) < 1e-5


def _map_files(tmp_path, n=160, seed=3):
    ev1, ev2, gt1, gt2 = tw.two_sessions(n=n, seed=seed)
    g1 = tw.MapOraclePoseGraph()
    pgs.feed(g1, ev1)
    pre = tw.scratch_prefix(str(tmp_path), f"map{seed}")
    tw.write_map(pre, g1.saved())
    return pre, ev2


def _compare(g, o, n_map, loaded_P):
    _, P, Q, _ = g.path()
    for i, k in enumerate(o.kfs):
        assert np.abs(P[i] - k["P"]).max() < TOL
        assert abs(opg.normalize_angle(opg.R2ypr(opg.quat_to_R(Q[i]))[0] - opg.R2ypr(k["R"])[0])) < TOL * 100
    assert np.array_equal(P[:n_map], loaded_P)
    info = g.info()
    assert info["iterations"] == o.last["iterations"] and info["successful"] == o.last["successful"]
    return info


def test_optimisation_with_a_loaded_map_matches_the_twin(tmp_path):
    from vins_mono_b200 import PoseGraph
    pre, ev2 = _map_files(tmp_path)
    g, o = PoseGraph(max_keyframes=512), tw.MapOraclePoseGraph()
    n = g.load(pre)
    assert o.load(tw.read_map(pre, with_points=False)) == n
    loaded_P = g.path()[1].copy()
    R0 = [opg.quat_to_R(q) for q in g.path()[2]]
    tw.feed_session(g, ev2, n)
    tw.feed_session(o, ev2, n)
    info = _compare(g, o, n, loaded_P)
    assert info["last_border"] == 0 and abs(info["final_cost"] - o.last["cost"]) <= 1e-12 * max(1.0, o.last["cost"])
    _, _, Q, _ = g.path()
    for i in range(o.earliest, n):
        want = opg.ypr2R(opg.R2ypr(opg.quat_to_R(opg.R_to_quat(R0[i]))))
        assert np.abs(opg.quat_to_R(Q[i]) - want).max() < 1e-12


def test_loops_onto_a_large_map_need_no_border(tmp_path):
    from vins_mono_b200 import PoseGraph
    n_map, n_new = 2000, 300
    rows = []
    for i in range(n_map):
        q = opg.R_to_quat(opg.ypr2R([0.1 * i, 1.0, -1.0]))
        rows.append(dict(index=i, stamp=0.1 * i, vio_T=[0.05 * i, 0.0, 0.0], pg_T=[0.05 * i, 0.0, 0.0], vio_Q=q, pg_Q=q,
                         loop_index=i - 40 if i % 97 == 50 else -1, loop_info=[0.1, 0, 0, 1, 0, 0, 0, 0.5] if i % 97 == 50 else [0] * 8,
                         kp=[], kpn=[], desc=[]))
    pre = tw.scratch_prefix(str(tmp_path))
    tw.write_map(pre, rows)
    g = PoseGraph(max_keyframes=2400)
    assert g.load(pre) == n_map
    for k in range(n_new):
        i = 6 * k + 7
        q = opg.R_to_quat(opg.ypr2R([0.1 * i + 20.0, 1.0, -1.0]))
        P = opg.ypr2R([20.0, 0, 0]) @ np.array([0.05 * i + 0.3, 0.2, 0.0]) + [1.0, 2.0, 0.0]
        li = np.r_[0.02, 0.01, 0.0, 1, 0, 0, 0, 0.3]
        g.add_keyframe(1000 + 0.1 * k, P, q, i, li)
    assert g.optimize() == 1
    g.sync()
    info = g.info()
    assert info["last_border"] == 0 and info["optimizations"] == 1 and info["iterations"] >= 1


def test_batch_with_and_without_maps_equals_standalone(tmp_path):
    from vins_mono_b200 import PoseGraph, PoseGraphBatch
    maps = [_map_files(tmp_path, 120, 3), _map_files(tmp_path, 120, 4)]
    plain = [pgs.make_run(150, n_anchors=6, seed=11)[0], pgs.make_run(150, n_anchors=6, seed=12)[0]]
    b = PoseGraphBatch(4, max_keyframes=512)
    singles = [PoseGraph(max_keyframes=512) for _ in range(4)]
    for k in range(2):
        b[k].load(maps[k][0])
        singles[k].load(maps[k][0])
    streams = [[e for e in maps[0][1]], [e for e in maps[1][1]], plain[0], plain[1]]
    for k, g in enumerate(singles):
        if k < 2:
            tw.feed_session(g, streams[k], 120)
        else:
            pgs.feed(g, streams[k])
    # the batch: every member takes its next event, then one batched optimisation for those with a loop
    pos = [0] * 4
    while any(pos[k] < len(streams[k]) for k in range(4)):
        act = np.zeros(4, np.int32)
        for k in range(4):
            while pos[k] < len(streams[k]):
                ev = streams[k][pos[k]]
                pos[k] += 1
                if ev[0] == "seq":
                    b[k].new_sequence()
                    continue
                _, stamp, P, Q, l, li = ev
                b[k].add_keyframe(stamp, P, Q, l, li)
                if l >= 0:
                    act[k] = 1
                break
        if act.any():
            b.optimize(act)
            b.sync()
    for k in range(4):
        _, P, Q, _ = b[k].path()
        _, Ps, Qs, _ = singles[k].path()
        assert np.array_equal(P, Ps) and np.array_equal(Q, Qs), k


def test_failed_loads_change_nothing(revisit, tmp_path):
    from vins_mono_b200 import PoseGraph
    from vins_mono_b200._abi import VinsError
    r = revisit
    ref = PoseGraph(max_keyframes=64)
    ref.enable_loop(_loop_cfg(r["seq"]))
    ref.load(r["prefix"])
    ref_pre = tw.scratch_prefix(str(tmp_path), "ref")
    ref.save(ref_pre)
    small = PoseGraph(max_keyframes=r["n"] - 1)
    with pytest.raises(VinsError) as e:
        small.load(r["prefix"])
    assert e.value.status == -4 and small.path()[0].size == 0
    g = PoseGraph(max_keyframes=64)
    g.enable_loop(_loop_cfg(r["seq"], max_corners=int(_rows(r["prefix"])[:, 25].max()) - 1))
    with pytest.raises(VinsError) as e:
        g.load(r["prefix"])
    assert e.value.status == -4 and "max_corners" in str(e.value) and g.path()[0].size == 0
    g = PoseGraph(max_keyframes=64)
    g.enable_loop(_loop_cfg(r["seq"]))
    g.add_keyframe(0.0, [0, 0, 0], [1, 0, 0, 0])
    with pytest.raises(VinsError) as e:
        g.load(r["prefix"])
    assert e.value.status == -1 and g.path()[0].size == 1
    # a load after failures behaves as if they never happened
    h = PoseGraph(max_keyframes=64)
    h.enable_loop(_loop_cfg(r["seq"]))
    with pytest.raises(VinsError):
        h.load(str(tmp_path / "missing") + os.sep)
    assert h.load(r["prefix"]) == r["n"]
    pre = tw.scratch_prefix(str(tmp_path), "after")
    h.save(pre)
    for f in os.listdir(ref_pre):
        assert open(ref_pre + f, "rb").read() == open(pre + f, "rb").read(), f
