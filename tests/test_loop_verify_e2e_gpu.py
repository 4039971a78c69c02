"""End to end on the GPU with loop verification inside the library: the estimator's key frames (the window pose
WINDOW_SIZE - 2 after each MARGIN_OLD) go into a PoseGraph with a yaw and translation drift injected into the VIO poses;
a ground-truth place recognition proposes an old key frame; both key frames are rendered (harness/loop_revisit.py: the
tracked landmarks are texture corners of the room) and attached; vp_find_connection decides.  An accepted loop goes to
vp_add_keyframe, its inliers to ve_set_relo_frame, and the estimator's relocalisation back through vp_update_loop.  The
loop-closed path must beat the drifted VIO path and match the numpy pose graph fed the same verified loops."""
import numpy as np
import pytest

from harness import loop_revisit, pipeline, synth
from oracle import loop_verify as olv
from oracle import pose_graph as opg

pytestmark = pytest.mark.gpu

TOL = 1e-12
INTR = [synth.FX, synth.FY, synth.CX, synth.CY, synth.K1, synth.K2, synth.P1, synth.P2]
YAW_RATE, T_RATE = 1.0, np.array([0.06, -0.04, 0.0])  # injected drift per second: degrees, metres


def _drift(t, P, Q):
    D = opg.ypr2R([YAW_RATE * t, 0, 0])
    return D @ P + T_RATE * t, D @ opg.quat_to_R(Q)


def test_verified_loops_close_the_estimator_trajectory():
    from vins_mono_b200 import Estimator, PoseGraph
    from vins_mono_b200.pose_graph import loop_config
    seq = synth.Sequence(seed=0, duration=12.0)
    pts = loop_revisit.corner_landmarks(seq, np.arange(0.2, 12.0, 0.5))
    msgs = synth.track_messages(seq, 110, max_feats=150, landmarks=pts)
    ids_at = {m[0]: m[1] for m in msgs}
    est = Estimator(tic=synth.TIC, ric=synth.RIC)
    est.set_seed(pipeline.gt_seed_rows(seq, [m[0] for m in msgs]), seq.ba, seq.bg)
    t_imu, acc, gyr = seq.imu()
    feeder = pipeline.ImuFeeder(t_imu, acc, gyr)
    g, o = PoseGraph(max_keyframes=256), opg.OraclePoseGraph()
    g.enable_loop(loop_config(seq.rows, seq.cols, INTR, synth.RIC, synth.TIC, olv.load_pattern(), 256, 16384))
    W = est.W
    stamps, vio, attached, relo_waiting = [], [], set(), None
    tried, accepted, relos = 0, [], 0
    for stamp, ids, d in msgs:
        feeder.feed(est, stamp)
        est.processImage(ids, d, stamp)
        info = est.info()
        if relo_waiting is not None:
            r = est.relo()
            if not r["pending"] and r["solves"] > relo_waiting[1]:
                li = np.r_[r["relo_relative_t"], r["relo_relative_q"], r["relo_relative_yaw"]]
                g.update_loop(relo_waiting[0], li)
                o.update_loop(relo_waiting[0], li)
                relos += 1
                relo_waiting = None
        if info["solver_flag"] != 1 or info["marginalization_flag"] != 0:
            continue
        st = est.states()[0][W - 2]
        t_kf = est.headers()[W - 2]
        P, R = _drift(t_kf, st[0:3], st[3:7])
        Q = opg.R_to_quat(R)
        idx = len(stamps)
        loop_index, li, res = -1, None, None
        cand = loop_revisit.revisit_candidate(seq, stamps, t_kf, max_dist=3.0, max_yaw=20.0)
        if cand is not None and relo_waiting is None:
            if cand not in attached:
                g.attach_keyframe(cand, vio[cand][0], vio[cand][1], seq.render(stamps[cand]), np.zeros((0, 3)), np.zeros((0, 2)),
                                  np.zeros((0, 2)), np.zeros(0))
                attached.add(cand)
            p3d, uv, norm, pid = loop_revisit.window_points(seq, t_kf, ids_at[t_kf], pts, P, R)
            g.attach_keyframe(idx, P, Q, seq.render(t_kf), p3d, uv, norm, pid)
            res = g.find_connection(idx, cand)
            tried += 1
            if res["accepted"]:
                loop_index, li = cand, res["loop_info"]
        idx_g, _, _ = g.add_keyframe(t_kf, P, Q, loop_index, li)
        o.add_keyframe(t_kf, P, Q, loop_index, li)
        assert idx_g == idx
        stamps.append(t_kf)
        vio.append((P, Q))
        if loop_index < 0:
            continue
        accepted.append((idx, loop_index, res["n_matches"], res["n_inliers"]))
        assert g.optimize() == 1 and o.optimize() == 1
        g.sync()
        old = g.keyframe(loop_index)
        pts_xyid = res["points"][np.argsort(res["points"][:, 2])]
        if est.setReloFrame(t_kf, idx, pts_xyid, old["P"], opg.quat_to_R(old["Q"])):
            relo_waiting = (idx, est.relo()["solves"])
    print(f"key frames {len(stamps)}, candidates verified {tried}, accepted (cur, old, matches, inliers) {accepted}, relocalisations {relos}")
    assert accepted, "no candidate was accepted"
    st_g, P_g, Q_g, _ = g.path()
    st_o, P_o, Q_o, _ = o.path()
    assert np.array_equal(st_g, st_o)
    assert np.abs(P_g - P_o).max() < TOL
    gt = np.array([seq.pose(t)[0] for t in st_g])
    vio_P = np.array([v[0] for v in vio])
    ate_vio = np.sqrt(np.mean(np.sum((vio_P - gt) ** 2, 1)))
    ate_loop = np.sqrt(np.mean(np.sum((P_g - gt) ** 2, 1)))
    print(f"ATE: VIO {ate_vio:.3f} m, loop-closed {ate_loop:.3f} m")
    assert ate_loop < ate_vio
