"""End to end on the GPU: the estimator's key frames go into a PoseGraph the way pose_graph_node receives them (the window
pose WINDOW_SIZE - 2 after each MARGIN_OLD, pubKeyframe in visualization.cpp), loops found between key frames come with
findConnection's relative pose, the loop message goes to the estimator (ve_set_relo_frame with the old key frame's
corrected pose), and ve_get_relocalization's relative pose comes back through vp_update_loop (relo_relative_pose_callback).
The corrected path must match the numpy pose graph fed the same inputs."""
import numpy as np
import pytest

from harness import pipeline, synth
from oracle import pose_graph as opg

pytestmark = pytest.mark.gpu

TOL = 1e-12


def _gt(seq, t):
    p, R, *_ = seq.pose(t)
    return p, R


def _candidate(seq, graph_stamps, t_cur, ids):
    """Old key frame for a loop at t_cur: at least 3 s older, within 3 m and 20 degrees of yaw, most matched points."""
    p1, R1 = _gt(seq, t_cur)
    best = None
    for idx, t in enumerate(graph_stamps):
        if t > t_cur - 3.0:
            break
        p0, R0 = _gt(seq, t)
        dyaw = opg.normalize_angle(opg.R2ypr(R1)[0] - opg.R2ypr(R0)[0])
        if abs(dyaw) >= 20.0 or np.linalg.norm(p1 - p0) >= 3.0:
            continue
        mp, _, _ = synth.loop_frame_matches(seq, t, ids, pixel_sigma=0.3, seed=idx)
        if len(mp) >= 40 and (best is None or len(mp) > best[1]):
            best = (idx, len(mp), mp)
    return best


@pytest.mark.parametrize("fast", [False, True])
def test_estimator_relocalisation_drives_the_pose_graph(fast):
    from vins_mono_b200 import Estimator, PoseGraph
    seq = synth.Sequence(seed=0, duration=12.0)
    msgs = synth.track_messages(seq, 110, max_feats=150)
    ids_at = {m[0]: m[1] for m in msgs}
    est = Estimator(tic=synth.TIC, ric=synth.RIC)
    est.set_seed(pipeline.gt_seed_rows(seq, [m[0] for m in msgs]), seq.ba, seq.bg)
    t_imu, acc, gyr = seq.imu()
    feeder = pipeline.ImuFeeder(t_imu, acc, gyr)
    g, o = PoseGraph(max_keyframes=256, fast_relocalization=fast), opg.OraclePoseGraph(fast_relocalization=fast)
    W = est.W
    stamps, loops_sent, updates, relo_waiting = [], 0, [], None
    rng = np.random.default_rng(1)
    for stamp, ids, d in msgs:
        feeder.feed(est, stamp)
        est.processImage(ids, d, stamp)
        info = est.info()
        if relo_waiting is not None:  # the solve after the loop message carried the relocalisation block
            r = est.relo()
            if not r["pending"] and r["solves"] > relo_waiting[1]:
                assert r["factors"] >= 20
                li = np.r_[r["relo_relative_t"], r["relo_relative_q"], r["relo_relative_yaw"]]
                g.update_loop(relo_waiting[0], li)
                o.update_loop(relo_waiting[0], li)
                updates.append(relo_waiting[0])
                relo_waiting = None
        if info["solver_flag"] != 1 or info["marginalization_flag"] != 0:
            continue
        st = est.states()[0][W - 2]
        t_kf = est.headers()[W - 2]
        loop_index, li, cand = -1, None, None
        if loops_sent < 3 and relo_waiting is None:
            cand = _candidate(seq, stamps, t_kf, ids_at[t_kf])
        if cand is not None:  # findConnection's result: the relative pose of the two key frames (PnP stands in: ground truth + noise)
            loop_index = cand[0]
            p0, R0 = _gt(seq, stamps[loop_index])
            p1, R1 = _gt(seq, t_kf)
            yaw = opg.normalize_angle(opg.R2ypr(R1)[0] - opg.R2ypr(R0)[0])
            li = np.r_[R0.T @ (p1 - p0) + rng.normal(0, 0.02, 3), opg.R_to_quat(R0.T @ R1), yaw + rng.normal(0, 0.3)]
        idx, P_g, Q_g = g.add_keyframe(t_kf, st[0:3], st[3:7], loop_index, li)
        idx_o, P_o, Q_o = o.add_keyframe(t_kf, st[0:3], st[3:7], loop_index, li)
        assert idx == idx_o == len(stamps)
        assert np.abs(P_g - P_o).max() < TOL
        stamps.append(t_kf)
        if cand is None:
            continue
        assert g.optimize() == 1 and o.optimize() == 1
        g.sync()
        loops_sent += 1
        # the loop message: this key frame's stamp and index, the matched points, the old key frame's corrected pose
        old = g.keyframe(loop_index)
        assert np.abs(old["P"] - o.kfs[loop_index]["P"]).max() < TOL
        found = est.setReloFrame(t_kf, idx, cand[2], old["P"], opg.quat_to_R(old["Q"]))
        assert found
        relo_waiting = (idx, est.relo()["solves"])
    assert loops_sent >= 2 and len(updates) >= 2, (loops_sent, updates)
    assert g.info()["optimizations"] == loops_sent
    # the later optimisations used the loop_info that vp_update_loop replaced
    assert np.array_equal(g.keyframe(updates[0])["loop_info"], o.kfs[updates[0]]["loop_info"])
    st_g, P, Q, sq = g.path()
    st_o, P_o, Q_o, sq_o = o.path()
    dP = np.abs(P - P_o).max()
    dQ = np.max([min(np.abs(a - b).max(), np.abs(a + b).max()) for a, b in zip(Q, Q_o)])
    r, t, yaw = g.drift()
    dd = max(np.abs(r - o.r_drift).max(), np.abs(t - o.t_drift).max(), abs(yaw - o.yaw_drift) / 180.0)
    print(f"key frames {len(P)}, loops {loops_sent}, loop updates {len(updates)}: dP={dP:.2e} dQ={dQ:.2e} drift={dd:.2e}")
    assert np.array_equal(st_g, st_o) and np.array_equal(sq, sq_o)
    assert dP < TOL and dQ < TOL and dd < TOL
