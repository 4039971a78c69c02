"""GPU checks of the 4-DoF pose graph (include/vinsb200/pose_graph.h) against the numpy restatement oracle/pose_graph.py:
the device residual / Jacobian of single edges, whole optimisations (iteration and successful-step counts, per-key-frame
yaw and t, costs, drift), capacity errors that leave the graph unchanged, the loop-closure effect on a drift-injected
run, batch members bit-identical to stand-alone handles, and bit-reproducible repeats."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from harness import pose_graph_synth as ps  # noqa: E402
from oracle import pose_graph as opg  # noqa: E402

pytestmark = pytest.mark.gpu

# Device vs oracle after whole optimisations.  The two solve the same damped systems in different summation orders
# (block Cholesky with a dense border vs a dense Cholesky).  Measured on an H100: at most 4e-15 in t, quaternion and drift
# over every case below; the tolerance leaves a few hundred times that.
TOL_X = 1e-12


def _vp():
    from vins_mono_b200 import PoseGraph, PoseGraphBatch, PoseGraphError, debug_four_dof_error
    return PoseGraph, PoseGraphBatch, PoseGraphError, debug_four_dof_error


def _line_events(n, loops, seed=0, seqs=()):
    """A wandering path of n key frames with VIO drift; loops = {k: j}; measurements from the ground truth."""
    rng = np.random.default_rng(seed)
    P = np.cumsum(rng.normal(0, 0.3, (n, 3)), axis=0)
    yaw = np.cumsum(rng.normal(0, 5.0, n))
    pitch, roll = rng.normal(0, 3.0, n), rng.normal(0, 3.0, n)
    R = [opg.ypr2R([yaw[k], pitch[k], roll[k]]) for k in range(n)]
    ye = np.cumsum(rng.normal(0, 0.3, n))
    pe = np.cumsum(rng.normal(0, 0.02, (n, 3)), axis=0)
    ev = []
    for k in range(n):
        if k in seqs:
            ev.append(("seq",))
        Rz = opg.ypr2R([ye[k], 0, 0])
        li, l = None, -1
        if k in loops:
            l = loops[k]
            rel_t = R[l].T @ (P[k] - P[l]) + rng.normal(0, 0.05, 3)
            rel_R = R[l].T @ R[k]
            rel_yaw = opg.normalize_angle(opg.R2ypr(R[k])[0] - opg.R2ypr(R[l])[0] + rng.normal(0, 1.0))
            rel_t = rel_t * min(1.0, 15.0 / max(np.linalg.norm(rel_t), 1e-9))
            if abs(rel_yaw) >= 29.0:
                rel_yaw = np.sign(rel_yaw) * 25.0
            li = np.r_[rel_t, opg.R_to_quat(rel_R), rel_yaw]
        ev.append(("kf", 0.1 * k, Rz @ P[k] + pe[k], opg.R_to_quat(Rz @ R[k]), l, li))
    return ev


def _run_pair(ev, fast=False, optimize_every=False):
    PoseGraph = _vp()[0]
    g, o = PoseGraph(max_keyframes=2048, fast_relocalization=fast), opg.OraclePoseGraph(fast_relocalization=fast)
    ps.feed(g, ev, optimize_every)
    ps.feed(o, ev, optimize_every)
    if not optimize_every:
        assert g.optimize() == 1 and o.optimize() == 1
        g.sync()
    return g, o


def _compare(g, o, tol=TOL_X):
    info = g.info()
    assert info["iterations"] == o.last["iterations"] and info["successful"] == o.last["successful"], (info, o.last)
    assert abs(info["initial_cost"] - o.last["cost0"]) <= 1e-9 * max(1.0, o.last["cost0"])
    assert abs(info["final_cost"] - o.last["cost"]) <= tol * max(1.0, o.last["cost"])
    st, P, Q, sq = g.path()
    st_o, P_o, Q_o, sq_o = o.path()
    assert np.array_equal(sq, sq_o)
    dP = np.abs(P - P_o).max()
    dQ = np.max([min(np.abs(a - b).max(), np.abs(a + b).max()) for a, b in zip(Q, Q_o)])
    r, t, yaw = g.drift()
    dd = max(np.abs(r - o.r_drift).max(), np.abs(t - o.t_drift).max(), abs(yaw - o.yaw_drift) / 180.0)
    print(f"n={info['last_n']} border={info['last_border']} it={info['iterations']} ok={info['successful']} "
          f"dP={dP:.2e} dQ={dQ:.2e} drift={dd:.2e}")
    assert dP < tol and dQ < tol and dd < tol, (dP, dQ, dd)
    return dP


@pytest.mark.parametrize("weighted,robust", [(0, 0), (1, 0), (1, 1)])
def test_edge_matches_oracle(weighted, robust):
    debug = _vp()[3]
    rng = np.random.default_rng(3)
    for trial in range(40):
        yi, yj = rng.uniform(-180, 180, 2)
        if trial % 4 == 0:
            yi, yj = 179.9, -179.8  # yaw difference across +-180
        xi, xj = np.r_[yi, rng.normal(0, 2, 3)], np.r_[yj, rng.normal(0, 2, 3)]
        meas = np.r_[rng.normal(0, 2, 3), rng.uniform(-20, 20)]
        pr = rng.uniform(-20, 20, 2)
        scale = 0.01 if trial % 2 else 1.0  # inside and outside the Huber threshold
        xj[1:] = xi[1:] + scale * (xj[1:] - xi[1:])
        r, J, c = debug(np.r_[xi, xj], np.r_[meas, pr], weighted, robust)
        ro, Jo, co = opg.four_dof(xi, xj, pr[0], pr[1], meas, bool(weighted), bool(robust))
        assert np.abs(r - ro).max() < 1e-12 and np.abs(J - Jo).max() < 1e-12 and abs(c - co) < 1e-12 * max(1, co)
        if not robust:  # the Jacobian against central differences
            x = np.r_[xi, xj]
            for col in range(8):
                h = 1e-6
                xp, xm = x.copy(), x.copy()
                xp[col] += h
                xm[col] -= h
                fd = (debug(xp, np.r_[meas, pr], weighted, 0)[0] - debug(xm, np.r_[meas, pr], weighted, 0)[0]) / (2 * h)
                assert np.abs(fd - J[:, col]).max() < 1e-6


SMALL = {  # n: loops {new end: anchor}; every anchor position mod 4 across the cases
    5: {4: 1},
    6: {5: 2, 4: 0},
    7: {6: 3, 5: 1},
    60: {30: 1, 34: 2, 41: 7, 50: 12, 55: 1, 58: 0, 59: 21},
}


@pytest.mark.parametrize("n", sorted(SMALL))
def test_small_graphs_match_oracle(n):
    _compare(*_run_pair(_line_events(n, SMALL[n], seed=n)))


def test_empty_border_matches_oracle():
    g, o = _run_pair(_line_events(40, {20: 0, 39: 0}, seed=5))
    assert g.info()["last_border"] == 0
    _compare(g, o)


def test_border_at_capacity_and_one_past():
    PoseGraph, _, PoseGraphError, _ = _vp()
    n = 300
    loops = {120 + k: 1 + k for k in range(88)}
    loops[299] = 0
    g, o = _run_pair(_line_events(n, loops, seed=8))
    assert g.info()["last_border"] == 352
    _compare(g, o)
    # 89 free anchors: VP_ERR_CAPACITY, and the graph behaves as if the call had not happened
    loops89 = dict(loops)
    loops89[298] = 100
    ev = _line_events(n, loops89, seed=8)
    g2 = PoseGraph(max_keyframes=2048)
    ps.feed(g2, ev, False)
    before = g2.path()
    with pytest.raises(PoseGraphError) as e:
        g2.optimize()
    assert e.value.status == -4
    after = g2.path()
    assert all(np.array_equal(a, b) for a, b in zip(before, after))
    assert g2.info()["optimizations"] == 0


def test_max_keyframes_is_a_capacity_error():
    PoseGraph, _, PoseGraphError, _ = _vp()
    g = PoseGraph(max_keyframes=8)
    ev = _line_events(9, {7: 1}, seed=2)
    for e in ev[:8]:
        g.add_keyframe(*e[1:])
    with pytest.raises(PoseGraphError) as err:
        g.add_keyframe(*ev[8][1:])
    assert err.value.status == -4
    assert g.info()["keyframes"] == 8
    assert g.optimize() == 1
    g.sync()
    assert g.info()["optimizations"] == 1


@pytest.mark.parametrize("n,anchors,kw", [
    (500, 24, {}),
    (500, 20, dict(breaks=(200,), same_anchor=4, anchor_as_new_end=True)),
    (500, 20, dict(tail_without_loop=40)),
    (2000, 88, {}),
])
def test_synthetic_runs_match_oracle(n, anchors, kw):
    ev, gt = ps.make_run(n, n_anchors=anchors, seed=n + anchors, **kw)
    g, o = _run_pair(ev)
    _compare(g, o)


def test_optimise_after_every_loop_matches_oracle():
    ev, gt = ps.make_run(300, n_anchors=8, seed=4, breaks=(150,))
    _compare(*_run_pair(ev, optimize_every=True))


@pytest.mark.parametrize("fast", [False, True])
def test_update_loop_matches_oracle(fast):
    ev = _line_events(80, {40: 3, 60: 10, 79: 20}, seed=9)
    g, o = _run_pair(ev, fast=fast, optimize_every=True)
    li = np.r_[0.1, -0.2, 0.05, 1, 0, 0, 0, 2.0]
    g.update_loop(60, li)
    o.update_loop(60, li)
    r, t, yaw = g.drift()
    assert np.abs(t - o.t_drift).max() < TOL_X and abs(yaw - o.yaw_drift) < TOL_X
    P = np.r_[1.0, 2.0, 3.0]
    Q = np.r_[1.0, 0, 0, 0]
    Pc, _ = g.correct_pose(P, Q)
    assert np.abs(Pc - (o.r_drift @ (o.w_r_vio @ P + o.w_t_vio) + o.t_drift)).max() < TOL_X


def test_loop_closure_reduces_ate():
    ev, gt = ps.make_run(600, n_anchors=40, seed=11, yaw_walk=0.15, pos_walk=0.01)
    PoseGraph = _vp()[0]
    g = PoseGraph(max_keyframes=2048)
    ps.feed(g, ev, True)
    _, P, _, _ = g.path()
    vio = np.array([e[2] for e in ev if e[0] == "kf"])

    def ate(X):
        return np.sqrt(np.mean(np.sum((X - X[0] - (gt - gt[0])) ** 2, axis=1)))

    ratio = ate(P) / ate(vio)
    print(f"ATE vio {ate(vio):.4f} m, loop-closed {ate(P):.4f} m, ratio {ratio:.3f}")
    assert ratio < 0.6


def test_batch_members_match_standalone_bit_for_bit():
    PoseGraph, PoseGraphBatch, _, _ = _vp()
    S = 64
    b = PoseGraphBatch(S, max_keyframes=512)
    runs = [ps.make_run(200 + 3 * k, n_anchors=4 + k % 9, seed=100 + k)[0] for k in range(S)]
    for k in range(S):
        ps.feed(b[k], runs[k], False)
    active = np.array([k % 5 != 3 for k in range(S)], np.int32)
    idle_before = {k: b[k].path() for k in range(S) if not active[k]}
    st = b.optimize(active)
    assert all(st[k] == (1 if active[k] else 0) for k in range(S))
    b.sync()
    for k, p in idle_before.items():
        assert all(np.array_equal(x, y) for x, y in zip(p, b[k].path()))
        assert b[k].info()["optimizations"] == 0
    for k in [0, 1, 7, 30, 62]:
        assert active[k]
        g = PoseGraph(max_keyframes=512)
        ps.feed(g, runs[k], False)
        g.optimize()
        g.sync()
        assert all(np.array_equal(x, y) for x, y in zip(g.path(), b[k].path())), k
        # a repeat run is bit-identical
        g2 = PoseGraph(max_keyframes=512)
        ps.feed(g2, runs[k], False)
        g2.optimize()
        assert all(np.array_equal(x, y) for x, y in zip(g.path(), g2.path())), k


def test_keyframes_added_while_an_optimisation_is_in_flight():
    """vp_add_keyframe never waits: key frames added after vp_optimize get the drift of the last collected optimisation, and
    are moved by the new drift when the result is collected (pose_graph.cpp:562-571)."""
    PoseGraph = _vp()[0]
    ev = _line_events(80, {40: 3, 70: 10}, seed=12)
    g, o = PoseGraph(max_keyframes=256), opg.OraclePoseGraph()
    ps.feed(g, ev[:70], True)  # the first loop's optimisation, collected
    ps.feed(o, ev[:70], True)
    g.add_keyframe(*ev[70][1:])
    o.add_keyframe(*ev[70][1:])
    g2, o2 = g, o
    assert g2.info()["optimizations"] == 1
    # second loop at key frame 70 is pending on both; the GPU graph enqueues it and keeps adding key frames
    o_pending = o2.pending
    assert g2.optimize() == 1
    stored = [g2.add_keyframe(*e[1:])[1] for e in ev[71:]]
    # the oracle adds the same key frames before its (synchronous) optimisation: they get the old drift too
    stored_o = [o2.add_keyframe(*e[1:])[1] for e in ev[71:]]
    assert o2.pending == o_pending
    for a, b in zip(stored, stored_o):
        assert np.abs(a - b).max() < TOL_X
    o2.optimize()
    g2.sync()
    _compare(g2, o2)
    _, P, _, _ = g2.path()
    assert np.abs(P[71:] - np.array(stored)).max() > 1e-6  # collected result moved them


def test_active_member_without_pending_work_is_untouched():
    _, PoseGraphBatch, _, _ = _vp()
    b = PoseGraphBatch(3, max_keyframes=256)
    runs = [_line_events(60, {40: 3, 59: 7}, seed=20 + k) for k in range(3)]
    for k in range(3):
        ps.feed(b[k], runs[k], False)
    assert list(b.optimize()) == [1, 1, 1]
    b.sync()
    before = [b[k].path() for k in range(3)]
    info = [b[k].info() for k in range(3)]
    e = _line_events(61, {40: 3, 59: 7, 60: 5}, seed=20)[-1]
    b[0].add_keyframe(*e[1:])  # only member 0 has something pending now
    st = b.optimize(np.array([1, 1, 1], np.int32))
    assert list(st) == [1, 0, 0]
    b.sync()
    for k in (1, 2):
        assert all(np.array_equal(x, y) for x, y in zip(before[k], b[k].path()))
        assert b[k].info() == info[k]
    assert b[0].info()["optimizations"] == 2


def test_later_optimisation_uses_the_updated_loop_info():
    PoseGraph = _vp()[0]
    ev = _line_events(90, {40: 3, 60: 10, 89: 20}, seed=14)
    new_li = np.r_[0.3, -0.2, 0.1, 1, 0, 0, 0, 4.0]

    def run(dev, update):
        gr = PoseGraph(max_keyframes=256) if dev else opg.OraclePoseGraph()
        ps.feed(gr, ev[:61], True)
        if update:
            gr.update_loop(60, new_li)
        ps.feed(gr, ev[61:], True)
        return gr

    g = run(True, True)
    o = run(False, True)
    _compare(g, o)
    assert np.array_equal(g.keyframe(60)["loop_info"], new_li)
    _, P_upd, _, _ = g.path()
    _, P_old, _, _ = run(True, False).path()
    assert np.abs(P_upd - P_old).max() > 1e-3  # the replaced measurement changed the later solve


def test_member_keeps_its_batch_alive_and_fails_cleanly_after_close(monkeypatch):
    import gc
    from vins_mono_b200 import VinsError, load_library
    _, PoseGraphBatch, _, _ = _vp()
    g = PoseGraphBatch(2, max_keyframes=8)[0]  # the batch itself is never bound to a name
    gc.collect()
    g.add_keyframe(0.0, [1, 2, 3], [1, 0, 0, 0])
    assert g.info()["keyframes"] == 1 and np.array_equal(g.path()[1], [[1, 2, 3]])
    b = PoseGraphBatch(2, max_keyframes=8)
    m = b[1]
    b.close()
    monkeypatch.setattr(load_library(), "vp_info", lambda *a: pytest.fail("a closed member reached the library"))
    with pytest.raises(VinsError):
        m.info()
