"""GPU checks of pose-graph optimisations whose border is larger than one CTA factors in shared memory (more than 88
free loop anchors, 352 border columns), against the numpy restatement oracle/pose_graph.py: whole optimisations on the
multi-CTA path (uncapped synthetic runs, chains up to 1024 anchors, sequence breaks, both fast_relocalization settings,
optimising after every loop across the route boundary), the anchor capacity, bit-identical results below the boundary
whatever the capacity, batches mixing both routes, and the loop-closure effect."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from harness import pose_graph_synth as ps  # noqa: E402
from oracle import pose_graph as opg  # noqa: E402

pytestmark = pytest.mark.gpu

# Device vs oracle after whole optimisations: the same damped systems solved in different summation orders (block
# Cholesky with a dense border, tiled on the tensor cores, vs numpy's dense Cholesky).
TOL_X = 1e-12
UNCAPPED = 10 ** 6
# The 1024-anchor chain (8220 unknowns) is the one case past 1e-12: 3.3e-12 in t and 6.0e-12 in the drift on an H100,
# after 5 iterations, with identical iteration and step counts and costs.  Its first damped system has condition number
# 1.3e4.  Two float64 dense Cholesky solves of that system (numpy's lower factor, as the oracle does, and LAPACK's upper
# one) have long-double residuals |A x + g| / (|A| |x|) of 7.8e-16 and 1.7e-15, and their steps still differ by 4.3e-14
# (unscaled).  A third summation order (the device's) differs by the same mechanism, compounded over the 5 accepted steps
# of a 2056-key-frame random walk.  So this case is held to 1e-11.
TOL_X_1024 = 1e-11


def _vp():
    from vins_mono_b200 import PoseGraph, PoseGraphBatch, PoseGraphError
    return PoseGraph, PoseGraphBatch, PoseGraphError


def _pair(ev, fast=False, optimize_every=False, max_keyframes=2100, max_anchors=1024):
    PoseGraph = _vp()[0]
    g = PoseGraph(max_keyframes=max_keyframes, fast_relocalization=fast, max_anchors=max_anchors)
    o = opg.OraclePoseGraph(fast_relocalization=fast)
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
    return info


def _same(g, h):
    return all(np.array_equal(x, y) for x, y in zip(g.path(), h.path())) and \
        all(np.array_equal(x, y) for x, y in zip(g.drift(), h.drift()))


def _chain_n(anchors):  # make_chain spreads the anchors over the first half and the loops over the second
    return max(300, 2 * anchors + 8)


@pytest.fixture(scope="module")
def run2000():
    ev, gt = ps.make_run(2000, n_anchors=UNCAPPED, seed=2)
    g, o = _pair(ev)
    return ev, gt, g, o


# 126 and 327 distinct anchors; the earliest is the range's constant key frame, the rest are free
@pytest.mark.parametrize("n,seed,anchors", [(1000, 1, 125), (2000, 2, 326)])
def test_uncapped_runs_match_oracle(n, seed, anchors, run2000):
    if n == 2000:
        _, _, g, o = run2000
    else:
        g, o = _pair(ps.make_run(n, n_anchors=UNCAPPED, seed=seed)[0])
    info = _compare(g, o)
    assert info["last_border"] == 4 * anchors


@pytest.mark.parametrize("anchors", [89, 96, 128, 257, 1024])
def test_chains_past_the_one_cta_border_match_oracle(anchors):
    n = _chain_n(anchors)
    g, o = _pair(ps.make_chain(n, anchors, seed=anchors), max_keyframes=max(n, 300))
    info = _compare(g, o, TOL_X_1024 if anchors == 1024 else TOL_X)
    assert info["last_border"] == 4 * anchors
    _, launches = g.timing()
    Tl = -(-(4 * anchors + 1) // 64)
    assert launches == 27 + 5 * (2 * Tl + 1), launches
    print(f"launches={launches}")


def test_sequence_breaks_match_oracle():
    ev, _ = ps.make_run(1000, n_anchors=UNCAPPED, seed=1, breaks=(500,), same_anchor=6, anchor_as_new_end=True)
    g, o = _pair(ev)
    assert _compare(g, o)["last_border"] > 352


@pytest.mark.parametrize("fast", [False, True])
def test_update_loop_past_the_one_cta_border_matches_oracle(fast):
    ev = ps.make_chain(300, 96, seed=31)
    loop_kfs = [k for k, e in enumerate(ev) if e[4] >= 0]
    g, o = _pair(ev[:-1], fast=fast)
    _compare(g, o)
    k = loop_kfs[-3]
    li = np.r_[ev[k][5][:7] + np.r_[0.1, -0.2, 0.05, 0, 0, 0, 0], ev[k][5][7] + 2.0]
    li[3:7] /= np.linalg.norm(li[3:7])
    g.update_loop(k, li)
    o.update_loop(k, li)
    r, t, yaw = g.drift()
    assert np.abs(t - o.t_drift).max() < TOL_X and abs(yaw - o.yaw_drift) < TOL_X
    P, Q = np.r_[1.0, 2.0, 3.0], np.r_[1.0, 0, 0, 0]
    Pc, _ = g.correct_pose(P, Q)
    assert np.abs(Pc - (o.r_drift @ (o.w_r_vio @ P + o.w_t_vio) + o.t_drift)).max() < TOL_X
    ps.feed(g, ev[-1:], True)  # the next optimisation uses the replaced measurement
    ps.feed(o, ev[-1:], True)
    assert _compare(g, o)["last_border"] == 4 * 96


def test_optimise_after_every_loop_across_the_boundary_matches_oracle():
    ev = ps.make_chain(240, 92, seed=7)
    PoseGraph = _vp()[0]
    g, o = PoseGraph(max_keyframes=256, max_anchors=92), opg.OraclePoseGraph()
    borders, worst = [], 0.0
    for e in ev:
        ps.feed(g, [e], True)
        ps.feed(o, [e], True)
        if e[4] >= 0:
            borders.append(g.info()["last_border"])
            worst = max(worst, float(np.abs(g.path()[1] - o.path()[1]).max()))
    print(f"worst dP over {len(borders)} optimisations: {worst:.2e}")
    assert min(borders) <= 352 < max(borders) == 4 * 92
    assert worst < TOL_X
    _compare(g, o)


def test_anchor_capacity():
    PoseGraph, _, PoseGraphError = _vp()
    A = 100
    g, o = _pair(ps.make_chain(300, A, seed=5), max_keyframes=300, max_anchors=A)
    assert _compare(g, o)["last_border"] == 4 * A
    g2 = PoseGraph(max_keyframes=300, max_anchors=A)
    ps.feed(g2, ps.make_chain(300, A + 1, seed=5), False)
    before, info = g2.path(), g2.info()
    with pytest.raises(PoseGraphError) as e:
        g2.optimize()
    assert e.value.status == -4 and f"at most {A}" in str(e.value)
    assert all(np.array_equal(a, b) for a, b in zip(before, g2.path()))
    assert g2.info() == info and info["optimizations"] == 0
    for bad in (-1, 1025):
        with pytest.raises(RuntimeError):
            PoseGraph(max_keyframes=64, max_anchors=bad)


@pytest.mark.parametrize("case", ["small", "352", "2000_88"])
def test_capacity_leaves_the_one_cta_route_bit_identical(case):
    PoseGraph = _vp()[0]
    if case == "small":
        ev = ps.make_chain(60, 7, seed=60)
    elif case == "352":
        ev = ps.make_chain(300, 88, seed=88)
    else:
        ev = ps.make_run(2000, n_anchors=88, seed=2088)[0]
    runs = []
    for cap in (0, 1024):
        g = PoseGraph(max_keyframes=2048, max_anchors=cap)
        ps.feed(g, ev, False)
        assert g.optimize() == 1
        g.sync()
        assert g.timing()[1] == 27
        runs.append(g)
    assert runs[0].info() == runs[1].info() and runs[0].info()["last_border"] <= 352
    assert _same(runs[0], runs[1])


def test_batch_mixing_routes_matches_standalone_bit_for_bit():
    PoseGraph, PoseGraphBatch, _ = _vp()
    cap_n, cap_a = 700, 160
    specs = [(600, 150), (400, 40), None, (500, 100), (300, 89), "inactive", (200, 12)]
    S = len(specs)
    evs = [ps.make_chain(s[0], s[1], seed=300 + k) if isinstance(s, tuple) else ps.make_chain(120, 4, seed=300 + k)
           for k, s in enumerate(specs)]
    evs[2] = [e[:4] + (-1, None) if e[0] == "kf" else e for e in evs[2]]  # no loop: nothing pending

    def batch_run():
        b = PoseGraphBatch(S, max_keyframes=cap_n, max_anchors=cap_a)
        for k in range(S):
            ps.feed(b[k], evs[k], False)
        active = np.array([s != "inactive" for s in specs], np.int32)
        idle = {k: (b[k].path(), b[k].info()) for k in (2, 5)}
        st = b.optimize(active)
        assert list(st) == [1, 1, 0, 1, 1, 0, 1], st
        b.sync()
        for k, (p, info) in idle.items():
            assert all(np.array_equal(x, y) for x, y in zip(p, b[k].path())) and b[k].info() == info
        return b

    b1, b2 = batch_run(), batch_run()
    Tl = -(-(4 * 150 + 1) // 64)
    assert b1.timing()[2] == 27 + 5 * (2 * Tl + 1)
    for k, s in enumerate(specs):
        if not isinstance(s, tuple):
            continue
        g = PoseGraph(max_keyframes=cap_n, max_anchors=cap_a)
        ps.feed(g, evs[k], False)
        g.optimize()
        g.sync()
        assert g.info()["last_border"] == 4 * s[1]
        assert g.timing()[1] == (27 if 4 * s[1] <= 352 else 27 + 5 * (2 * -(-(4 * s[1] + 1) // 64) + 1))
        assert _same(g, b1[k]) and b1[k].info() == g.info(), k
        assert _same(b1[k], b2[k]), k


def test_loop_closure_reduces_ate_past_the_one_cta_border(run2000):
    ev, gt, g, o = run2000
    vio = np.array([e[2] for e in ev if e[0] == "kf"])

    def ate(X):
        return np.sqrt(np.mean(np.sum((X - X[0] - (gt - gt[0])) ** 2, axis=1)))

    a_dev, a_ora, a_vio = ate(g.path()[1]), ate(o.path()[1]), ate(vio)
    print(f"border={g.info()['last_border']} ATE vio {a_vio:.4f} m, loop-closed {a_dev:.4f} m (oracle {a_ora:.4f} m), "
          f"ratio {a_dev / a_vio:.3f}")
    assert abs(a_dev - a_ora) < 1e-9
    assert a_dev < a_vio
