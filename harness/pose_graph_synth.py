"""Synthetic pose-graph runs: key frames along a synth.Sequence ground truth (a path that revisits itself), VIO poses with
an injected yaw and position random-walk drift (pitch and roll exact), loop edges between key frames at least
`min_gap` indices apart that are spatially close, measured as the ground-truth relative pose plus noise.

make_run() returns a list of events for PoseGraph / OraclePoseGraph:
  ("seq",)                                        new_sequence()
  ("kf", stamp, P, Q_wxyz, loop_index, loop_info8) add_keyframe(...)
and the ground-truth positions of the key frames."""
from __future__ import annotations

import numpy as np

from harness import synth


def _rz(deg):
    a = np.deg2rad(deg)
    return np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1.0]])


def _ypr(R):
    n, o, a = R[:, 0], R[:, 1], R[:, 2]
    y = np.arctan2(n[1], n[0])
    return np.rad2deg(y)


def make_run(n, n_anchors=10, seed=0, dt=0.25, min_gap=50, radius=0.6, yaw_walk=0.05, pos_walk=0.004, t_noise=0.01,
             yaw_noise=0.2, breaks=(), same_anchor=0, anchor_as_new_end=False, tail_without_loop=0):
    """n key frames, loops onto about n_anchors distinct anchors.  breaks: key-frame indices that start a new sequence.
    same_anchor: extra loops onto already used anchors.  anchor_as_new_end: the first anchor also gets a loop of its own
    onto an older key frame.  tail_without_loop: the last k key frames form a sequence of their own with no loop."""
    rng = np.random.default_rng(seed)
    seq = synth.Sequence(seed=seed % 7, duration=n * dt + 1.0)
    P_gt, R_gt = [], []
    for k in range(n):
        p, R, *_ = seq.pose(0.5 + k * dt)
        P_gt.append(p)
        R_gt.append(R)
    P_gt, R_gt = np.array(P_gt), np.array(R_gt)
    yaw_err = np.cumsum(rng.normal(0, yaw_walk, n))
    pos_err = np.cumsum(rng.normal(0, pos_walk, (n, 3)), axis=0)
    brk = set(breaks)
    if tail_without_loop:
        brk.add(n - tail_without_loop)
    seg = np.cumsum([1 if k in brk else 0 for k in range(n)])
    # VIO frame of each sequence restarts at its first key frame
    P_vio, R_vio = np.zeros((n, 3)), np.zeros((n, 3, 3))
    for k in range(n):
        Rz = _rz(yaw_err[k])
        P_vio[k] = Rz @ P_gt[k] + pos_err[k]
        R_vio[k] = Rz @ R_gt[k]
    # loops
    cand = {}
    yaw_gt = np.array([_ypr(R) for R in R_gt])
    for k in range(min_gap, n):
        if tail_without_loop and k >= n - tail_without_loop:
            break
        d = np.linalg.norm(P_gt[:k - min_gap + 1] - P_gt[k], axis=1)
        dyaw = np.abs((yaw_gt[k] - yaw_gt[:k - min_gap + 1] + 180.0) % 360.0 - 180.0)
        d[dyaw > 20.0] = np.inf  # the loop gate accepts |relative yaw| < 30 degrees
        j = int(np.argmin(d))
        if d[j] < radius:
            cand[k] = j
    loops, anchors = {}, []
    keys = sorted(cand)
    stride = max(1, len(keys) // max(1, n_anchors))
    for k in keys[::stride]:
        j = cand[k]
        if j in anchors or any(abs(j - a) < 2 for a in anchors) or j in loops:
            continue
        if len(anchors) >= n_anchors:
            break
        loops[k] = j
        anchors.append(j)
    free = [k for k in keys if k not in loops]
    extra = 0
    for k in free:
        older = [a for a in anchors if a <= k - min_gap]
        if extra >= same_anchor or not older:
            continue
        loops[k] = older[extra % len(older)]
        extra += 1
    if anchor_as_new_end and anchors:
        a = max(anchors)
        if a >= min_gap:
            d = np.linalg.norm(P_gt[:a - min_gap + 1] - P_gt[a], axis=1)
            loops[a] = int(np.argmin(d))
    events = []
    for k in range(n):
        if k in brk:
            events.append(("seq",))
        li, l = None, -1
        if k in loops:
            l = loops[k]
            Rj = R_gt[l]
            rel_t = Rj.T @ (P_gt[k] - P_gt[l]) + rng.normal(0, t_noise, 3)
            rel_R = Rj.T @ R_gt[k]
            rel_yaw = _ypr(R_gt[k]) - _ypr(Rj) + rng.normal(0, yaw_noise)
            rel_yaw = (rel_yaw + 180.0) % 360.0 - 180.0
            li = np.r_[rel_t, synth.rot_to_quat_wxyz(rel_R), rel_yaw]
        events.append(("kf", 0.5 + k * dt, P_vio[k], synth.rot_to_quat_wxyz(R_vio[k]), l, li))
    return events, P_gt


def feed(graph, events, optimize_every=True):
    """Drives a PoseGraph or OraclePoseGraph with the events; optimises (and waits) after every key frame with a loop."""
    for ev in events:
        if ev[0] == "seq":
            graph.new_sequence()
            continue
        _, stamp, P, Q, l, li = ev
        graph.add_keyframe(stamp, P, Q, l, li)
        if optimize_every and l >= 0:
            graph.optimize()
            if hasattr(graph, "sync"):
                graph.sync()


def make_chain(n, n_anchors, seed=0, n_loops=None):
    """A random-walk path of n key frames with VIO drift and loops onto exactly n_anchors distinct anchors (spread over
    the first half; the loops start in the second half, one or more per anchor), measured from the ground truth.
    Key frame 0 is the earliest anchor as well, so the range is the whole graph.  Returns the events."""
    rng = np.random.default_rng(seed)
    P = np.cumsum(rng.normal(0, 0.3, (n, 3)), axis=0)
    yaw = np.cumsum(rng.normal(0, 3.0, n))
    R = [synth._rz(np.deg2rad(yaw[k])) @ synth._ry(np.deg2rad(rng.normal(0, 3))) @ synth._rx(np.deg2rad(rng.normal(0, 3)))
         for k in range(n)]
    ye, pe = np.cumsum(rng.normal(0, 0.1, n)), np.cumsum(rng.normal(0, 0.01, (n, 3)), axis=0)
    anchors = [0] + list(np.linspace(1, n // 2 - 1, n_anchors).astype(int)) if n_anchors else [0]
    srcs = np.linspace(n // 2 + 1, n - 1, max(n_loops or len(anchors), len(anchors))).astype(int)
    loops = {int(k): int(anchors[i % len(anchors)]) for i, k in enumerate(srcs)}
    events = []
    for k in range(n):
        li, l = None, -1
        if k in loops:
            l = loops[k]
            rel_t = R[l].T @ (P[k] - P[l])
            rel_t = rel_t * min(1.0, 15.0 / max(np.linalg.norm(rel_t), 1e-9)) + rng.normal(0, 0.02, 3)
            rel_yaw = float(np.clip((yaw[k] - yaw[l] + 180.0) % 360.0 - 180.0, -25, 25)) + rng.normal(0, 0.5)
            li = np.r_[rel_t, synth.rot_to_quat_wxyz(R[l].T @ R[k]), rel_yaw]
        Rz = _rz(ye[k])
        events.append(("kf", 0.1 * k, Rz @ P[k] + pe[k], synth.rot_to_quat_wxyz(Rz @ R[k]), l, li))
    return events
