"""numpy twin of pose-graph reuse: the reference's saved-map format (savePoseGraph / loadPoseGraph,
pose_graph/src/pose_graph.cpp:697-870) and oracle/pose_graph.py's restatement extended with a loaded map (the loaded
key-frame constructor, keyframe.cpp:44-70, and optimize4DoF's `sequence == 0` constants, pose_graph.cpp:473).  Edges
between two constant key frames are left out of the minimiser, as Ceres removes such residual blocks before it
minimises (they are only its fixed cost).  Test infrastructure only."""
from __future__ import annotations

import os

import numpy as np

import oracle.pose_graph as opg

ROW = " %d" + " %f" * 15 + " %d" + " %f" * 8 + " %d\n"


# ---- the format
def desc_line(words):
    """boost::dynamic_bitset's operator<<: bit 255 first.  words: 4 uint64, bit i in word i // 64."""
    bits = [(int(words[(255 - j) >> 6]) >> ((255 - j) & 63)) & 1 for j in range(256)]
    return "".join("1" if b else "0" for b in bits) + "\n"


def parse_desc(line):
    assert len(line) == 256 and set(line) <= {"0", "1"}, "descriptor line"
    w = [0, 0, 0, 0]
    for j, ch in enumerate(line):
        if ch == "1":
            w[(255 - j) >> 6] |= 1 << ((255 - j) & 63)
    return np.array(w, np.uint64)


def write_map(prefix, kfs):
    """kfs: dicts with index, stamp, vio_T, pg_T, vio_Q, pg_Q (w x y z), loop_index, loop_info, kp (n, 2), kpn (n, 2),
    desc (n, 4) uint64."""
    with open(prefix + "pose_graph.txt", "w") as f:
        for k in kfs:
            n = len(k["kp"])
            f.write(ROW % (k["index"], k["stamp"], *k["vio_T"], *k["pg_T"], *k["vio_Q"], *k["pg_Q"], k["loop_index"], *k["loop_info"], n))
            with open(prefix + "%d_briefdes.dat" % k["index"], "w") as fb, open(prefix + "%d_keypoints.txt" % k["index"], "w") as fk:
                for i in range(n):
                    fb.write(desc_line(k["desc"][i]))
                    fk.write("%f %f %f %f\n" % (float(k["kp"][i][0]), float(k["kp"][i][1]), float(k["kpn"][i][0]), float(k["kpn"][i][1])))


def read_map(prefix, with_points=True):
    kfs = []
    for line in open(prefix + "pose_graph.txt").read().split("\n"):
        if not line.strip():
            continue
        t = line.split()
        assert len(t) == 26, "pose_graph.txt line"
        v = [float(x) for x in t]
        k = dict(index=int(t[0]), stamp=v[1], vio_T=np.array(v[2:5]), pg_T=np.array(v[5:8]), vio_Q=np.array(v[8:12]),
                 pg_Q=np.array(v[12:16]), loop_index=int(t[16]), loop_info=np.array(v[17:25]), n=int(t[25]))
        assert k["index"] == len(kfs) and -1 <= k["loop_index"] < k["index"]
        if with_points:
            rows = [r.split() for r in open(prefix + "%d_keypoints.txt" % k["index"]).read().split("\n") if r.strip()]
            assert len(rows) == k["n"]
            p = np.array([[float(x) for x in r] for r in rows], np.float64).reshape(-1, 4).astype(np.float32)
            k["kp"], k["kpn"] = p[:, :2], p[:, 2:]
            des = open(prefix + "%d_briefdes.dat" % k["index"]).read()
            assert len(des) == 257 * k["n"]
            k["desc"] = np.array([parse_desc(des[257 * i:257 * i + 256]) for i in range(k["n"])], np.uint64).reshape(-1, 4)
        kfs.append(k)
    return kfs


# ---- the restatement
class MapProblem(opg.Problem):
    """optimize4DoF's problem of one range with a constant mask: the edges between two constants are dropped."""

    def __init__(self, vio_P, vio_R, seq, loops, const):
        super().__init__(vio_P, vio_R, seq, loops)
        self.const = np.asarray(const, bool)
        self.edges = [e for e in self.edges if not (self.const[e[0]] and self.const[e[1]])]

    def solve(self, max_iterations=5, function_tolerance=1e-6):
        n = self.n
        free = np.flatnonzero(~self.const)
        cols = np.concatenate([np.arange(4 * i, 4 * i + 4) for i in free]) if len(free) else np.zeros(0, int)
        x = self.x0.copy()
        lin, cost = self.evaluate(x)
        cost0 = cost
        radius, dec, scale = 1e4, 2.0, None
        need_lin, converged, it, succ = True, False, 0, 0
        H = g = None
        while it < max_iterations and not converged and len(free) and n >= 2:
            if need_lin:
                lin, _ = self.evaluate(x)
                Hf, gf = np.zeros((4 * n, 4 * n)), np.zeros(4 * n)
                for (a, b, r, J) in lin:
                    idx = np.r_[4 * a:4 * a + 4, 4 * b:4 * b + 4]
                    Hf[np.ix_(idx, idx)] += J.T @ J
                    gf[idx] += J.T @ r
                Hu, gu = Hf[np.ix_(cols, cols)], gf[cols]
                if scale is None:
                    scale = 1.0 / (1.0 + np.sqrt(np.diag(Hu)))
                H, g = Hu * np.outer(scale, scale), gu * scale
                need_lin = False
                if np.max(np.abs(gu)) <= 1e-10:
                    converged = True
                    break
            A = H + np.diag(np.clip(np.diag(H), 1e-6, 1e32) / radius)
            it += 1
            try:
                Lc = np.linalg.cholesky(A)
                ds = -np.linalg.solve(Lc.T, np.linalg.solve(Lc, g))
                ok = np.all(np.isfinite(ds))
            except np.linalg.LinAlgError:
                ok = False
            mc = 0.0
            if ok:
                d = ds * scale
                dfull = np.zeros((n, 4))
                dfull[free] = d.reshape(-1, 4)
                for (a, b, r, J) in lin:
                    jd = J @ np.r_[dfull[a], dfull[b]]
                    mc -= jd @ (r + 0.5 * jd)
                ok = mc > 0 and np.isfinite(mc)
            if not ok:
                radius /= dec
                dec *= 2
                if radius < 1e-32:
                    break
                continue
            xc = x.copy()
            for i in free:
                xc[i, 0] = opg.normalize_angle(x[i, 0] + dfull[i, 0])
                xc[i, 1:] = x[i, 1:] + dfull[i, 1:]
            _, cc = self.evaluate(xc, jac=False)
            if np.linalg.norm(d) <= 1e-8 * (np.linalg.norm(x[free]) + 1e-8):
                converged = True
                continue
            change = cost - cc
            if np.isfinite(cc) and abs(change) <= function_tolerance * cost:
                if change > 0:
                    x, cost, succ = xc, cc, succ + 1
                converged = True
                continue
            rho = change / mc
            if np.isfinite(cc) and rho > 1e-3:
                x, cost, succ = xc, cc, succ + 1
                radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - (2 * rho - 1) ** 3))
                dec, need_lin = 2.0, True
            else:
                radius /= dec
                dec *= 2
                if radius < 1e-32:
                    break
        return x, dict(iterations=it, successful=succ, cost0=cost0, cost=cost, converged=converged)


class MapOraclePoseGraph(opg.OraclePoseGraph):
    """OraclePoseGraph with load(): loaded key frames are sequence 0 and constant in every optimisation."""

    def load(self, kfs):
        assert not self.kfs
        for m in kfs:
            R = opg.quat_to_R(m["pg_Q"])  # not normalised
            li = np.asarray(m["loop_info"], float)
            self.kfs.append(dict(stamp=m["stamp"], seq=0, has_loop=m["loop_index"] != -1, loop_index=m["loop_index"], loop_info=li.copy(),
                                 vio_P=np.array(m["pg_T"], float), vio_R=R.copy(), P=np.array(m["pg_T"], float), R=R.copy()))
            if m["loop_index"] != -1 and (self.earliest == -1 or m["loop_index"] < self.earliest):
                self.earliest = m["loop_index"]
        return len(kfs)

    def saved(self):
        """The rows vp_save writes (without points)."""
        return [dict(index=i, stamp=k["stamp"], vio_T=k["vio_P"], pg_T=k["P"], vio_Q=opg.R_to_quat(k["vio_R"]), pg_Q=opg.R_to_quat(k["R"]),
                     loop_index=k["loop_index"] if k["has_loop"] else -1, loop_info=k["loop_info"], kp=[], kpn=[], desc=[])
                for i, k in enumerate(self.kfs)]

    def problem(self):
        first, cur = self.earliest, self.pending
        rng = self.kfs[first:cur + 1]
        loops = [(k["loop_index"] - first, np.r_[k["loop_info"][:3], k["loop_info"][7]]) if k["has_loop"] else None for k in rng]
        const = [i == 0 or k["seq"] == 0 for i, k in enumerate(rng)]
        return MapProblem([k["vio_P"] for k in rng], [k["vio_R"] for k in rng], [k["seq"] for k in rng], loops, const)


def two_sessions(n=160, seed=3, yaw0=35.0, offset=(4.0, -2.0, 0.5), loop_every=8, dt=0.25):
    """Session 1: harness.pose_graph_synth.make_run(n, seed).  Session 2 revisits the same path (same ground truth) with
    its own VIO drift, in a VIO frame turned by yaw0 and moved by offset, and without loops of its own; its key frame k
    loops onto session-1 key frame k - 2 every loop_every key frames (global index = n_map + k once loaded).  Returns
    (events 1, events 2 with loop indices into the map, ground truth 1, ground truth 2)."""
    from harness import pose_graph_synth as pgs
    from harness import synth
    ev1, gt1 = pgs.make_run(n, seed=seed, dt=dt)
    ev2, gt2 = pgs.make_run(n, n_anchors=0, seed=seed + 7, dt=dt)  # same synth.Sequence (seed % 7), other drift
    sq = synth.Sequence(seed=seed % 7, duration=n * dt + 1.0)
    R_gt = [sq.pose(0.5 + k * dt)[1] for k in range(n)]
    rng = np.random.default_rng(seed + 100)
    Rz = opg.ypr2R([yaw0, 0, 0])
    out, k = [], 0
    for ev in ev2:
        if ev[0] != "kf":
            continue
        _, stamp, P, Q, _, _ = ev
        P2, Q2 = Rz @ P + np.asarray(offset), opg.R_to_quat(Rz @ opg.quat_to_R(Q))
        l, li = -1, None
        if k >= 2 and k % loop_every == 0:
            l = k - 2
            Rj = R_gt[l]
            rel_t = Rj.T @ (gt2[k] - gt1[l]) + rng.normal(0, 0.01, 3)
            rel_R = Rj.T @ R_gt[k]
            rel_yaw = opg.R2ypr(R_gt[k])[0] - opg.R2ypr(Rj)[0] + rng.normal(0, 0.2)
            li = np.r_[rel_t, synth.rot_to_quat_wxyz(rel_R), (rel_yaw + 180.0) % 360.0 - 180.0]
        out.append(("kf", 1000.0 + stamp, P2, Q2, l, li))
        k += 1
    return ev1, out, gt1, gt2


def feed_session(graph, events, n_map, optimize=True):
    """Session-2 events into a graph holding a map of n_map key frames (loop targets are map indices)."""
    for _, stamp, P, Q, l, li in events:
        graph.add_keyframe(stamp, P, Q, l, li)
        if optimize and l >= 0:
            graph.optimize()
            if hasattr(graph, "sync"):
                graph.sync()


def ate(P, gt):
    """RMS position error after the best rigid alignment (Umeyama, no scale)."""
    P, gt = np.asarray(P, float), np.asarray(gt, float)
    mp, mg = P.mean(0), gt.mean(0)
    U, _, Vt = np.linalg.svd((gt - mg).T @ (P - mp))
    D = np.diag([1, 1, np.sign(np.linalg.det(U @ Vt))])
    R = U @ D @ Vt
    return float(np.sqrt(np.mean(np.sum((gt - (mg + (P - mp) @ R.T)) ** 2, axis=1))))


def scratch_prefix(d, name="map"):
    os.makedirs(os.path.join(d, name), exist_ok=True)
    return os.path.join(d, name) + os.sep
