"""numpy restatement of the reference's pose graph (pose_graph/src/pose_graph.cpp, pose_graph.h): addKeyFrame with the
loop already found, updateKeyFrameLoop, and optimize4DoF including the Ceres 1.14 Levenberg-Marquardt loop in the form
vins_mono_b200/csrc/initial.cpp's sfm_bundle restates (Jacobi scaling fixed at the first Jacobian, radius 1e4, the
1 - (2 rho - 1)^3 rule, diagonal clamp [1e-6, 1e32], tolerances 1e-6 / 1e-8 / 1e-10).  The normal equations are
solved densely.  Test infrastructure only."""
from __future__ import annotations

import numpy as np

HUBER_A = 0.1


def ypr2R(ypr):
    y, p, r = np.asarray(ypr, float) / 180.0 * np.pi
    Rz = np.array([[np.cos(y), -np.sin(y), 0], [np.sin(y), np.cos(y), 0], [0, 0, 1.0]])
    Ry = np.array([[np.cos(p), 0, np.sin(p)], [0, 1.0, 0], [-np.sin(p), 0, np.cos(p)]])
    Rx = np.array([[1.0, 0, 0], [0, np.cos(r), -np.sin(r)], [0, np.sin(r), np.cos(r)]])
    return Rz @ Ry @ Rx


def R2ypr(R):
    n, o, a = R[:, 0], R[:, 1], R[:, 2]
    y = np.arctan2(n[1], n[0])
    p = np.arctan2(-n[2], n[0] * np.cos(y) + n[1] * np.sin(y))
    r = np.arctan2(a[0] * np.sin(y) - a[1] * np.cos(y), -o[0] * np.sin(y) + o[1] * np.cos(y))
    return np.array([y, p, r]) / np.pi * 180.0


def quat_to_R(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def R_to_quat(R):
    t = np.trace(R)
    if t > 0:
        s = np.sqrt(t + 1.0)
        w = 0.5 * s
        s = 0.5 / s
        q = np.array([w, (R[2, 1] - R[1, 2]) * s, (R[0, 2] - R[2, 0]) * s, (R[1, 0] - R[0, 1]) * s])
    else:
        i = 0
        if R[1, 1] > R[0, 0]:
            i = 1
        if R[2, 2] > R[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        s = np.sqrt(R[i, i] - R[j, j] - R[k, k] + 1.0)
        c = np.zeros(3)
        c[i] = 0.5 * s
        s = 0.5 / s
        w = (R[k, j] - R[j, k]) * s
        c[j] = (R[j, i] + R[i, j]) * s
        c[k] = (R[k, i] + R[i, k]) * s
        q = np.array([w, *c])
    return q


def normalize_angle(a):
    return a - 360.0 if a > 180.0 else (a + 360.0 if a < -180.0 else a)


def four_dof(xi, xj, pitch_i, roll_i, meas, weighted=False, robust=False):
    """FourDOFError / FourDOFWeightError (pose_graph.h:159-248): x = yaw (degrees), t.  Returns (r, J 4x8, cost) with the
    HuberLoss(0.1) corrector applied when robust (residual and Jacobian times sqrt(rho'))."""
    R = ypr2R([xi[0], pitch_i, roll_i])
    d = np.asarray(xj[1:4], float) - np.asarray(xi[1:4], float)
    r = np.zeros(4)
    r[:3] = R.T @ d - np.asarray(meas[:3], float)
    r[3] = normalize_angle(xj[0] - xi[0] - meas[3])
    w = 1.0
    if weighted:
        r[3] = r[3] / 10.0
        w = 0.1
    J = np.zeros((4, 8))
    dR = np.array([-R[1], R[0], np.zeros(3)])
    J[:3, 0] = np.pi / 180.0 * (dR.T @ d)
    J[:3, 1:4] = -R.T
    J[:3, 5:8] = R.T
    J[3, 0], J[3, 4] = -w, w
    s = float(r @ r)
    if not robust:
        return r, J, 0.5 * s
    b = HUBER_A * HUBER_A
    rho, rho1 = s, 1.0
    if s > b:
        q = np.sqrt(s)
        rho, rho1 = 2.0 * HUBER_A * q - b, max(np.finfo(float).tiny, HUBER_A / q)
    sc = np.sqrt(rho1)
    return r * sc, J * sc, 0.5 * rho


def huber_rho(s):
    b = HUBER_A * HUBER_A
    return s if s <= b else 2.0 * HUBER_A * np.sqrt(s) - b


class Problem:
    """The optimize4DoF problem of one range: x0 (n x 4: yaw, t), pitch / roll, edges (older, newer, meas 4, loop)."""

    def __init__(self, vio_P, vio_R, seq, loops):
        n = len(vio_P)
        self.n = n
        self.ypr = np.array([R2ypr(quat_to_R(R_to_quat(R))) for R in vio_R])
        self.x0 = np.column_stack([self.ypr[:, 0], np.asarray(vio_P, float)])
        self.edges = []
        for i in range(n):
            for j in range(1, 5):
                if i - j >= 0 and seq[i] == seq[i - j]:
                    Rb = quat_to_R(R_to_quat(vio_R[i - j]))
                    m = np.r_[Rb.T @ (self.x0[i, 1:] - self.x0[i - j, 1:]), self.x0[i, 0] - self.x0[i - j, 0]]
                    self.edges.append((i - j, i, m, False))
            if loops[i] is not None:
                l, m = loops[i]
                self.edges.append((l, i, np.asarray(m, float), True))

    def evaluate(self, x, jac=True):
        out, cost = [], 0.0
        for (a, b, m, lp) in self.edges:
            r, J, c = four_dof(x[a], x[b], self.ypr[a, 1], self.ypr[a, 2], m, lp, lp)
            out.append((a, b, r, J))
            cost += c
        return out, cost

    def robust_residuals(self, xfree):
        """Residual vector whose half squared norm is the cost (scipy's minimum check): each loop block scaled to
        sqrt(rho(|r|^2)) r / |r|."""
        x = self.x0.copy()
        x[1:] = xfree.reshape(-1, 4)
        res = []
        for (a, b, m, lp) in self.edges:
            r, _, _ = four_dof(x[a], x[b], self.ypr[a, 1], self.ypr[a, 2], m, lp, False)
            if lp:
                s = float(r @ r)
                r = r * (np.sqrt(huber_rho(s)) / np.sqrt(s)) if s > 0 else r
            res.append(r)
        return np.concatenate(res)

    def solve(self, max_iterations=5, function_tolerance=1e-6):
        """Ceres LM (sfm_bundle's restatement); key frame 0 constant.  Returns x, summary dict.  Tests raise
        max_iterations and lower function_tolerance to run it to convergence."""
        n, nx = self.n, 4 * (self.n - 1)
        x = self.x0.copy()
        lin, cost = self.evaluate(x)
        cost0 = cost
        radius, dec = 1e4, 2.0
        scale = None
        need_lin, converged, it, succ = True, False, 0, 0
        H = g = None

        def assemble(lin):
            H = np.zeros((4 * n, 4 * n))
            g = np.zeros(4 * n)
            for (a, b, r, J) in lin:
                idx = np.r_[4 * a:4 * a + 4, 4 * b:4 * b + 4]
                H[np.ix_(idx, idx)] += J.T @ J
                g[idx] += J.T @ r
            return H[4:, 4:], g[4:]

        while it < max_iterations and not converged and nx > 0:
            if need_lin:
                lin, _ = self.evaluate(x)
                Hu, gu = assemble(lin)
                if scale is None:
                    scale = 1.0 / (1.0 + np.sqrt(np.diag(Hu)))
                H = Hu * np.outer(scale, scale)
                g = gu * scale
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
                d = (ds * scale).reshape(-1, 4)
                dfull = np.vstack([np.zeros(4), d])
                for (a, b, r, J) in lin:
                    jd = J @ np.r_[dfull[a] if a > 0 else np.zeros(4), dfull[b]]
                    mc -= jd @ (r + 0.5 * jd)
                ok = mc > 0 and np.isfinite(mc)
            if not ok:
                radius /= dec
                dec *= 2
                if radius < 1e-32:
                    break
                continue
            xc = x.copy()
            for i in range(1, n):
                xc[i, 0] = normalize_angle(x[i, 0] + dfull[i, 0])
                xc[i, 1:] = x[i, 1:] + dfull[i, 1:]
            _, cc = self.evaluate(xc, jac=False)
            if np.linalg.norm(d) <= 1e-8 * (np.linalg.norm(x[1:]) + 1e-8):
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
                dec = 2.0
                need_lin = True
            else:
                radius /= dec
                dec *= 2
                if radius < 1e-32:
                    break
        return x, dict(iterations=it, successful=succ, cost0=cost0, cost=cost, converged=converged)


def _gate(li):
    return abs(li[7]) < 30.0 and np.linalg.norm(li[:3]) < 20.0


class OraclePoseGraph:
    """PoseGraph bookkeeping (pose_graph.cpp:42-167, 403-579, 889-923) with a synchronous optimize()."""

    def __init__(self, fast_relocalization=False, max_iterations=5):
        self.fast, self.max_iterations = fast_relocalization, max_iterations
        self.kfs = []
        self.sequence, self.sequence_cnt, self.sequence_loop = 1, 0, [0]
        self.w_r_vio, self.w_t_vio = np.eye(3), np.zeros(3)
        self.r_drift, self.t_drift, self.yaw_drift = np.eye(3), np.zeros(3), 0.0
        self.earliest, self.pending = -1, -1
        self.last = None

    def new_sequence(self):
        if self.kfs and self.kfs[-1]["seq"] == self.sequence:
            self.sequence += 1

    def add_keyframe(self, stamp, P, Q, loop_index=-1, loop_info=None):
        kf = dict(stamp=stamp, seq=self.sequence, has_loop=False, loop_index=-1, loop_info=np.zeros(8))
        if self.sequence_cnt != kf["seq"]:
            self.sequence_cnt += 1
            self.sequence_loop.append(0)
            self.w_r_vio, self.w_t_vio = np.eye(3), np.zeros(3)
            self.r_drift, self.t_drift = np.eye(3), np.zeros(3)
        kf["vio_P"] = self.w_r_vio @ np.asarray(P, float) + self.w_t_vio
        kf["vio_R"] = self.w_r_vio @ quat_to_R(Q)
        idx = len(self.kfs)
        if loop_index >= 0 and _gate(np.asarray(loop_info, float)):
            li = np.asarray(loop_info, float)
            kf.update(has_loop=True, loop_index=loop_index, loop_info=li.copy())
            if self.earliest > loop_index or self.earliest == -1:
                self.earliest = loop_index
            old = self.kfs[loop_index]
            w_P = old["vio_R"] @ li[:3] + old["vio_P"]
            w_R = old["vio_R"] @ quat_to_R(li[3:7])
            shift_yaw = R2ypr(w_R)[0] - R2ypr(kf["vio_R"])[0]
            shift_r = ypr2R([shift_yaw, 0, 0])
            shift_t = w_P - w_R @ kf["vio_R"].T @ kf["vio_P"]
            if old["seq"] != kf["seq"] and self.sequence_loop[kf["seq"]] == 0:
                self.w_r_vio, self.w_t_vio = shift_r, shift_t
                kf["vio_P"] = shift_r @ kf["vio_P"] + shift_t
                kf["vio_R"] = shift_r @ kf["vio_R"]
                for o in self.kfs:
                    if o["seq"] == kf["seq"]:
                        o["vio_P"] = shift_r @ o["vio_P"] + shift_t
                        o["vio_R"] = shift_r @ o["vio_R"]
                self.sequence_loop[kf["seq"]] = 1
            self.pending = idx
        kf["P"] = self.r_drift @ kf["vio_P"] + self.t_drift
        kf["R"] = self.r_drift @ kf["vio_R"]
        self.kfs.append(kf)
        return idx, kf["P"].copy(), R_to_quat(kf["R"])

    def update_loop(self, index, loop_info):
        kf, li = self.kfs[index], np.asarray(loop_info, float)
        if not _gate(li):
            return
        kf["loop_info"] = li.copy()
        if self.fast:
            old = self.kfs[kf["loop_index"]]
            w_P = old["R"] @ li[:3] + old["P"]
            w_R = old["R"] @ quat_to_R(li[3:7])
            self.yaw_drift = R2ypr(w_R)[0] - R2ypr(kf["vio_R"])[0]
            self.r_drift = ypr2R([self.yaw_drift, 0, 0])
            self.t_drift = w_P - w_R @ kf["vio_R"].T @ kf["vio_P"]

    def problem(self):
        first, cur = self.earliest, self.pending
        rng = self.kfs[first:cur + 1]
        loops = [(k["loop_index"] - first, np.r_[k["loop_info"][:3], k["loop_info"][7]]) if k["has_loop"] else None for k in rng]
        return Problem([k["vio_P"] for k in rng], [k["vio_R"] for k in rng], [k["seq"] for k in rng], loops)

    def optimize(self, max_iterations=None, function_tolerance=1e-6):
        if self.pending < 0:
            return 0
        first, cur = self.earliest, self.pending
        pb = self.problem()
        x, info = pb.solve(self.max_iterations if max_iterations is None else max_iterations, function_tolerance)
        for i in range(pb.n):
            k = self.kfs[first + i]
            k["R"] = ypr2R([x[i, 0], pb.ypr[i, 1], pb.ypr[i, 2]])
            k["P"] = x[i, 1:].copy()
        ck = self.kfs[cur]
        self.yaw_drift = R2ypr(ck["R"])[0] - R2ypr(ck["vio_R"])[0]
        self.r_drift = ypr2R([self.yaw_drift, 0, 0])
        self.t_drift = ck["P"] - self.r_drift @ ck["vio_P"]
        for k in self.kfs[cur + 1:]:
            k["P"] = self.r_drift @ k["vio_P"] + self.t_drift
            k["R"] = self.r_drift @ k["vio_R"]
        self.pending = -1
        self.last = dict(info, n=pb.n, x=x)
        return 1

    def path(self):
        return (np.array([k["stamp"] for k in self.kfs]), np.array([k["P"] for k in self.kfs]),
                np.array([R_to_quat(k["R"]) for k in self.kfs]), np.array([k["seq"] for k in self.kfs]))
