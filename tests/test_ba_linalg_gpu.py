"""The BA solver's dense linear algebra on the device against float64 / long-double references: the step's packed Cholesky
with the right-hand side carried as row n and the backward solve (ba_step_kernel's fetch / factor / solve sequence, both
placements of the factor, the retry's re-fetch), the Schur reduction (ba_reduce_kernel and the single-CTA recomputation of
the linear-solver retry) and the marginalisation solve (marg_solve_kernel).  tests/hostlib/ba_linalg_dev.cu compiles the
production code of ba_kernels.cu into a test library; the trust region of the solve hides a slightly wrong step, so the
end-to-end tests alone would not see most of what is checked here."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from test_sym_eig import floor_ref
from vins_mono_b200 import build as vb_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostlib", "ba_linalg_dev.cu")
U = 2.0 ** -53
BA_MAX_D = 352
OJ_BASE, OJ_FULL, LW_BASE, LW_FULL, IMUJ_STRIDE = 34, 48, 36, 120, 480
gpu = pytest.mark.gpu

P_D = ctypes.POINTER(ctypes.c_double)
P_I = ctypes.POINTER(ctypes.c_int)


def compile_lib(out):
    # the flags of the product's ba_*.cu objects
    subprocess.check_call(["nvcc", *vb_build.NVCC_FLAGS, "--fmad=true", "-shared", "-o", str(out), SRC],
                          stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)


def test_library_compiles(tmp_path):
    """Cross-compiles the test library for sm_90a (no GPU needed), so it cannot rot on machines without one."""
    out = tmp_path / "libbalinalg.so"
    compile_lib(out)
    assert out.stat().st_size > 0


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    out = tmp_path_factory.mktemp("balinalg") / "libbalinalg.so"
    compile_lib(out)
    l = ctypes.CDLL(str(out))
    l.t_factor.argtypes = [ctypes.c_int, P_I, P_D, P_D, P_D, P_D, P_D, P_D, ctypes.c_int, P_D, P_D, P_I]
    l.t_reduce.argtypes = [P_I, P_I, P_I, P_I, P_D, P_D, P_D, ctypes.c_int, ctypes.c_int, P_I, P_I, P_I, P_D, P_D, P_D,
                           ctypes.c_double, ctypes.c_double] + [P_D] * 8
    l.t_marg_solve.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, P_D, P_D, ctypes.c_int, P_D, P_D, P_D, P_D, P_D]
    return l


def dp(a):
    return a.ctypes.data_as(P_D) if a is not None else None


def ip(a):
    return a.ctypes.data_as(P_I)


# ------------------------------------------------------------------------------------------------------------------------
# A. Cholesky and solve

# every n of one and two blocks, the block boundary at 64, the reduced systems of W = 10, 20, 22 (with and without the
# extrinsic, td and relocalisation columns) and the capacity
W_SIZES = {15 * (W + 1) + k for W in (10, 20, 22) for k in (0, 1, 6, 7, 12, 13)}
SIZES = sorted(set(range(1, 41)) | {63, 64, 65, 351, 352} | {d for d in W_SIZES if d <= BA_MAX_D})


def packed(A):
    return np.ascontiguousarray(A[np.tril_indices(A.shape[0])])


def unpack(p, n):
    L = np.zeros((n, n))
    L[np.tril_indices(n)] = p
    return L


def factor(lib, members, smem, refetch=None):
    """members: list of (A, b, diag, scale, mu); refetch: the systems the second factorisation reads (or None).
    Returns [(L, y, flag_first, flag_final)] per member."""
    ns = np.array([m[0].shape[0] for m in members], np.int32)
    A = np.concatenate([packed(m[0]) for m in members])
    A2 = np.concatenate([packed(r) for r in refetch]) if refetch is not None else None
    b, dg, sc = (np.concatenate([m[k] for m in members]) for k in (1, 2, 3))
    mu = np.array([m[4] for m in members], np.float64)
    Lo = np.full(len(A), np.nan)
    yo = np.full(int(ns.sum()), np.nan)
    fl = np.full(2 * len(ns), -1, np.int32)
    err = lib.t_factor(len(ns), ip(ns), dp(A), dp(A2), dp(b), dp(dg), dp(sc), dp(mu), int(smem), dp(Lo), dp(yo), ip(fl))
    assert err == 0, f"CUDA error {err}"
    out, po, vo = [], 0, 0
    for k, n in enumerate(ns):
        out.append((unpack(Lo[po:po + n * (n + 1) // 2], n), yo[vo:vo + n], fl[2 * k], fl[2 * k + 1]))
        po += n * (n + 1) // 2
        vo += n
    return out


def spd_ba_like(n, rng):
    """J^T J with row scales over six decades, Jacobi-scaled, as the step sees it (E = its diagonal, mu small)."""
    J = rng.standard_normal((n + 8, n)) * np.logspace(0, 6, n + 8)[:, None]
    H = J.T @ J
    s = 1.0 / (1.0 + np.sqrt(np.diag(H)))
    A = s[:, None] * H * s[None, :]
    A = (A + A.T) / 2
    scale = rng.uniform(0.5, 2.0, n)
    diag = np.sqrt(np.clip(np.diag(A), 1e-6, 1e32)) * scale
    return A, rng.standard_normal(n), diag, scale, 1e-4


def spd_well(n, rng):
    B = rng.standard_normal((n, n))
    A = B @ B.T / n + np.eye(n)
    return A, rng.standard_normal(n), np.ones(n), np.ones(n), 1e-3


def regularised(m):
    A, b, diag, scale, mu = m
    return A + np.diag(mu * (diag * diag) / (scale * scale))


def solve_ref(A, b):
    """A^-1 b with one step of refinement on a long-double residual."""
    c = np.linalg.cholesky(A)
    sol = lambda r: np.linalg.solve(c.T, np.linalg.solve(c, r))
    y = sol(b)
    r = (b.astype(np.longdouble) - A.astype(np.longdouble) @ y.astype(np.longdouble)).astype(np.float64)
    return y + sol(r), c


def check_factor(m, res):
    """The gates of one factorisation; returns a failure message or None."""
    L, y, f0, f1 = res
    n = L.shape[0]
    A = regularised(m)
    if f1 != 1:
        return f"n={n}: flag {f1}"
    Ll = L.astype(np.longdouble)
    resid = np.abs(A.astype(np.longdouble) - Ll @ Ll.T).max()
    if not resid <= 4 * n * U * np.abs(A).max():
        return f"n={n}: |A - L L^T| = {float(resid):.3e}, max|A| = {np.abs(A).max():.3e}"
    yref, Lref = solve_ref(A, m[1])
    kappa = np.linalg.cond(A)
    if kappa <= 1e3:
        if not np.abs(L - Lref).max() <= 1e-13 * np.abs(L).max():
            return f"n={n}: |L - Lref| = {np.abs(L - Lref).max():.3e}"
        if not np.abs(y - yref).max() <= 1e-12 * np.abs(yref).max():
            return f"n={n}: |y - yref| = {np.abs(y - yref).max():.3e}, |yref| = {np.abs(yref).max():.3e}"
    elif not np.linalg.norm(y - yref) <= 10 * n * U * kappa * np.linalg.norm(yref):
        return f"n={n}: |y - yref| / |yref| = {np.linalg.norm(y - yref) / np.linalg.norm(yref):.3e}, kappa = {kappa:.2e}"
    return None


@gpu
@pytest.mark.parametrize("kind", ["ba_like", "well_conditioned"])
@pytest.mark.parametrize("placement", ["smem", "global"])
def test_cholesky_solve(lib, placement, kind):
    """Every size in one batch (factor in shared memory, filled by the bulk copy, wherever the step would put it there; in
    global memory everywhere else), against the float64 reference; the batch twice and every member solo, bit for bit."""
    smem = placement == "smem"
    fits = {n for n in SIZES if lib.t_step_smem_fits(n)}
    # global memory: the sizes the step does not keep in shared memory, plus a few small ones
    sizes = sorted(fits) if smem else sorted((set(SIZES) - fits) | {1, 8, 13, 40})
    assert sizes
    rng = np.random.default_rng(11 if kind == "ba_like" else 12)
    gen = spd_ba_like if kind == "ba_like" else spd_well
    members = [gen(n, rng) for n in sizes]
    if kind == "well_conditioned":
        assert all(np.linalg.cond(regularised(m)) <= 1e3 for m in members)
    res = factor(lib, members, smem)
    again = factor(lib, members, smem)
    fails = [msg for m, r in zip(members, res) if (msg := check_factor(m, r))]
    for m, r, r2 in zip(members, res, again):
        n = m[0].shape[0]
        if not (np.array_equal(r[0], r2[0]) and np.array_equal(r[1], r2[1])):
            fails.append(f"n={n}: two runs differ")
        solo = factor(lib, [m], smem)[0]
        if not (np.array_equal(r[0], solo[0]) and np.array_equal(r[1], solo[1]) and r[3] == solo[3]):
            fails.append(f"n={n}: batch member differs from its solo run")
    assert not fails, "\n".join(fails)


def ldl_exact(n, k, dk, rng):
    """A = L0 diag(d) L0^T with a small-integer unit lower L0 and d = 1 except d_k = dk: exact in float64."""
    L0 = np.tril(rng.integers(-1, 2, (n, n)).astype(np.float64), -1) + np.eye(n)
    d = np.ones(n)
    d[k] = dk
    return (L0 * d) @ L0.T


def pivots(n):
    """every k mod 8 in the first block, a middle block and the (partial) last block"""
    ks = set(range(min(8, n)))
    if n > 24:
        ks |= set(range(8 * (n // 16), 8 * (n // 16) + 8))
    ks |= set(range(8 * ((n - 1) // 8), n))
    return sorted(ks)


@gpu
@pytest.mark.parametrize("placement", ["smem", "global"])
@pytest.mark.parametrize("n", [8, 13, 172])
def test_cholesky_flags_failure(lib, placement, n):
    """A non-positive pivot at any position, or a NaN / +inf on the diagonal, clears the flag; the same matrices with a
    positive pivot factorise."""
    smem = placement == "smem"
    if smem and not lib.t_step_smem_fits(n):
        pytest.skip("the step keeps this size in global memory")
    rng = np.random.default_rng(n)
    ks = pivots(n)
    one = lambda A: (A, np.ones(n), np.ones(n), np.ones(n), 0.0)
    for dk in (-1.0, 0.0, 1.0):
        mats = [ldl_exact(n, k, dk, np.random.default_rng(1000 * n + k)) for k in ks]
        res = factor(lib, [one(A) for A in mats], smem)
        flags = [r[3] for r in res]
        assert flags == [1 if dk > 0 else 0] * len(ks), (dk, list(zip(ks, flags)))
        if dk > 0:
            assert all(r[0].shape == (n, n) and np.abs(r[0] @ r[0].T - A).max() <= 4 * n * U * np.abs(A).max()
                       for r, A in zip(res, mats))
    for bad in (np.nan, np.inf):
        mats = []
        for k in sorted({0, n // 2, n - 1}):
            A = ldl_exact(n, k, 1.0, rng)
            A[k, k] = bad
            mats.append(A)
        assert [r[3] for r in factor(lib, [one(A) for A in mats], smem)] == [0] * len(mats), bad


@gpu
@pytest.mark.parametrize("placement", ["smem", "global"])
def test_cholesky_refetch(lib, placement):
    """The retry's sequence: a failed factorisation of A1, plain stores of A2 over the packed source by the CTA, a second
    fetch (the bulk copy again in shared memory, mbarrier phase flipped) and factorisation: bit for bit the solo result for A2."""
    smem = placement == "smem"
    sizes = [n for n in (1, 5, 8, 13, 64, 165, 172, 178) if lib.t_step_smem_fits(n) == smem or n <= 13]
    rng = np.random.default_rng(3)
    for n in sizes:
        m2 = spd_ba_like(n, rng)
        A1 = ldl_exact(n, n // 2, -1.0, rng)
        m1 = (A1,) + m2[1:]
        r = factor(lib, [m1], smem, refetch=[m2[0]])[0]
        solo = factor(lib, [m2], smem)[0]
        assert r[2] == 0 and r[3] == 1, (n, r[2], r[3])
        assert np.array_equal(r[0], solo[0]) and np.array_equal(r[1], solo[1]), n


# ------------------------------------------------------------------------------------------------------------------------
# B. Schur reduction

def hii_index(i, j):
    return i * 6 - i * (i - 1) // 2 + (j - i)


def reduce_problem(W, ex, td, relo, L, seed, sort=True):
    """Synthetic linearisation records derived from random per-observation Jacobians (the definitions of ba_eval_kernel),
    plus the Jacobians themselves for the reference."""
    rng = np.random.default_rng(seed)
    F = W + 1
    D = 15 * F + 6 * ex + td
    col_ex = 15 * F if ex else -1
    col_td = 15 * F + 6 * ex if td else -1
    col_relo = -1
    if relo:
        col_relo = D
        D += 6
    anchors = np.sort(rng.integers(0, W, L)) if L else np.zeros(0, int)
    nobs = np.array([rng.integers(1, W - a + 1) for a in anchors], int)
    has_relo = (rng.random(L) < 0.15).astype(int) if relo else np.zeros(L, int)
    if relo and L:
        has_relo[L // 2] = 1
    order = np.arange(L) if sort else rng.permutation(L)
    anchors, nobs, has_relo = anchors[order], nobs[order], has_relo[order]
    rows = nobs + has_relo
    start = np.concatenate([[0], np.cumsum(rows)]).astype(np.int32)
    M = int(start[-1])
    wide = ex or td
    oj, lw = (OJ_FULL, LW_FULL) if wide else (OJ_BASE, LW_BASE)
    Ji = rng.standard_normal((M, 2, 6))
    Jj = rng.standard_normal((M, 2, 6))
    Jex = rng.standard_normal((M, 2, 6)) * 0.5 if ex else np.zeros((M, 2, 6))
    Jtd = rng.standard_normal((M, 2)) * 3 if td else np.zeros((M, 2))
    Jl = rng.standard_normal((M, 2)) * np.repeat(rng.uniform(0.05, 2.0, L), rows)[:, None] if M else np.zeros((0, 2))
    r = rng.standard_normal((M, 2))
    if L:  # a landmark with a tiny Hll: the 1e-6 floor of lm_inv_lambda's diagonal
        l = L // 3
        Jl[start[l]:start[l + 1]] *= 1e-5
    lm = np.repeat(np.arange(L), rows)
    t = np.arange(M) - np.repeat(start[:-1], rows)  # row within the landmark
    is_relo = (t == np.repeat(rows, rows) - 1) & (np.repeat(has_relo, rows) == 1)
    Jtd[is_relo] = 0.0  # the match is a plain projection factor: no time-offset Jacobian
    obsJ = np.zeros((M, oj))
    obsJ[:, 0:12] = Ji.reshape(M, 12)
    obsJ[:, 12:24] = Jj.reshape(M, 12)
    obsJ[:, 24:26] = r
    obsJ[:, 26:28] = Jl
    obsJ[:, 28:34] = np.einsum("mki,mk->mi", Jj, Jl)
    if wide:
        obsJ[:, 34:46] = Jex.reshape(M, 12)
        obsJ[:, 46:48] = Jtd
    lmW = np.zeros((L, lw))
    seg = lambda x: np.add.reduceat(x, start[:-1], axis=0) if M else np.zeros((L,) + x.shape[1:])
    HiiF = seg(np.einsum("mki,mkj->mij", Ji, Ji))
    for i in range(6):
        for j in range(i, 6):
            lmW[:, hii_index(i, j)] = HiiF[:, i, j]
    lmW[:, 21:27] = seg(np.einsum("mki,mk->mi", Ji, r))
    lmW[:, 27:33] = seg(np.einsum("mki,mk->mi", Ji, Jl))
    lmW[:, 33] = seg((Jl * Jl).sum(1))
    lmW[:, 34] = seg((Jl * r).sum(1))
    if wide:
        lmW[:, 36:72] = seg(np.einsum("mki,mkj->mij", Ji, Jex)).reshape(L, 36)
        HeeF = seg(np.einsum("mki,mkj->mij", Jex, Jex))
        for i in range(6):
            for j in range(i, 6):
                lmW[:, 72 + hii_index(i, j)] = HeeF[:, i, j]
        lmW[:, 93:99] = seg(np.einsum("mki,mk->mi", Jex, r))
        lmW[:, 99:105] = seg(np.einsum("mki,mk->mi", Jex, Jl))
        lmW[:, 105:111] = seg(np.einsum("mki,mk->mi", Ji, Jtd))
        lmW[:, 111:117] = seg(np.einsum("mki,mk->mi", Jex, Jtd))
        lmW[:, 117] = seg((Jtd * Jtd).sum(1))
        lmW[:, 118] = seg((Jtd * r).sum(1))
        lmW[:, 119] = seg((Jtd * Jl).sum(1))
    imuJ = np.zeros((W, IMUJ_STRIDE))
    imuJ[:, :450] = rng.standard_normal((W, 450))
    imuJ[:, 450:465] = rng.standard_normal((W, 15))
    imuJ[:, 466] = 1.0
    if W > 1:
        imuJ[1, 466] = 0.0  # a skipped factor
    # prior over a subset of the blocks
    blocks = [(0, 0), (1, 0), (0, 1), (1, 2)] + ([(2, 0)] if ex else []) + ([(3, 0)] if td else [])
    sizes = {0: 6, 1: 9, 2: 6, 3: 1}
    off = np.concatenate([[0], np.cumsum([sizes[b[0]] for b in blocks])]).astype(np.int32)
    pn = int(off[-1])
    Jp = rng.standard_normal((pn + 3, pn))
    pA = Jp.T @ Jp
    gpr = rng.standard_normal(pn)
    return dict(W=W, F=F, D=D, L=L, M=M, ex=ex, td=td, relo=relo, col_ex=col_ex, col_td=col_td, col_relo=col_relo,
                anchors=anchors.astype(np.int32), start=start, has_relo=has_relo.astype(np.int32), obsJ=obsJ, lmW=lmW, imuJ=imuJ,
                Ji=Ji, Jj=Jj, Jex=Jex, Jtd=Jtd, Jl=Jl, r=r, lm=lm, t=t, is_relo=is_relo,
                ptype=np.array([b[0] for b in blocks], np.int32), pindex=np.array([b[1] for b in blocks], np.int32),
                poff=off[:-1].copy(), pA=pA, gpr=gpr, scale=rng.uniform(0.3, 3.0, D + L))


def reduce_reference(pb, mu, first):
    """Hpp, S = Hpp - Hpl (Hll + mu E)^-1 Hlp, gp and gred = gp - Hpl (Hll + mu E)^-1 gl in long double, assembled from the
    Jacobians."""
    ld = np.longdouble
    D, L, M, F = pb["D"], pb["L"], pb["M"], pb["F"]
    H = np.zeros(D * D, ld)
    g = np.zeros(D, ld)
    Hpl = np.zeros((D, L), ld)
    if M:
        an = pb["anchors"][pb["lm"]]
        fj = an + pb["t"] + 1
        cols = [6 * an[:, None] + np.arange(6)]
        cj = np.where(pb["is_relo"][:, None], pb["col_relo"] + np.arange(6), 6 * np.minimum(fj, F - 1)[:, None] + np.arange(6))
        cols.append(cj)
        Jc = [pb["Ji"], pb["Jj"]]
        if pb["ex"]:
            cols.append(np.broadcast_to(pb["col_ex"] + np.arange(6), (M, 6)))
            Jc.append(pb["Jex"])
        if pb["td"]:
            cols.append(np.full((M, 1), pb["col_td"]))
            Jc.append(pb["Jtd"][:, :, None])
        C = np.concatenate(cols, 1)
        J = np.concatenate(Jc, 2).astype(ld)  # M x 2 x K
        outer = np.einsum("mki,mkj->mij", J, J)
        np.add.at(H, (C[:, :, None] * D + C[:, None, :]).ravel(), outer.ravel())
        np.add.at(g, C.ravel(), np.einsum("mki,mk->mi", J, pb["r"].astype(ld)).ravel())
        wl = np.einsum("mki,mk->mi", J, pb["Jl"].astype(ld))
        np.add.at(Hpl, (C.ravel(), np.repeat(pb["lm"], C.shape[1])), wl.ravel())
    H = H.reshape(D, D)
    for k in range(pb["W"]):
        rec = pb["imuJ"][k]
        if rec[466] == 0.0:
            continue
        c = np.concatenate([6 * k + np.arange(6), 6 * F + 9 * k + np.arange(9), 6 * (k + 1) + np.arange(6), 6 * F + 9 * (k + 1) + np.arange(9)])
        Jw = rec[:450].reshape(15, 30).astype(ld)
        H[np.ix_(c, c)] += Jw.T @ Jw
        g[c] += Jw.T @ rec[450:465].astype(ld)
    pc = np.concatenate([(6 * idx + np.arange(6)) if ty == 0 else (6 * F + 9 * idx + np.arange(9)) if ty == 1 else
                         (pb["col_ex"] + np.arange(6)) if ty == 2 else np.array([pb["col_td"]])
                         for ty, idx in zip(pb["ptype"], pb["pindex"])])
    H[np.ix_(pc, pc)] += pb["pA"].astype(ld)
    g[pc] += pb["gpr"].astype(ld)
    Jl = pb["Jl"].astype(ld)
    hll = np.zeros(L, ld)
    gl = np.zeros(L, ld)
    if M:
        np.add.at(hll, pb["lm"], (Jl * Jl).sum(1))
        np.add.at(gl, pb["lm"], (Jl * pb["r"].astype(ld)).sum(1))
    s = 1 / (1 + np.sqrt(hll)) if first else pb["scale"][D:].astype(ld)
    E = np.clip(hll * s * s, 1e-6, 1e32) / (s * s)
    inv = 1 / (hll + mu * E)
    S = H - (Hpl * inv) @ Hpl.T
    gs = Hpl @ (inv * gl)
    return H, S, g, g - gs, gs


def run_reduce(lib, pb, mu, mu2, first):
    D, L = pb["D"], pb["L"]
    shape = np.array([pb["W"], L, pb["M"], pb["ex"], pb["td"], pb["relo"], int(pb["ex"] or pb["td"]), first], np.int32)
    out = [np.zeros(D * D), np.zeros(D * D), np.zeros(D * (D + 1) // 2), np.zeros(D), np.zeros(D),
           np.zeros(D * D), np.zeros(D * (D + 1) // 2), np.zeros(D)]
    err = lib.t_reduce(ip(shape), ip(pb["anchors"]), ip(pb["start"]), ip(pb["has_relo"]), dp(pb["obsJ"]), dp(pb["lmW"]),
                       dp(pb["imuJ"]), len(pb["gpr"]), len(pb["ptype"]), ip(pb["ptype"]), ip(pb["pindex"]), ip(pb["poff"]),
                       dp(pb["pA"]), dp(pb["gpr"]), dp(pb["scale"]), mu, mu2, *[dp(o) for o in out])
    assert err == 0, f"CUDA error {err}"
    Hf, S, Spk, gred, gp, S2, Spk2, gred2 = out
    return dict(H=Hf.reshape(D, D), S=S.reshape(D, D), Spk=Spk, gred=gred, gp=gp, S2=S2.reshape(D, D), Spk2=Spk2, gred2=gred2)


# W, ex, td, relo, L, mu, first, sorted by anchor (relocalisation only where 15 F + 6 ex + td + 6 <= BA_MAX_D)
RED_CASES = [
    (3, 0, 0, 0, 0, 1e-4, 1, True),
    (3, 1, 1, 1, 1, 1e3, 0, True),
    (3, 1, 0, 0, 37, 1e-4, 0, True),
    (3, 0, 1, 1, 1025, 1e3, 1, False),
    (10, 0, 1, 0, 37, 1e3, 1, True),
    (10, 1, 1, 0, 1023, 1e-4, 1, True),
    (10, 1, 1, 1, 1024, 1e3, 0, True),
    (10, 0, 0, 1, 1025, 1e-4, 0, True),
    (10, 1, 0, 1, 2300, 1e3, 1, True),
    (20, 1, 1, 1, 1025, 1e-4, 1, True),
    (20, 0, 0, 0, 2300, 1e3, 0, True),
    (20, 1, 0, 0, 1024, 1e-4, 0, False),
    (22, 1, 1, 0, 2300, 1e-4, 1, True),
    (22, 0, 1, 1, 1025, 1e3, 0, True),
    (22, 0, 0, 1, 37, 1e-4, 1, False),
]


@gpu
@pytest.mark.parametrize("W,ex,td,relo,L,mu,first,srt", RED_CASES)
def test_schur_reduction(lib, W, ex, td, relo, L, mu, first, srt):
    if relo:
        assert 15 * (W + 1) + 6 * ex + td + 6 <= BA_MAX_D
    pb = reduce_problem(W, ex, td, relo, L, seed=W * 10007 + L + 7 * ex + 3 * td + relo, sort=srt)
    mu2 = 1e3 if mu < 1 else 1e-4
    got = run_reduce(lib, pb, mu, mu2, first)
    other = run_reduce(lib, pb, mu2, mu, first)  # ba_reduce_kernel at mu2
    H, S, gp, gred, gs = (x.astype(np.float64) for x in reduce_reference(pb, mu, first))
    _, S_2, _, gred_2, gs_2 = (x.astype(np.float64) for x in reduce_reference(pb, mu2, first))
    hs = np.abs(H).max()
    gsc = max(np.abs(gp).max(), np.abs(gs).max(), np.abs(gs_2).max())
    D = pb["D"]
    tril = np.tril_indices(D)
    assert np.abs(got["H"] - H).max() <= 1e-13 * hs
    assert np.abs(got["gp"] - gp).max() <= 1e-13 * gsc
    for name, Sd, Spk, gd, Sr, gr in (("reduce", got["S"], got["Spk"], got["gred"], S, gred),
                                      ("single", got["S2"], got["Spk2"], got["gred2"], S_2, gred_2),
                                      ("reduce mu2", other["S"], other["Spk"], other["gred"], S_2, gred_2)):
        assert np.abs(Sd - Sr).max() <= 1e-13 * hs, (name, np.abs(Sd - Sr).max() / hs)
        assert np.abs(gd - gr).max() <= 1e-13 * gsc, (name, np.abs(gd - gr).max() / gsc)
        assert np.array_equal(Sd, Sd.T), name
        assert np.array_equal(Spk, Sd[tril]), name
    assert np.abs(got["S2"] - other["S"]).max() <= 1e-13 * hs
    assert np.abs(got["gred2"] - other["gred"]).max() <= 1e-13 * gsc
    assert np.array_equal(other["H"], got["H"])


# ------------------------------------------------------------------------------------------------------------------------
# C. Marginalisation solve

EPS = 1e-8


def marg_system(md, nl, n, t_pd, rng):
    """[m_dense | n_lm landmarks | n kept], H = sum of per-factor J^T J: a dense factor without landmarks and per-landmark
    factors (so the landmark block is exactly diagonal).  The kept columns have a 4-dimensional null space, as the prior's
    gauge; one landmark has d <= eps; without t_pd two dense columns are equal, which makes T singular."""
    P = md + nl + n
    Z = np.linalg.qr(rng.standard_normal((n, 4)))[0]
    proj = np.eye(n) - Z @ Z.T  # kept Jacobians J_n proj: J_n Z = 0

    def factor_rows(k, lm):
        J = np.zeros((k, P))
        J[:, :md] = rng.standard_normal((k, md))
        J[:, md + nl:] = (rng.standard_normal((k, n)) * rng.uniform(0.05, 1.0, n)) @ proj
        if lm is not None:
            J[:, md + lm] = rng.standard_normal(k) * (1e-5 if lm == nl // 2 and nl else 1.0)
        return J

    Js = [factor_rows(2 * md + n + 8, None)] + [factor_rows(3, c) for c in range(nl)]
    H = sum(J.T @ J for J in Js)
    b = sum(J.T @ rng.standard_normal(J.shape[0]) for J in Js)
    if not t_pd:
        H[1, :] = H[0, :]
        H[:, 1] = H[:, 0]
        b[1] = b[0]
    return H, b


def marg_reference(H, b, md, nl, n):
    """Landmarks with d > eps eliminated (long double), then T+ by eigh (eigenvalues > eps), A' = W_nn - W_nm T+ W_mn."""
    ld = np.longdouble
    q = np.r_[0:md, md + nl:md + nl + n]
    W = H[np.ix_(q, q)].astype(ld)
    bw = b[q].astype(ld)
    for c in range(nl):
        d = H[md + c, md + c]
        if d > EPS:
            w = H[q, md + c].astype(ld)
            W -= np.outer(w, w) / d
            bw -= w * (b[md + c] / ld(d))
    W = W.astype(np.float64)
    bw = bw.astype(np.float64)
    tw, tv = np.linalg.eigh(W[:md, :md])
    keep = tw > EPS
    Tp = (tv[:, keep] / tw[keep]) @ tv[:, keep].T
    A = W[md:, md:] - W[md:, :md] @ Tp @ W[:md, md:]
    return A, bw[md:] - W[md:, :md] @ Tp @ bw[:md]


def joint_reference(H, b, md, nl, n):
    """marginalization_factor.cpp's joint pseudo-inverse of the whole marginalised block (landmarks with d <= eps left out)."""
    mcols = [i for i in range(md)] + [md + c for c in range(nl) if H[md + c, md + c] > EPS]
    r = np.arange(md + nl, md + nl + n)
    Amm = H[np.ix_(mcols, mcols)]
    w, V = np.linalg.eigh((Amm + Amm.T) / 2)
    keep = w > EPS
    Ainv = (V[:, keep] / w[keep]) @ V[:, keep].T
    Arm = H[np.ix_(r, mcols)]
    return H[np.ix_(r, r)] - Arm @ Ainv @ Arm.T, b[r] - Arm @ Ainv @ b[mcols]


# kept columns around the n <= 96 template switch, the shipped window (75, 76) and the largest window (W = 22 with extrinsic
# and td: 6 W + 16 = 148, the largest prior config_valid admits)
@gpu
@pytest.mark.parametrize("n", [69, 75, 76, 96, 97, 136, 142, 148])
@pytest.mark.parametrize("md", [6, 15])
def test_marg_solve(lib, md, n):
    """The marginalisation solve on both routes of the reduced system (shared memory wherever it fits, global memory
    always), with T positive definite (Cholesky path) and singular (eigen path), against the two-stage reference."""
    fails = []
    for nl in (0, 1, 16, 17, 300):
        for t_pd in (True, False):
            rng = np.random.default_rng(md * 100000 + n * 1000 + nl * 2 + t_pd)
            H, b = marg_system(md, nl, n, t_pd, rng)
            Ar, br = marg_reference(H, b, md, nl, n)
            rA, rg, rc, w = floor_ref(Ar, br)
            if t_pd:  # the two-stage reference is the joint pseudo-inverse where the marginalised block is nonsingular
                Aj, bj = joint_reference(H, b, md, nl, n)
                assert np.abs(Aj - Ar).max() <= 1e-10 * np.abs(H).max() and np.abs(bj - br).max() <= 1e-9 * np.abs(b).max()
            Am = np.triu(H)
            scale = np.abs(H).max()
            tau = max(1e-12 * np.abs(Ar).sum(1).max(), 4 * EPS)
            assert (w < 0.3 * tau).sum() == 4 and not np.any((w >= 0.3 * tau) & (w < 3 * tau))
            for wig in (0, 1) if not lib.t_marg_w_in_global(md, n) else (1,):
                Aout, Araw = np.zeros(n * n), np.zeros(n * n)
                gout, cout, graw = np.zeros(n), np.zeros(1), np.zeros(n + 7)
                err = lib.t_marg_solve(md, nl, n, dp(Am), dp(b), wig, dp(Aout), dp(gout), dp(cout), dp(Araw), dp(graw))
                assert err == 0, f"CUDA error {err}"
                tag = f"nl={nl} t_pd={t_pd} w_in_global={wig}"
                checks = [("Araw", np.abs(Araw.reshape(n, n) - (Ar + Ar.T) / 2).max() <= 1e-13 * scale),
                          ("Aout", np.abs(Aout.reshape(n, n) - rA).max() <= 1e-13 * scale),
                          ("gout", np.abs(gout - rg).max() <= 1e-9 * np.abs(b).max()),
                          ("cout", abs(cout[0] - rc) <= 1e-5 * rc),
                          ("floor pairs", graw[n + 1] == (-1 if wig else 4))]
                fails += [f"{tag}: {name}" for name, ok in checks if not ok]
    assert not fails, "\n".join(fails)
