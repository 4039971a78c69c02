// Test entry points for the dense linear algebra of the BA solver: the step's packed Cholesky and triangular solve, the
// Schur reduction (ba_reduce_kernel and the single-CTA recomputation of the linear-solver retry) and the marginalisation
// solve.  The production kernels and device functions are compiled in from ba_kernels.cu; each entry point takes host
// arrays, allocates, launches, copies back, frees and returns the CUDA error code (tests/test_ba_linalg_gpu.py).
#include "../../vins_mono_b200/csrc/ba_kernels.cu"

#include <vector>

using namespace vb;

namespace ba_linalg_test {

struct FactorJob {  // one member of a t_factor batch
    int n;
    double* spk;         // packed source, ba_spk_doubles(n) (what ba_reduce_kernel writes)
    const double* spk2;  // refetch: the system the second factorisation reads, or null
    const double* gred;
    const double* diag;
    const double* scale;
    double mu;
    double* work;        // global placement: ba_work_layout(n, 0).total
    double* L;           // out: packed factor, n (n + 1) / 2
    double* y;           // out: (S + mu E)^-1 gred
    int* flag;           // out: [0] first factorisation, [1] the one whose factor is returned
};

// One CTA per member, the fetch / factor / solve sequence of ba_step_kernel.  With spk2, the first factorisation is followed
// by the retry's sequence: plain stores of spk2 over spk by every thread, the proxy fence, and a second fetch (a bulk copy
// again in the shared-memory placement, with the mbarrier phase flipped).
__global__ void __launch_bounds__(512) t_factor_kernel(const FactorJob* __restrict__ jobs, int use_smem) {
    extern __shared__ __align__(16) double chol_smem[];
    __shared__ double rdiag[BA_MAX_D], ysm[BA_MAX_D], linv[(BA_MAX_D / CHOL_NB) * 64];
    __shared__ int flag;
    __shared__ __align__(8) unsigned long long copy_bar;
    __shared__ BaProblem sp;  // the fields the step's fetch reads: Spk, gred, diag, scale
    const FactorJob& jb = jobs[blockIdx.x];
    const int D = jb.n, npk = D * (D + 1) / 2, tid = threadIdx.x, nt = blockDim.x;
    unsigned copy_phase = 0;
    if (tid == 0) {
        mbar_init(&copy_bar, 1);
        sp.Spk = jb.spk;
        sp.gred = const_cast<double*>(jb.gred);
        sp.diag = const_cast<double*>(jb.diag);
        sp.scale = const_cast<double*>(jb.scale);
    }
    __syncthreads();
    double* Lp = use_smem ? chol_smem + CHOL_NB * CHOL_PS : jb.work + ba_work_layout(D, 0).Lp;
    bool copy_in_flight = false;
    if (use_smem) {  // issued before the fetch, as the step does
        if (tid == 0) bulk_g2s_chunked(Lp, jb.spk, spk_copy_bytes(D), 8192u, &copy_bar);
        copy_in_flight = true;
    }
    step_load_system(sp, Lp, jb.mu, D, use_smem != 0, copy_in_flight, &copy_bar, copy_phase);
    bool ok = cholesky_packed(Lp, chol_smem, D, rdiag, linv, &flag, D + 1);
    if (tid == 0) jb.flag[0] = ok ? 1 : 0;
    if (jb.spk2) {
        __syncthreads();
        for (int i = tid; i < npk; i += nt) jb.spk[i] = jb.spk2[i];
        fence_proxy_async_global();
        step_load_system(sp, Lp, jb.mu, D, use_smem != 0, copy_in_flight, &copy_bar, copy_phase);
        ok = cholesky_packed(Lp, chol_smem, D, rdiag, linv, &flag, D + 1);
    }
    if (ok) step_solve(Lp, linv, D, ysm);
    for (int i = tid; i < npk; i += nt) jb.L[i] = Lp[i];
    for (int i = tid; i < D; i += nt) jb.y[i] = ok ? ysm[i] : 0.0;
    if (tid == 0) jb.flag[1] = ok ? 1 : 0;
}

__global__ void __launch_bounds__(512) t_reduce_single_kernel(const BaSeq* __restrict__ seqs, double mu) {
    __shared__ BaProblem sp;
    const BaSeq& q = seqs[0];
    load_desc(&sp, &q.p);
    reduce_single_cta(sp, sp.acc[q.st.cur], mu, q.st.first);
}

// device allocations of one entry point, freed on return
struct DevArena {
    std::vector<void*> ptrs;
    cudaError_t err = cudaSuccess;
    template <class T>
    T* alloc(size_t count, const T* src = nullptr, int fill = 0) {
        void* p = nullptr;
        const size_t bytes = (count ? count : 1) * sizeof(T);
        if (err == cudaSuccess) err = cudaMalloc(&p, bytes);
        if (err != cudaSuccess) return nullptr;
        ptrs.push_back(p);
        err = src ? cudaMemcpy(p, src, count * sizeof(T), cudaMemcpyHostToDevice) : cudaMemset(p, fill, bytes);
        return static_cast<T*>(p);
    }
    template <class T>
    void get(T* dst, const T* src, size_t count) {
        if (err == cudaSuccess) err = cudaMemcpy(dst, src, count * sizeof(T), cudaMemcpyDeviceToHost);
    }
    ~DevArena() {
        for (void* p : ptrs) cudaFree(p);
    }
};

int finish(DevArena& m) {
    if (m.err == cudaSuccess) m.err = cudaGetLastError();
    if (m.err == cudaSuccess) m.err = cudaDeviceSynchronize();
    return (int)m.err;
}

}  // namespace ba_linalg_test

using namespace ba_linalg_test;

extern "C" {

// Whether ba_step_kernel keeps the packed factor of this D in shared memory on the current device (launch_ba_solve's rule).
int t_step_smem_fits(int D) {
    std::lock_guard<std::mutex> lock(g_cfg_mutex);
    DeviceCfg& c = device_cfg_locked();
    const size_t chol_bytes = sizeof(double) * ((size_t)(D + 1) * (D + 2) / 2 + CHOL_NB * CHOL_PS);
    return chol_bytes + (size_t)c.step_static + 256 <= (size_t)c.smem_limit ? 1 : 0;
}

int t_marg_w_in_global(int md, int n) { return marg_w_in_global(md, n); }

// S members in one launch.  Member k has size n[k]; its packed lower triangle (n (n + 1) / 2 doubles) and n-vectors are
// consecutive in A (A2: the refetched system, or null), b, diag, scale, L and y.  flag: 2 per member.
int t_factor(int S, const int* n, const double* A, const double* A2, const double* b, const double* diag, const double* scale,
             const double* mu, int use_smem, double* L, double* y, int* flag) {
    DevArena m;
    std::vector<FactorJob> jobs(S);
    std::vector<double*> dL(S), dy(S);
    int* dflag = m.alloc<int>(2 * (size_t)S);
    size_t po = 0, vo = 0;
    int nmax = 1;
    for (int k = 0; k < S; k++) {
        const int D = n[k];
        const size_t np = (size_t)D * (D + 1) / 2;
        nmax = std::max(nmax, D);
        FactorJob& j = jobs[k];
        j.n = D;
        j.spk = m.alloc<double>(ba_spk_doubles(D));
        if (m.err == cudaSuccess) m.err = cudaMemcpy(j.spk, A + po, np * sizeof(double), cudaMemcpyHostToDevice);
        j.spk2 = A2 ? m.alloc<double>(np, A2 + po) : nullptr;
        j.gred = m.alloc<double>(D, b + vo);
        j.diag = m.alloc<double>(D, diag + vo);
        j.scale = m.alloc<double>(D, scale + vo);
        j.mu = mu[k];
        j.work = use_smem ? nullptr : m.alloc<double>(ba_work_layout(D, 0).total);
        j.L = dL[k] = m.alloc<double>(np);
        j.y = dy[k] = m.alloc<double>(D);
        j.flag = dflag + 2 * k;
        po += np;
        vo += D;
    }
    const FactorJob* djobs = m.alloc<FactorJob>(S, jobs.data());
    const size_t panel = sizeof(double) * CHOL_NB * CHOL_PS;
    const size_t dyn = use_smem ? panel + sizeof(double) * (size_t)(nmax + 1) * (nmax + 2) / 2 : panel;
    if (m.err == cudaSuccess) m.err = cudaFuncSetAttribute(t_factor_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
    if (m.err == cudaSuccess) t_factor_kernel<<<S, 512, dyn>>>(djobs, use_smem);
    int e = finish(m);
    po = vo = 0;
    for (int k = 0; k < S; k++) {
        const size_t np = (size_t)n[k] * (n[k] + 1) / 2;
        m.get(L + po, dL[k], np);
        m.get(y + vo, dy[k], n[k]);
        po += np;
        vo += n[k];
    }
    m.get(flag, dflag, 2 * (size_t)S);
    return e ? e : (int)m.err;
}

// ba_reduce_kernel at mu (its production grid), then reduce_single_cta at mu2 on the same records.
// shape: W, L, M, est_ex, est_td, relo, wide records (oj = OJ_FULL, lw = LW_FULL), first.  The prior has pn rows and pnb
// blocks (ptype, pindex, poff, pA pn x pn, gpr pn).  Out (NaN where nothing was written): from ba_reduce_kernel Hfull, S
// (D x D), Spk (D (D + 1) / 2), gred, gp (D); from reduce_single_cta S2, Spk2, gred2.
int t_reduce(const int* shape, const int* lm_anchor, const int* lm_start, const int* lm_relo, const double* obsJ, const double* lmW,
             const double* imuJ, int pn, int pnb, const int* ptype, const int* pindex, const int* poff, const double* pA,
             const double* gpr, const double* scale, double mu, double mu2, double* Hfull, double* S, double* Spk, double* gred,
             double* gp, double* S2, double* Spk2, double* gred2) {
    DevArena m;
    const int W = shape[0], L = shape[1], M = shape[2], F = W + 1;
    BaSeq q{};
    BaDims& d = q.p.dims;
    d.W = W;
    d.L = L;
    d.M = M;
    d.est_ex = shape[3];
    d.est_td = shape[4];
    d.col_sb = 6 * F;
    d.col_ex = d.est_ex ? 15 * F : -1;
    d.col_td = d.est_td ? 15 * F + 6 * d.est_ex : -1;
    d.D = 15 * F + 6 * d.est_ex + d.est_td;
    d.col_relo = -1;
    if (shape[5]) {
        d.col_relo = d.D;
        d.D += 6;
    }
    d.oj = shape[6] ? OJ_FULL : OJ_BASE;
    d.lw = shape[6] ? LW_FULL : LW_BASE;
    const int D = d.D;
    const size_t npk = (size_t)D * (D + 1) / 2;
    q.active = 1;
    q.st.mu = mu;
    q.st.first = shape[7];
    q.st.cur = 0;
    BaProblem& p = q.p;
    BaAccum& a = p.acc[0];
    a.obsJ = m.alloc<double>((size_t)M * d.oj, obsJ);
    a.lmW = m.alloc<double>((size_t)L * d.lw, lmW);
    a.imuJ = m.alloc<double>((size_t)W * IMUJ_STRIDE, imuJ);
    std::vector<double> gpr_h(BA_PRIOR_COST + 8, 0.0);
    for (int i = 0; i < pn; i++) gpr_h[i] = gpr[i];
    a.gpr = m.alloc<double>(gpr_h.size(), gpr_h.data());
    a.gp = m.alloc<double>(D, nullptr, 0xff);
    p.acc[1] = a;
    p.lm_anchor = m.alloc<int>(L, lm_anchor);
    p.lm_start = m.alloc<int>((size_t)L + 1, lm_start);
    p.lm_relo = m.alloc<int>(L, lm_relo);
    p.prior.n = pn;
    p.prior.nblocks = pnb;
    p.prior.type = m.alloc<int>(pnb, ptype);
    p.prior.index = m.alloc<int>(pnb, pindex);
    p.prior.off = m.alloc<int>(pnb, poff);
    p.prior.A = m.alloc<double>((size_t)pn * pn, pA);
    p.S = m.alloc<double>((size_t)D * D, nullptr, 0xff);
    p.Spk = m.alloc<double>(ba_spk_doubles(D), nullptr, 0xff);
    p.Hfull = m.alloc<double>((size_t)D * D, nullptr, 0xff);
    p.gred = m.alloc<double>(D, nullptr, 0xff);
    p.scale = m.alloc<double>((size_t)D + L, scale);
    BaSeq* dq = m.alloc<BaSeq>(1);
    p.st = dq ? &dq->st : nullptr;
    if (m.err == cudaSuccess) m.err = cudaMemcpy(dq, &q, sizeof(BaSeq), cudaMemcpyHostToDevice);
    BatchShape sh{};
    sh.S = 1;
    sh.W = W;
    sh.D = D;
    sh.est_ex = d.est_ex;
    sh.est_td = d.est_td;
    sh.any_relo = shape[5];
    if (m.err == cudaSuccess) launch_reduce(dq, sh, 0);
    int e = finish(m);
    m.get(Hfull, p.Hfull, (size_t)D * D);
    m.get(S, p.S, (size_t)D * D);
    m.get(Spk, p.Spk, npk);
    m.get(gred, p.gred, D);
    m.get(gp, a.gp, D);
    if (e == 0 && m.err == cudaSuccess) {
        cudaMemset(p.S, 0xff, sizeof(double) * D * D);
        cudaMemset(p.Spk, 0xff, sizeof(double) * npk);
        cudaMemset(p.gred, 0xff, sizeof(double) * D);
        t_reduce_single_kernel<<<1, 512>>>(dq, mu2);
        e = finish(m);
    }
    m.get(S2, p.S, (size_t)D * D);
    m.get(Spk2, p.Spk, npk);
    m.get(gred2, p.gred, D);
    return e ? e : (int)m.err;
}

// marg_solve_kernel on one member: Am (P x P, upper triangle read) and bm (P) with P = md + nl + n, eps = 1e-8.
// Out: Aout, Araw (n x n), gout (n), cout (1), graw (n + BA_MARG_DIAG).
int t_marg_solve(int md, int nl, int n, const double* Am, const double* bm, int w_in_global, double* Aout, double* gout,
                 double* cout, double* Araw, double* graw) {
    DevArena m;
    const int P = md + nl + n, q = md + n;
    BaSeq s{};
    s.active = 1;
    s.do_marg = 1;
    MargPlan& mp = s.mp;
    mp.P = P;
    mp.m_dense = md;
    mp.n_lm = nl;
    mp.n = n;
    mp.w_in_global = w_in_global;
    mp.Am = m.alloc<double>((size_t)P * P, Am);
    mp.bm = m.alloc<double>(P, bm);
    mp.Aout = m.alloc<double>((size_t)n * n, nullptr, 0xff);
    mp.gout = m.alloc<double>(n, nullptr, 0xff);
    mp.cout = m.alloc<double>(1, nullptr, 0xff);
    mp.Araw = m.alloc<double>((size_t)n * n, nullptr, 0xff);
    mp.graw = m.alloc<double>((size_t)n + BA_MARG_DIAG, nullptr, 0xff);
    mp.Wglobal = m.alloc<double>((size_t)q * q, nullptr, 0xff);
    const BaSeq* dq = m.alloc<BaSeq>(1, &s);
    BatchShape sh{};
    sh.S = 1;
    sh.max_md = md;
    sh.max_n = n;
    sh.w_in_global = w_in_global;
    const size_t smem = prepare_marg_solve(sh);
    if (m.err == cudaSuccess) marg_solve_kernel<<<1, MARG_THREADS, smem>>>(dq, 1e-8);
    const int e = finish(m);
    m.get(Aout, mp.Aout, (size_t)n * n);
    m.get(gout, mp.gout, n);
    m.get(cout, mp.cout, 1);
    m.get(Araw, mp.Araw, (size_t)n * n);
    m.get(graw, mp.graw, (size_t)n + BA_MARG_DIAG);
    return e ? e : (int)m.err;
}

}  // extern "C"
