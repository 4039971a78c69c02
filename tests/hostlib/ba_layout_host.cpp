// Test-only host check of the BA path's buffer layouts (vins_mono_b200/csrc/ba_layout.h): every layout the batch sizes,
// carves, writes and reads, evaluated over the window sizes, optional blocks and landmark counts the estimator accepts.
#include "../../vins_mono_b200/csrc/ba_layout.h"

#include <algorithm>
#include <cstdio>
#include <string>
#include <vector>

namespace {

struct Region {
    const char* name;
    size_t off, len;  // in the layout's unit
};

struct Checker {
    std::string first;
    long checks = 0, failures = 0;
    void fail(const char* what, const char* name, int W, int L) {
        if (failures++ == 0) {
            char buf[256];
            std::snprintf(buf, sizeof buf, "%s: %s (W=%d, L=%d)", what, name, W, L);
            first = buf;
        }
    }
    void expect(bool ok, const char* what, int W, int L) {
        checks++;
        if (!ok) fail(what, "", W, L);
    }
    // the regions are pairwise disjoint, inside [0, total), and start on a multiple of `align` units
    void layout(const char* what, std::vector<Region> rs, size_t total, size_t align, int W, int L) {
        std::sort(rs.begin(), rs.end(), [](const Region& a, const Region& b) { return a.off < b.off; });
        for (size_t i = 0; i < rs.size(); i++) {
            checks++;
            if (rs[i].off + rs[i].len > total) fail(what, rs[i].name, W, L);
            if (rs[i].off % align) fail(what, rs[i].name, W, L);
            if (i && rs[i].len && rs[i - 1].off + rs[i - 1].len > rs[i].off) fail(what, rs[i].name, W, L);
        }
    }
};

}  // namespace

// Returns the number of failed checks; writes the number of checks and the first failure.
extern "C" long check_ba_layouts(int Lmax, long* n_checks, char* msg, int msg_len) {
    using namespace vb;
    Checker c;
    const size_t D16 = 2;  // doubles per 16 bytes
    for (int W = 3; W <= 22; W++) {
        const int F = W + 1;
        // config_valid's window limit is the solvers' capacity
        c.expect(6 * W + 16 <= BA_MAX_PRIOR_N && 15 * F + 7 <= BA_MAX_D, "window within the solver capacity", W, 0);
        // member capacity as create_member sizes it: one relocalisation match per landmark on top of the tracks, every
        // optional column block, a prior with two speed-bias blocks
        const int Mmax = Lmax * F, Dcap = 15 * F + 6 + 1 + 6, nmax = 6 * F + 9 * 2 + 6 + 1;
        const BaInLayout in_max = ba_in_layout_max(W, Lmax, Mmax);
        const size_t out_max = ba_out_reserve(F, Lmax, true);
        c.expect(ba_states_layout(F, 0).lam <= ba_states_layout(BA_MAX_FRAMES, 0).lam, "ba_finish_kernel's staging", W, 0);

        // workspaces sized at the capacity
        const BaAccLayout a = ba_acc_layout(W, Lmax, Mmax, Dcap);
        c.layout("acc", {{"obsJ", a.obsJ, (size_t)Mmax * OJ_FULL}, {"lmW", a.lmW, (size_t)Lmax * LW_FULL},
                         {"imuJ", a.imuJ, (size_t)W * IMUJ_STRIDE}, {"gpr", a.gpr, BA_PRIOR_COST + 1},
                         {"gp", a.gp, (size_t)Dcap}, {"cost", a.cost, 1}},
                 a.total, 1, W, Lmax);
        c.layout("acc records", {{"obsJ", a.obsJ, 0}, {"lmW", a.lmW, 0}, {"imuJ", a.imuJ, 0}, {"gpr", a.gpr, 0}, {"gp", a.gp, 0}},
                 a.total, D16, W, Lmax);
        const BaPriorLayout pr = ba_prior_layout(nmax);
        c.layout("prior", {{"A", pr.A, (size_t)nmax * nmax}, {"g0", pr.g0, (size_t)nmax}, {"c0", pr.c0, 1},
                           {"x0", pr.x0, 9 * (size_t)BA_MAX_PRIOR_BLOCKS}},
                 pr.total, 1, W, 0);
        c.expect(6 * W + 16 <= nmax, "prior capacity", W, 0);
        const BaMargLayout m = ba_marg_layout(nmax, Lmax);
        const size_t q = (size_t)nmax + BA_MARG_MAX_DENSE;
        c.layout("marg", {{"Am", m.Am, m.P * m.P}, {"bm", m.bm, m.P}, {"Araw", m.Araw, (size_t)nmax * nmax},
                          {"graw", m.graw, (size_t)nmax + BA_MARG_DIAG}, {"Wglobal", m.Wglobal, q * q}},
                 m.total, 1, W, Lmax);
        const BaVecLayout v = ba_vec_layout(Dcap, Lmax);
        const size_t Nv = (size_t)Dcap + Lmax;
        c.layout("vec", {{"scale", v.scale, Nv}, {"diag", v.diag, Nv}, {"grad", v.grad, Nv}, {"gn", v.gn, Nv}}, v.total, 1, W, Lmax);
        const size_t work_alloc = ba_work_layout(Dcap, Lmax).total, spk_alloc = ba_spk_doubles(Dcap);
        for (int Dx = 1; Dx <= Dcap; Dx++) {  // every reduced dimension, odd packed counts included
            const size_t npk = (size_t)Dx * (Dx + 1) / 2, copied = (npk + 1) & ~(size_t)1;
            c.expect(copied <= spk_alloc && (copied * sizeof(double)) % 16 == 0, "Spk slack covers the bulk copy", W, Dx);
        }

        for (int ex = 0; ex <= 1; ex++)
            for (int td = 0; td <= 1; td++)
                for (int relo_req = 0; relo_req <= 1; relo_req++)
                    for (int L : {0, 1, Lmax}) {
                        // the relocalisation gate of stage_frame
                        const int D0 = 15 * F + 6 * ex + td;
                        const bool relo = relo_req && D0 + 6 <= BA_MAX_D;
                        const int D = D0 + (relo ? 6 : 0);
                        c.expect(D <= BA_MAX_D && D <= Dcap, "columns within capacity", W, L);
                        const int M = L * F;  // every track at full length, plus its relocalisation match
                        // states
                        const BaStatesLayout s = ba_states_layout(F, L);
                        c.layout("states", {{"pose", (size_t)s.pose, 7 * (size_t)F}, {"sb", (size_t)s.sb, 9 * (size_t)F}, {"ex", (size_t)s.ex, 7},
                                            {"td", (size_t)s.td, 1}, {"lam", (size_t)s.lam, (size_t)L}, {"relo", (size_t)s.relo, 7}},
                                 s.total, 1, W, L);
                        c.expect(s.total <= ba_states_layout(F, Lmax).total, "states fit the x[1] allocation", W, L);
                        // output block
                        const BaOutLayout o = ba_out_layout(F, L, relo);
                        c.layout("out", {{"state", 0, (sizeof(SolverState) + 7) / 8}, {"frames", (size_t)o.frames, (size_t)BA_OUT_FRAME * F},
                                         {"ex", (size_t)o.ex, BA_OUT_EX}, {"depths", (size_t)o.depths, (size_t)L},
                                         {"relo", (size_t)o.relo, relo ? (size_t)BA_OUT_RELO : 0}},
                                 o.total, 1, W, L);
                        const size_t reserve = ba_out_reserve(F, L, relo);
                        c.expect(reserve >= (size_t)o.total && reserve % D16 == 0, "output block reserve", W, L);
                        c.expect(reserve <= out_max, "output block within the at-capacity reserve", W, L);
                        // input block, with and without a solve
                        for (int solve = 0; solve <= 1; solve++)
                            for (size_t n_jobs : {(size_t)0, (size_t)1, (size_t)4 * F})
                                for (size_t n_rec : {(size_t)0, (size_t)1, (size_t)4096})
                                    for (size_t n_lm : {(size_t)0, (size_t)L}) {
                                        const BaInLayout il = ba_in_layout(W, n_jobs, n_rec, L, M, n_lm, solve != 0);
                                        std::vector<Region> rs = {{"jobs", il.jobs, n_jobs * sizeof(PreintJob)},
                                                                  {"samples", il.samples, n_rec * 7 * sizeof(double)}};
                                        if (solve) {
                                            rs.push_back({"ints", il.ints, sizeof(int) * (3 * (size_t)L + 1 + M + W)});
                                            rs.push_back({"dbls", il.dbls, sizeof(double) * (6 * (size_t)L + 6 * (size_t)M)});
                                            rs.push_back({"states", il.states, sizeof(double) * s.total});
                                            rs.push_back({"marg", il.marg, sizeof(int) * 2 * n_lm});
                                        }
                                        c.layout("input block", rs, il.total, 16, W, L);
                                        c.expect(il.total % 16 == 0 && il.total <= in_max.total, "input block within the at-capacity size", W, L);
                                        if (!solve || n_jobs != 1 || n_rec != 1) continue;
                                        // the bound arrays, host side (the device side is the same function at another base)
                                        std::vector<double> buf(il.total / sizeof(double) + 2);
                                        unsigned char* base = reinterpret_cast<unsigned char*>(buf.data());
                                        const BaInPtrs p = ba_in_bind(base, il);
                                        auto at = [&](const void* ptr) { return (size_t)(static_cast<const unsigned char*>(ptr) - base); };
                                        c.layout("bound input block",
                                                 {{"jobs", at(p.jobs), sizeof(PreintJob)}, {"samples", at(p.samples), 7 * sizeof(double)},
                                                  {"lm_anchor", at(p.lm_anchor), 4 * (size_t)L}, {"lm_start", at(p.lm_start), 4 * (size_t)(L + 1)},
                                                  {"ob_frame", at(p.ob_frame), 4 * (size_t)M}, {"imu_slot", at(p.imu_slot), 4 * (size_t)W},
                                                  {"lm_relo", at(p.lm_relo), 4 * (size_t)L}, {"lm_pts", at(p.lm_pts), 16 * (size_t)L},
                                                  {"lm_vel", at(p.lm_vel), 16 * (size_t)L}, {"lm_td", at(p.lm_td), 8 * (size_t)L},
                                                  {"lm_row", at(p.lm_row), 8 * (size_t)L}, {"ob_pts", at(p.ob_pts), 16 * (size_t)M},
                                                  {"ob_vel", at(p.ob_vel), 16 * (size_t)M}, {"ob_td", at(p.ob_td), 8 * (size_t)M},
                                                  {"ob_row", at(p.ob_row), 8 * (size_t)M}, {"states", at(p.states), 8 * (size_t)s.total},
                                                  {"marg_lms", at(p.marg_lms), 4 * n_lm}, {"marg_col_lm", at(p.marg_col_lm), 4 * n_lm}},
                                                 il.total, 4, W, L);
                                    }
                        // ba_step_kernel's scratch at this frame's D and L, inside the capacity allocation
                        const BaWorkLayout w = ba_work_layout(D, L);
                        const size_t N = (size_t)D + L;
                        c.layout("work", {{"u", w.u, N}, {"y", w.y, N}, {"delta", w.delta, N}, {"Lp", w.Lp, (size_t)(D + 1) * (D + 2) / 2}},
                                 w.total, 1, W, L);
                        c.expect(w.total <= work_alloc, "work within the allocation", W, L);
                    }
    }
    if (n_checks) *n_checks = c.checks;
    if (msg && msg_len > 0) std::snprintf(msg, (size_t)msg_len, "%s", c.first.c_str());
    return c.failures;
}
