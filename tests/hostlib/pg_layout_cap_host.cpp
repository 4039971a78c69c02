// Host check of the pose graph's workspace and arena layouts (vins_mono_b200/csrc/pg_layout.h) at a given anchor
// capacity, compiled with g++ by tests/test_pose_graph_border_cpu.py: the workspace regions are disjoint and inside
// total, W holds the linearisation's edge scratch, the multi-CTA path's regions (U, Ud, yb) exist exactly when the
// capacity exceeds PG_MAX_D columns and are 16-byte aligned, every input block up to the capacity fits the arena's
// reserve with 16-byte aligned arrays, and the default capacity gives the same layouts as the calls without it.
#include <cstdio>
#include <vector>

#include "pg_layout.h"

using namespace vb;

namespace {

struct Reg {
    size_t begin, end;
};

bool disjoint_inside(const std::vector<Reg>& r, size_t total, const char* what, char* msg, int cap) {
    for (size_t i = 0; i < r.size(); i++) {
        if (r[i].end > total || r[i].begin > r[i].end) {
            snprintf(msg, cap, "%s: region %zu [%zu, %zu) vs total %zu", what, i, r[i].begin, r[i].end, total);
            return false;
        }
        for (size_t j = 0; j < i; j++)
            if (r[i].begin < r[j].end && r[j].begin < r[i].end && r[i].begin != r[i].end && r[j].begin != r[j].end) {
                snprintf(msg, cap, "%s: regions %zu and %zu overlap", what, j, i);
                return false;
            }
    }
    return true;
}

}  // namespace

extern "C" long check_pg_layouts_cap(int cap_n, int cap_anchors, long* checked, char* msg, int cap) {
    long fails = 0, n_checked = 0;
    const PgWorkLayout w = pg_work_layout(cap_n, cap_anchors);
    const size_t n = cap_n, nsb = pg_num_sb(cap_n), D = 4 * (size_t)cap_anchors, Dp = D + 1;
    const size_t Dps = (D < (size_t)PG_MAX_D ? D : PG_MAX_D) + 1, Np = pg_tile_np((int)D);
    const size_t Wsz = 16 * nsb * Dp > 180 * n ? 16 * nsb * Dp : 180 * n;
    const std::vector<Reg> regs = {
        {w.state, w.state + PG_STATE_DOUBLES}, {w.x, w.x + 4 * n},       {w.xc, w.xc + 4 * n},         {w.dx, w.dx + 4 * n},
        {w.scale, w.scale + 4 * n},            {w.ypr, w.ypr + 3 * n},   {w.smeas, w.smeas + 16 * n},  {w.blk, w.blk + PG_BLK_KF * n},
        {w.g, w.g + 4 * n},                    {w.L, w.L + 256 * nsb},   {w.F, w.F + 256 * nsb},       {w.W, w.W + Wsz},
        {w.start, w.start + (Dp + 1) / 2},     {w.Sp, w.Sp + Dps * (Dps + 1) / 2},
        {w.U, w.U + Np * Np},                  {w.Ud, w.Ud + Np * PG_TILE}, {w.yb, w.yb + (Np ? D : 0)}};
    if (!disjoint_inside(regs, w.total, "workspace", msg, cap)) fails++;
    n_checked++;
    if ((D > (size_t)PG_MAX_D) != (Np > 0) || (Np && (Np % PG_TILE || Np < Dp))) {
        snprintf(msg, cap, "multi-CTA regions at D = %zu: Np = %zu", D, Np);
        fails++;
    }
    if (w.U % 2 || w.Ud % 2 || w.yb % 2) {  // in doubles: even = 16-byte aligned
        snprintf(msg, cap, "multi-CTA regions not 16-byte aligned: U %zu Ud %zu yb %zu", w.U, w.Ud, w.yb);
        fails++;
    }
    n_checked++;
    for (int nb = 0; nb <= cap_anchors; nb += (nb < 8 ? 1 : 37)) {
        const PgInLayout il = pg_in_layout(cap_n, nb);
        const size_t arrays[] = {il.pose, il.loop, il.seq, il.loop_idx, il.bslot, il.lfirst, il.lnext, il.anchors, il.total};
        for (size_t a : arrays)
            if (a % 16) {
                snprintf(msg, cap, "input block n=%d nb=%d: array at byte %zu not 16-byte aligned", cap_n, nb, a);
                fails++;
            }
        if (il.total > pg_in_layout(cap_n, cap_anchors).total) {
            snprintf(msg, cap, "input block n=%d nb=%d does not fit the capacity reserve", cap_n, nb);
            fails++;
        }
        n_checked++;
    }
    for (int S : {1, 3, 64}) {
        if (pg_hdr_layout(S).total + (size_t)S * pg_in_layout(cap_n, cap_anchors).total > pg_arena_bytes(S, cap_n, cap_anchors)) {
            snprintf(msg, cap, "arena S=%d", S);
            fails++;
        }
        if (pg_arena_bytes(S, cap_n) != pg_arena_bytes(S, cap_n, PG_MAX_ANCHORS)) {
            snprintf(msg, cap, "arena S=%d: the default capacity differs from PG_MAX_ANCHORS", S);
            fails++;
        }
        n_checked++;
    }
    if (pg_work_layout(cap_n).total != pg_work_layout(cap_n, PG_MAX_ANCHORS).total) {
        snprintf(msg, cap, "workspace: the default capacity differs from PG_MAX_ANCHORS");
        fails++;
    }
    *checked = n_checked + 1;
    return fails;
}
