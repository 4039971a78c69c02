// Host check of the pose graph's buffer layouts (vins_mono_b200/csrc/pg_layout.h), compiled with g++ by
// tests/test_pose_graph_cpu.py: for key-frame counts up to the capacity and border sizes up to PG_MAX_ANCHORS, every
// layout's regions are disjoint, inside its total and (input arena) 16-byte aligned; a launch of every member at capacity
// fits the arena; the workspace holds the linearisation's edge scratch inside W.
#include <cstdio>
#include <vector>

#include "pg_layout.h"

using namespace vb;

namespace {

struct Reg {
    size_t begin, end;
};

bool disjoint_inside(std::vector<Reg> r, size_t total, bool align16, const char* what, char* msg, int cap) {
    for (size_t i = 0; i < r.size(); i++) {
        if (r[i].end > total || r[i].begin > r[i].end || (align16 && r[i].begin % 16)) {
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

extern "C" long check_pg_layouts(int cap_n, long* checked, char* msg, int cap) {
    long fails = 0, n_checked = 0;
    for (int n = 2; n <= cap_n; n += (n < 40 ? 1 : 37)) {
        for (int nb = 0; nb <= PG_MAX_ANCHORS && nb < n; nb += (nb < 8 ? 1 : 11)) {
            const PgInLayout il = pg_in_layout(n, nb);
            const size_t d = sizeof(double), i = sizeof(int);
            if (!disjoint_inside({{il.pose, il.pose + 7 * n * d}, {il.loop, il.loop + 4 * n * d}, {il.seq, il.seq + n * i},
                                  {il.loop_idx, il.loop_idx + n * i}, {il.bslot, il.bslot + n * i}, {il.lfirst, il.lfirst + n * i},
                                  {il.lnext, il.lnext + n * i}, {il.anchors, il.anchors + nb * i}},
                                 il.total, true, "input block", msg, cap))
                fails++;
            if (il.total % 16 || il.total > pg_in_layout(cap_n, PG_MAX_ANCHORS).total) {
                snprintf(msg, cap, "input block n=%d nb=%d does not fit the capacity reserve", n, nb);
                fails++;
            }
            const PgOutLayout ol = pg_out_layout(n);
            if (ol.total % 2 || ol.summary + PG_SUMMARY > ol.total || ol.total > pg_out_layout(cap_n).total) {
                snprintf(msg, cap, "output block n=%d", n);
                fails++;
            }
            n_checked++;
        }
    }
    for (int S : {1, 2, 7, 64}) {
        const PgHdrLayout h = pg_hdr_layout(S);
        const size_t i = sizeof(int), ll = sizeof(long long);
        if (!disjoint_inside({{0, i}, {h.member, h.member + S * i}, {h.n, h.n + S * i}, {h.nb, h.nb + S * i},
                              {h.in_off, h.in_off + S * ll}, {h.out_off, h.out_off + S * ll}},
                             h.total, false, "header", msg, cap))
            fails++;
        if (h.total + (size_t)S * pg_in_layout(cap_n, PG_MAX_ANCHORS).total > pg_arena_bytes(S, cap_n)) {
            snprintf(msg, cap, "arena S=%d", S);
            fails++;
        }
        n_checked++;
    }
    const PgWorkLayout w = pg_work_layout(cap_n);
    const size_t n = cap_n, nsb = pg_num_sb(cap_n), Dp = PG_MAX_D + 1;
    if (!disjoint_inside({{w.state * 8, (w.state + PG_STATE_DOUBLES) * 8}, {w.x * 8, (w.x + 4 * n) * 8}, {w.xc * 8, (w.xc + 4 * n) * 8},
                          {w.dx * 8, (w.dx + 4 * n) * 8}, {w.scale * 8, (w.scale + 4 * n) * 8}, {w.ypr * 8, (w.ypr + 3 * n) * 8},
                          {w.smeas * 8, (w.smeas + 16 * n) * 8}, {w.blk * 8, (w.blk + PG_BLK_KF * n) * 8}, {w.g * 8, (w.g + 4 * n) * 8},
                          {w.L * 8, (w.L + 256 * nsb) * 8}, {w.F * 8, (w.F + 256 * nsb) * 8}, {w.W * 8, (w.W + 16 * nsb * Dp) * 8},
                          {w.start * 8, w.start * 8 + Dp * sizeof(int)}, {w.Sp * 8, (w.Sp + Dp * (Dp + 1) / 2) * 8}},
                         w.total * 8, false, "workspace", msg, cap))
        fails++;
    if (180 * n > 16 * nsb * Dp) {  // the linearisation's edge scratch (5 edges x 36 doubles per key frame) lives in W
        snprintf(msg, cap, "edge scratch does not fit W");
        fails++;
    }
    *checked = n_checked + 1;
    return fails;
}
