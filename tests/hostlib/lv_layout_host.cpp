// Host check of the loop-verification layouts (vins_mono_b200/csrc/lv_layout.h), compiled with g++ by
// tests/test_loop_verify_cpu.py: every region of a slot, a staging block, an attach scratch and a verification scratch is
// 16-byte aligned, disjoint from the others and inside the total, for capacities up to the limits; the result block
// holds its header and list.
#include <cstdio>
#include <vector>

#include "lv_layout.h"

using namespace vb;

namespace {
struct Reg {
    size_t begin, end;
};
bool ok(const std::vector<Reg>& r, size_t total, const char* what, char* msg, int cap) {
    for (size_t i = 0; i < r.size(); i++) {
        if (r[i].end > total || r[i].begin % 16 || r[i].begin > r[i].end) {
            snprintf(msg, cap, "%s: region %zu [%zu, %zu) total %zu", what, i, r[i].begin, r[i].end, total);
            return false;
        }
        for (size_t j = 0; j < i; j++)
            if (r[i].begin < r[j].end && r[j].begin < r[i].end) {
                snprintf(msg, cap, "%s: regions %zu and %zu overlap", what, j, i);
                return false;
            }
    }
    return total % 16 == 0;
}
}  // namespace

extern "C" long check_lv_layouts(long* checked, char* msg, int cap) {
    long fails = 0, n = 0;
    for (int w : {1, 2, 25, 150, 1000, LV_CAP_WINDOW})
        for (int c : {1, 7, 4096, 16384, LV_CAP_CORNERS}) {
            const LvSlotLayout s = lv_slot_layout(w, c);
            if (!ok({{0, sizeof(LvSlotHdr)}, {s.p3d, s.p3d + 12 * (size_t)w}, {s.uv, s.uv + 8 * (size_t)w}, {s.norm, s.norm + 8 * (size_t)w},
                     {s.id, s.id + 8 * (size_t)w}, {s.wdesc, s.wdesc + 32 * (size_t)w}, {s.kp, s.kp + 8 * (size_t)c},
                     {s.kpn, s.kpn + 8 * (size_t)c}, {s.kdesc, s.kdesc + 32 * (size_t)c}},
                    s.total, "slot", msg, cap))
                fails++;
            if (lv_arena_bytes(3, 5, w, c) != 15 * s.total) fails++;
            n++;
        }
    for (int rows : {8, 97, 480, LV_MAX_ROWS})
        for (int cols : {8, 131, 752, LV_MAX_COLS})
            for (int w : {1, 150, LV_CAP_WINDOW}) {
                const LvStageLayout st = lv_stage_layout(rows, cols, w);
                const size_t px = (size_t)rows * cols;
                if (!ok({{0, sizeof(LvSlotHdr)}, {st.img, st.img + px}, {st.p3d, st.p3d + 12 * (size_t)w}, {st.uv, st.uv + 8 * (size_t)w},
                         {st.norm, st.norm + 8 * (size_t)w}, {st.id, st.id + 8 * (size_t)w}},
                        st.total, "stage", msg, cap))
                    fails++;
                const LvAttachLayout a = lv_attach_layout(rows, cols);
                if (!ok({{a.blur, a.blur + px}, {a.score, a.score + px}, {a.keep, a.keep + px}, {a.rowcnt, a.rowcnt + 4 * (size_t)rows},
                         {a.status, a.status + 8}},
                        a.total, "attach scratch", msg, cap))
                    fails++;
                n++;
            }
    for (int w : {1, 26, 150, LV_CAP_WINDOW}) {
        const LvConnLayout c = lv_conn_layout(w);
        if (!ok({{0, 16}, {c.win_match, c.win_match + 4 * (size_t)w}, {c.midx, c.midx + 4 * (size_t)w},
                 {c.hyp_cnt, c.hyp_cnt + 4 * (size_t)LV_HYP}, {c.hyp_pose, c.hyp_pose + 96 * (size_t)LV_HYP}},
                c.total, "verification scratch", msg, cap))
            fails++;
        if (lv_result_doubles(w) != (size_t)LV_RES_LIST + 3 * (size_t)w || LV_RES_RQ + 9 > LV_RES_LIST || LV_RES_T + 3 > LV_RES_RQ ||
            LV_RES_R + 9 > LV_RES_T || LV_RES_LOOP + 8 > LV_RES_R)
            fails++;
        n++;
    }
    *checked = n;
    return fails;
}
