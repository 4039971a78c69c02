// Host access to the saved pose-graph format (vins_mono_b200/csrc/pg_map.cpp), compiled with g++ together with it by
// tests/test_pose_graph_map_cpu.py: read a map, write one back, and hand the parsed values to Python.
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "pg_map.h"

using namespace vb;

namespace {
void put(const std::string& s, char* msg, int cap) { std::snprintf(msg, cap, "%s", s.c_str()); }
}  // namespace

// Reads src and writes it under dst.  Returns the key-frame count or the status of the failed step.
extern "C" int pgmap_copy(const char* src, const char* dst, int with_points, int max_keyframes, int max_corners, char* msg, int cap) {
    std::vector<MapKeyFrame> kfs;
    std::string err;
    int rc = map_read(src, with_points != 0, max_keyframes, max_corners, &kfs, &err);
    if (!rc) rc = map_write(dst, kfs, with_points != 0, &err);
    put(err, msg, cap);
    return rc ? rc : (int)kfs.size();
}

// Reads src: rows (26 doubles per key frame, in the file's column order), then for every keypoint in key-frame order
// pts (pixel x y, normalised x y as float) and desc (4 words).  Returns the key-frame count or the status.
extern "C" int pgmap_read(const char* src, int with_points, int max_keyframes, int max_corners, double* rows, int cap_rows, float* pts,
                          unsigned long long* desc, int cap_pts, char* msg, int cap) {
    std::vector<MapKeyFrame> kfs;
    std::string err;
    const int rc = map_read(src, with_points != 0, max_keyframes, max_corners, &kfs, &err);
    put(err, msg, cap);
    if (rc) return rc;
    if ((int)kfs.size() > cap_rows) return -100;
    int p = 0;
    for (size_t i = 0; i < kfs.size(); i++) {
        const MapKeyFrame& k = kfs[i];
        double* r = rows + 26 * i;
        r[0] = k.index;
        r[1] = k.stamp;
        std::memcpy(r + 2, k.vio_T, 24);
        std::memcpy(r + 5, k.pg_T, 24);
        std::memcpy(r + 8, k.vio_Q, 32);
        std::memcpy(r + 12, k.pg_Q, 32);
        r[16] = k.loop_index;
        std::memcpy(r + 17, k.loop_info, 64);
        r[25] = k.n_kp;
        for (size_t j = 0; j < k.kp.size() / 2; j++, p++) {
            if (p >= cap_pts) return -100;
            pts[4 * p] = k.kp[2 * j];
            pts[4 * p + 1] = k.kp[2 * j + 1];
            pts[4 * p + 2] = k.kpn[2 * j];
            pts[4 * p + 3] = k.kpn[2 * j + 1];
            for (int w = 0; w < 4; w++) desc[4 * p + w] = k.desc[4 * j + w];
        }
    }
    return (int)kfs.size();
}
