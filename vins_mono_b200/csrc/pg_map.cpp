// The saved pose-graph format (pg_map.h).
#include "pg_map.h"

#include <cstdio>
#include <cstring>
#include <memory>

#include "vinsb200/pose_graph.h"

namespace vb {
namespace {

using File = std::unique_ptr<FILE, int (*)(FILE*)>;

File open(const std::string& path, const char* mode) { return File(std::fopen(path.c_str(), mode), std::fclose); }

bool read_all(const std::string& path, std::string* s) {
    File f = open(path, "rb");
    if (!f) return false;
    char buf[1 << 16];
    size_t n;
    s->clear();
    while ((n = std::fread(buf, 1, sizeof(buf), f.get())) > 0) s->append(buf, n);
    return !std::ferror(f.get());
}

// the lines of s that hold more than white space, with their 1-based line numbers
std::vector<std::pair<int, std::string>> content_lines(const std::string& s) {
    std::vector<std::pair<int, std::string>> out;
    size_t b = 0;
    for (int ln = 1; b < s.size(); ln++) {
        size_t e = s.find('\n', b);
        if (e == std::string::npos) e = s.size();
        std::string line = s.substr(b, e - b);
        if (line.find_first_not_of(" \t\r") != std::string::npos) out.emplace_back(ln, std::move(line));
        b = e + 1;
    }
    return out;
}

bool only_space(const char* p) {
    for (; *p; p++)
        if (*p != ' ' && *p != '\t' && *p != '\r') return false;
    return true;
}

int fail(std::string* err, int rc, const std::string& msg) {
    *err = msg;
    return rc;
}

std::string where(const std::string& path, int line) { return path + ":" + std::to_string(line) + ": "; }

}  // namespace

int map_write(const std::string& prefix, const std::vector<MapKeyFrame>& kfs, bool with_points, std::string* err) {
    const std::string path = prefix + "pose_graph.txt";
    File f = open(path, "w");
    if (!f) return fail(err, VP_ERR_INVALID, "vp_save: cannot write " + path);
    for (const MapKeyFrame& k : kfs) {
        const int n = with_points ? k.n_kp : 0;
        std::fprintf(f.get(), " %d %f %f %f %f %f %f %f %f %f %f %f %f %f %f %f %d %f %f %f %f %f %f %f %f %d\n", k.index, k.stamp,
                     k.vio_T[0], k.vio_T[1], k.vio_T[2], k.pg_T[0], k.pg_T[1], k.pg_T[2], k.vio_Q[0], k.vio_Q[1], k.vio_Q[2], k.vio_Q[3],
                     k.pg_Q[0], k.pg_Q[1], k.pg_Q[2], k.pg_Q[3], k.loop_index, k.loop_info[0], k.loop_info[1], k.loop_info[2],
                     k.loop_info[3], k.loop_info[4], k.loop_info[5], k.loop_info[6], k.loop_info[7], n);
        const std::string bp = prefix + std::to_string(k.index) + "_briefdes.dat", kp = prefix + std::to_string(k.index) + "_keypoints.txt";
        File fb = open(bp, "wb"), fk = open(kp, "w");
        if (!fb) return fail(err, VP_ERR_INVALID, "vp_save: cannot write " + bp);
        if (!fk) return fail(err, VP_ERR_INVALID, "vp_save: cannot write " + kp);
        char line[257];
        line[256] = '\n';
        for (int i = 0; i < n; i++) {
            const uint64_t* d = k.desc.data() + 4 * (size_t)i;
            for (int j = 0; j < 256; j++) line[j] = (d[(255 - j) >> 6] >> ((255 - j) & 63)) & 1 ? '1' : '0';
            std::fwrite(line, 1, sizeof(line), fb.get());
            std::fprintf(fk.get(), "%f %f %f %f\n", k.kp[2 * i], k.kp[2 * i + 1], k.kpn[2 * i], k.kpn[2 * i + 1]);
        }
        if (std::ferror(fb.get()) || std::fclose(fb.release())) return fail(err, VP_ERR_INVALID, "vp_save: cannot write " + bp);
        if (std::ferror(fk.get()) || std::fclose(fk.release())) return fail(err, VP_ERR_INVALID, "vp_save: cannot write " + kp);
    }
    if (std::ferror(f.get()) || std::fclose(f.release())) return fail(err, VP_ERR_INVALID, "vp_save: cannot write " + path);
    return 0;
}

int map_read(const std::string& prefix, bool with_points, int max_keyframes, int max_corners, std::vector<MapKeyFrame>* out,
             std::string* err) {
    const std::string path = prefix + "pose_graph.txt";
    std::string text;
    if (!read_all(path, &text)) return fail(err, VP_ERR_INVALID, "vp_load: cannot read " + path);
    std::vector<MapKeyFrame> kfs;
    for (const auto& [ln, line] : content_lines(text)) {
        if ((int)kfs.size() >= max_keyframes)
            return fail(err, VP_ERR_CAPACITY, where(path, ln) + "more than max_keyframes = " + std::to_string(max_keyframes) + " key frames");
        MapKeyFrame k;
        double* li = k.loop_info;
        int used = -1;
        const int got = std::sscanf(line.c_str(), "%d %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %lf %d %lf %lf %lf %lf %lf %lf %lf %lf %d%n",
                                    &k.index, &k.stamp, &k.vio_T[0], &k.vio_T[1], &k.vio_T[2], &k.pg_T[0], &k.pg_T[1], &k.pg_T[2],
                                    &k.vio_Q[0], &k.vio_Q[1], &k.vio_Q[2], &k.vio_Q[3], &k.pg_Q[0], &k.pg_Q[1], &k.pg_Q[2], &k.pg_Q[3],
                                    &k.loop_index, &li[0], &li[1], &li[2], &li[3], &li[4], &li[5], &li[6], &li[7], &k.n_kp, &used);
        if (got != 26 || used < 0 || !only_space(line.c_str() + used))
            return fail(err, VP_ERR_INVALID, where(path, ln) + "truncated or unparsable key-frame line");
        if (k.index != (int)kfs.size())
            return fail(err, VP_ERR_INVALID, where(path, ln) + "index " + std::to_string(k.index) + ", expected " + std::to_string(kfs.size()));
        if (k.loop_index < -1 || k.loop_index >= k.index)
            return fail(err, VP_ERR_INVALID, where(path, ln) + "loop_index " + std::to_string(k.loop_index) + " does not name an earlier key frame");
        if (k.n_kp < 0) return fail(err, VP_ERR_INVALID, where(path, ln) + "negative keypoint count");
        if (with_points && k.n_kp > max_corners)
            return fail(err, VP_ERR_CAPACITY, where(path, ln) + std::to_string(k.n_kp) + " keypoints, at most max_corners = " + std::to_string(max_corners));
        kfs.push_back(std::move(k));
    }
    if (with_points) {
        std::string s;
        for (MapKeyFrame& k : kfs) {
            const size_t n = (size_t)k.n_kp;
            const std::string kp = prefix + std::to_string(k.index) + "_keypoints.txt";
            if (!read_all(kp, &s)) return fail(err, VP_ERR_INVALID, "vp_load: cannot read " + kp);
            const auto lines = content_lines(s);
            if (lines.size() != n)
                return fail(err, VP_ERR_INVALID, kp + ": " + std::to_string(lines.size()) + " keypoint lines, the key frame lists " + std::to_string(n));
            k.kp.resize(2 * n);
            k.kpn.resize(2 * n);
            for (size_t i = 0; i < n; i++) {
                double v[4];
                int used = -1;
                const char* c = lines[i].second.c_str();
                if (std::sscanf(c, "%lf %lf %lf %lf%n", &v[0], &v[1], &v[2], &v[3], &used) != 4 || used < 0 || !only_space(c + used))
                    return fail(err, VP_ERR_INVALID, where(kp, lines[i].first) + "truncated or unparsable keypoint line");
                k.kp[2 * i] = (float)v[0];
                k.kp[2 * i + 1] = (float)v[1];
                k.kpn[2 * i] = (float)v[2];
                k.kpn[2 * i + 1] = (float)v[3];
            }
            const std::string bp = prefix + std::to_string(k.index) + "_briefdes.dat";
            if (!read_all(bp, &s)) return fail(err, VP_ERR_INVALID, "vp_load: cannot read " + bp);
            k.desc.assign(4 * n, 0);
            size_t p = 0;
            for (size_t i = 0; i < n; i++, p += 257) {
                if (s.size() < p + 257 || s[p + 256] != '\n')
                    return fail(err, VP_ERR_INVALID, where(bp, (int)i + 1) + "not a line of 256 '0' / '1' characters");
                uint64_t* d = k.desc.data() + 4 * i;
                for (int j = 0; j < 256; j++) {
                    const char ch = s[p + j];
                    if (ch != '0' && ch != '1') return fail(err, VP_ERR_INVALID, where(bp, (int)i + 1) + "not a line of 256 '0' / '1' characters");
                    if (ch == '1') d[(255 - j) >> 6] |= (uint64_t)1 << ((255 - j) & 63);
                }
            }
            if (p != s.size())
                return fail(err, VP_ERR_INVALID, bp + ": more descriptor data than the key frame's " + std::to_string(n) + " keypoints");
        }
    }
    *out = std::move(kfs);
    return 0;
}

}  // namespace vb
