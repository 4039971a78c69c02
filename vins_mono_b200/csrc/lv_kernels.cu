// Loop verification on the device (KeyFrame::findConnection and what it needs, pose_graph/src/keyframe.cpp):
//   attach   GaussianBlur 9x9 sigma 2 (OpenCV's 8-bit fixed-point path), FAST-9 + non-maximum suppression (cv::FAST, 20),
//            ordered corner compaction, liftProjective of the corners (PINHOLE, MEI, KANNALA_BRANDT: camera_lift.h), BRIEF on
//            the window points and on the corners
//   connect  brute-force Hamming matching (searchByBRIEFDes), PnP-RANSAC in float64 (one warp per hypothesis, 6-point
//            DLT, consensus count, Gauss-Newton refit on the best consensus set), relative pose and the loop gate.
// Every stage up to the matches is integer (or float32 where the reference is) and bit-exact; no sum uses atomics.  The
// member / job index is the last grid dimension of every kernel.
#include <cstdint>

#include "camera_lift.h"
#include "lv_kernels.h"
#include "lv_layout.h"

namespace vb {
namespace {

constexpr int BLUR_TX = 32, BLUR_TY = 16, BLUR_R = 4;
// OpenCV's fixed-point 9-tap Gaussian for sigma 2 (8 fraction bits, sum 256): getGaussianKernelBitExact rounded with error
// diffusion, centre = 256 - the rest
__constant__ int c_gauss[9] = {7, 17, 32, 46, 52, 46, 32, 17, 7};
// the FAST circle of radius 3 in cyclic order
__constant__ int c_circle[16][2] = {{0, 3}, {1, 3}, {2, 2}, {3, 1}, {3, 0}, {3, -1}, {2, -2}, {1, -3},
                                    {0, -3}, {-1, -3}, {-2, -2}, {-3, -1}, {-3, 0}, {-3, 1}, {-2, 2}, {-1, 3}};

// BORDER_REFLECT_101 for the halo of a tile.  The last tile's halo reaches past n + R where the tile overhangs the image;
// those outputs are discarded, and clamping to [-R, n - 1 + R] first keeps their loads inside the image (n > R).
__device__ __forceinline__ int reflect101(int i, int n) {
    i = min(max(i, -BLUR_R), n - 1 + BLUR_R);
    i = i < 0 ? -i : i;
    return i >= n ? 2 * (n - 1) - i : i;
}

// rows x cols, uint8 -> uint8: row pass exact in 16 bits, column pass in 32 bits, (v + 2^15) >> 16
__global__ void lv_blur_kernel(const char* stage, char* scratch, size_t stage_stride, size_t scratch_stride, int rows, int cols) {
    __shared__ uint8_t in[BLUR_TY + 2 * BLUR_R][BLUR_TX + 2 * BLUR_R];
    __shared__ uint16_t hrow[BLUR_TY + 2 * BLUR_R][BLUR_TX];
    const uint8_t* img = reinterpret_cast<const uint8_t*>(stage + blockIdx.z * stage_stride + lv_stage_layout(rows, cols, 0).img);
    uint8_t* out = reinterpret_cast<uint8_t*>(scratch + blockIdx.z * scratch_stride + lv_attach_layout(rows, cols).blur);
    const int x0 = blockIdx.x * BLUR_TX - BLUR_R, y0 = blockIdx.y * BLUR_TY - BLUR_R;
    const int tid = threadIdx.y * BLUR_TX + threadIdx.x;
    for (int i = tid; i < (BLUR_TY + 2 * BLUR_R) * (BLUR_TX + 2 * BLUR_R); i += BLUR_TX * BLUR_TY) {
        const int yy = i / (BLUR_TX + 2 * BLUR_R), xx = i % (BLUR_TX + 2 * BLUR_R);
        in[yy][xx] = img[(size_t)reflect101(y0 + yy, rows) * cols + reflect101(x0 + xx, cols)];
    }
    __syncthreads();
    for (int yy = threadIdx.y; yy < BLUR_TY + 2 * BLUR_R; yy += BLUR_TY) {
        unsigned s = 0;
        for (int k = 0; k < 9; k++) s += c_gauss[k] * in[yy][threadIdx.x + k];
        hrow[yy][threadIdx.x] = (uint16_t)s;
    }
    __syncthreads();
    const int x = blockIdx.x * BLUR_TX + threadIdx.x, y = blockIdx.y * BLUR_TY + threadIdx.y;
    if (x >= cols || y >= rows) return;
    unsigned s = 0;
    for (int k = 0; k < 9; k++) s += (unsigned)c_gauss[k] * hrow[threadIdx.y + k][threadIdx.x];
    out[(size_t)y * cols + x] = (uint8_t)((s + 32768u) >> 16);
}

// FAST-9 score map on the raw image: 0 where no corner, else max(t, best 9-arc margin) - 1 (cornerScore<16>)
__global__ void lv_fast_score_kernel(const char* stage, char* scratch, size_t stage_stride, size_t scratch_stride, int rows, int cols) {
    const uint8_t* img = reinterpret_cast<const uint8_t*>(stage + blockIdx.z * stage_stride + lv_stage_layout(rows, cols, 0).img);
    uint8_t* score = reinterpret_cast<uint8_t*>(scratch + blockIdx.z * scratch_stride + lv_attach_layout(rows, cols).score);
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
    if (x >= cols) return;
    int sc = 0;
    if (x >= 3 && x < cols - 3 && y >= 3 && y < rows - 3) {
        const int v = img[(size_t)y * cols + x];
        int d[16];
#pragma unroll
        for (int k = 0; k < 16; k++) d[k] = v - img[(size_t)(y + c_circle[k][1]) * cols + x + c_circle[k][0]];
        int dark = -1000, bright = -1000;  // best arc minimum of v - p and of p - v
#pragma unroll
        for (int s = 0; s < 16; s++) {
            int mn = 1000, mx = -1000;
#pragma unroll
            for (int j = 0; j < 9; j++) {
                const int e = d[(s + j) & 15];
                mn = min(mn, e);
                mx = max(mx, e);
            }
            dark = max(dark, mn);
            bright = max(bright, -mx);
        }
        if (dark > LV_FAST_THRESHOLD || bright > LV_FAST_THRESHOLD) sc = max(LV_FAST_THRESHOLD, max(dark, bright)) - 1;
    }
    score[(size_t)y * cols + x] = (uint8_t)sc;
}

// non-maximum suppression: a corner survives when its score is strictly greater than its 8 neighbours'; per-row counts
__global__ void lv_fast_nms_kernel(char* scratch, size_t scratch_stride, int rows, int cols) {
    const LvAttachLayout al = lv_attach_layout(rows, cols);
    char* sc = scratch + blockIdx.z * scratch_stride;
    const uint8_t* score = reinterpret_cast<const uint8_t*>(sc + al.score);
    uint8_t* keep = reinterpret_cast<uint8_t*>(sc + al.keep);
    const int y = blockIdx.y;
    int count = 0;
    for (int x0 = 0; x0 < cols; x0 += blockDim.x) {
        const int x = x0 + threadIdx.x;
        int k = 0;
        if (x < cols) {
            const int s = score[(size_t)y * cols + x];
            if (s > 0) {  // corners lie at least 3 pixels inside, so every neighbour exists
                k = 1;
                for (int dy = -1; dy <= 1; dy++)
                    for (int dx = -1; dx <= 1; dx++)
                        if ((dx || dy) && s <= score[(size_t)(y + dy) * cols + x + dx]) k = 0;
            }
            keep[(size_t)y * cols + x] = (uint8_t)k;
        }
        count += __syncthreads_count(k);
    }
    if (threadIdx.x == 0) reinterpret_cast<int*>(sc + al.rowcnt)[y] = count;
}

struct Intr {
    double v[9];
};

// One CTA per attach: exclusive scan of the row counts, then (when the corners fit) the corners in row-major order, the
// window arrays and the header into the slot.
__global__ void __launch_bounds__(1024, 1) lv_fast_compact_kernel(const char* stage, char* scratch, char* slot, size_t stage_stride,
                                                               size_t scratch_stride, size_t slot_stride, int rows, int cols,
                                                               int max_window, int max_corners) {
    __shared__ int base[LV_MAX_ROWS];
    const LvAttachLayout al = lv_attach_layout(rows, cols);
    const LvStageLayout st = lv_stage_layout(rows, cols, max_window);
    const LvSlotLayout sl = lv_slot_layout(max_window, max_corners);
    const char* sg = stage + blockIdx.z * stage_stride;
    char* sc = scratch + blockIdx.z * scratch_stride;
    char* out = slot + blockIdx.z * slot_stride;
    const int t = threadIdx.x;
    base[t] = t < rows ? reinterpret_cast<const int*>(sc + al.rowcnt)[t] : 0;
    __syncthreads();
    for (int off = 1; off < LV_MAX_ROWS; off <<= 1) {  // inclusive scan
        const int v = t >= off ? base[t - off] : 0;
        __syncthreads();
        base[t] += v;
        __syncthreads();
    }
    const int total = base[LV_MAX_ROWS - 1];
    const bool overflow = total > max_corners;
    int* status = reinterpret_cast<int*>(sc + al.status);
    if (t == 0) {
        status[0] = total;
        status[1] = overflow;
    }
    if (overflow) return;
    const uint8_t* keep = reinterpret_cast<const uint8_t*>(sc + al.keep);
    float* kp = reinterpret_cast<float*>(out + sl.kp);
    const int lane = t & 31, warp = t >> 5;
    for (int y = warp; y < rows; y += 32) {
        int pos = y ? base[y - 1] : 0;
        for (int x0 = 0; x0 < cols; x0 += 32) {
            const int x = x0 + lane;
            const bool k = x < cols && keep[(size_t)y * cols + x];
            const unsigned b = __ballot_sync(0xffffffffu, k);
            if (k) {
                const int p = pos + __popc(b & ((1u << lane) - 1));
                kp[2 * p] = (float)x;
                kp[2 * p + 1] = (float)y;
            }
            pos += __popc(b);
        }
    }
    const LvSlotHdr* sh = reinterpret_cast<const LvSlotHdr*>(sg);
    const int n = sh->n_win;
    for (int i = t; i < 3 * n; i += blockDim.x) reinterpret_cast<float*>(out + sl.p3d)[i] = reinterpret_cast<const float*>(sg + st.p3d)[i];
    for (int i = t; i < 2 * n; i += blockDim.x) {
        reinterpret_cast<float*>(out + sl.uv)[i] = reinterpret_cast<const float*>(sg + st.uv)[i];
        reinterpret_cast<float*>(out + sl.norm)[i] = reinterpret_cast<const float*>(sg + st.norm)[i];
    }
    for (int i = t; i < n; i += blockDim.x) reinterpret_cast<double*>(out + sl.id)[i] = reinterpret_cast<const double*>(sg + st.id)[i];
    if (t == 0) {
        LvSlotHdr* h = reinterpret_cast<LvSlotHdr*>(out);
        for (int k = 0; k < 3; k++) h->vio_P[k] = sh->vio_P[k];
        for (int k = 0; k < 4; k++) h->vio_Q[k] = sh->vio_Q[k];
        h->n_win = n;
        h->n_corners = total;
        h->attached = 1;
    }
}

constexpr int LIFT_THREADS = 128;

// liftProjective / z of the compacted corners (computeBRIEFPoint, keyframe.cpp:108), one thread per corner, stored as float
// like the reference's cv::Point2f.  A grid over max_corners; nothing to do when the corners overflowed.
__global__ void __launch_bounds__(LIFT_THREADS) lv_lift_kernel(const char* scratch, char* slot, size_t scratch_stride, size_t slot_stride,
                                                               int rows, int cols, int max_window, int max_corners, Intr intr,
                                                               int camera_model, double xi) {
    const LvSlotLayout sl = lv_slot_layout(max_window, max_corners);
    const int* status = reinterpret_cast<const int*>(scratch + blockIdx.z * scratch_stride + lv_attach_layout(rows, cols).status);
    if (status[1]) return;
    const int p = blockIdx.x * LIFT_THREADS + threadIdx.x;
    if (p >= status[0]) return;
    char* out = slot + blockIdx.z * slot_stride;
    const float* kp = reinterpret_cast<const float*>(out + sl.kp);
    float* kpn = reinterpret_cast<float*>(out + sl.kpn);
    double X, Y;
    lift_projective(camera_model, intr.v, xi, (double)kp[2 * p], (double)kp[2 * p + 1], X, Y);
    kpn[2 * p] = (float)X;
    kpn[2 * p + 1] = (float)Y;
}

// BRIEF (DVision BRIEF::compute on the blurred image): one warp per point; blockIdx.y = 0 window points (staging uv),
// 1 corners (slot).  Bit i = r * 32 + lane of round r; words assembled from the ballots.
__global__ void lv_brief_kernel(const char* stage, const char* scratch, char* slot, size_t stage_stride, size_t scratch_stride,
                                size_t slot_stride, const int* pattern, int rows, int cols, int max_window, int max_corners) {
    __shared__ int4 pat[LV_BITS];
    for (int i = threadIdx.x; i < LV_BITS; i += blockDim.x) pat[i] = reinterpret_cast<const int4*>(pattern)[i];
    __syncthreads();
    const LvAttachLayout al = lv_attach_layout(rows, cols);
    const LvSlotLayout sl = lv_slot_layout(max_window, max_corners);
    const char* sg = stage + blockIdx.z * stage_stride;
    const char* sc = scratch + blockIdx.z * scratch_stride;
    char* out = slot + blockIdx.z * slot_stride;
    const int* status = reinterpret_cast<const int*>(sc + al.status);
    if (status[1]) return;
    const bool win = blockIdx.y == 0;
    const int n = win ? reinterpret_cast<const LvSlotHdr*>(sg)->n_win : status[0];
    const float* pts = win ? reinterpret_cast<const float*>(sg + lv_stage_layout(rows, cols, max_window).uv)
                           : reinterpret_cast<const float*>(out + sl.kp);
    unsigned long long* desc = reinterpret_cast<unsigned long long*>(out + (win ? sl.wdesc : sl.kdesc));
    const uint8_t* im = reinterpret_cast<const uint8_t*>(sc + al.blur);
    const int lane = threadIdx.x & 31, wpb = blockDim.x >> 5;
    for (int p = blockIdx.x * wpb + (threadIdx.x >> 5); p < n; p += gridDim.x * wpb) {
        const float px = pts[2 * p], py = pts[2 * p + 1];
        unsigned long long w[LV_WORDS] = {0, 0, 0, 0};
#pragma unroll
        for (int r = 0; r < LV_BITS / 32; r++) {
            const int4 q = pat[r * 32 + lane];
            const int x1 = (int)__fadd_rn(px, (float)q.x), y1 = (int)__fadd_rn(py, (float)q.y);
            const int x2 = (int)__fadd_rn(px, (float)q.z), y2 = (int)__fadd_rn(py, (float)q.w);
            bool bit = false;
            if (x1 >= 0 && x1 < cols && y1 >= 0 && y1 < rows && x2 >= 0 && x2 < cols && y2 >= 0 && y2 < rows)
                bit = im[(size_t)y1 * cols + x1] < im[(size_t)y2 * cols + x2];
            const unsigned b = __ballot_sync(0xffffffffu, bit);
            w[r >> 1] |= (unsigned long long)b << (32 * (r & 1));
        }
        if (lane < LV_WORDS) desc[(size_t)LV_WORDS * p + lane] = lane == 0 ? w[0] : lane == 1 ? w[1] : lane == 2 ? w[2] : w[3];
    }
}

// ---- verification

// searchByBRIEFDes: one CTA per job, one warp per window point; each lane keeps the first smallest distance of its
// strided corners, the warp takes the lexicographic minimum (distance, index), i.e. the first index of the smallest
// distance.  Then warp 0 lists the matched window points in window order.
__global__ void __launch_bounds__(1024) lv_match_kernel(const char* arena, const long long* jobs, char* scratch, size_t scratch_stride,
                                                        int max_window, int max_corners) {
    const LvSlotLayout sl = lv_slot_layout(max_window, max_corners);
    const LvConnLayout cl = lv_conn_layout(max_window);
    const int j = blockIdx.z;
    const char* cur = arena + jobs[2 * j];
    const char* old = arena + jobs[2 * j + 1];
    char* sc = scratch + j * scratch_stride;
    const int nw = reinterpret_cast<const LvSlotHdr*>(cur)->n_win, nc = reinterpret_cast<const LvSlotHdr*>(old)->n_corners;
    const unsigned long long* wd = reinterpret_cast<const unsigned long long*>(cur + sl.wdesc);
    const unsigned long long* kd = reinterpret_cast<const unsigned long long*>(old + sl.kdesc);
    int* win_match = reinterpret_cast<int*>(sc + cl.win_match);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int w = warp; w < nw; w += nwarps) {
        const unsigned long long a0 = wd[4 * w], a1 = wd[4 * w + 1], a2 = wd[4 * w + 2], a3 = wd[4 * w + 3];
        int best = LV_MATCH_INIT, bi = -1;
        for (int c = lane; c < nc; c += 32) {
            const int d = __popcll(a0 ^ kd[4 * c]) + __popcll(a1 ^ kd[4 * c + 1]) + __popcll(a2 ^ kd[4 * c + 2]) + __popcll(a3 ^ kd[4 * c + 3]);
            if (d < best) {
                best = d;
                bi = c;
            }
        }
        for (int o = 16; o; o >>= 1) {
            const int ob = __shfl_xor_sync(0xffffffffu, best, o), oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oi >= 0 && (ob < best || (ob == best && (bi < 0 || oi < bi)))) {
                best = ob;
                bi = oi;
            }
        }
        if (lane == 0) win_match[w] = (bi >= 0 && best < LV_MATCH_ACCEPT) ? bi : -1;
    }
    __syncthreads();
    if (warp == 0) {
        int* midx = reinterpret_cast<int*>(sc + cl.midx);
        int pos = 0;
        for (int w0 = 0; w0 < nw; w0 += 32) {
            const int w = w0 + lane;
            const bool m = w < nw && win_match[w] >= 0;
            const unsigned b = __ballot_sync(0xffffffffu, m);
            if (m) midx[pos + __popc(b & ((1u << lane) - 1))] = w;
            pos += __popc(b);
        }
        if (lane == 0) reinterpret_cast<int*>(sc)[0] = pos;
    }
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {  // splitmix64 finaliser
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    return z ^ (z >> 31);
}

// cyclic Jacobi on the symmetric n x n matrix a (row-major, destroyed: its diagonal ends as the eigenvalues); v = the
// eigenvectors as columns.  One thread.
__device__ __noinline__ void jacobi_eig(double* a, double* v, int n) {
    for (int i = 0; i < n * n; i++) v[i] = (i / n == i % n) ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 30; sweep++) {
        double off = 0, dia = 0;
        for (int p = 0; p < n; p++)
            for (int q = 0; q < n; q++) (p == q ? dia : off) += a[p * n + q] * a[p * n + q];
        if (off <= 1e-30 * dia) break;
        for (int p = 0; p < n - 1; p++)
            for (int q = p + 1; q < n; q++) {
                const double apq = a[p * n + q];
                if (apq == 0.0) continue;
                const double theta = (a[q * n + q] - a[p * n + p]) / (2.0 * apq);
                const double tt = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
                for (int k = 0; k < n; k++) {  // columns p, q
                    const double akp = a[k * n + p], akq = a[k * n + q];
                    a[k * n + p] = c * akp - s * akq;
                    a[k * n + q] = s * akp + c * akq;
                }
                for (int k = 0; k < n; k++) {  // rows p, q
                    const double apk = a[p * n + k], aqk = a[q * n + k];
                    a[p * n + k] = c * apk - s * aqk;
                    a[q * n + k] = s * apk + c * aqk;
                }
                for (int k = 0; k < n; k++) {
                    const double vkp = v[k * n + p], vkq = v[k * n + q];
                    v[k * n + p] = c * vkp - s * vkq;
                    v[k * n + q] = s * vkp + c * vkq;
                }
            }
    }
}

struct Match {
    const float* p3d;      // cur window 3-D points
    const float* kpn;      // old corners, normalised
    const int* win_match;  // window point -> old corner
    const int* midx;       // matched window points
};
__device__ __forceinline__ void load_match(const Match& m, int i, double* X, double* u) {
    const int w = m.midx[i], c = m.win_match[w];
    X[0] = m.p3d[3 * w];
    X[1] = m.p3d[3 * w + 1];
    X[2] = m.p3d[3 * w + 2];
    u[0] = m.kpn[2 * c];
    u[1] = m.kpn[2 * c + 1];
}
__device__ __forceinline__ double reproj2(const double* P, const double* X, const double* u) {
    const double x = P[0] * X[0] + P[1] * X[1] + P[2] * X[2] + P[9];
    const double y = P[3] * X[0] + P[4] * X[1] + P[5] * X[2] + P[10];
    const double z = P[6] * X[0] + P[7] * X[1] + P[8] * X[2] + P[11];
    const double ex = x / z - u[0], ey = y / z - u[1];
    return ex * ex + ey * ey;
}
__device__ Match job_match(const char* arena, const long long* jobs, const char* sc, int j, int max_window, int max_corners) {
    const LvSlotLayout sl = lv_slot_layout(max_window, max_corners);
    const LvConnLayout cl = lv_conn_layout(max_window);
    return Match{reinterpret_cast<const float*>(arena + jobs[2 * j] + sl.p3d), reinterpret_cast<const float*>(arena + jobs[2 * j + 1] + sl.kpn),
                 reinterpret_cast<const int*>(sc + cl.win_match), reinterpret_cast<const int*>(sc + cl.midx)};
}

constexpr int HYP_WARPS = 4;

// One warp per hypothesis: LV_SAMPLE distinct correspondences drawn from a counter-based stream (hypothesis, draw), a
// DLT on them (lane 0), then every lane scores its strided correspondences; count = squared error <= threshold^2.
__global__ void __launch_bounds__(HYP_WARPS * 32) lv_pnp_hyp_kernel(const char* arena, const long long* jobs, char* scratch,
                                                                    size_t scratch_stride, int max_window, int max_corners) {
    __shared__ double work[HYP_WARPS][2 * 144];
    __shared__ double pose[HYP_WARPS][12];
    __shared__ double smp[HYP_WARPS][LV_SAMPLE][5];  // the sample: X (3), u (2)
    const LvConnLayout cl = lv_conn_layout(max_window);
    const int j = blockIdx.z, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, h = blockIdx.x * HYP_WARPS + warp;
    char* sc = scratch + j * scratch_stride;
    const int n = reinterpret_cast<const int*>(sc)[0];
    if (n <= LV_MIN_LOOP_NUM || h >= LV_HYP) return;
    const Match m = job_match(arena, jobs, sc, j, max_window, max_corners);
    if (lane == 0) {
        int idx[LV_SAMPLE];
        unsigned long long ctr = 0;
        for (int k = 0; k < LV_SAMPLE; k++) {
            for (;;) {
                const int c = (int)(mix64(0x9e3779b97f4a7c15ull * (unsigned long long)(h + 1) + ctr++) % (unsigned long long)n);
                bool dup = false;
                for (int q = 0; q < k; q++) dup |= idx[q] == c;
                if (!dup) {
                    idx[k] = c;
                    break;
                }
            }
        }
        double(*X)[5] = smp[warp];
        double c3[3] = {0, 0, 0}, sc3 = 0;
        for (int k = 0; k < LV_SAMPLE; k++) {
            load_match(m, idx[k], X[k], X[k] + 3);
            for (int q = 0; q < 3; q++) c3[q] += X[k][q] / LV_SAMPLE;
        }
        for (int k = 0; k < LV_SAMPLE; k++)
            sc3 += sqrt((X[k][0] - c3[0]) * (X[k][0] - c3[0]) + (X[k][1] - c3[1]) * (X[k][1] - c3[1]) + (X[k][2] - c3[2]) * (X[k][2] - c3[2])) / LV_SAMPLE;
        const double s = sc3 > 0 ? 1.7320508075688772 / sc3 : 1.0;
        double* A = work[warp];
        double* V = work[warp] + 144;
        for (int i = 0; i < 144; i++) A[i] = 0;
        for (int k = 0; k < LV_SAMPLE; k++) {  // rows [Xn 1 0 0 -u Xn -u], [0 Xn 1 -v Xn -v]; unknowns P row-major 3 x 4
            const double Xn[4] = {s * (X[k][0] - c3[0]), s * (X[k][1] - c3[1]), s * (X[k][2] - c3[2]), 1.0};
            for (int r = 0; r < 2; r++) {
                double row[12];
                for (int q = 0; q < 4; q++) {
                    row[q] = r == 0 ? Xn[q] : 0.0;
                    row[4 + q] = r == 1 ? Xn[q] : 0.0;
                    row[8 + q] = -X[k][3 + r] * Xn[q];
                }
#pragma unroll 1
                for (int a = 0; a < 12; a++)
                    for (int b = 0; b < 12; b++) A[a * 12 + b] += row[a] * row[b];
            }
        }
        jacobi_eig(A, V, 12);
        int mi = 0;
        for (int i = 1; i < 12; i++)
            if (A[i * 12 + i] < A[mi * 12 + mi]) mi = i;
        double P[12];  // de-normalised: P [s I, -s c; 0 1]
        for (int r = 0; r < 3; r++) {
            const double* pr = &V[0];
            double p4 = V[(4 * r + 3) * 12 + mi];
            for (int q = 0; q < 3; q++) {
                P[3 * r + q] = s * pr[(4 * r + q) * 12 + mi];
                p4 -= s * pr[(4 * r + q) * 12 + mi] * c3[q];
            }
            P[9 + r] = p4;
        }
        const double det = P[0] * (P[4] * P[8] - P[5] * P[7]) - P[1] * (P[3] * P[8] - P[5] * P[6]) + P[2] * (P[3] * P[7] - P[4] * P[6]);
        if (det < 0)
            for (int i = 0; i < 12; i++) P[i] = -P[i];
        // polar factor of M = P[:, :3]: R = M (M^T M)^(-1/2), scale = mean singular value
        double* B = work[warp];
        double* E = work[warp] + 16;
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) B[a * 3 + b] = P[a] * P[b] + P[3 + a] * P[3 + b] + P[6 + a] * P[6 + b];
        jacobi_eig(B, E, 3);
        double isq[9], sv = 0;
        for (int a = 0; a < 3; a++) sv += sqrt(fmax(B[a * 3 + a], 0.0)) / 3;
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) {
                double acc = 0;
                for (int k = 0; k < 3; k++) acc += E[a * 3 + k] * E[b * 3 + k] / sqrt(fmax(B[k * 3 + k], 1e-300));
                isq[a * 3 + b] = acc;
            }
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) pose[warp][3 * a + b] = P[3 * a] * isq[b] + P[3 * a + 1] * isq[3 + b] + P[3 * a + 2] * isq[6 + b];
        for (int r = 0; r < 3; r++) pose[warp][9 + r] = P[9 + r] / sv;
    }
    __syncwarp();
    double P[12];
    for (int i = 0; i < 12; i++) P[i] = pose[warp][i];
    int count = 0;
    const double thr2 = LV_PNP_THRESHOLD * LV_PNP_THRESHOLD;
    for (int i0 = 0; i0 < n; i0 += 32) {
        const int i = i0 + lane;
        bool in = false;
        if (i < n) {
            double X[3], u[2];
            load_match(m, i, X, u);
            in = reproj2(P, X, u) <= thr2;  // false for NaN
        }
        count += __popc(__ballot_sync(0xffffffffu, in));
    }
    if (lane == 0) {
        reinterpret_cast<int*>(sc + cl.hyp_cnt)[h] = count;
        double* hp = reinterpret_cast<double*>(sc + cl.hyp_pose) + 12 * h;
        for (int i = 0; i < 12; i++) hp[i] = P[i];
    }
}

constexpr int REFIT_THREADS = 128;

__device__ void rodrigues(const double* w, double* R) {
    const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
    const double a = th < 1e-12 ? 1.0 : sin(th) / th, b = th < 1e-12 ? 0.5 : (1.0 - cos(th)) / (th * th);
    const double K[9] = {0, -w[2], w[1], w[2], 0, -w[0], -w[1], w[0], 0};
    for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) {
            double kk = 0;
            for (int k = 0; k < 3; k++) kk += K[3 * i + k] * K[3 * k + j];
            R[3 * i + j] = (i == j ? 1.0 : 0.0) + a * K[3 * i + j] + b * kk;
        }
}

__device__ double yaw_deg(const double* R) {  // Utility::R2ypr(R).x()
    return atan2(R[3], R[0]) * (180.0 / 3.14159265358979323846);
}

// One CTA per job: the best hypothesis (most consensus, lowest index on ties), its consensus set, Gauss-Newton on the
// reprojection error over that set (float64, fixed-order tree sums), the old key frame's pose and findConnection's gate.
__global__ void __launch_bounds__(REFIT_THREADS) lv_pnp_refit_kernel(const char* arena, const long long* jobs, char* scratch,
                                                                     size_t scratch_stride, double* result, size_t result_stride,
                                                                     int max_window, int max_corners, Intr ext_r, Intr ext_t) {
    __shared__ double red[27][REFIT_THREADS];
    __shared__ double P[12];
    __shared__ uint8_t inl[LV_CAP_WINDOW];
    __shared__ int s_best, s_stop;
    const LvConnLayout cl = lv_conn_layout(max_window);
    const LvSlotLayout sl = lv_slot_layout(max_window, max_corners);
    const int j = blockIdx.z, t = threadIdx.x;
    char* sc = scratch + j * scratch_stride;
    double* res = result + j * result_stride;
    const int n = reinterpret_cast<const int*>(sc)[0];
    const char* cur = arena + jobs[2 * j];
    if (t == 0) {
        for (int i = 0; i < LV_RES_LIST; i++) res[i] = 0;
        res[1] = n;
        int best = -1, bc = 0;
        if (n > LV_MIN_LOOP_NUM)
            for (int h = 0; h < LV_HYP; h++) {
                const int c = reinterpret_cast<const int*>(sc + cl.hyp_cnt)[h];
                if (c > bc) {
                    bc = c;
                    best = h;
                }
            }
        s_best = best;
        res[4] = best;
        if (best >= 0)
            for (int i = 0; i < 12; i++) P[i] = reinterpret_cast<const double*>(sc + cl.hyp_pose)[12 * best + i];
    }
    __syncthreads();
    if (s_best < 0) return;
    const Match m = job_match(arena, jobs, sc, j, max_window, max_corners);
    const double thr2 = LV_PNP_THRESHOLD * LV_PNP_THRESHOLD;
    int n_in = 0;
    for (int i0 = 0; i0 < n; i0 += REFIT_THREADS) {
        const int i = i0 + t;
        bool in = false;
        if (i < n) {
            double X[3], u[2];
            load_match(m, i, X, u);
            in = reproj2(P, X, u) <= thr2;
            inl[i] = in;
        }
        n_in += __syncthreads_count(in);
    }
    for (int it = 0; it < LV_REFIT_ITERS; it++) {
        double acc[27];
        for (int k = 0; k < 27; k++) acc[k] = 0;
        for (int i = t; i < n; i += REFIT_THREADS) {
            if (!inl[i]) continue;
            double X[3], u[2];
            load_match(m, i, X, u);
            const double RX[3] = {P[0] * X[0] + P[1] * X[1] + P[2] * X[2], P[3] * X[0] + P[4] * X[1] + P[5] * X[2],
                                  P[6] * X[0] + P[7] * X[1] + P[8] * X[2]};
            const double x = RX[0] + P[9], y = RX[1] + P[10], z = RX[2] + P[11], iz = 1.0 / z;
            const double r[2] = {x * iz - u[0], y * iz - u[1]};
            // d(proj)/d(Xc) and d(Xc)/d(omega) = -[RX]x (R <- exp(omega) R), d(Xc)/dt = I
            const double dp[2][3] = {{iz, 0, -x * iz * iz}, {0, iz, -y * iz * iz}};
            const double dw[3][3] = {{0, RX[2], -RX[1]}, {-RX[2], 0, RX[0]}, {RX[1], -RX[0], 0}};
            double J[2][6];
            for (int a = 0; a < 2; a++) {
                for (int b = 0; b < 3; b++) J[a][b] = dp[a][0] * dw[0][b] + dp[a][1] * dw[1][b] + dp[a][2] * dw[2][b];
                for (int b = 0; b < 3; b++) J[a][3 + b] = dp[a][b];
            }
            int k = 0;
            for (int a = 0; a < 6; a++)
                for (int b = a; b < 6; b++) acc[k++] += J[0][a] * J[0][b] + J[1][a] * J[1][b];
            for (int a = 0; a < 6; a++) acc[21 + a] += J[0][a] * r[0] + J[1][a] * r[1];
        }
        for (int k = 0; k < 27; k++) red[k][t] = acc[k];
        __syncthreads();
        for (int w = REFIT_THREADS / 2; w; w >>= 1) {
            if (t < w)
                for (int k = 0; k < 27; k++) red[k][t] += red[k][t + w];
            __syncthreads();
        }
        if (t == 0) {
            double H[36], g[6], L[36] = {0};
            int k = 0;
            for (int a = 0; a < 6; a++)
                for (int b = a; b < 6; b++) H[6 * a + b] = H[6 * b + a] = red[k++][0];
            for (int a = 0; a < 6; a++) g[a] = -red[21 + a][0];
            bool ok = true;
            for (int a = 0; a < 6 && ok; a++) {  // Cholesky
                for (int b = 0; b <= a; b++) {
                    double s = H[6 * a + b];
                    for (int q = 0; q < b; q++) s -= L[6 * a + q] * L[6 * b + q];
                    if (a == b) {
                        if (!(s > 0)) ok = false;
                        else L[6 * a + a] = sqrt(s);
                    } else
                        L[6 * a + b] = s / L[6 * b + b];
                }
            }
            s_stop = !ok;
            if (ok) {
                double y[6], d[6];
                for (int a = 0; a < 6; a++) {
                    double s = g[a];
                    for (int q = 0; q < a; q++) s -= L[6 * a + q] * y[q];
                    y[a] = s / L[6 * a + a];
                }
                for (int a = 5; a >= 0; a--) {
                    double s = y[a];
                    for (int q = a + 1; q < 6; q++) s -= L[6 * q + a] * d[q];
                    d[a] = s / L[6 * a + a];
                }
                double dR[9], R[9];
                rodrigues(d, dR);
                for (int a = 0; a < 3; a++)
                    for (int b = 0; b < 3; b++) R[3 * a + b] = dR[3 * a] * P[b] + dR[3 * a + 1] * P[3 + b] + dR[3 * a + 2] * P[6 + b];
                for (int i = 0; i < 9; i++) P[i] = R[i];
                for (int a = 0; a < 3; a++) P[9 + a] += d[3 + a];
            }
        }
        __syncthreads();
        if (s_stop) break;
    }
    if (t == 0) {
        // PnP_R_old = R_pnp^T ric^T, PnP_T_old = -R_pnp^T t_pnp - PnP_R_old tic (PnPRANSAC's tail)
        const LvSlotHdr* ch = reinterpret_cast<const LvSlotHdr*>(cur);
        double Rwc[9], Twc[3], Ro[9], To[3];
        for (int a = 0; a < 3; a++) {
            for (int b = 0; b < 3; b++) Rwc[3 * a + b] = P[3 * b + a];
            Twc[a] = -(P[a] * P[9] + P[3 + a] * P[10] + P[6 + a] * P[11]);
        }
        for (int a = 0; a < 3; a++)
            for (int b = 0; b < 3; b++) Ro[3 * a + b] = Rwc[3 * a] * ext_r.v[3 * b] + Rwc[3 * a + 1] * ext_r.v[3 * b + 1] + Rwc[3 * a + 2] * ext_r.v[3 * b + 2];
        for (int a = 0; a < 3; a++) To[a] = Twc[a] - (Ro[3 * a] * ext_t.v[0] + Ro[3 * a + 1] * ext_t.v[1] + Ro[3 * a + 2] * ext_t.v[2]);
        // the current key frame's VIO rotation from its quaternion (w x y z)
        const double qw = ch->vio_Q[0], qx = ch->vio_Q[1], qy = ch->vio_Q[2], qz = ch->vio_Q[3];
        const double qn = sqrt(qw * qw + qx * qx + qy * qy + qz * qz);
        const double w_ = qw / qn, x_ = qx / qn, y_ = qy / qn, z_ = qz / qn;
        const double tx = 2 * x_, ty = 2 * y_, tz = 2 * z_;
        const double Rc[9] = {1 - (ty * y_ + tz * z_), ty * x_ - tz * w_, tz * x_ + ty * w_,
                              ty * x_ + tz * w_, 1 - (tx * x_ + tz * z_), tz * y_ - tx * w_,
                              tz * x_ - ty * w_, tz * y_ + tx * w_, 1 - (tx * x_ + ty * y_)};
        double rt[3], rq[9];
        for (int a = 0; a < 3; a++) {
            rt[a] = 0;
            for (int k = 0; k < 3; k++) rt[a] += Ro[3 * k + a] * (ch->vio_P[k] - To[k]);
            for (int b = 0; b < 3; b++) rq[3 * a + b] = Ro[a] * Rc[b] + Ro[3 + a] * Rc[3 + b] + Ro[6 + a] * Rc[6 + b];
        }
        double yaw = yaw_deg(Rc) - yaw_deg(Ro);
        if (yaw > 180.0) yaw -= 360.0;
        else if (yaw < -180.0) yaw += 360.0;
        const double tn = sqrt(rt[0] * rt[0] + rt[1] * rt[1] + rt[2] * rt[2]);
        const bool accepted = n_in > LV_MIN_LOOP_NUM && fabs(yaw) < 30.0 && tn < 20.0;
        res[0] = accepted;
        res[2] = n_in;
        res[3] = n_in;
        for (int a = 0; a < 3; a++) res[LV_RES_LOOP + a] = rt[a];
        res[LV_RES_LOOP + 7] = yaw;
        for (int i = 0; i < 9; i++) res[LV_RES_R + i] = Ro[i];
        for (int a = 0; a < 3; a++) res[LV_RES_T + a] = To[a];
        for (int i = 0; i < 9; i++) res[LV_RES_RQ + i] = rq[i];
    }
    if (t < 32) {  // the consensus set in window order: old normalised x, y and the feature id
        const double* ids = reinterpret_cast<const double*>(cur + sl.id);
        double* list = res + LV_RES_LIST;
        int pos = 0;
        for (int i0 = 0; i0 < n; i0 += 32) {
            const int i = i0 + t;
            const bool in = i < n && inl[i];
            const unsigned b = __ballot_sync(0xffffffffu, in);
            if (in) {
                double X[3], u[2];
                load_match(m, i, X, u);
                const int p = pos + __popc(b & ((1u << t) - 1));
                list[3 * p] = u[0];
                list[3 * p + 1] = u[1];
                list[3 * p + 2] = ids[m.midx[i]];
            }
            pos += __popc(b);
        }
    }
}

// ---- vp_load: one CTA per loaded key frame copies its staged block into its slot (16-byte words; every array of both
//      layouts is 16-byte aligned and the copies are whole words of the block, which the staging zero-pads)
__global__ void __launch_bounds__(256) lv_scatter_kernel(char* arena, const char* staged, int max_window, int max_corners) {
    const long long* job = reinterpret_cast<const long long*>(staged) + 2 * blockIdx.x;
    char* slot = arena + job[0];
    const char* blk = staged + job[1];
    const LvSlotHdr h = *reinterpret_cast<const LvSlotHdr*>(blk);
    const LvSlotLayout sl = lv_slot_layout(max_window, max_corners);
    const LvLoadLayout ll = lv_load_layout(h.n_corners);
    auto copy = [&](size_t dst, size_t src, size_t bytes) {
        const uint4* s = reinterpret_cast<const uint4*>(blk + src);
        uint4* d = reinterpret_cast<uint4*>(slot + dst);
        for (size_t i = threadIdx.x; i < bytes / 16; i += blockDim.x) d[i] = s[i];
    };
    copy(0, 0, lv_align16(sizeof(LvSlotHdr)));
    copy(sl.kp, ll.kp, lv_align16(8 * (size_t)h.n_corners));
    copy(sl.kpn, ll.kpn, lv_align16(8 * (size_t)h.n_corners));
    copy(sl.kdesc, ll.kdesc, 32 * (size_t)h.n_corners);
}

}  // namespace

void launch_lv_scatter(char* arena, const char* staged, int n_kf, int max_window, int max_corners, cudaStream_t s) {
    if (n_kf > 0) lv_scatter_kernel<<<n_kf, 256, 0, s>>>(arena, staged, max_window, max_corners);
}

void launch_lv_lift(const LvAttachLaunch& L, cudaStream_t s) {
    Intr in;
    for (int i = 0; i < 8; i++) in.v[i] = L.intrinsics[i];
    lv_lift_kernel<<<dim3((L.max_corners + LIFT_THREADS - 1) / LIFT_THREADS, 1, 1), LIFT_THREADS, 0, s>>>(
        L.scratch, L.slot, lv_attach_layout(L.rows, L.cols).total, lv_slot_layout(L.max_window, L.max_corners).total, L.rows, L.cols,
        L.max_window, L.max_corners, in, L.camera_model, L.xi);
}

int launch_lv_attach(const LvAttachLaunch& L, cudaStream_t s, cudaEvent_t* ev) {
    const size_t stage_stride = lv_stage_layout(L.rows, L.cols, L.max_window).total, scratch_stride = lv_attach_layout(L.rows, L.cols).total;
    const size_t slot_stride = lv_slot_layout(L.max_window, L.max_corners).total;
    if (ev) cudaEventRecord(ev[0], s);
    lv_blur_kernel<<<dim3((L.cols + BLUR_TX - 1) / BLUR_TX, (L.rows + BLUR_TY - 1) / BLUR_TY, 1), dim3(BLUR_TX, BLUR_TY), 0, s>>>(
        L.stage, L.scratch, stage_stride, scratch_stride, L.rows, L.cols);
    if (ev) cudaEventRecord(ev[1], s);
    lv_fast_score_kernel<<<dim3((L.cols + 127) / 128, L.rows, 1), 128, 0, s>>>(L.stage, L.scratch, stage_stride, scratch_stride, L.rows, L.cols);
    lv_fast_nms_kernel<<<dim3(1, L.rows, 1), 256, 0, s>>>(L.scratch, scratch_stride, L.rows, L.cols);
    lv_fast_compact_kernel<<<dim3(1, 1, 1), 1024, 0, s>>>(L.stage, L.scratch, L.slot, stage_stride, scratch_stride, slot_stride, L.rows,
                                                           L.cols, L.max_window, L.max_corners);
    launch_lv_lift(L, s);
    if (ev) cudaEventRecord(ev[2], s);
    lv_brief_kernel<<<dim3(64, 2, 1), 256, 0, s>>>(L.stage, L.scratch, L.slot, stage_stride, scratch_stride, slot_stride, L.pattern, L.rows,
                                                    L.cols, L.max_window, L.max_corners);
    if (ev) cudaEventRecord(ev[3], s);
    return 6;
}

int launch_lv_connect(const LvConnLaunch& L, cudaStream_t s, cudaEvent_t* ev, int match) {
    Intr r, t;
    for (int i = 0; i < 9; i++) r.v[i] = L.ric[i];
    for (int i = 0; i < 8; i++) t.v[i] = i < 3 ? L.tic[i] : 0.0;
    int launches = 0;
    if (ev) cudaEventRecord(ev[0], s);
    if (match) {
        lv_match_kernel<<<dim3(1, 1, L.n_jobs), 1024, 0, s>>>(L.arena, L.jobs, L.scratch, L.scratch_stride, L.max_window, L.max_corners);
        launches++;
    }
    if (ev) cudaEventRecord(ev[1], s);
    lv_pnp_hyp_kernel<<<dim3(LV_HYP / HYP_WARPS, 1, L.n_jobs), HYP_WARPS * 32, 0, s>>>(L.arena, L.jobs, L.scratch, L.scratch_stride,
                                                                                       L.max_window, L.max_corners);
    if (ev) cudaEventRecord(ev[2], s);
    lv_pnp_refit_kernel<<<dim3(1, 1, L.n_jobs), REFIT_THREADS, 0, s>>>(L.arena, L.jobs, L.scratch, L.scratch_stride, L.result,
                                                                       L.result_stride, L.max_window, L.max_corners, r, t);
    if (ev) cudaEventRecord(ev[3], s);
    return launches + 2;
}

}  // namespace vb
