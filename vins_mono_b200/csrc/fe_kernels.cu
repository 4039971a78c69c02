// Front-end image kernels for sm_90a (feature_tracker hot path, SURVEY.md §8 rows a3, a4, a7, a8).
//
// Every kernel reproduces the integer / IEEE-f32 arithmetic of the OpenCV routine the reference calls
// (feature_tracker/src/feature_tracker.cpp:87-93 CLAHE, :113 calcOpticalFlowPyrLK, :66 circle,
// :149 goodFeaturesToTrack) operation by operation, so results are bit-identical to a plain CPU evaluation:
// no FMA contraction where OpenCV's baseline build has none (explicit __fmul_rn/__fadd_rn), integer
// window sums accumulated exactly.  All of this is HBM/L2-bound byte and integer work; nothing here is
// GEMM shaped, so no tensor cores.
#include "cuda_check.h"
#include "fe_kernels.h"

#include <cfloat>
#include <cstdint>

namespace vb {

__device__ __forceinline__ int reflect101(int p, int len) {
    if (len == 1) return 0;
    while (p < 0 || p >= len) p = p < 0 ? -p : 2 * (len - 1) - p;
    return p;
}

__device__ __forceinline__ uint8_t sat_u8(float v) {
    int i = __float2int_rn(v);  // cvRound: round-half-even
    return (uint8_t)min(max(i, 0), 255);
}

// ---------------------------------------------------------------------------------------------
// CLAHE step 1: one CTA per tile -> 256-entry LUT (histogram, clip, redistribute, cumulative sum).
// Image reads are coalesced along rows; per-warp shared histograms keep atomics off a single bank set.
__global__ void __launch_bounds__(256) clahe_lut_kernel(const FeSeq* __restrict__ seqs, int rows, int cols,
                                                        int tiles_x, int tw, int th, int clip, float lut_scale) {
    const FeSeq& q = seqs[blockIdx.y];
    if (!q.track || !q.equalize) return;
    const uint8_t* __restrict__ src = q.raw;
    const int pitch = q.raw_pitch;
    uint8_t* __restrict__ lut = q.lut;
    __shared__ int wh[8][256];
    __shared__ int red[8];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x;
    for (int i = tid; i < 8 * 256; i += 256) (&wh[0][0])[i] = 0;
    __syncthreads();
    for (int y = warp; y < th; y += 8) {
        const int sy = reflect101(ty * th + y, rows);
        const uint8_t* row = src + (size_t)sy * pitch;
        for (int x = lane; x < tw; x += 32) {
            const int sx = reflect101(tx * tw + x, cols);
            atomicAdd(&wh[warp][row[sx]], 1);
        }
    }
    __syncthreads();
    int h = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) h += wh[w][tid];
    int over = 0;
    if (clip > 0 && h > clip) {
        over = h - clip;
        h = clip;
    }
    // block sum of `over`
    int s = over;
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    int clipped = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) clipped += red[w];
    if (clip > 0) {
        const int redist = clipped / 256;
        int residual = clipped - redist * 256;
        h += redist;
        if (residual != 0) {
            const int step = max(256 / residual, 1);
            // bins 0, step, 2*step, ... (first `residual` of them that are < 256) get one more count
            if (tid % step == 0 && tid / step < residual) h += 1;
        }
    }
    // inclusive scan of h over 256 threads
    int v = h;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += t;
    }
    __syncthreads();
    if (lane == 31) red[warp] = v;
    __syncthreads();
    int base = 0;
    for (int w = 0; w < warp; w++) base += red[w];
    v += base;
    lut[(size_t)blockIdx.x * 256 + tid] = sat_u8(__fmul_rn((float)v, lut_scale));
}

// CLAHE step 2: bilinear blend of the four neighbouring tile LUTs, 4 pixels per thread.
__global__ void __launch_bounds__(256) clahe_apply_kernel(const FeSeq* __restrict__ seqs, int rows, int cols, int tiles_x,
                                                          int tiles_y, float inv_tw, float inv_th) {
    const FeSeq& q = seqs[blockIdx.z];
    if (!q.track) return;
    const uint8_t* __restrict__ src = q.raw;
    const int spitch = q.raw_pitch;
    const uint8_t* __restrict__ lut = q.lut;
    uint8_t* __restrict__ dst = const_cast<uint8_t*>(q.forw.img[0]);
    const int dpitch = q.forw.pitch[0];
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int y = blockIdx.y;
    if (x0 >= cols) return;
    if (!q.equalize) {  // EQUALIZE = 0: forw_img = img (feature_tracker.cpp:94-95)
        for (int k = 0; k < 4; k++)
            if (x0 + k < cols) dst[(size_t)y * dpitch + x0 + k] = src[(size_t)y * spitch + x0 + k];
        return;
    }
    const float tyf = __fsub_rn(__fmul_rn((float)y, inv_th), 0.5f);
    int ty1 = (int)floorf(tyf);
    const float ya = __fsub_rn(tyf, (float)ty1), ya1 = __fsub_rn(1.0f, ya);
    int ty2 = min(ty1 + 1, tiles_y - 1);
    ty1 = max(ty1, 0);
    const uint8_t* p1 = lut + (size_t)ty1 * tiles_x * 256;
    const uint8_t* p2 = lut + (size_t)ty2 * tiles_x * 256;
    uint8_t in[4], out[4];
    const bool full = (x0 + 3 < cols) && ((spitch & 3) == 0) && ((dpitch & 3) == 0);
    if (full)
        *reinterpret_cast<uchar4*>(in) = *reinterpret_cast<const uchar4*>(src + (size_t)y * spitch + x0);
    else
        for (int k = 0; k < 4; k++) in[k] = x0 + k < cols ? src[(size_t)y * spitch + x0 + k] : 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int x = x0 + k;
        const float txf = __fsub_rn(__fmul_rn((float)x, inv_tw), 0.5f);
        int tx1 = (int)floorf(txf);
        const float xa = __fsub_rn(txf, (float)tx1), xa1 = __fsub_rn(1.0f, xa);
        int tx2 = min(tx1 + 1, tiles_x - 1);
        tx1 = max(tx1, 0);
        const int v = in[k];
        const float l11 = (float)__ldg(p1 + tx1 * 256 + v), l12 = (float)__ldg(p1 + tx2 * 256 + v);
        const float l21 = (float)__ldg(p2 + tx1 * 256 + v), l22 = (float)__ldg(p2 + tx2 * 256 + v);
        const float top = __fadd_rn(__fmul_rn(l11, xa1), __fmul_rn(l12, xa));
        const float bot = __fadd_rn(__fmul_rn(l21, xa1), __fmul_rn(l22, xa));
        out[k] = sat_u8(__fadd_rn(__fmul_rn(top, ya1), __fmul_rn(bot, ya)));
    }
    if (full)
        *reinterpret_cast<uchar4*>(dst + (size_t)y * dpitch + x0) = *reinterpret_cast<uchar4*>(out);
    else
        for (int k = 0; k < 4; k++)
            if (x0 + k < cols) dst[(size_t)y * dpitch + x0 + k] = out[k];
}

// ---------------------------------------------------------------------------------------------
// pyrDown: [1 4 6 4 1]^2, reflect-101, (sum + 128) >> 8.  One thread per output pixel; the 5x5
// footprint is served by L1 (source level <= 361 KB, read once from HBM).
__global__ void __launch_bounds__(256) pyrdown_kernel(const FeSeq* __restrict__ seqs, int level, int use_cur) {
    const FeSeq& q = seqs[blockIdx.z];
    if (!q.track) return;
    const PyramidView& pv = use_cur ? q.cur : q.forw;  // use_cur: the debug entry builds both pyramids
    if (level > pv.nlev) return;
    const uint8_t* __restrict__ src = pv.img[level - 1];
    const int rows = pv.rows[level - 1], cols = pv.cols[level - 1], spitch = pv.pitch[level - 1];
    uint8_t* __restrict__ dst = const_cast<uint8_t*>(pv.img[level]);
    const int drows = pv.rows[level], dcols = pv.cols[level], dpitch = pv.pitch[level];
    const int dx = blockIdx.x * blockDim.x + threadIdx.x;
    const int dy = blockIdx.y * blockDim.y + threadIdx.y;
    if (dx >= dcols || dy >= drows) return;
    int xs[5];
#pragma unroll
    for (int i = 0; i < 5; i++) xs[i] = reflect101(2 * dx + i - 2, cols);
    int acc = 0;
    const int k[5] = {1, 4, 6, 4, 1};
#pragma unroll
    for (int j = 0; j < 5; j++) {
        const uint8_t* row = src + (size_t)reflect101(2 * dy + j - 2, rows) * spitch;
        const int r = row[xs[0]] + row[xs[4]] + 4 * (row[xs[1]] + row[xs[3]]) + 6 * row[xs[2]];
        acc += k[j] * r;
    }
    dst[(size_t)dy * dpitch + dx] = (uint8_t)((acc + 128) >> 8);
}

// ---------------------------------------------------------------------------------------------
// Pyramidal Lucas-Kanade, one 128-thread CTA per point, all levels inside one launch.
// Mirrors OpenCV's LKTrackerInvoker including the float accumulation structure of its x86 (CV_SIMD128) build: per window
// row 16 pixels go through four float lanes and 5 through a scalar float, lanes are combined as (l0 + l2) + (l1 + l3); the
// per-pixel terms are produced by all threads, the (inherently sequential) float chains run on 15 / 10 threads.  Results
// are bit-identical to cv2 4.13 (tests/test_frontend_gpu.py checks the golden digests of the cv2-backed twin).  Per level the CTA stages the
// 24x24 previous-image neighbourhood in shared memory, derives the Scharr gradient there (zero outside
// the image, reflect-101 inside), builds the 21x21 int16 patch + gradient patch, then iterates on a cached
// 40x40 region of the next image.  The 441-pixel window is spread over 4 warps (the track count of a frame, 150,
// matches the SM count, so a point per CTA puts one warp on each scheduler of an SM; a warp per point left three
// of the four schedulers idle and the kernel bound by one warp's issue latency).  Reductions are warp shuffles
// on 64-bit integers + a 4-entry shared-memory exchange; every thread then evaluates the same scalar update,
// so control flow stays CTA-uniform.
#define LK_WARPS 4
#define LK_RS 40                 // next-image search region cached per level: 22x22 window + 9 px margin each side
struct LkSmem {
    uint8_t tile[24 * 24];       // previous-level neighbourhood
    uint8_t region[LK_RS * LK_RS];  // next-level search region (reflect-101 padded coordinates)
    int16_t deriv[22 * 22 * 2];  // Scharr dx,dy at the 22x22 bilinear source positions
    int16_t iwin[441];
    int16_t dwin[441 * 2];
    int px[441], py[441];        // (J - I) Ix and (J - I) Iy of every window pixel (exact integers)
    float chain[16];
};

__global__ void __launch_bounds__(32 * LK_WARPS) lk_track_kernel(const FeSeq* __restrict__ seqs, int max_iter, double eps2,
                                                                 float min_eig_thr) {
    __shared__ LkSmem sm;
    constexpr int NT = 32 * LK_WARPS;
    const FeSeq& q = seqs[blockIdx.y];
    const int lane = threadIdx.x;  // index within the CTA that owns point p
    const int wl = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int p = blockIdx.x;
    if (!q.track || p >= q.n_pts) return;
    const PyramidView& prev = q.cur;
    const PyramidView& next = q.forw;
    const float* __restrict__ prev_pts = q.pts_in;
    float* __restrict__ next_pts = q.pts_out;
    uint8_t* __restrict__ status = q.status;
    const int img_rows = prev.rows[0], img_cols = prev.cols[0];
    const int W = 21;
    const float half = 10.f;
    const float FLT_SCALE = 1.f / (1 << 20);
    const float px0 = prev_pts[2 * p], py0 = prev_pts[2 * p + 1];
    float outx = 0.f, outy = 0.f;  // nextPts[ptidx]
    int st = 1;
    for (int level = prev.nlev; level >= 0; level--) {
        const uint8_t* I = prev.img[level];
        const uint8_t* J = next.img[level];
        const int rows = prev.rows[level], cols = prev.cols[level], pitch = prev.pitch[level];
        const float sc = 1.f / (float)(1 << level);  // exact power of two
        float ppx = __fmul_rn(px0, sc), ppy = __fmul_rn(py0, sc);
        float nx, ny;
        if (level == prev.nlev) {
            nx = ppx;
            ny = ppy;
        } else {
            nx = __fmul_rn(outx, 2.f);
            ny = __fmul_rn(outy, 2.f);
        }
        outx = nx;
        outy = ny;
        ppx = __fsub_rn(ppx, half);
        ppy = __fsub_rn(ppy, half);
        const int ipx = (int)floorf(ppx), ipy = (int)floorf(ppy);
        if (ipx < -W || ipx >= cols || ipy < -W || ipy >= rows) {
            if (level == 0) st = 0;
            continue;
        }
        float a = __fsub_rn(ppx, (float)ipx), b = __fsub_rn(ppy, (float)ipy);
        int iw00 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), __fsub_rn(1.f, b)), 16384.f));
        int iw01 = __float2int_rn(__fmul_rn(__fmul_rn(a, __fsub_rn(1.f, b)), 16384.f));
        int iw10 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), b), 16384.f));
        int iw11 = 16384 - iw00 - iw01 - iw10;
        // stage the 24x24 neighbourhood, origin (ipy-1, ipx-1), reflect-101 padding
        __syncthreads();
        for (int i = lane; i < 24 * 24; i += NT) {
            const int ty = i / 24, tx = i - ty * 24;
            sm.tile[i] = I[(size_t)reflect101(ipy - 1 + ty, rows) * pitch + reflect101(ipx - 1 + tx, cols)];
        }
        __syncthreads();
        // Scharr gradient at the 22x22 positions (calcSharrDeriv); zero outside the image
        for (int i = lane; i < 22 * 22; i += NT) {
            const int dyi = i / 22, dxi = i - dyi * 22;
            const int gy = ipy + dyi, gx = ipx + dxi;
            int ddx = 0, ddy = 0;
            if (gx >= 0 && gx < cols && gy >= 0 && gy < rows) {
                const uint8_t* t = &sm.tile[dyi * 24 + dxi];  // top-left of the 3x3 around (dyi+1, dxi+1)
                const int p00 = t[0], p01 = t[1], p02 = t[2];
                const int p10 = t[24], p12 = t[26];
                const int p20 = t[48], p21 = t[49], p22 = t[50];
                ddx = ((p02 + p22) * 3 + p12 * 10) - ((p00 + p20) * 3 + p10 * 10);
                ddy = ((p20 - p00) + (p22 - p02)) * 3 + (p21 - p01) * 10;
            }
            sm.deriv[2 * i] = (int16_t)ddx;
            sm.deriv[2 * i + 1] = (int16_t)ddy;
        }
        __syncthreads();
        for (int i = lane; i < 441; i += NT) {
            const int y = i / 21, x = i - y * 21;
            const uint8_t* t = &sm.tile[(y + 1) * 24 + (x + 1)];
            const int ival = (t[0] * iw00 + t[1] * iw01 + t[24] * iw10 + t[25] * iw11 + (1 << 8)) >> 9;
            const int16_t* d = &sm.deriv[2 * (y * 22 + x)];
            const int ixval = (d[0] * iw00 + d[2] * iw01 + d[44] * iw10 + d[46] * iw11 + (1 << 13)) >> 14;
            const int iyval = (d[1] * iw00 + d[3] * iw01 + d[45] * iw10 + d[47] * iw11 + (1 << 13)) >> 14;
            sm.iwin[i] = (int16_t)ival;
            sm.dwin[2 * i] = (int16_t)ixval;
            sm.dwin[2 * i + 1] = (int16_t)iyval;
        }
        __syncthreads();
        // window sums A11, A12, A22: 12 lane chains (quantity q, lane j: pixels j, 4+j, 8+j, 12+j of every row, float product
        // then float add) and 3 scalar-tail chains (pixels 16..20, integer product converted to float)
        if (lane < 15) {
            const int qi = lane < 12 ? lane >> 2 : lane - 12, j = lane & 3;
            float acc = 0.f;
            // the terms of a batch of rows are formed first (independent loads and products), then added in order: only the
            // additions sit on the dependent chain
            if (lane < 12) {
                for (int y0 = 0; y0 < 21; y0 += 3) {
                    float term[12];
#pragma unroll
                    for (int u = 0; u < 12; u++) {
                        const int i = (y0 + (u >> 2)) * 21 + 4 * (u & 3) + j;
                        // A11: Ix Ix, A12: Ix Iy, A22: Iy Iy, as index selects (no divergent paths inside the chain warp)
                        const float fa = (float)sm.dwin[2 * i + (qi == 2)], fb = (float)sm.dwin[2 * i + (qi != 0)];
                        term[u] = __fmul_rn(fa, fb);
                    }
#pragma unroll
                    for (int u = 0; u < 12; u++) acc = __fadd_rn(acc, term[u]);
                }
            } else {
                for (int y0 = 0; y0 < 21; y0 += 3) {
                    float term[15];
#pragma unroll
                    for (int u = 0; u < 15; u++) {
                        const int i = (y0 + u / 5) * 21 + 16 + u % 5;
                        const int ia = sm.dwin[2 * i + (qi == 2)], ib = sm.dwin[2 * i + (qi != 0)];
                        term[u] = __int2float_rn(ia * ib);
                    }
#pragma unroll
                    for (int u = 0; u < 15; u++) acc = __fadd_rn(acc, term[u]);
                }
            }
            sm.chain[lane] = acc;
        }
        __syncthreads();
        float A11, A12, A22;
        {
            const float* c = sm.chain;
            A11 = __fmul_rn(__fadd_rn(c[12], __fadd_rn(__fadd_rn(c[0], c[2]), __fadd_rn(c[1], c[3]))), FLT_SCALE);
            A12 = __fmul_rn(__fadd_rn(c[13], __fadd_rn(__fadd_rn(c[4], c[6]), __fadd_rn(c[5], c[7]))), FLT_SCALE);
            A22 = __fmul_rn(__fadd_rn(c[14], __fadd_rn(__fadd_rn(c[8], c[10]), __fadd_rn(c[9], c[11]))), FLT_SCALE);
        }
        float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
        const float dif = __fsub_rn(A11, A22);
        const float disc = __fadd_rn(__fmul_rn(dif, dif), __fmul_rn(__fmul_rn(4.f, A12), A12));
        const float min_eig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(disc)), (float)(2 * W * W));
        if (min_eig < min_eig_thr || D < FLT_EPSILON) {
            if (level == 0) st = 0;
            continue;
        }
        D = __fdiv_rn(1.f, D);
        nx = __fsub_rn(nx, half);
        ny = __fsub_rn(ny, half);
        float pdx = 0.f, pdy = 0.f;
        int ry0 = 0, rx0 = 0;
        bool have_region = false;
        for (int j = 0; j < max_iter; j++) {
            const int inx = (int)floorf(nx), iny = (int)floorf(ny);
            if (inx < -W || inx >= cols || iny < -W || iny >= rows) {
                if (level == 0) st = 0;
                break;
            }
            a = __fsub_rn(nx, (float)inx);
            b = __fsub_rn(ny, (float)iny);
            iw00 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), __fsub_rn(1.f, b)), 16384.f));
            iw01 = __float2int_rn(__fmul_rn(__fmul_rn(a, __fsub_rn(1.f, b)), 16384.f));
            iw10 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), b), 16384.f));
            iw11 = 16384 - iw00 - iw01 - iw10;
            // the 22x22 tile the window needs: served from the cached region, which is (re)loaded around the
            // current position only when the window walks out of it
            if (!have_region || inx < rx0 || inx + 22 > rx0 + LK_RS || iny < ry0 || iny + 22 > ry0 + LK_RS) {
                ry0 = iny - (LK_RS - 22) / 2;
                rx0 = inx - (LK_RS - 22) / 2;
                __syncthreads();
                for (int i = lane; i < LK_RS * LK_RS; i += NT) {
                    const int ty = i / LK_RS, tx = i - ty * LK_RS;
                    sm.region[i] = J[(size_t)reflect101(ry0 + ty, rows) * pitch + reflect101(rx0 + tx, cols)];
                }
                __syncthreads();
                have_region = true;
            }
            const uint8_t* rbase = &sm.region[(iny - ry0) * LK_RS + (inx - rx0)];
            auto mismatch = [&](int y, int x, int& px, int& py) {  // (J - I) * (Ix, Iy) of one window pixel, exact integers
                const int i = y * 21 + x;
                const uint8_t* t = rbase + y * LK_RS + x;
                const int diff = ((t[0] * iw00 + t[1] * iw01 + t[LK_RS] * iw10 + t[LK_RS + 1] * iw11 + (1 << 8)) >> 9) - sm.iwin[i];
                px = diff * sm.dwin[2 * i];
                py = diff * sm.dwin[2 * i + 1];
            };
            // every thread forms the integer products of its window pixels; the chain threads pair them up
            for (int w = lane; w < 441; w += NT) {
                const int y = w / 21, x = w - 21 * y;
                int ax, ay;
                mismatch(y, x, ax, ay);
                sm.px[w] = ax;
                sm.py[w] = ay;
            }
            __syncthreads();
            if (lane < 10) {
                float acc = 0.f;
                if (lane < 8) {  // lane chains: X / Y of pixel pair (k, k + 4), rows in order, block 0 then block 1
                    const int* src = ((lane & 1) ? sm.py : sm.px) + (lane >> 1);
                    for (int y0 = 0; y0 < 21; y0 += 7) {
                        float term[14];
#pragma unroll
                        for (int u = 0; u < 14; u++) {  // integer pair sum -> float, like v_dotprod + v_cvt_f32
                            const int* q2 = src + (y0 + (u >> 1)) * 21 + 8 * (u & 1);
                            term[u] = __int2float_rn(q2[0] + q2[4]);
                        }
#pragma unroll
                        for (int u = 0; u < 14; u++) acc = __fadd_rn(acc, term[u]);
                    }
                } else {
                    const int* src = lane == 8 ? sm.px : sm.py;
                    for (int y0 = 0; y0 < 21; y0 += 3) {
                        float term[15];
#pragma unroll
                        for (int u = 0; u < 15; u++) term[u] = __int2float_rn(src[(y0 + u / 5) * 21 + 16 + u % 5]);
#pragma unroll
                        for (int u = 0; u < 15; u++) acc = __fadd_rn(acc, term[u]);
                    }
                }
                sm.chain[lane] = acc;
            }
            __syncthreads();
            // qb0 = {X0, Y0, X1, Y1}, qb1 = {X2, Y2, X3, Y3}; q = qb0 + qb1; b1 = tail + (q0 + q2), b2 = tail + (q1 + q3)
            const float* c = sm.chain;
            const float q0 = __fadd_rn(c[0], c[4]), q1 = __fadd_rn(c[1], c[5]), q2 = __fadd_rn(c[2], c[6]), q3 = __fadd_rn(c[3], c[7]);
            const float fb1 = __fmul_rn(__fadd_rn(c[8], __fadd_rn(q0, q2)), FLT_SCALE);
            const float fb2 = __fmul_rn(__fadd_rn(c[9], __fadd_rn(q1, q3)), FLT_SCALE);
            const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb2), __fmul_rn(A22, fb1)), D);
            const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, fb1), __fmul_rn(A11, fb2)), D);
            nx = __fadd_rn(nx, dx);
            ny = __fadd_rn(ny, dy);
            outx = __fadd_rn(nx, half);
            outy = __fadd_rn(ny, half);
            if (__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)) <= eps2) break;
            if (j > 0 && fabs((double)__fadd_rn(dx, pdx)) < 0.01 && fabs((double)__fadd_rn(dy, pdy)) < 0.01) {
                outx = __fsub_rn(outx, __fmul_rn(dx, 0.5f));
                outy = __fsub_rn(outy, __fmul_rn(dy, 0.5f));
                break;
            }
            pdx = dx;
            pdy = dy;
        }
    }
    if (lane == 0) {
        // FeatureTracker::readImage's inBorder() cull is fused here (feature_tracker.cpp:5-11,115-117)
        if (st) {
            const int ix = __float2int_rn(outx), iy = __float2int_rn(outy);
            if (!(1 <= ix && ix < img_cols - 1 && 1 <= iy && iy < img_rows - 1)) st = 0;
        }
        next_pts[2 * p] = outx;
        next_pts[2 * p + 1] = outy;
        status[p] = (uint8_t)st;
    }
}

// ---------------------------------------------------------------------------------------------
// Mask: 255 (or the fisheye mask) with a filled cv::circle of radius r at every kept track.
// halfw[d] = half width of the rasterised disc at row offset |d| (midpoint algorithm, host-computed).
// Mask start: 255 everywhere, or the fisheye mask (feature_tracker.cpp:38-41); also clears the detection counters.
__global__ void __launch_bounds__(256) mask_init_kernel(const FeSeq* __restrict__ seqs, int rows, int cols) {
    const FeSeq& q = seqs[blockIdx.y];
    if (!q.detect) return;
    const size_t n16 = (size_t)rows * cols / 16, total = (size_t)rows * cols;
    uint4* m16 = reinterpret_cast<uint4*>(q.mask);
    const uint4* s16 = reinterpret_cast<const uint4*>(q.mask_init);
    const size_t stride = (size_t)gridDim.x * blockDim.x, i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    for (size_t i = i0; i < n16; i += stride) m16[i] = s16 ? s16[i] : make_uint4(~0u, ~0u, ~0u, ~0u);
    for (size_t i = n16 * 16 + i0; i < total; i += stride) q.mask[i] = q.mask_init ? q.mask_init[i] : (uint8_t)255;
    if (i0 == 0) {
        q.count[FE_COUNT_CANDIDATES] = 0;
        q.count[FE_COUNT_SELECTED] = 0;
        *q.maxv = 0u;
    }
}

__global__ void __launch_bounds__(128) mask_discs_kernel(const FeSeq* __restrict__ seqs, int rows, int cols, int radius,
                                                         const int* __restrict__ halfw) {
    const FeSeq& q = seqs[blockIdx.y];
    const int c = blockIdx.x;
    if (!q.detect || c >= q.n_centres) return;
    uint8_t* __restrict__ mask = q.mask;
    const int pitch = cols;
    const int* __restrict__ centres = q.centres;
    const int cx = centres[2 * c], cy = centres[2 * c + 1];
    const int side = 2 * radius + 1;
    for (int i = threadIdx.x; i < side * side; i += blockDim.x) {
        const int dy = i / side - radius, dx = i % side - radius;
        const int y = cy + dy, x = cx + dx;
        if (y < 0 || y >= rows || x < 0 || x >= cols) continue;
        if (abs(dx) <= halfw[abs(dy)]) mask[(size_t)y * pitch + x] = 0;
    }
}

// ---------------------------------------------------------------------------------------------
// Shi-Tomasi min-eigenvalue map (cornerMinEigenVal, blockSize 3, Sobel 3) + masked global max.
// 32x16 output tile per CTA; image tile with a 2-pixel halo in shared memory; Sobel products for the
// (tile+1 ring) positions are evaluated at reflect-101 *positions* (the box filter mirrors the
// derivative images, not the source).  Box sums in double exactly like OpenCV's CV_64F sum type.
#define ME_TW 32
#define ME_TH 16

__device__ __forceinline__ unsigned f32_sortable(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(ME_TW* ME_TH) min_eig_kernel(const FeSeq* __restrict__ seqs, int rows, int cols, float k1, float k2) {
    const FeSeq& q = seqs[blockIdx.z];
    if (!q.detect) return;
    const uint8_t* __restrict__ img = q.det_img;
    const int pitch = q.det_pitch;
    const uint8_t* __restrict__ mask = q.use_mask ? q.mask : nullptr;
    const int mpitch = cols, epitch = cols;
    float* __restrict__ eig = q.eig;
    unsigned* __restrict__ max_sortable = q.maxv;
    __shared__ uint8_t tile[(ME_TH + 4) * (ME_TW + 4)];
    // the derivative products are staged already widened to double (the box filter sums them in double like OpenCV's CV_64F
    // sum type): one conversion per staged element instead of nine per output pixel
    __shared__ double sxx[(ME_TH + 2) * (ME_TW + 2)], sxy[(ME_TH + 2) * (ME_TW + 2)], syy[(ME_TH + 2) * (ME_TW + 2)];
    __shared__ unsigned wmax[ME_TW * ME_TH / 32];
    const int tx0 = blockIdx.x * ME_TW, ty0 = blockIdx.y * ME_TH;
    const int tid = threadIdx.y * ME_TW + threadIdx.x;
    const int TWP = ME_TW + 4;
    // tile index (j,i) <-> image coordinate (ty0-2+j, tx0-2+i), stored value = img at reflect-101 coordinate
    for (int i = tid; i < (ME_TH + 4) * TWP; i += ME_TW * ME_TH) {
        const int j = i / TWP, ii = i - j * TWP;
        tile[i] = img[(size_t)reflect101(ty0 - 2 + j, rows) * pitch + reflect101(tx0 - 2 + ii, cols)];
    }
    __syncthreads();
    const int DW = ME_TW + 2;
    for (int i = tid; i < (ME_TH + 2) * DW; i += ME_TW * ME_TH) {
        const int j = i / DW, ii = i - j * DW;
        // derivative position p = (ty0-1+j, tx0-1+ii); evaluate Sobel at q = reflect101(p)
        if (ty0 - 1 + j > rows || tx0 - 1 + ii > cols) {  // beyond the 1-pixel ring of the image: unused
            sxx[i] = sxy[i] = syy[i] = 0.0;
            continue;
        }
        const int qy = reflect101(ty0 - 1 + j, rows), qx = reflect101(tx0 - 1 + ii, cols);
        // neighbours of q, reflected on the image, then mapped to tile indices
        const int ym = reflect101(qy - 1, rows) - (ty0 - 2), y0 = qy - (ty0 - 2), yp = reflect101(qy + 1, rows) - (ty0 - 2);
        const int xm = reflect101(qx - 1, cols) - (tx0 - 2), x0 = qx - (tx0 - 2), xp = reflect101(qx + 1, cols) - (tx0 - 2);
        const float pmm = tile[ym * TWP + xm], pm0 = tile[ym * TWP + x0], pmp = tile[ym * TWP + xp];
        const float p0m = tile[y0 * TWP + xm], p0p = tile[y0 * TWP + xp];
        const float ppm = tile[yp * TWP + xm], pp0 = tile[yp * TWP + x0], ppp = tile[yp * TWP + xp];
        // Sobel dx: rows [-1 0 1] exact, then column [k1 k2 k1] as  k2*r0 + k1*(r- + r+)
        const float rm = __fsub_rn(pmp, pmm), r0 = __fsub_rn(p0p, p0m), rp = __fsub_rn(ppp, ppm);
        const float gx = __fadd_rn(__fmul_rn(k2, r0), __fmul_rn(k1, __fadd_rn(rm, rp)));
        // Sobel dy: rows [k1 k2 k1] tap by tap (k1*a + k2*b) + k1*c, then column difference
        const float sm_ = __fadd_rn(__fadd_rn(__fmul_rn(k1, pmm), __fmul_rn(k2, pm0)), __fmul_rn(k1, pmp));
        const float sp_ = __fadd_rn(__fadd_rn(__fmul_rn(k1, ppm), __fmul_rn(k2, pp0)), __fmul_rn(k1, ppp));
        const float gy = __fsub_rn(sp_, sm_);
        sxx[i] = (double)__fmul_rn(gx, gx);
        sxy[i] = (double)__fmul_rn(gx, gy);
        syy[i] = (double)__fmul_rn(gy, gy);
    }
    __syncthreads();
    const int x = tx0 + threadIdx.x, y = ty0 + threadIdx.y;
    unsigned key = 0;  // sortable encoding of -inf side: 0 is below every real float
    if (x < cols && y < rows) {
        double sa = 0, sb = 0, sc = 0;
#pragma unroll
        for (int j = 0; j < 3; j++) {
            const int o = (threadIdx.y + j) * DW + threadIdx.x;
            const double ra = __dadd_rn(__dadd_rn(sxx[o], sxx[o + 1]), sxx[o + 2]);
            const double rb = __dadd_rn(__dadd_rn(sxy[o], sxy[o + 1]), sxy[o + 2]);
            const double rc = __dadd_rn(__dadd_rn(syy[o], syy[o + 1]), syy[o + 2]);
            sa = __dadd_rn(sa, ra);
            sb = __dadd_rn(sb, rb);
            sc = __dadd_rn(sc, rc);
        }
        const float a = __fmul_rn((float)sa, 0.5f), b = (float)sb, c = __fmul_rn((float)sc, 0.5f);
        const float d = __fsub_rn(a, c);
        const float e = __fsub_rn(__fadd_rn(a, c), __fsqrt_rn(__fadd_rn(__fmul_rn(d, d), __fmul_rn(b, b))));
        eig[(size_t)y * epitch + x] = e;
        if (!mask || mask[(size_t)y * mpitch + x]) key = f32_sortable(e);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
    if ((tid & 31) == 0) wmax[tid >> 5] = key;
    __syncthreads();
    if (tid == 0) {
        unsigned m = 0;
        for (int w = 0; w < ME_TW * ME_TH / 32; w++) m = max(m, wmax[w]);
        if (m) atomicMax(max_sortable, m);
    }
}

// Candidate collection: interior pixels with thresholded eig != 0, equal to the 3x3 max of the
// thresholded map, and mask != 0.  Key = (eig bits << 32) | linear offset: eig > thr >= 0 so the float
// bit pattern orders like the value; ties resolve on the larger offset first (greaterThanPtr).
__global__ void __launch_bounds__(256) gftt_candidates_kernel(const FeSeq* __restrict__ seqs, int rows, int cols, double quality,
                                                              int capacity) {
    const FeSeq& q = seqs[blockIdx.z];
    if (!q.detect) return;
    const float* __restrict__ eig = q.eig;
    const int epitch = cols, mpitch = cols;
    const uint8_t* __restrict__ mask = q.use_mask ? q.mask : nullptr;
    const unsigned* __restrict__ max_sortable = q.maxv;
    unsigned long long* __restrict__ keys = q.keys;
    int* __restrict__ count = q.count + FE_COUNT_CANDIDATES;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x < 1 || y < 1 || x >= cols - 1 || y >= rows - 1) return;
    const unsigned ms = *max_sortable;
    float max_val = 0.f;
    if (ms) max_val = __uint_as_float((ms & 0x80000000u) ? (ms & 0x7fffffffu) : ~ms);
    const float thr = (float)__dmul_rn((double)max_val, quality);
    const float v = eig[(size_t)y * epitch + x];
    if (!(v > thr) || v == 0.f) return;
    if (mask && !mask[(size_t)y * mpitch + x]) return;
    float m = v;
#pragma unroll
    for (int j = -1; j <= 1; j++)
#pragma unroll
        for (int i = -1; i <= 1; i++) {
            float w = eig[(size_t)(y + j) * epitch + (x + i)];
            w = w > thr ? w : 0.f;
            m = fmaxf(m, w);
        }
    if (v != m) return;
    const int slot = atomicAdd(count, 1);
    if (slot < capacity)
        keys[slot] = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned)(y * cols + x);
}

// Descending bitonic sort of the candidate keys by one CTA; keys live in shared memory when they fit.
__global__ void __launch_bounds__(1024) sort_keys_desc_kernel(const FeSeq* __restrict__ seqs, int capacity) {
    extern __shared__ unsigned long long sk[];
    const FeSeq& q = seqs[blockIdx.x];
    if (!q.detect) return;
    unsigned long long* __restrict__ keys = q.keys;
    const int* __restrict__ count = q.count + FE_COUNT_CANDIDATES;
    int n = min(*count, capacity);
    int npad = 1;
    while (npad < n) npad <<= 1;
    if (npad < 2) return;
    const bool in_smem = npad <= SORT_SMEM_KEYS;
    unsigned long long* a = in_smem ? sk : keys;
    if (in_smem) {
        for (int i = threadIdx.x; i < npad; i += blockDim.x) sk[i] = i < n ? keys[i] : 0ull;
    } else {
        for (int i = n + threadIdx.x; i < npad; i += blockDim.x) keys[i] = 0ull;  // capacity is a power of two
    }
    __syncthreads();
    for (int k = 2; k <= npad; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < npad; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long x = a[i], y = a[l];
                    const bool desc = (i & k) == 0;
                    if (desc ? (x < y) : (x > y)) {
                        a[i] = y;
                        a[l] = x;
                    }
                }
            }
            __syncthreads();
        }
    if (in_smem)
        for (int i = threadIdx.x; i < n; i += blockDim.x) keys[i] = sk[i];
}

// Greedy minimum-distance selection over the sorted candidates (goodFeaturesToTrack tail), one warp.
// 32 candidates at a time: each lane tests its candidate against the corners already kept (3x3 cells
// of a cell_size grid), then the batch is resolved in priority order with shuffles, so the result is
// exactly the sequential greedy scan.
#define SEL_CELL_CAP 8
__global__ void __launch_bounds__(32) gftt_select_kernel(const FeSeq* __restrict__ seqs, int capacity, int cols, int rows,
                                                         float min_dist, int cell, int gw, int gh) {
    const FeSeq& q = seqs[blockIdx.x];
    if (!q.detect) return;
    const unsigned long long* __restrict__ keys = q.keys;
    const int* __restrict__ count = q.count + FE_COUNT_CANDIDATES;
    const int max_corners = q.max_corners;
    int* __restrict__ cell_cnt = q.cell_cnt;
    short2* __restrict__ cell_pts = q.cell_pts;
    float* __restrict__ out_pts = q.new_pts;
    int* __restrict__ out_n = q.count + FE_COUNT_SELECTED;
    const int lane = threadIdx.x;
    const int n = min(*count, capacity);
    for (int i = lane; i < gw * gh; i += 32) cell_cnt[i] = 0;
    __syncwarp();
    const float md2 = __fmul_rn(min_dist, min_dist);
    int kept = 0;
    for (int base = 0; base < n && kept < max_corners; base += 32) {
        const int idx = base + lane;
        int x = 0, y = 0, xc = 0, yc = 0;
        bool good = idx < n;
        if (good) {
            const unsigned off = (unsigned)(keys[idx] & 0xffffffffull);
            y = off / cols;
            x = off - y * cols;
            xc = x / cell;
            yc = y / cell;
            const int x1 = max(0, xc - 1), y1 = max(0, yc - 1), x2 = min(gw - 1, xc + 1), y2 = min(gh - 1, yc + 1);
            for (int yy = y1; yy <= y2 && good; yy++)
                for (int xx = x1; xx <= x2 && good; xx++) {
                    const int c = yy * gw + xx, m = cell_cnt[c];
                    for (int k = 0; k < m; k++) {
                        const short2 q = cell_pts[c * SEL_CELL_CAP + k];
                        const float dx = (float)(x - q.x), dy = (float)(y - q.y);
                        if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < md2) {
                            good = false;
                            break;
                        }
                    }
                }
        }
        // resolve inside the batch, in order
        unsigned alive = __ballot_sync(0xffffffffu, good);
        for (int i = 0; i < 32; i++) {
            if (!((alive >> i) & 1u)) continue;  // uniform
            const int xi = __shfl_sync(0xffffffffu, x, i), yi = __shfl_sync(0xffffffffu, y, i);
            if (lane > i && good) {
                const float dx = (float)(x - xi), dy = (float)(y - yi);
                if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) < md2) good = false;
            }
            alive = __ballot_sync(0xffffffffu, good);
        }
        // append survivors in lane order, cut at max_corners
        const int rank = __popc(alive & ((1u << lane) - 1u));
        if (good && kept + rank < max_corners) {
            const int c = yc * gw + xc;
            const int slot = atomicAdd(&cell_cnt[c], 1);
            if (slot < SEL_CELL_CAP) cell_pts[c * SEL_CELL_CAP + slot] = make_short2((short)x, (short)y);
            out_pts[2 * (kept + rank)] = (float)x;
            out_pts[2 * (kept + rank) + 1] = (float)y;
        }
        kept = min(max_corners, kept + __popc(alive));
        __syncwarp();
    }
    if (lane == 0) *out_n = kept;
}

// ---------------------------------------------------------------------------------------------
// launch wrappers: one launch per stage for the whole batch (member = last grid dimension)
void launch_track(const FeSeq* seqs, const FeShape& sh, cudaStream_t s, int* launches, KernelProfile* prof) {
    KernelProfile none;
    if (!prof) prof = &none;
    if (!sh.any_track) return;
    const int rows = sh.rows, cols = sh.cols;
    int n = 0;
    prof->begin(s);
    if (sh.any_equalize) {
        const int tiles_x = 8, tiles_y = 8;
        int ext_rows = rows, ext_cols = cols;
        if (cols % tiles_x != 0 || rows % tiles_y != 0) {
            ext_rows = rows + (tiles_y - rows % tiles_y);
            ext_cols = cols + (tiles_x - cols % tiles_x);
        }
        const int tw = ext_cols / tiles_x, th = ext_rows / tiles_y, area = tw * th;
        const float lut_scale = 255.f / (float)area;
        int clip = (int)(3.0 * area / 256);
        clip = clip < 1 ? 1 : clip;
        clahe_lut_kernel<<<dim3(tiles_x * tiles_y, sh.S), 256, 0, s>>>(seqs, rows, cols, tiles_x, tw, th, clip, lut_scale);
        clahe_apply_kernel<<<dim3((cols + 4 * 256 - 1) / (4 * 256), rows, sh.S), 256, 0, s>>>(seqs, rows, cols, tiles_x, tiles_y,
                                                                                               1.0f / tw, 1.0f / th);
        n += 2;
    } else {
        clahe_apply_kernel<<<dim3((cols + 4 * 256 - 1) / (4 * 256), rows, sh.S), 256, 0, s>>>(seqs, rows, cols, 8, 8, 1.f, 1.f);
        n += 1;
    }
    prof->end(0, s, n);
    prof->begin(s);
    int r = rows, c = cols;
    for (int l = 1; l <= sh.nlev; l++) {
        r = (r + 1) / 2;
        c = (c + 1) / 2;
        pyrdown_kernel<<<dim3((c + 31) / 32, (r + 7) / 8, sh.S), dim3(32, 8), 0, s>>>(seqs, l, 0);
        n++;
    }
    prof->end(1, s, sh.nlev);
    if (sh.max_pts > 0) {
        const double eps = 0.01;
        prof->begin(s);
        lk_track_kernel<<<dim3(sh.max_pts, sh.S), 32 * LK_WARPS, 0, s>>>(seqs, 30, eps * eps, 1e-4f);
        prof->end(2, s);
        n++;
    }
    if (launches) *launches += n;
}

void launch_pyramid_only(const FeSeq* seqs, const FeShape& sh, int use_cur, cudaStream_t s) {
    int r = sh.rows, c = sh.cols;
    for (int l = 1; l <= sh.nlev; l++) {
        r = (r + 1) / 2;
        c = (c + 1) / 2;
        pyrdown_kernel<<<dim3((c + 31) / 32, (r + 7) / 8, sh.S), dim3(32, 8), 0, s>>>(seqs, l, use_cur);
    }
}

void launch_lk_only(const FeSeq* seqs, const FeShape& sh, cudaStream_t s) {
    if (sh.max_pts <= 0) return;
    const double eps = 0.01;
    lk_track_kernel<<<dim3(sh.max_pts, sh.S), 32 * LK_WARPS, 0, s>>>(seqs, 30, eps * eps, 1e-4f);
}

void launch_detect(const FeSeq* seqs, const FeShape& sh, const int* halfw, cudaStream_t s, int* launches, KernelProfile* prof) {
    KernelProfile none;
    if (!prof) prof = &none;
    if (!sh.any_detect) return;
    const int rows = sh.rows, cols = sh.cols;
    int n = 0;
    prof->begin(s);
    mask_init_kernel<<<dim3(32, sh.S), 256, 0, s>>>(seqs, rows, cols);
    n++;
    if (sh.max_centres > 0) {
        mask_discs_kernel<<<dim3(sh.max_centres, sh.S), 128, 0, s>>>(seqs, rows, cols, sh.min_dist, halfw);
        n++;
    }
    prof->end(3, s, n);
    const double scale = 1.0 / ((double)(1 << 2) * 3 * 255.0);
    prof->begin(s);
    min_eig_kernel<<<dim3((cols + ME_TW - 1) / ME_TW, (rows + ME_TH - 1) / ME_TH, sh.S), dim3(ME_TW, ME_TH), 0, s>>>(
        seqs, rows, cols, (float)scale, (float)(2.0 * scale));
    prof->end(4, s);
    prof->begin(s);
    gftt_candidates_kernel<<<dim3((cols + 31) / 32, (rows + 7) / 8, sh.S), dim3(32, 8), 0, s>>>(seqs, rows, cols, 0.01, sh.key_capacity);
    raise_dynamic_smem((const void*)sort_keys_desc_kernel, SORT_SMEM_KEYS * (int)sizeof(unsigned long long));
    sort_keys_desc_kernel<<<sh.S, 1024, SORT_SMEM_KEYS * sizeof(unsigned long long), s>>>(seqs, sh.key_capacity);
    const int cell = (int)lrint((double)sh.min_dist);
    const int gw = (cols + cell - 1) / cell, gh = (rows + cell - 1) / cell;
    gftt_select_kernel<<<sh.S, 32, 0, s>>>(seqs, sh.key_capacity, cols, rows, (float)sh.min_dist, cell, gw, gh);
    prof->end(5, s, 3);
    n += 4;
    if (launches) *launches += n;
}

}  // namespace vb
