// Internal launch interface of the front-end kernels (fe_kernels.cu).  Every launch serves a whole batch: `seqs` is a
// device array of per-member descriptors, the member index is the last grid dimension (a stand-alone tracker is a batch
// of one).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "kprof.h"

namespace vb {

constexpr int MAX_PYR_LEVELS = 5;
constexpr int SORT_SMEM_KEYS = 16384;  // 128 KB of 64-bit candidate keys sorted inside one CTA's shared memory
// A member's counter slot (FeSeq::count, FE_COUNT_SLOT ints): Shi-Tomasi candidates found, corners selected, and the
// maximum of the min-eigenvalue map as a sortable unsigned (FeSeq::maxv points at it)
enum : int { FE_COUNT_CANDIDATES = 0, FE_COUNT_SELECTED = 1, FE_COUNT_MAXV = 2, FE_COUNT_SLOT = 4 };

struct PyramidView {
    const uint8_t* img[MAX_PYR_LEVELS];
    int rows[MAX_PYR_LEVELS], cols[MAX_PYR_LEVELS], pitch[MAX_PYR_LEVELS];
    int nlev;  // index of the coarsest level (levels 0..nlev)
};

struct FeSeq {  // one member's work of one image step
    int track;         // build the forw pyramid from `raw` and track n_pts points cur -> forw
    int detect;        // setMask discs + goodFeaturesToTrack on det_img
    int equalize;      // CLAHE (EQUALIZE), else level 0 = raw
    int raw_pitch;
    const uint8_t* raw;   // the new frame (device memory)
    uint8_t* lut;         // 64 x 256 CLAHE tile LUTs
    PyramidView cur, forw;
    int n_pts, use_mask;
    const float* pts_in;  // n_pts x 2
    float* pts_out;
    uint8_t* status;
    // detection
    const uint8_t* det_img;  // level 0 of the forw pyramid (or a raw frame for the test entry)
    int det_pitch, n_centres;
    uint8_t* mask;           // rows x cols
    const uint8_t* mask_init;// fisheye mask or null (255)
    const int* centres;      // n_centres x 2 kept tracks (rounded)
    float* eig;
    unsigned long long* keys;
    int* count;              // counter slot: [FE_COUNT_CANDIDATES], [FE_COUNT_SELECTED]
    unsigned* maxv;          // count + FE_COUNT_MAXV
    int* cell_cnt;
    short2* cell_pts;
    float* new_pts;          // max_corners x 2
    int max_corners, pad;
};

struct FeShape {
    int S, rows, cols, nlev;
    int max_pts, max_centres;
    int any_track, any_detect, any_equalize;
    int min_dist, key_capacity;
};

// profile slots: 0 clahe (lut + apply), 1 pyrdown, 2 lk_track, 3 mask, 4 min_eig, 5 candidates + sort + select
void launch_track(const FeSeq* seqs, const FeShape& sh, cudaStream_t s, int* launches, KernelProfile* prof = nullptr);
void launch_detect(const FeSeq* seqs, const FeShape& sh, const int* halfw, cudaStream_t s, int* launches, KernelProfile* prof = nullptr);
// test entries
void launch_pyramid_only(const FeSeq* seqs, const FeShape& sh, int use_cur, cudaStream_t s);
void launch_lk_only(const FeSeq* seqs, const FeShape& sh, cudaStream_t s);

}  // namespace vb
