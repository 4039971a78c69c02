// Layouts of the packed buffers of the 4-DoF pose-graph solver (pg_kernels.cu, pose_graph.cpp): the batch input arena
// (one host-to-device copy per launch), a member's input block inside it, the output arena (one device-to-host copy) and
// the per-member device workspace.  Each layout is defined here once, as offsets computed from the sizes it depends on;
// whatever sizes, carves, writes or reads one of these buffers goes through it.  Host and device code share it;
// tests/hostlib/pg_layout_host.cpp checks it with g++.
#pragma once
#include <cstddef>

#include "ba_types.h"

#ifdef __CUDACC__
#define PG_LAYOUT_FN __host__ __device__ constexpr inline
#else
#define PG_LAYOUT_FN constexpr inline
#endif

namespace vb {

// The border (the dense Schur complement of the loop anchors) has 4 columns per free anchor.  Borders of at most PG_MAX_D
// columns (the BA step's dense system size) are factored in one CTA in shared memory; larger ones by the multi-CTA
// path in global memory (tile storage, PG_TILE x PG_TILE tiles).  A graph's anchor capacity (vp_config::max_anchors)
// is PG_MAX_ANCHORS by default and at most PG_CAP_ANCHORS.
constexpr int PG_MAX_D = BA_MAX_D;
constexpr int PG_MAX_ANCHORS = PG_MAX_D / 4;
constexpr int PG_CAP_ANCHORS = 1024;
constexpr int PG_TILE = 64;
// Super-blocks of the chain: 4 consecutive key frames, 16 unknowns.
constexpr int PG_SB = 4, PG_SBD = 16;
// Per key frame of the assembled normal equations: diagonal block | 4 blocks to the key frames 1..4 back | loop block.
constexpr int PG_BLK = 16, PG_BLK_DIAG = 0, PG_BLK_BACK = 16, PG_BLK_LOOP = 80, PG_BLK_KF = 96;
// Solver summary at the end of a member's output block (doubles):
//   iterations, successful steps, initial cost, final cost, converged, border columns, key frames,
//   largest gradient component at the last linearisation
constexpr int PG_SUMMARY = 8;

PG_LAYOUT_FN size_t pg_align16(size_t bytes) { return (bytes + 15) & ~(size_t)15; }
PG_LAYOUT_FN int pg_num_sb(int n) { return (n + PG_SB - 1) / PG_SB; }

// ---- a member's input block, in bytes, every array 16-byte aligned:
//      VIO pose n x 7 (t, q wxyz) | loop measurement n x 4 (t, yaw) | sequence n | loop target (local, -1) n |
//      border slot (-1 when not a free anchor) n | first loop edge into the key frame (its source, -1) n |
//      next loop edge into the same anchor (source, -1) n | anchor key frames nb (local index, ascending)
struct PgInLayout {
    size_t pose, loop, seq, loop_idx, bslot, lfirst, lnext, anchors, total;
};
PG_LAYOUT_FN PgInLayout pg_in_layout(int n, int nb) {
    PgInLayout o{0, 0, 0, 0, 0, 0, 0, 0, 0};
    o.loop = pg_align16((size_t)7 * n * sizeof(double));
    o.seq = o.loop + pg_align16((size_t)4 * n * sizeof(double));
    o.loop_idx = o.seq + pg_align16((size_t)n * sizeof(int));
    o.bslot = o.loop_idx + pg_align16((size_t)n * sizeof(int));
    o.lfirst = o.bslot + pg_align16((size_t)n * sizeof(int));
    o.lnext = o.lfirst + pg_align16((size_t)n * sizeof(int));
    o.anchors = o.lnext + pg_align16((size_t)n * sizeof(int));
    o.total = o.anchors + pg_align16((size_t)nb * sizeof(int));
    return o;
}

// ---- the batch input arena of one launch, in bytes: header | member blocks.  The header lists, per active slot b
//      (grid.y of every kernel), the member index, n, nb, the byte / double offsets of its input and output blocks and
//      nc, the number of constant key frames (local 0 .. nc - 1; every other key frame is free).
struct PgHdrLayout {
    size_t member, n, nb, in_off, out_off, nc, total;
};
PG_LAYOUT_FN PgHdrLayout pg_hdr_layout(int S) {
    PgHdrLayout o{0, 0, 0, 0, 0, 0, 0};
    o.member = pg_align16(sizeof(int));  // [0] = number of active slots
    o.n = o.member + pg_align16((size_t)S * sizeof(int));
    o.nb = o.n + pg_align16((size_t)S * sizeof(int));
    o.in_off = o.nb + pg_align16((size_t)S * sizeof(int));
    o.out_off = o.in_off + pg_align16((size_t)S * sizeof(long long));
    o.nc = o.out_off + pg_align16((size_t)S * sizeof(long long));
    o.total = o.nc + pg_align16((size_t)S * sizeof(int));
    return o;
}
// bytes of the arena: the header plus every member at capacity
PG_LAYOUT_FN size_t pg_arena_bytes(int S, int cap_n, int cap_anchors = PG_MAX_ANCHORS) {
    return pg_hdr_layout(S).total + (size_t)S * pg_in_layout(cap_n, cap_anchors).total;
}

// ---- a member's output block, in doubles: yaw (degrees) and t per key frame of the range (n x 4) | summary.
//      An even count, so consecutive blocks stay 16-byte aligned.
struct PgOutLayout {
    size_t x, summary, total;
};
PG_LAYOUT_FN PgOutLayout pg_out_layout(int n) {
    return PgOutLayout{0, (size_t)4 * n, (((size_t)4 * n + PG_SUMMARY) + 1) & ~(size_t)1};
}

// ---- solver state of a member (in its workspace): written by the setup kernel, advanced by the update kernel
struct PgState {
    double radius, decrease, cost, cost0, cost_c, model_change, xnorm, gmax;
    int iter, successful, need_lin, first, done, converged, step_ok, lin_fail;
};
constexpr int PG_STATE_DOUBLES = (int)((sizeof(PgState) + sizeof(double) - 1) / sizeof(double));

// ---- a member's device workspace at capacity cap_n key frames and cap_anchors free anchors, in doubles.  W (the chain's
//      border columns L^-1 B and L^-1 r as column D) has (D + 1) columns at run time; it is sized for the capacity and
//      also holds the linearisation's edge scratch (180 doubles per key frame).  Sp is the packed border system of the
//      one-CTA path (D <= PG_MAX_D).  U and yb exist only when the capacity exceeds PG_MAX_D columns: U is the border
//      system [S z] of the multi-CTA path, its upper triangle in a Np x Np row-major square (Np = D + 1 rounded up to
//      PG_TILE, z in column D), factored in place except for its diagonal tiles, whose factors go to Ud (one
//      PG_TILE x PG_TILE tile per panel, stacked); yb is the border part of the step.  These are 16-byte aligned.
struct PgWorkLayout {
    size_t state, x, xc, dx, scale, ypr, smeas, blk, g, L, F, W, start, Sp, U, Ud, yb, total;
};
PG_LAYOUT_FN size_t pg_max_sz(size_t a, size_t b) { return a > b ? a : b; }
PG_LAYOUT_FN size_t pg_even(size_t d) { return (d + 1) & ~(size_t)1; }
// columns of the square holding U for a border of D columns (0 on the one-CTA path)
PG_LAYOUT_FN int pg_tile_np(int D) { return D > PG_MAX_D ? (D + 1 + PG_TILE - 1) / PG_TILE * PG_TILE : 0; }
PG_LAYOUT_FN PgWorkLayout pg_work_layout(int cap_n, int cap_anchors = PG_MAX_ANCHORS) {
    const size_t n = (size_t)cap_n, nsb = (size_t)pg_num_sb(cap_n), D = 4 * (size_t)cap_anchors, Dp = D + 1;
    const size_t Dps = (D < (size_t)PG_MAX_D ? D : (size_t)PG_MAX_D) + 1, Np = (size_t)pg_tile_np((int)D);
    PgWorkLayout o{};
    o.state = 0;
    o.x = (PG_STATE_DOUBLES + 1) & ~1;
    o.xc = o.x + 4 * n;                                   // candidate point
    o.dx = o.xc + 4 * n;                                  // step (unscaled)
    o.scale = o.dx + 4 * n;                               // Jacobi scaling
    o.ypr = o.scale + 4 * n;                              // yaw, pitch, roll of the VIO pose (degrees)
    o.smeas = o.ypr + 3 * n;                              // sequential-edge measurements: 4 edges x (t, yaw)
    o.blk = o.smeas + 16 * n;                             // assembled blocks, PG_BLK_KF per key frame
    o.g = o.blk + (size_t)PG_BLK_KF * n;                  // gradient (scaled)
    o.L = o.g + 4 * n;                                    // chain factor: 16 x 16 per super-block
    o.F = o.L + 256 * nsb;                                // chain off-diagonal factor blocks
    o.W = o.F + 256 * nsb;                                // 16 nsb x (D + 1), row-major
    o.start = o.W + pg_max_sz(16 * nsb * Dp, 180 * n);    // first super-block of each W column (ints, Dp of them)
    o.Sp = o.start + (((Dp + 1) / 2 + 1) & ~(size_t)1);   // packed border system (D + 1 rows: S | z)
    o.U = pg_even(o.Sp + ((Dps * (Dps + 1) / 2 + 1) & ~(size_t)1));
    o.Ud = o.U + Np * Np;
    o.yb = o.Ud + Np * PG_TILE;
    o.total = o.yb + (Np ? pg_even(D) : 0);
    return o;
}

}  // namespace vb
