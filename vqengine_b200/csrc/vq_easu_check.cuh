// vq_easu_check.cuh — which EASU kernel vq_fsr_easu launches, and whether its constants keep every tap inside what that
// kernel can address. Host code only: vq_post.cu calls it before any launch, and tests/host_check/easu_check_host.cpp builds
// the same source with g++ so that tests/test_post_domain.py sweeps it on the CPU.
//
// The kernels place output pixel o of an axis at easu_pos(o) = fl(fl(o * scale) + bias), take 'f' = floor(easu_pos(o)) and
// read the 12 texels f-1 .. f+2. fl(o * scale) and fl(. + bias) are monotone in o, so floor(easu_pos(0)) and
// floor(easu_pos(out - 1)) bound 'f' over the whole axis. Constants are refused when
//   * any of con0 is not finite;
//   * a tap leaves [-W, 2W) x [-H, 2H), W = max(in.width, 3), H = max(in.height, 3): load_addr's WRAP folds a tap back into
//     the image with one add or subtract, which is right only in that range (images under 3 texels use the general % and
//     any tap in the range);
//   * the up path (0 < scale <= 1 on both axes, not the exact 2x) would need more candidate 'f' texels per 32 x 8 output tile
//     than its shared-memory arrays hold (ncx > 32 or ncy > 8). The fused post kernel (vq_post_process) runs the up path on
//     its 30 x 14 display tiles widened by RCAS's 1-pixel ring and holds 32 x 16 candidates: check(..., FUSED_UP_TILE).
// Every con0 that FsrEasuCon builds for the image (viewport <= input size) passes: its taps lie in [-2, width + 1].
#pragma once
#include <math.h>

namespace vqeasu {

enum Path { EASU_GENERIC = 0, EASU_UP = 1, EASU_2X = 2 };
enum Verdict { EASU_OK = 0, EASU_NONFINITE = 1, EASU_TAPS_OUTSIDE = 2, EASU_TILE_FOOTPRINT = 3 };
constexpr int UP_TILE_X = 32, UP_TILE_Y = 8;   // easu_up_kernel's output tile and its candidate-texel capacity

// The up path's output tiles along x and y, the ring of extra outputs EASU computes around each (clipped to the output), and
// the candidate 'f' texels the kernel can hold per widened tile
struct UpTile { int x, y, ring, cap_x, cap_y; };
constexpr UpTile EASU_UP_TILE = {UP_TILE_X, UP_TILE_Y, 0, UP_TILE_X, UP_TILE_Y};   // easu_up_kernel
constexpr UpTile FUSED_UP_TILE = {30, 14, 1, 32, 16};                              // post_fsr_up_kernel (vq_post.cu)

// the kernels' easu_pos (__fmul_rn then __fadd_rn); the product goes through a volatile so that no host compiler fuses it
inline float pos(int o, float scale, float bias) {
    volatile float p = (float)o * scale;
    return p + bias;
}

inline Path path(const float c[4], int in_w, int in_h, int out_w, int out_h) {
    if (c[0] == 0.5f && c[1] == 0.5f && c[2] == -0.25f && c[3] == -0.25f && out_w == 2 * in_w && out_h == 2 * in_h) return EASU_2X;
    if (c[0] > 0.0f && c[1] > 0.0f && c[0] <= 1.0f && c[1] <= 1.0f) return EASU_UP;
    return EASU_GENERIC;
}

// largest number of candidate 'f' texels over the up path's tiles of `tile` outputs along one axis, each widened by `ring`
// outputs on both sides and clipped to [0, n_out)
inline int max_candidates(float scale, float bias, int n_out, int tile, int ring = 0) {
    int worst = 0;
    for (int o0 = 0; o0 < n_out; o0 += tile) {
        const int of = o0 - ring > 0 ? o0 - ring : 0;
        const int ol = o0 + tile - 1 + ring < n_out - 1 ? o0 + tile - 1 + ring : n_out - 1;
        const int n = (int)floorf(pos(ol, scale, bias)) - (int)floorf(pos(of, scale, bias)) + 1;
        worst = n > worst ? n : worst;
    }
    return worst;
}

// 'f' of the first and last output along one axis inside [-size + 1, 2 * size - 3], size = max(texels, 3).
// Deliberately the same rule for both address modes: CLAMP could take any finite tap, but constants that land outside this
// range were not built for these images under either mode, and one rule keeps the contract in vqcuda.h mode-independent.
inline bool axis_ok(float scale, float bias, int n_in, int n_out) {
    const double size = n_in > 3 ? n_in : 3;
    const double f0 = floor((double)pos(0, scale, bias)), f1 = floor((double)pos(n_out - 1, scale, bias));
    const double lo = (f0 < f1 ? f0 : f1) - 1.0, hi = (f0 < f1 ? f1 : f0) + 2.0;
    return lo >= -size && hi < 2.0 * size;
}

// c = con0 (scale x, scale y, bias x, bias y); ncx / ncy (may be null) receive the up path's largest tile footprint, 0 elsewhere;
// `tile` is the up path's tiling (easu_up_kernel's unless given)
inline Verdict check(const float c[4], int in_w, int in_h, int out_w, int out_h, int* ncx = nullptr, int* ncy = nullptr,
                     const UpTile& tile = EASU_UP_TILE) {
    if (ncx) *ncx = 0;
    if (ncy) *ncy = 0;
    for (int i = 0; i < 4; ++i)
        if (!isfinite(c[i])) return EASU_NONFINITE;
    if (!axis_ok(c[0], c[2], in_w, out_w) || !axis_ok(c[1], c[3], in_h, out_h)) return EASU_TAPS_OUTSIDE;
    if (path(c, in_w, in_h, out_w, out_h) != EASU_UP) return EASU_OK;
    const int nx = max_candidates(c[0], c[2], out_w, tile.x, tile.ring), ny = max_candidates(c[1], c[3], out_h, tile.y, tile.ring);
    if (ncx) *ncx = nx;
    if (ncy) *ncy = ny;
    return nx <= tile.cap_x && ny <= tile.cap_y ? EASU_OK : EASU_TILE_FOOTPRINT;
}

// The input rows the kernels read for output rows [rb, re) of an axis that axis_ok accepts: the taps f-1 .. f+2 of every
// 'f' = floor(pos(y)), folded into [0, n_in) as load_addr folds them (wrap: modulo n_in; otherwise clamped), as up to two
// increasing, disjoint, non-adjacent [begin, end) ranges in r[0..3]. Returns their count (0 for an empty range).
// 'f' is monotone in y, so the taps span [min f - 1, max f + 2] with f at rb and re - 1; every row of that span is read when
// consecutive outputs' 'f' differ by at most 4 (|scale| <= 4: every FsrEasuCon with output >= input / 4), a superset otherwise.
// Under wrap a span shorter than the image folds into at most two pieces: the top band of a 2x upscale also reads the last
// input rows, the bottom band the first ones.
inline int source_rows(float scale, float bias, bool wrap, int n_in, int rb, int re, int r[4]) {
    if (rb >= re) return 0;
    const int fa = (int)floorf(pos(rb, scale, bias)), fb = (int)floorf(pos(re - 1, scale, bias));
    int lo = (fa < fb ? fa : fb) - 1, hi = (fa < fb ? fb : fa) + 2;          // inclusive, unfolded
    if (!wrap) {
        lo = lo < 0 ? 0 : (lo > n_in - 1 ? n_in - 1 : lo);
        hi = hi < 0 ? 0 : (hi > n_in - 1 ? n_in - 1 : hi);
        r[0] = lo; r[1] = hi + 1;
        return 1;
    }
    if (hi - lo + 1 >= n_in) { r[0] = 0; r[1] = n_in; return 1; }
    const int a = (lo % n_in + n_in) % n_in, b = a + (hi - lo);             // folded start; end before the second fold
    if (b < n_in) { r[0] = a; r[1] = b + 1; return 1; }
    r[0] = 0; r[1] = b - n_in + 1;                                          // < a: the span is shorter than the image
    r[2] = a; r[3] = n_in;
    return 2;
}

}  // namespace vqeasu
