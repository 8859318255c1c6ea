// act16.cuh -- layout of the 16-bit saved activations / gradients of the training path (round 2).
//
// Why: with fp32 row-major activations the backward of one 256-wide layer moved ~5 KB per point through
// HBM (forward store 1 KB, wgrad reads dY + X 2 KB, dgrad reads dY and writes dX 2 KB) and both tensor-core
// kernels spent most of their warps converting / transposing fp32 into MMA operands (round-1 ncu: 4.4 TB/s,
// tensor pipe 38 %).  Here every per-point tensor of the training path is stored ONCE, as fp16, in the
// layout the MMAs consume directly:
//
//   "T32" layout of a (P, F) tensor, F % 8 == 0, P padded to a multiple of 128:
//        element (p, f)  ->  16-bit index  ((p / 32) * (F / 8) + f / 8) * 256 + (p % 32) * 8 + f % 8
//   i.e. tiles of 32 points; inside a tile one 16-byte cell per (8-feature group, point), cells of a group
//   contiguous over the 32 points.  A tile is F * 64 bytes, contiguous.
//
//   * a warp whose lanes are 32 consecutive points writes / reads one 8-feature group as 512 contiguous
//     bytes; eight consecutive points of one group are 128 contiguous bytes -- the rows of a wgmma register
//     fragment or accumulator fragment: no transposition;
//   * a tile copied to shared memory verbatim (one cp.async.bulk) IS a wgmma operand in the SWIZZLE_NONE
//     canonical layout: 8 points x 16 bytes = one 128-byte core matrix,
//       - MN-major (M or N = features, K = points): LBO (K direction, next 8 points) = 128 B,
//         SBO (MN direction, next 8 features) = 512 B          -> the wgrad contraction  dW = dY^T X
//       - K-major  (M = points, K = features): SBO = 128 B, LBO = 512 B     (not used: dgrad keeps A in registers);
//   * 2.5 KB per point and layer instead of 5 KB, and no converter warps.
//
// Precision: activations are post-ReLU values < 65504 (saturated), rounded to nearest fp16 (11 bits);
// gradients are stored as fp16 x 2^k with a per-tensor power-of-two scale chosen ON THE DEVICE from a
// rigorous bound (measured max |dY| of the previous layer x max column L1 norm of the weights), so nothing
// overflows and the top of the range is used; wgrad divides the scale out of its fp32 accumulators.
// The layer-to-layer gradient chain carries a second fp16 plane with the rounding residual (hi + lo = 22
// bits; dgrad16.cu), so the only 11-bit roundings a weight gradient sees are ONE of its layer's gradient
// and ONE of its layer's input.  Weights enter dgrad as fp16 hi + lo.  Measured effect on the parameter
// gradients: tests/test_gpu_round2.py, tests/test_gpu_backward.py (<= 1e-3 per tensor vs autograd through
// the fp32 oracle).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace snb {

constexpr int kA16Tile = 32;                 // points per T32 tile
__host__ __device__ constexpr long long a16_pad(long long n_points) { return (n_points + 127) / 128 * 128; }
// byte offset of the 16-byte cell (point p, feature group f8) of a (P, F) tensor
__host__ __device__ __forceinline__ size_t a16_cell(long long p, int f8, int F) {
  return ((size_t)(p >> 5) * (F >> 3) + f8) * 512 + (size_t)(p & 31) * 16;
}

// ---- saved activations of one field pass (snb_field_forward_train16): one buffer, sections in this order
//   enc  (Ppad, 64)  dir (Ppad, 32)  h1..h8 (8 x (Ppad, 256))  g (Ppad, 128)      fp16, T32
//   mask (8 layers x 8 words x Ppad) uint32: bit c of word w of layer l, point p = [h_{l+1}[p][32 w + c] > 0] (fp32 test)
struct Act16Layout {
  size_t enc, dir, h[8], g, mask, total;
};
__host__ __device__ inline Act16Layout make_act16_layout(long long n_points) {
  const size_t pp = (size_t)a16_pad(n_points);
  Act16Layout L{};
  size_t off = 0;
  L.enc = off; off += pp * 64 * 2;
  L.dir = off; off += pp * 32 * 2;
  for (int l = 0; l < 8; ++l) { L.h[l] = off; off += pp * 256 * 2; }
  L.g = off; off += pp * 128 * 2;
  L.mask = off; off += (size_t)8 * 8 * pp * 4;
  L.total = off;
  return L;
}
// mask word (layer l, word w, point p)
__host__ __device__ __forceinline__ size_t a16_mask_index(int l, int w, long long p, long long ppad) {
  return ((size_t)l * 8 + w) * (size_t)ppad + (size_t)p;
}

// ---- workspace of one backward pass (snb_field_backward16)
//   dS (Ppad,128) | hg (Ppad,8) | dYa (Ppad,256) | dYb (Ppad,256)   fp16 T32, hi planes
//   dS_lo | dYa_lo | dYb_lo                                            residual planes of the gradient chain
//   fold (SNB_BWD_WS_FLOATS floats) | state (kBwdStateFloats floats)
constexpr int kBwdStateFloats = 64;
struct Bwd16Layout {
  size_t ds, hg, dya, dyb, ds_lo, dya_lo, dyb_lo, fold, state, total;
};
__host__ __device__ inline Bwd16Layout make_bwd16_layout(long long n_points) {
  const size_t pp = (size_t)a16_pad(n_points);
  Bwd16Layout L{};
  size_t off = 0;
  L.ds = off; off += pp * 128 * 2;
  L.hg = off; off += pp * 8 * 2;
  L.dya = off; off += pp * 256 * 2;
  L.dyb = off; off += pp * 256 * 2;
  L.ds_lo = off; off += pp * 128 * 2;
  L.dya_lo = off; off += pp * 256 * 2;
  L.dyb_lo = off; off += pp * 256 * 2;
  L.fold = off; off += (size_t)(2 * 128 * 256 + 128) * 4;
  L.state = off; off += (size_t)kBwdStateFloats * 4;
  L.total = (off + 255) & ~(size_t)255;
  return L;
}
// state words (floats unless noted; "amax" entries are uint32 bit patterns raised with atomicMax)
enum {
  ST_AMAX_G = 0,      // max |g_raw| (real units)
  ST_AMAX_DS = 1,     // max |dS * scale[DS]|
  ST_AMAX_H0 = 2,     // +l: max |dH_l * scale[H_l]|, l = 0..7
  ST_SCALE_HG = 10,   // scale of the head-gradient cells [gp_r, gp_g, gp_b, g_sigma]
  ST_SCALE_DS = 11,
  ST_SCALE_H0 = 12,   // +l, l = 0..7
  ST_L1_FOLD = 20,    // max column L1 norm of W' (dS -> dH_7)
  ST_L1_L0 = 21,      // +l: of W_l[:, col_off:+256] (dH_l -> dH_{l-1}), l = 1..7
  ST_EVEC_MAX = 29,   // max |w_sigma|
  ST_WR_L1 = 30,      // max_j sum_c |W_rgb[c][j]|
};

// largest power of two s with s * bound <= target (bound > 0), clamped to a sane exponent range
__host__ __device__ __forceinline__ float pow2_scale(float bound, float target) {
  if (!(bound > 0.f) || !(bound < 3.0e38f)) return 1.0f;
  int e;
  const float m = frexpf(target / bound, &e);   // target / bound = m * 2^e, m in [0.5, 1)
  (void)m;
  e -= 1;                                        // 2^(e-1) <= target / bound
  if (e > 100) e = 100;
  if (e < -100) e = -100;
  return ldexpf(1.0f, e);
}
constexpr float kA16Target = 16384.0f;           // bound * scale <= 2^14: 4x head-room below fp16's 65504

__device__ __forceinline__ uint32_t pack_half2_sat(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

}  // namespace snb
