// wgrad_tc.cu -- weight gradients of one nn.Linear from fp32 row-major operands, on Hopper tensor cores.
//
//   dW[n][col_off + k] += sum_p dY[p][n] * X[p][k]      db[n] += sum_p dY[p][n]
//
// (reference: autograd of `nn.Linear` inside models/nerf.py:105-148; driver: field_bwd.cu.)
// dY (P, N) and X (P, ldx) are the plain row-major fp32 tensors the fp32-storage training forward /
// dgrad chain leave in HBM.
//
// As an MMA the reduction runs over POINTS:  D[m = out feature][n' = in feature] += A[m][p] B[n'][p],
// and both operands enter as bf16 hi + lo planes (gradients span fp32's exponent range; the 3-product
// split  x*w ~ xh*wh + xl*wh + xh*wl  keeps ~16 significand bits per operand, the gradient parity bar is
// 1e-3 per tensor).
//
// CTA (x, y): the 32-point tiles of slice x, out-feature block y (128 rows).  Per tile, all 256 threads
// load the fp32 rows (16-byte loads), split them and store 16-byte cells of the T32 layout (act16.cuh) --
// a cell is 8 features of one point, so a tile in shared memory IS the MN-major SWIZZLE_NONE canonical
// wgmma operand (LBO 128 B: next 8 points, SBO 512 B: next 8 features).  Two tile buffers: the conversion
// of tile i overlaps the wgmmas of tile i - 1.  Two warpgroups (M = 64 out features each, N = in features,
// K = 16 points) accumulate in registers for the whole slice; the same pass sums the bias gradient in fp32
// and, for the dgrad that follows, emits [X > 0] as (P, 8) words.  Epilogue: fp32 reductions from the
// fragments (split-P reduction), pairs of columns as one red.v2 where aligned.
// Roofline: HBM, 4 (N + K) bytes per point (X is read once per out-feature block).
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace snb {
using namespace wg;

namespace {

constexpr int kWtThreads = 256;

template <int FB>
struct WtGeo {
  static constexpr int kDyPlane = 128 * 32 * 2;        // one 128-feature x 32-point bf16 plane
  static constexpr int kXPlane = FB * 32 * 2;
  static constexpr int kBufBytes = 2 * kDyPlane + 2 * kXPlane;   // dY hi, dY lo, X hi, X lo
  static constexpr int kSmemBytes = 2 * kBufBytes + 1024;
};

struct WgradTcArgs {
  const float* dY; int N;
  const float* X; int ldx; int K;
  float* dW; int ldw; int col_off;
  float* db;                         // nullable
  uint32_t* x_pos_bits;              // nullable, K = 256 only: (P, 8) words, bit c of word w = [X[p][32 w + c] > 0]
  long long P;
  long long n_tiles, tiles_per_cta;
};

template <int FB>
__device__ __forceinline__ void wgmma_mn_bf16(float (&d)[FB / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (FB == 256) wgmma_m64n256_bf16_mn(d, a, b, acc);
  else if constexpr (FB == 64) wgmma_m64n64_bf16_mn(d, a, b, acc);
  else wgmma_m64n32_bf16_mn(d, a, b, acc);
}

// 8 fp32 values -> a 16-byte bf16 hi cell and the matching lo cell
__device__ __forceinline__ void split8_bf16(const float (&v)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const __nv_bfloat162 b = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
    h[j] = *reinterpret_cast<const uint32_t*>(&b);
    const __nv_bfloat162 r = __floats2bfloat162_rn(v[2 * j] - __low2float(b), v[2 * j + 1] - __high2float(b));
    l[j] = *reinterpret_cast<const uint32_t*>(&r);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

template <int FB>
__global__ void __launch_bounds__(kWtThreads, 1) wgrad_tc_kernel(WgradTcArgs a) {
  using G = WtGeo<FB>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint8_t pos[32][FB / 8];             // [X > 0] of one tile, one byte per 8-feature cell
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mb = blockIdx.y;
  const long long t_begin = (long long)blockIdx.x * a.tiles_per_cta;
  const long long t_end = t_begin + a.tiles_per_cta < a.n_tiles ? t_begin + a.tiles_per_cta : a.n_tiles;
  const int n_my = t_end > t_begin ? (int)(t_end - t_begin) : 0;
  if (n_my == 0) return;
  const bool emit_bits = a.x_pos_bits != nullptr && mb == 0;
  const int wgi = warp >> 2, wq = warp & 3, g = lane >> 2, tq = lane & 3;

  float bs[8];                                     // bias partial sums of feature group tid % 16
#pragma unroll
  for (int j = 0; j < 8; ++j) bs[j] = 0.f;
  float acc[FB / 2];
#pragma unroll
  for (int i = 0; i < FB / 2; ++i) acc[i] = 0.f;

  for (int i = 0; i < n_my; ++i) {
    // every thread of both warpgroups has passed the wait that retired tile i - 2, the last reader of this buffer
    // (and the previous tile's sign bits have been read out of pos[])
    __syncthreads();
    unsigned char* buf = smem + (size_t)(i & 1) * G::kBufBytes;
    unsigned char* dy_hi = buf;
    unsigned char* dy_lo = buf + G::kDyPlane;
    unsigned char* x_hi = buf + 2 * G::kDyPlane;
    unsigned char* x_lo = x_hi + G::kXPlane;
    const long long p0 = (t_begin + i) * 32;
    // ---- dY block: 16 feature groups x 32 points, two cells per thread (same group: the bias sums stay in registers)
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int e = tid + c * kWtThreads, grp = e & 15, p = e >> 4;
      const long long pt = p0 + p;
      float v[8];
      if (pt < a.P) {
        const float4* src = reinterpret_cast<const float4*>(a.dY + pt * a.N + mb * 128 + grp * 8);
        const float4 u0 = __ldg(src), u1 = __ldg(src + 1);
        v[0] = u0.x; v[1] = u0.y; v[2] = u0.z; v[3] = u0.w; v[4] = u1.x; v[5] = u1.y; v[6] = u1.z; v[7] = u1.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) v[j] = 0.f;
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) bs[j] += v[j];
      uint4 h, l;
      split8_bf16(v, h, l);
      *reinterpret_cast<uint4*>(dy_hi + grp * 512 + p * 16) = h;
      *reinterpret_cast<uint4*>(dy_lo + grp * 512 + p * 16) = l;
    }
    // ---- X tile: FB / 8 feature groups x 32 points
    for (int e = tid; e < (FB / 8) * 32; e += kWtThreads) {
      const int grp = e % (FB / 8), p = e / (FB / 8);
      const long long pt = p0 + p;
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = 0.f;
      if (pt < a.P) {
        const float* src = a.X + pt * a.ldx + grp * 8;
        if (grp * 8 + 8 <= a.K) {
          const float4 u0 = __ldg(reinterpret_cast<const float4*>(src)), u1 = __ldg(reinterpret_cast<const float4*>(src) + 1);
          v[0] = u0.x; v[1] = u0.y; v[2] = u0.z; v[3] = u0.w; v[4] = u1.x; v[5] = u1.y; v[6] = u1.z; v[7] = u1.w;
        } else {
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = grp * 8 + j < a.K ? __ldg(src + j) : 0.f;
        }
      }
      if (FB == 256 && emit_bits) {
        uint32_t b = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) b |= (v[j] > 0.f ? 1u : 0u) << j;
        pos[p][grp] = (uint8_t)b;
      }
      uint4 h, l;
      split8_bf16(v, h, l);
      *reinterpret_cast<uint4*>(x_hi + grp * 512 + p * 16) = h;
      *reinterpret_cast<uint4*>(x_lo + grp * 512 + p * 16) = l;
    }
    fence_proxy_async_smem();     // generic-proxy smem writes -> visible to the wgmmas
    __syncthreads();
    if (FB == 256 && emit_bits) {
      // thread = (point tid / 8, word tid % 8): four bytes of the tile's sign bits -> one word
      const int p = tid >> 3, w = tid & 7;
      const long long pt = p0 + p;
      if (pt < a.P)
        a.x_pos_bits[pt * 8 + w] = (uint32_t)pos[p][4 * w] | ((uint32_t)pos[p][4 * w + 1] << 8) |
                                   ((uint32_t)pos[p][4 * w + 2] << 16) | ((uint32_t)pos[p][4 * w + 3] << 24);
    }
    wgmma_fence();
    const uint32_t ah = smem_u32(dy_hi) + wgi * (8 * 512), al = smem_u32(dy_lo) + wgi * (8 * 512);
    const uint32_t bh = smem_u32(x_hi), bl = smem_u32(x_lo);
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      const uint64_t dah = make_smem_desc(ah + ks * 256, 128, 512), dal = make_smem_desc(al + ks * 256, 128, 512);
      const uint64_t dbh = make_smem_desc(bh + ks * 256, 128, 512), dbl = make_smem_desc(bl + ks * 256, 128, 512);
      wgmma_mn_bf16<FB>(acc, dah, dbh, (i > 0 || ks > 0) ? 1u : 0u);
      wgmma_mn_bf16<FB>(acc, dal, dbh, 1u);
      wgmma_mn_bf16<FB>(acc, dah, dbl, 1u);
    }
    wgmma_commit();
    wgmma_wait<1>();              // tile i - 1 has retired
  }
  wgmma_wait<0>();

  if (a.db != nullptr) {
    // threads t and t ^ 16 of a warp share a feature group; then one atomic per warp and feature
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = bs[j] + __shfl_xor_sync(0xffffffffu, bs[j], 16);
      if (lane < 16) atomicAdd(a.db + mb * 128 + (tid & 15) * 8 + j, v);
    }
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int m = mb * 128 + wgi * 64 + wq * 16 + g + 8 * rr;
    float* dst = a.dW + (size_t)m * a.ldw + a.col_off;
#pragma unroll
    for (int j = 0; j < FB / 8; ++j) {
      const int k = 8 * j + 2 * tq;
      if (k < a.K) red_add_pair(dst + k, acc[4 * j + 2 * rr], acc[4 * j + 2 * rr + 1], k + 1 < a.K);
    }
  }
}

template <int FB>
int launch_wgrad_tc(WgradTcArgs a, cudaStream_t st) {
  using G = WtGeo<FB>;
  static SmemOptIn optin;
  if (int rc = ensure_smem(wgrad_tc_kernel<FB>, optin, G::kSmemBytes, "wgrad_tc")) return rc;
  const int blocks = a.N / 128;
  long long ctas = (sm_count() + blocks - 1) / blocks;
  if (ctas > a.n_tiles) ctas = a.n_tiles;
  a.tiles_per_cta = (a.n_tiles + ctas - 1) / ctas;
  ctas = (a.n_tiles + a.tiles_per_cta - 1) / a.tiles_per_cta;
  wgrad_tc_kernel<FB><<<dim3((unsigned)ctas, blocks), kWtThreads, G::kSmemBytes, st>>>(a);
  return check_launch("wgrad_tc_kernel");
}

}  // namespace

int run_wgrad_tc(const float* dY, int N, const float* X, int ldx, int K, float* dW, int ldw, int col_off, float* db,
                 uint32_t* x_pos_bits, long long P, cudaStream_t st) {
  if (P == 0) return SNB_OK;
  if (x_pos_bits != nullptr && K != 256) return fail(SNB_ERR_INVALID, "run_wgrad_tc: mask bits need K = 256");
  if (((reinterpret_cast<uintptr_t>(dY) | reinterpret_cast<uintptr_t>(X)) & 15) != 0)
    return fail(SNB_ERR_INVALID, "run_wgrad_tc: dY and X must be 16-byte aligned");
  WgradTcArgs a{dY, N, X, ldx, K, dW, ldw, col_off, db, x_pos_bits, P, (P + 31) / 32, 0};
  if (N != 256 && N != 128) return fail(SNB_ERR_INVALID, "run_wgrad_tc: unsupported out features N=%d", N);
  if (ldx == 256 && K == 256) return launch_wgrad_tc<256>(a, st);
  if (ldx == 64 && K <= 64) return launch_wgrad_tc<64>(a, st);
  if (ldx == 32 && K <= 32) return launch_wgrad_tc<32>(a, st);
  return fail(SNB_ERR_INVALID, "run_wgrad_tc: unsupported shape N=%d K=%d ldx=%d", N, K, ldx);
}

}  // namespace snb
