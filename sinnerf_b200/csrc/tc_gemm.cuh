// tc_gemm.cuh -- the wgmma GEMM of the semantic-loss ViT (vit.cu) and the patch discriminator (disc.cu).
//
// C[z][m][n] = epi(alpha * sum_k A[z](m, k) B[z](n, k)): fp32 operands read through strides (or packed 16-bit weight
// planes for B), 64 x 64 output tile per warpgroup, 64-deep K chunks staged through shared memory, fp32 accumulate.
// The operand arithmetic is a template parameter: fp16 hi + lo with three products (fp32 parity), or one fp16 or one
// bf16 product.  Everything is internal to the including source file.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace snb {
namespace {
using namespace wg;

// operand arithmetic of the GEMMs
enum { kSplit = 0, kF16 = 1, kBf16 = 2 };
int mode_of(int precision) {
  switch (precision) {
    case SNB_PREC_FP32: case SNB_PREC_F16X3: case SNB_PREC_BF16X3: return kSplit;
    case SNB_PREC_F16: return kF16;
    case SNB_PREC_BF16: return kBf16;
    default: return -1;
  }
}

// to fp16's finite range; NaN stays NaN (fminf / fmaxf would return the bound)
__device__ __forceinline__ float clamp_f16(float x) {
  float y;
  asm("max.NaN.f32 %0, %1, 0fC77FE000;\n\tmin.NaN.f32 %0, %0, 0f477FE000;" : "=f"(y) : "f"(x));
  return y;
}

// two fp32 values -> the packed 16-bit pair(s) of the mode (lo only in split mode)
template <int kMode>
__device__ __forceinline__ void cvt2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  if constexpr (kMode == kBf16) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = 0u;
  } else {
    x0 = clamp_f16(x0);
    x1 = clamp_f16(x1);
    const __half2 h = __floats2half2_rn(x0, x1);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    lo = 0u;
    if constexpr (kMode == kSplit) {
      const __half2 l = __floats2half2_rn(x0 - __low2float(h), x1 - __high2float(h));
      lo = *reinterpret_cast<const uint32_t*>(&l);
    }
  }
}

// ------------------------------------------------------------------ GEMM
// C[z][m][n] = epi(alpha * sum_k A[z](m, k) B[z](n, k)), z = z1 * nz2 + z2.  A: fp32, element (m, k) at
// A + z1 a_z1 + z2 a_z2 + m a_m + k a_k.  B: fp32 likewise (kBF32), or a packed weight (hi / lo planes).
enum { EPI_STORE = 0, EPI_RESID, EPI_GELU, EPI_GELU_BWD, EPI_EMBED };
struct Gemm {
  const float* A; long long a_z1, a_z2, a_m, a_k;
  const float* Bf; const uint16_t* Bh; const uint16_t* Bl;
  long long b_z1, b_z2, b_n, b_k;
  float* C; long long c_z1, c_z2, c_m;
  int M, N, K, nz2;
  int a_vec, b_vec;     // contiguous, 16-byte aligned 8-element runs along k: vector loads
  float alpha;
  int epi;
  const float* bias;    // (N) or null
  const float* aux;     // EPI_RESID: residual rows (row stride aux_m); EPI_GELU_BWD: saved pre-activations
  float* aux_out;       // EPI_GELU: pre-activations (row stride aux_m), may be null
  long long aux_m;
  const float* pos;     // EPI_EMBED: pos_embed; row m of image z gets pos_embed[m + 1]
  const float* alpha_dev;   // run_gemm<kMode, true>: a further scale read from the device (1 / sigma of a spectral norm)
};

constexpr int kTile = 64, kChunk = 64, kGemmThreads = 128;
constexpr long long kMaxGemmRows = 65535ll * kTile;   // M tiles along grid.y, at most 65535 of them
constexpr int kPlaneBytes = kTile * kChunk * 2;   // one 64 x 64 16-bit operand tile

__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float gelu_grad_f(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.70710678118654752f));
  const float pdf = expf(-0.5f * x * x) * 0.39894228040143268f;
  return cdf + x * pdf;
}

__device__ __forceinline__ void load8_f32(const float* base, long long s_row, long long s_k, int row, int rows, int k,
                                          int K, bool vec, float (&v)[8]) {
  if (row < rows && vec && k + 8 <= K) {
    const float4* p = reinterpret_cast<const float4*>(base + row * s_row + k);
    const float4 a = __ldg(p), b = __ldg(p + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = (row < rows && k + e < K) ? __ldg(base + row * s_row + (long long)(k + e) * s_k) : 0.f;
  }
}

__device__ __forceinline__ uint4 load8_u16(const uint16_t* base, long long s_row, long long s_k, int row, int rows,
                                           int k, int K, bool vec) {
  if (row < rows && vec && k + 8 <= K) return __ldg(reinterpret_cast<const uint4*>(base + row * s_row + k));
  uint32_t w[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const uint32_t x0 = (row < rows && k + 2 * e < K) ? __ldg(base + row * s_row + (long long)(k + 2 * e) * s_k) : 0u;
    const uint32_t x1 = (row < rows && k + 2 * e + 1 < K) ? __ldg(base + row * s_row + (long long)(k + 2 * e + 1) * s_k) : 0u;
    w[e] = x0 | (x1 << 16);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}

template <int kMode>
__device__ __forceinline__ void cvt8(const float (&v)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) cvt2<kMode>(v[2 * i], v[2 * i + 1], h[i], l[i]);
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

template <int kMode>
__device__ __forceinline__ void mma(float (&acc)[32], uint64_t a, uint64_t b) {
  if constexpr (kMode == kBf16) wgmma_m64n64_bf16(acc, a, b);
  else wgmma_m64n64_f16(acc, a, b);
}

// One warpgroup per 64 x 64 tile of C.  Each 64-deep K chunk is staged in the no-swizzle K-major core-matrix layout:
// element (r, k) at (r / 8) 1024 + (k / 8) 128 + (r % 8) 16 + (k % 8) 2 bytes.  The next chunk's global loads are
// issued while the current chunk's wgmmas run.
template <int kMode, bool kBF32, bool kScaleDev>
__global__ void __launch_bounds__(kGemmThreads) vit_gemm_kernel(const Gemm g) {
  constexpr int kPlanes = kMode == kSplit ? 2 : 1;
  __shared__ __align__(128) unsigned char sA[kPlanes][kPlaneBytes];
  __shared__ __align__(128) unsigned char sB[kPlanes][kPlaneBytes];
  const int tid = threadIdx.x;
  const int z1 = blockIdx.z / g.nz2, z2 = blockIdx.z % g.nz2;
  const int m0 = blockIdx.y * kTile, n0 = blockIdx.x * kTile;
  const float* A = g.A + z1 * g.a_z1 + z2 * g.a_z2 + (long long)m0 * g.a_m;
  const long long boff = z1 * g.b_z1 + z2 * g.b_z2 + (long long)n0 * g.b_n;
  const int rows_a = g.M - m0, rows_b = g.N - n0;

  float va[4][8], vb[4][8];
  uint4 ph[4], pl[4];
  auto fetch = [&](int kc) {
    const int k0 = kc * kChunk;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int u = tid + kGemmThreads * j, r = u >> 3, k = k0 + (u & 7) * 8;
      load8_f32(A, g.a_m, g.a_k, r, rows_a, k, g.K, g.a_vec, va[j]);
      if constexpr (kBF32) {
        load8_f32(g.Bf + boff, g.b_n, g.b_k, r, rows_b, k, g.K, g.b_vec, vb[j]);
      } else {
        ph[j] = load8_u16(g.Bh + boff, g.b_n, g.b_k, r, rows_b, k, g.K, g.b_vec);
        if constexpr (kMode == kSplit) pl[j] = load8_u16(g.Bl + boff, g.b_n, g.b_k, r, rows_b, k, g.K, g.b_vec);
      }
    }
  };

  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  const int nk = (g.K + kChunk - 1) / kChunk;
  fetch(0);
  for (int kc = 0; kc < nk; ++kc) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int u = tid + kGemmThreads * j, r = u >> 3, kg = u & 7;
      const int off = (r >> 3) * 1024 + kg * 128 + (r & 7) * 16;
      uint4 h, l;
      cvt8<kMode>(va[j], h, l);
      *reinterpret_cast<uint4*>(sA[0] + off) = h;
      if constexpr (kMode == kSplit) *reinterpret_cast<uint4*>(sA[kPlanes - 1] + off) = l;
      if constexpr (kBF32) {
        cvt8<kMode>(vb[j], h, l);
      } else {
        h = ph[j];
        l = pl[j];
      }
      *reinterpret_cast<uint4*>(sB[0] + off) = h;
      if constexpr (kMode == kSplit) *reinterpret_cast<uint4*>(sB[kPlanes - 1] + off) = l;
    }
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int s = 0; s < kChunk / 16; ++s) {
      const uint64_t ah = make_smem_desc(smem_u32(sA[0]) + s * 256, 128, 1024);
      const uint64_t bh = make_smem_desc(smem_u32(sB[0]) + s * 256, 128, 1024);
      if constexpr (kMode == kSplit) {
        const uint64_t al = make_smem_desc(smem_u32(sA[kPlanes - 1]) + s * 256, 128, 1024);
        const uint64_t bl = make_smem_desc(smem_u32(sB[kPlanes - 1]) + s * 256, 128, 1024);
        mma<kMode>(acc, al, bh);
        mma<kMode>(acc, ah, bl);
      }
      mma<kMode>(acc, ah, bh);
    }
    wgmma_commit();
    if (kc + 1 < nk) fetch(kc + 1);
    wgmma_wait<0>();
    __syncthreads();
  }

  // epilogue: thread t of warp w holds rows 16 w + t / 4 (+ 8), columns 8 j + 2 (t % 4) + {0, 1}
  const int warp = tid >> 5, lane = tid & 31;
  float* C = g.C + z1 * g.c_z1 + z2 * g.c_z2;
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int m = m0 + 16 * warp + (lane >> 2) + 8 * rr;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int n = n0 + 8 * j + 2 * (lane & 3) + e;
        if (n >= g.N) continue;
        float v = acc[4 * j + 2 * rr + e] * g.alpha;
        if constexpr (kScaleDev) v *= __ldg(g.alpha_dev);
        if (g.bias != nullptr) v += g.bias[n];
        float* dst = C + m * g.c_m + n;
        switch (g.epi) {
          case EPI_RESID: *dst = g.aux[m * g.aux_m + n] + v; break;
          case EPI_GELU:
            if (g.aux_out != nullptr) g.aux_out[m * g.aux_m + n] = v;
            *dst = gelu_f(v);
            break;
          case EPI_GELU_BWD: *dst = v * gelu_grad_f(g.aux[m * g.aux_m + n]); break;
          case EPI_EMBED: *dst = v + g.pos[(long long)(m + 1) * SNB_VIT_DIM + n]; break;
          default: *dst = v;
        }
      }
    }
  }
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <int kMode, bool kScaleDev = false>
int run_gemm(Gemm g, int nz, cudaStream_t st) {
  if (g.M <= 0 || g.N <= 0 || nz <= 0) return SNB_OK;
  if (g.nz2 <= 0) g.nz2 = 1;
  g.a_vec = g.a_k == 1 && aligned16(g.A) && g.a_m % 4 == 0 && g.a_z1 % 4 == 0 && g.a_z2 % 4 == 0;
  if (g.M > kMaxGemmRows || nz > 65535)
    return fail(SNB_ERR_INVALID, "vit_gemm_kernel: %d x %d x %d GEMM over %d matrices exceeds the launch grid (at most "
                "%lld rows, 65535 matrices)", g.M, g.N, g.K, nz, kMaxGemmRows);
  const dim3 grid((g.N + kTile - 1) / kTile, (g.M + kTile - 1) / kTile, nz);
  if (g.Bf != nullptr) {
    g.b_vec = g.b_k == 1 && aligned16(g.Bf) && g.b_n % 4 == 0 && g.b_z1 % 4 == 0 && g.b_z2 % 4 == 0;
    vit_gemm_kernel<kMode, true, kScaleDev><<<grid, kGemmThreads, 0, st>>>(g);
  } else {
    g.b_vec = g.b_k == 1 && aligned16(g.Bh) && (g.Bl == nullptr || aligned16(g.Bl)) && g.b_n % 8 == 0 &&
              g.b_z1 % 8 == 0 && g.b_z2 % 8 == 0;
    vit_gemm_kernel<kMode, false, kScaleDev><<<grid, kGemmThreads, 0, st>>>(g);
  }
  return check_launch("vit_gemm_kernel");
}

Gemm gemm(int M, int N, int K) {
  Gemm g{};
  g.M = M; g.N = N; g.K = K; g.nz2 = 1; g.alpha = 1.f; g.epi = EPI_STORE;
  return g;
}

}  // namespace
}  // namespace snb
