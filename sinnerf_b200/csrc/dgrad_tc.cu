// dgrad_tc.cu -- input gradients of one nn.Linear from / to fp32 row-major tensors, on Hopper tensor cores.
//
//   dX[p][k] = ( sum_n dY[p][n] W[n][col_off + k]  +  extra[p] evec[k] ) * [mask[p][k] > 0]        k < 256
//
// (reference: autograd through models/nerf.py:105-148; driver: field_bwd.cu.)
// dY (P, N) with N = 256 or 128, mask = sign bits of the saved post-ReLU input of
// the layer (32 B per point, emitted by the wgrad kernel that reads that input anyway), extra/evec =
// the sigma head's rank-1 term at h8.  dY and dX are plain row-major fp32.
//
// Mapping (dgrad16.cu's): CTA (x, y) owns 128-point tiles x, x + gridDim.x, ... and output columns
// [128 y, +128); W^T of those columns is converted once to bf16 hi + lo and stays resident in shared memory
// (128 KB at N = 256); two warpgroups (wgmma M = 64 points each, N = 128) take A from registers: each thread
// loads its fragment's fp32 pairs (8 points of a warp read 32 contiguous bytes each), splits them into bf16
// hi + lo and issues the register-operand wgmma.  bf16 3-product split (hi*hi + lo*hi + hi*lo), fp32
// accumulate: gradients need fp32's range.
//
// HBM per point and layer: dY 4N + 32 B of mask in, dX 1 KB out: HBM-bound.
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace snb {
using namespace wg;

namespace {

constexpr int kDtTile = 128;
constexpr int kDtThreads = 256;

struct DgradTcArgs {
  const float* dY;
  const float* W; int ldw; int col_off;   // nn.Linear weight (N, ldw); inputs [col_off, col_off + 256)
  const uint32_t* mask_bits;       // (P,8) nullable: bit c of word w = [input[p][32 w + c] > 0] (wgrad_tc emits it)
  const float* extra; int extra_stride;   // nullable per-point scalar
  const float* evec;               // (256), with extra
  float* dX;                       // (P, 256)
  long long P;
};

template <int NRED>
struct DtSmem {
  // W^T planes of this CTA's 128 output columns: [hi|lo][n8][128 rows = output columns k][8 n], bf16
  static constexpr int kPlaneBytes = (NRED / 8) * 128 * 16;
  alignas(128) unsigned char b[2][kPlaneBytes];
  alignas(16) float evec[128];
};

__device__ __forceinline__ void bf16_split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - __low2float(h), x1 - __high2float(h));
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

template <int NRED>
__global__ void __launch_bounds__(kDtThreads, 1) dgrad_tc_kernel(DgradTcArgs a) {
  using S = DtSmem<NRED>;
  constexpr int kSteps = NRED / 16;
  extern __shared__ unsigned char smem_raw[];
  S& s = *reinterpret_cast<S*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int kh = blockIdx.y;
  const long long ntiles = (a.P + kDtTile - 1) / kDtTile;

  for (int i = tid; i < 128; i += kDtThreads) s.evec[i] = a.evec != nullptr ? a.evec[kh * 128 + i] : 0.f;
  for (int t = tid; t < (NRED / 8) * 128; t += kDtThreads) {
    const int row = t & 127, n8 = t >> 7;
    const int k = kh * 128 + row;
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float w0 = __ldg(a.W + (size_t)(n8 * 8 + 2 * j) * a.ldw + a.col_off + k);
      const float w1 = __ldg(a.W + (size_t)(n8 * 8 + 2 * j + 1) * a.ldw + a.col_off + k);
      bf16_split_pair(w0, w1, h[j], l[j]);
    }
    const int off = n8 * (128 * 16) + row * 16;
    *reinterpret_cast<uint4*>(s.b[0] + off) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(s.b[1] + off) = make_uint4(l[0], l[1], l[2], l[3]);
  }
  fence_proxy_async_smem();
  __syncthreads();

  const int wgi = warp >> 2, wq = warp & 3, g = lane >> 2, tq = lane & 3;
  const uint32_t bh0 = smem_u32(s.b[0]), bl0 = smem_u32(s.b[1]);
  float acc[64];
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long pt0 = tile * kDtTile + wgi * 64 + wq * 16 + g;    // rows pt0 and pt0 + 8 of this thread
    const bool in0 = pt0 < a.P, in1 = pt0 + 8 < a.P;
    // fragments of one K16 step: (row, k 2tq..+1) and (row, k 2tq+8..+9) of rows pt0, pt0 + 8, as bf16 hi + lo
    auto load_a = [&](int ks, uint32_t (&fh)[4], uint32_t (&fl)[4]) {
      const int c = 16 * ks + 2 * tq;
      const float2 z = make_float2(0.f, 0.f);
      const float2 v0 = in0 ? __ldg(reinterpret_cast<const float2*>(a.dY + pt0 * NRED + c)) : z;
      const float2 v1 = in1 ? __ldg(reinterpret_cast<const float2*>(a.dY + (pt0 + 8) * NRED + c)) : z;
      const float2 v2 = in0 ? __ldg(reinterpret_cast<const float2*>(a.dY + pt0 * NRED + c + 8)) : z;
      const float2 v3 = in1 ? __ldg(reinterpret_cast<const float2*>(a.dY + (pt0 + 8) * NRED + c + 8)) : z;
      bf16_split_pair(v0.x, v0.y, fh[0], fl[0]);
      bf16_split_pair(v1.x, v1.y, fh[1], fl[1]);
      bf16_split_pair(v2.x, v2.y, fh[2], fl[2]);
      bf16_split_pair(v3.x, v3.y, fh[3], fl[3]);
    };
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    // kB K16 steps per batch, two register sets: a register-A wgmma reads its fragment asynchronously, so a set
    // is refilled only after wgmma.wait_group has retired the batch that used it
    constexpr int kB = 4, kBatches = kSteps / kB;
    static_assert(kSteps % kB == 0, "K16 steps per batch");
    uint32_t fh[2][kB][4], fl[2][kB][4];
    auto load_batch = [&](int set, int b) {
#pragma unroll
      for (int i = 0; i < kB; ++i) load_a(b * kB + i, fh[set][i], fl[set][i]);
    };
    load_batch(0, 0);
#pragma unroll
    for (int b = 0; b < kBatches; ++b) {
      const int set = b & 1;
      wgmma_fence();
#pragma unroll
      for (int i = 0; i < kB; ++i) {
        const int ks = b * kB + i;
        const uint64_t dbh = make_smem_desc(bh0 + ks * 2 * (128 * 16), 128 * 16, 128);
        const uint64_t dbl = make_smem_desc(bl0 + ks * 2 * (128 * 16), 128 * 16, 128);
        wgmma_m64n128_bf16_rs(acc, fh[set][i], dbh, ks > 0 ? 1u : 0u);
        wgmma_m64n128_bf16_rs(acc, fl[set][i], dbh, 1u);
        wgmma_m64n128_bf16_rs(acc, fh[set][i], dbl, 1u);
      }
      wgmma_commit();
      if (b + 1 < kBatches) {
        wgmma_wait<1>();            // batch b - 1 (the other register set) has retired
        load_batch(set ^ 1, b + 1);
      }
    }
    wgmma_wait<0>();
    // ---- epilogue: (+ sigma term) * mask -> dX rows
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long pt = pt0 + 8 * rr;
      if (pt >= a.P) continue;
      const float ex = a.extra != nullptr ? a.extra[pt * a.extra_stride] : 0.f;
      uint32_t mw[4] = {~0u, ~0u, ~0u, ~0u};
      if (a.mask_bits != nullptr) {
        const uint4 m = __ldg(reinterpret_cast<const uint4*>(a.mask_bits + pt * 8) + kh);
        mw[0] = m.x; mw[1] = m.y; mw[2] = m.z; mw[3] = m.w;
      }
      float* dst = a.dX + pt * 256 + kh * 128;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + 2 * tq;
        const float2 e = *reinterpret_cast<const float2*>(s.evec + c);
        const float x0 = (mw[c >> 5] >> (c & 31)) & 1u ? fmaf(ex, e.x, acc[4 * j + 2 * rr]) : 0.f;
        const float x1 = (mw[c >> 5] >> ((c & 31) + 1)) & 1u ? fmaf(ex, e.y, acc[4 * j + 2 * rr + 1]) : 0.f;
        *reinterpret_cast<float2*>(dst + c) = make_float2(x0, x1);
      }
    }
  }
}

template <int NRED>
int launch_dgrad_tc(const DgradTcArgs& a, cudaStream_t st) {
  static SmemOptIn optin;
  const int smem = (int)sizeof(DtSmem<NRED>) + 1024;
  if (int rc = ensure_smem(dgrad_tc_kernel<NRED>, optin, smem, "dgrad_tc")) return rc;
  const long long ntiles = (a.P + kDtTile - 1) / kDtTile;
  long long ctas = (sm_count() + 1) / 2;          // two column halves per tile
  if (ctas > ntiles) ctas = ntiles;
  dgrad_tc_kernel<NRED><<<dim3((unsigned)ctas, 2), kDtThreads, smem, st>>>(a);
  return check_launch("dgrad_tc_kernel");
}

}  // namespace

// run_dgrad (field_bwd.cu) on tensor cores; the ReLU mask arrives as the bit matrix run_wgrad_tc emitted
int run_dgrad_tc(const float* dY, int N, const float* W, int ldw, int col_off, const uint32_t* mask_bits,
                 const float* extra, int extra_stride, const float* evec, float* dX, long long P, cudaStream_t st) {
  if (P == 0) return SNB_OK;
  DgradTcArgs a{dY, W, ldw, col_off, mask_bits, extra, extra_stride, evec, dX, P};
  if (N == 256) return launch_dgrad_tc<256>(a, st);
  if (N == 128) return launch_dgrad_tc<128>(a, st);
  return fail(SNB_ERR_INVALID, "run_dgrad_tc: unsupported reduction length %d", N);
}

}  // namespace snb
