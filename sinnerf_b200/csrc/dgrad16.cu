// dgrad16.cu -- input gradients of one nn.Linear from / to 16-bit T32 tensors (act16.cuh), on tensor cores.
//
//   dX[p][k] = ( sum_n dY[p][n] W[n][col_off + k]  +  extra[p] evec[k] ) * [mask[p][k]]        k < 256
//
// (reference: autograd through models/nerf.py:105-148.)  A CTA owns 128 points (two warpgroups, wgmma M = 64) and
// one 128-column half of the output; W^T of that half is resident in shared memory; the operands are already
// 16-bit in HBM:
//   * dY (Ppad, N) fp16 in the T32 layout, stored as true * s_in: lane = point, an 8-feature cell is 16 bytes,
//     the 8 points of a register fragment row are 128 contiguous bytes: dY goes from HBM straight into the
//     wgmma A fragments (register operand form), no conversion, no transposition;
//   * the gradient CHAIN (dgrad -> dgrad) is carried as fp16 hi + lo planes (22 bits), so rounding does not
//     accumulate over the 8 layers; the wgrad of each layer reads only the hi plane -- its error is ONE fp16
//     rounding of that layer's gradient, whatever the depth (measured: hi-only chains reached 1.1e-3 on the first
//     layer's weights, hi + lo 2e-4; the parity bar is 1e-3).  The driver (bwd16.cu) carries the lo plane from dS
//     down to dH_4 and runs the four lowest hops hi-only: kLoIn / kLoOut say whether dY / dX have it;
//   * W^T as fp16 hi + lo; products hi*hi + lo*hi + hi*lo (2 without the lo plane);
//   * the epilogue multiplies by the power-of-two ratio s_out / s_in, adds the sigma head's rank-1 term,
//     applies the ReLU mask (bit words the forward wrote, 32 B per point), rounds to fp16 and writes cells of
//     the output T32 tensor -- 4 x 512 contiguous bytes per warp and 32 columns; it also raises the running
//     max |dX * s_out| that the NEXT layer's scale is derived from.
//   * s_out = the largest power of two with  (max |dY| / s_in) * (max column L1 norm of W) [+ max |extra| max |evec|]
//     * s_out <= 2^14: a rigorous bound, so the fp16 stores cannot overflow; chosen identically by every CTA
//     from three device scalars (no host round trip).
// HBM per point and layer: 4 N + 32 B in, 1 KB out with the lo plane (the fp32 version moved the same bytes but
// spent its warps converting them, and its wgrad read 2 KB where wgrad16 reads 1 KB); 2 N + 32 in, 512 B out without.
#include <cuda_fp16.h>

#include "act16.cuh"

#include "common.cuh"
#include "wgmma.cuh"

namespace snb {
using namespace wg;

namespace {

constexpr int kDgTile = 128;                 // points per CTA tile (two warpgroups of 64, wgmma M = 64)
constexpr int kDgThreads = 256;

struct Dgrad16Args {
  const unsigned char* dY;         // (Ppad, NRED) fp16 T32, stored as true * state[st_scale_in]
  const unsigned char* dY_lo;      // same shape: fp16(true * s - hi) (kLo)
  const float* W; int ldw; int col_off;   // nn.Linear weight (NRED, ldw); inputs [col_off, col_off + 256)
  const uint32_t* mask;            // (8 words, Ppad) nullable: bit c of word w = [input[p][32 w + c] > 0]
  const float* extra; int extra_stride;   // nullable per-point scalar (true units)
  const float* evec;               // (256), with extra
  unsigned char* dX;               // (Ppad, 256) fp16 T32, stored as true * state[st_scale_out]
  unsigned char* dX_lo;            // residual plane (kLo)
  float* state;                    // Bwd16 state words (act16.cuh)
  int st_amax_in, st_scale_in, st_l1, st_amax_out, st_scale_out;
  long long P, ppad;
};

template <int NRED>
struct Dg16Smem {
  // W^T planes of this CTA's 128 output columns: [hi|lo][n8 = n / 8][128 rows = output columns k][8 n]
  // (the K-major canonical layout of the wgmma B operand: N = k, K = n)
  static constexpr int kPlaneBytes = (NRED / 8) * 128 * 16;
  alignas(128) unsigned char b[2][kPlaneBytes];
  alignas(16) float evec[128];
};

__device__ __forceinline__ void f16_split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  const __half2 h = __floats2half2_rn(x0, x1);
  hi = *reinterpret_cast<const uint32_t*>(&h);
  const float2 b = __half22float2(h);
  const __half2 l = __floats2half2_rn(x0 - b.x, x1 - b.y);
  lo = *reinterpret_cast<const uint32_t*>(&l);
}

// kLoIn: dY comes with its residual plane (3 products); kLoOut: dX is written with its residual plane.
// CTA (x, y): output columns [128 y, +128) of the point tiles x, x + gridDim.x, ...; W^T of those columns is
// resident in shared memory (fp16 hi + lo), the A operand (dY cells) goes from HBM straight into the wgmma
// register fragments -- a fragment row is 16 contiguous bytes of one T32 cell, 8 points of a warp's load are
// 128 contiguous bytes.
template <int NRED, bool kLoIn, bool kLoOut>
__global__ void __launch_bounds__(kDgThreads, 1) dgrad16_kernel(Dgrad16Args a) {
  constexpr bool kLo = kLoIn;
  using S = Dg16Smem<NRED>;
  constexpr int kSteps = NRED / 16;
  extern __shared__ unsigned char smem_raw[];
  S& s = *reinterpret_cast<S*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int kh = blockIdx.y;                      // output column half
  const long long ntiles = (a.P + kDgTile - 1) / kDgTile;

  // ---------------- one-time setup: resident W^T of this half
  for (int i = tid; i < 128; i += kDgThreads) s.evec[i] = a.evec != nullptr ? a.evec[kh * 128 + i] : 0.f;
  // task = (n8 block, output column): 8 consecutive reduction rows n of one input column k
  for (int t = tid; t < (NRED / 8) * 128; t += kDgThreads) {
    const int row = t & 127, n8 = t >> 7;
    const int k = kh * 128 + row;
    uint32_t h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float w0 = __ldg(a.W + (size_t)(n8 * 8 + 2 * j) * a.ldw + a.col_off + k);
      const float w1 = __ldg(a.W + (size_t)(n8 * 8 + 2 * j + 1) * a.ldw + a.col_off + k);
      f16_split_pair(w0, w1, h[j], l[j]);
    }
    const int off = n8 * (128 * 16) + row * 16;
    *reinterpret_cast<uint4*>(s.b[0] + off) = make_uint4(h[0], h[1], h[2], h[3]);
    *reinterpret_cast<uint4*>(s.b[1] + off) = make_uint4(l[0], l[1], l[2], l[3]);
  }
  fence_proxy_async_smem();
  __syncthreads();
  // output scale: every thread of every CTA derives the same power of two from three device scalars
  const float s_in = a.state[a.st_scale_in];
  float bound = __uint_as_float(reinterpret_cast<const uint32_t*>(a.state)[a.st_amax_in]) / s_in * a.state[a.st_l1];
  if (a.extra != nullptr)
    bound += __uint_as_float(reinterpret_cast<const uint32_t*>(a.state)[ST_AMAX_G]) * a.state[ST_EVEC_MAX];
  const float s_out = pow2_scale(bound, kA16Target);
  const float ratio = s_out / s_in;
  if (blockIdx.x == 0 && blockIdx.y == 0 && tid == 0) a.state[a.st_scale_out] = s_out;

  const int wgi = warp >> 2, wq = warp & 3, g = lane >> 2, tq = lane & 3;
  const uint32_t bh0 = smem_u32(s.b[0]), bl0 = smem_u32(s.b[1]);
  float amax = 0.f;
  float acc[64];
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long pt0 = tile * kDgTile + wgi * 64 + wq * 16 + g;    // rows pt0 and pt0 + 8 of this thread
    const bool in0 = pt0 < a.ppad, in1 = pt0 + 8 < a.ppad;
    // A fragments of one K16 step: cells (pt, 2 ks) and (pt, 2 ks + 1), 32-bit word tq of each
    auto load_a = [&](const unsigned char* base, int ks, uint32_t (&f)[4]) {
      const size_t o0 = a16_cell(pt0, 2 * ks, NRED) + 4 * tq, o1 = a16_cell(pt0 + 8, 2 * ks, NRED) + 4 * tq;
      f[0] = in0 ? __ldg(reinterpret_cast<const uint32_t*>(base + o0)) : 0u;
      f[1] = in1 ? __ldg(reinterpret_cast<const uint32_t*>(base + o1)) : 0u;
      f[2] = in0 ? __ldg(reinterpret_cast<const uint32_t*>(base + o0 + 512)) : 0u;
      f[3] = in1 ? __ldg(reinterpret_cast<const uint32_t*>(base + o1 + 512)) : 0u;
    };
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    // A fragments of kB consecutive K16 steps per batch, two register sets: a register-A wgmma reads its fragment
    // asynchronously, so a set is refilled only after wgmma.wait_group has retired the batch that used it
    constexpr int kB = 4, kBatches = kSteps / kB;
    static_assert(kSteps % kB == 0, "K16 steps per batch");
    uint32_t fh[2][kB][4], fl[2][kLo ? kB : 1][4];
    auto load_batch = [&](int set, int b) {
#pragma unroll
      for (int i = 0; i < kB; ++i) {
        load_a(a.dY, b * kB + i, fh[set][i]);
        if (kLo) load_a(a.dY_lo, b * kB + i, fl[set][kLo ? i : 0]);
      }
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
        wgmma_m64n128_f16_rs(acc, fh[set][i], dbh, ks > 0 ? 1u : 0u);
        if (kLo) wgmma_m64n128_f16_rs(acc, fl[set][kLo ? i : 0], dbh, 1u);
        wgmma_m64n128_f16_rs(acc, fh[set][i], dbl, 1u);
      }
      wgmma_commit();
      if (b + 1 < kBatches) {
        wgmma_wait<1>();            // batch b - 1 (the other register set) has retired
        load_batch(set ^ 1, b + 1);
      }
    }
    wgmma_wait<0>();
    // ---- epilogue: scale, (+ sigma term), mask, fp16 hi (+ lo) -> dX cells
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long pt = pt0 + 8 * rr;
      const bool live = pt < a.P, inbuf = pt < a.ppad;
      const float ex = (live && a.extra != nullptr) ? a.extra[pt * a.extra_stride] * s_out : 0.f;
      uint32_t mw[4] = {~0u, ~0u, ~0u, ~0u};
      if (live && a.mask != nullptr) {
#pragma unroll
        for (int w = 0; w < 4; ++w) mw[w] = __ldg(a.mask + (size_t)(kh * 4 + w) * (size_t)a.ppad + pt);
      }
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int c = 8 * j + 2 * tq;                   // column inside this half
        const float2 e = *reinterpret_cast<const float2*>(s.evec + c);
        float x0 = fmaf(ex, e.x, acc[4 * j + 2 * rr] * ratio);
        float x1 = fmaf(ex, e.y, acc[4 * j + 2 * rr + 1] * ratio);
        x0 = (mw[c >> 5] >> (c & 31)) & 1u ? x0 : 0.f;
        x1 = (mw[c >> 5] >> ((c & 31) + 1)) & 1u ? x1 : 0.f;
        if (!live) { x0 = 0.f; x1 = 0.f; }
        amax = fmaxf(amax, fmaxf(fabsf(x0), fabsf(x1)));
        const uint32_t o = pack_half2_sat(x0, x1);
        const int k = kh * 128 + c;
        if (inbuf) {
          *reinterpret_cast<uint32_t*>(a.dX + a16_cell(pt, k >> 3, 256) + (k & 7) * 2) = o;
          if (kLoOut) {
            const float2 hv = __half22float2(*reinterpret_cast<const __half2*>(&o));
            *reinterpret_cast<uint32_t*>(a.dX_lo + a16_cell(pt, k >> 3, 256) + (k & 7) * 2) = pack_half2_sat(x0 - hv.x, x1 - hv.y);
          }
        }
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, off));
  if (lane == 0 && amax > 0.f)
    atomicMax(reinterpret_cast<uint32_t*>(a.state) + a.st_amax_out, __float_as_uint(amax == amax ? fminf(amax, 65504.f) : 65504.f));
}

template <int NRED, bool kLoIn, bool kLoOut>
int launch_dgrad16(const Dgrad16Args& a, cudaStream_t st) {
  static SmemOptIn optin;
  const int smem = (int)sizeof(Dg16Smem<NRED>) + 1024;
  if (int rc = ensure_smem(dgrad16_kernel<NRED, kLoIn, kLoOut>, optin, smem, "dgrad16")) return rc;
  const int sms = sm_count();
  const long long ntiles = (a.P + kDgTile - 1) / kDgTile;
  long long ctas = (sms + 1) / 2;                 // two column halves per tile
  if (ctas > ntiles) ctas = ntiles;
  dgrad16_kernel<NRED, kLoIn, kLoOut><<<dim3((unsigned)ctas, 2), kDgThreads, smem, st>>>(a);
  return check_launch("dgrad16_kernel");
}

}  // namespace

// dY (Ppad, N) -> dX (Ppad, 256), fp16 T32 hi (+ lo) planes; scales and running maxima live in `state` (act16.cuh).
// dY_lo / dX_lo NULL = that tensor has no residual plane (hi-only).
int run_dgrad16(const void* dY, const void* dY_lo, int N, const float* W, int ldw, int col_off, const uint32_t* mask,
                const float* extra, int extra_stride, const float* evec, void* dX, void* dX_lo, float* state, int st_amax_in,
                int st_scale_in, int st_l1, int st_amax_out, int st_scale_out, long long P, cudaStream_t st) {
  if (P == 0) return SNB_OK;
  Dgrad16Args a{reinterpret_cast<const unsigned char*>(dY), reinterpret_cast<const unsigned char*>(dY_lo), W, ldw, col_off, mask,
                extra, extra_stride, evec, reinterpret_cast<unsigned char*>(dX), reinterpret_cast<unsigned char*>(dX_lo), state,
                st_amax_in, st_scale_in, st_l1, st_amax_out, st_scale_out, P, a16_pad(P)};
  const bool li = dY_lo != nullptr, lo = dX_lo != nullptr;
  if (N == 256) {
    if (li && lo) return launch_dgrad16<256, true, true>(a, st);
    if (li) return launch_dgrad16<256, true, false>(a, st);
    if (!lo) return launch_dgrad16<256, false, false>(a, st);
  }
  if (N == 128 && li && lo) return launch_dgrad16<128, true, true>(a, st);   // the direction layer: dS -> dH_8
  if (!li && lo) return fail(SNB_ERR_INVALID, "run_dgrad16: a residual plane cannot be produced from a hi-only input chain");
  return fail(SNB_ERR_INVALID, "run_dgrad16: no kernel for reduction length %d with these residual planes", N);
}

}  // namespace snb
