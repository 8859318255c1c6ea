// wgrad16.cu -- weight gradients of one nn.Linear from 16-bit T32 operands (act16.cuh), on tensor cores.
//
//   dW[n][col_off + k] += (1 / scale) * sum_p dY[p][n] X[p][k]        db[n] += (1 / scale) * sum_p dY[p][n]
//   optional head rows:  dH[r][k] += (1 / scale2) * sum_p (hg[p][r] + hg[p][r + 4]) X[p][k],  r < 4   (sigma / rgb head
//                        weights; features r + 4 of the hg cell hold the fp16 rounding residual of feature r)
//
// (reference: autograd of `nn.Linear` inside models/nerf.py:105-148.)  dY, X and hg are fp16 tensors in
// the T32 layout: a 32-point tile copied verbatim into shared memory IS the MN-major SWIZZLE_NONE canonical
// wgmma operand, so the whole kernel is
//   producer (thread 0)           cp.async.bulk of the tile's dY block (128 features x 64 B) and X block (FB x 64 B)
//                                 into a kStages-deep ring (mbarrier complete_tx);
//   two warpgroups                per tile 2 K-steps (K = 16 points) of wgmma SS, M = 64 out features each,
//                                 N = FB, into register accumulators that live for the CTA's whole slice of
//                                 points; one product (fp16 x fp16, fp32 accumulate); column sums of the dY tile
//                                 (the bias gradient) from shared memory while the MMAs run; at the end scaled
//                                 fp32 reductions from the fragments (split-P reduction; column pairs as red.v2).
// No converter warps, no transposition, every HBM byte read once: 2 (FA + FB) bytes per point
// (1 KB for a 256 x 256 layer; the fp32 version moved 2 KB and converted all of it in registers).
// Roofline: HBM (the fp32 reductions of the epilogue are per CTA, independent of the number of points).
#include "act16.cuh"
#include "common.cuh"
#include "wgmma.cuh"

namespace snb {
using namespace wg;

namespace {

constexpr int kW16Threads = 256;   // two warpgroups: out-feature rows [64 w, +64) of the CTA's 128-row block

// NM: 128-row out-feature blocks of dY (FA = 128 NM; 0 = head rows only); FB: X features (MMA N); kHead: hg operand
template <int NM, int FB, bool kHead>
struct W16Geo {
  static constexpr int kFA = 128 * NM;
  static constexpr int kDyBytes = 128 * 64, kXBytes = FB * 64, kHgBytes = kHead ? 512 : 0;   // per 32-point tile
  static constexpr int kStageBytes = kDyBytes + kXBytes + kHgBytes;
  static constexpr int kStagesRaw = (160 * 1024) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024;
  static_assert(kStages >= 2 && kSmemBytes <= 227 * 1024, "shared memory");
  static_assert(FB == 32 || FB == 64 || FB == 128 || FB == 256, "MMA N");
};

struct W16Args {
  const unsigned char* dY;     // (Ppad, FA) fp16 T32 (unused when NM == 0)
  const unsigned char* X;      // (Ppad, FB) fp16 T32
  const unsigned char* hg;     // (Ppad, 8)  fp16 T32 (kHead)
  int K;                       // valid columns of X (<= FB)
  float* dW; int ldw; int col_off;
  float* db;                   // nullable
  const float* scale;          // device: dY is stored as true * (*scale)
  float* dH[8];                // kHead: destination row pointers (nullable per row)
  const float* scale2;         // device: scale of hg
  long long n_tiles;           // 32-point tiles (Ppad / 32)
  long long tiles_per_cta;
};

template <int FB>
__device__ __forceinline__ void wgmma_mn(float (&d)[FB / 2], uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (FB == 256) wgmma_m64n256_f16_mn(d, a, b, acc);
  else if constexpr (FB == 128) wgmma_m64n128_f16_mn(d, a, b, acc);
  else if constexpr (FB == 64) wgmma_m64n64_f16_mn(d, a, b, acc);
  else wgmma_m64n32_f16_mn(d, a, b, acc);
}

// CTA (x, y): out-feature block y (y == NM: the head rows) over the 32-point tiles of slice x.  Thread 0 bulk-copies
// each tile's dY block (128 features x 32 points = 8 KB, contiguous in T32) and X (FB x 64 B) into a ring; a tile
// copied verbatim IS the MN-major SWIZZLE_NONE canonical operand (LBO = 128 B: next 8 points, SBO = 512 B: next 8
// features).  wgmma M = 64 out features per warpgroup, N = FB in features, K = 16 points; the accumulators live in
// registers for the CTA's whole slice; epilogue: scaled fp32 reductions straight from the fragments (column pairs
// as one red.v2 where the address is 8-byte aligned).
template <int NM, int FB, bool kHead>
__global__ void __launch_bounds__(kW16Threads, 1) wgrad16_kernel(W16Args a) {
  using G = W16Geo<NM, FB, kHead>;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* ring = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ uint64_t full[G::kStages], empty[G::kStages];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mb = blockIdx.y;
  const bool head = kHead && mb == NM;
  const long long t_begin = (long long)blockIdx.x * a.tiles_per_cta;
  const long long t_end = t_begin + a.tiles_per_cta < a.n_tiles ? t_begin + a.tiles_per_cta : a.n_tiles;
  const int n_my = t_end > t_begin ? (int)(t_end - t_begin) : 0;
  if (n_my == 0) return;

  if (tid == 0) {
    for (int i = 0; i < G::kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kW16Threads / 32); }
    fence_mbar_init();
  }
  __syncthreads();
  int next_load = 0;
  auto produce = [&](int upto) {
    for (; next_load < n_my && next_load < upto; ++next_load) {
      const int st = next_load % G::kStages;
      mbar_wait(&empty[st], ((next_load / G::kStages) & 1) ^ 1);
      unsigned char* dst = ring + (size_t)st * G::kStageBytes;
      const long long t = t_begin + next_load;
      const uint32_t bytes = (head ? 512 : G::kDyBytes) + G::kXBytes;
      mbar_arrive_expect_tx(&full[st], bytes);
      if (head) bulk_g2s(dst, a.hg + (size_t)t * 512, 512, &full[st]);
      else bulk_g2s(dst, a.dY + ((size_t)t * (G::kFA / 8) + mb * 16) * 512, G::kDyBytes, &full[st]);
      for (int o = 0; o < G::kXBytes; o += 16384)
        bulk_g2s(dst + G::kDyBytes + o, a.X + (size_t)t * G::kXBytes + o, G::kXBytes - o < 16384 ? G::kXBytes - o : 16384, &full[st]);
    }
  };
  if (tid == 0) produce(G::kStages);
  __syncwarp();

  const int wgi = warp >> 2, wq = warp & 3, g = lane >> 2, tq = lane & 3;
  // bias: thread = (feature group tid / 16 of this block, points 2 (tid % 16) + {0, 1} of every tile)
  float bs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bs[j] = 0.f;
  const bool do_bias = !head && a.db != nullptr;
  float acc[FB / 2];
#pragma unroll
  for (int i = 0; i < FB / 2; ++i) acc[i] = 0.f;
  int pend = -1;
  for (int i = 0; i < n_my; ++i) {
    const int st = i % G::kStages;
    mbar_wait(&full[st], (i / G::kStages) & 1);
    const unsigned char* tile = ring + (size_t)st * G::kStageBytes;
    const uint32_t base = smem_u32(tile);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
      // head rows: the 8 head-gradient features as all 8 row groups of A (SBO = 0): rows 8..63 repeat rows 0..7
      const uint64_t ad = head ? make_smem_desc(base + ks * 256, 128, 0)
                               : make_smem_desc(base + wgi * (8 * 512) + ks * 256, 128, 512);
      const uint64_t bd = make_smem_desc(base + G::kDyBytes + ks * 256, 128, 512);
      wgmma_mn<FB>(acc, ad, bd, (i > 0 || ks > 0) ? 1u : 0u);
    }
    wgmma_commit();
    if (do_bias) {
      const int grp = tid >> 4, p2 = (tid & 15) * 2;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const uint4 c = *reinterpret_cast<const uint4*>(tile + grp * 512 + (p2 + q) * 16);
        const uint32_t w[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[j]));
          bs[2 * j] += f.x; bs[2 * j + 1] += f.y;
        }
      }
    }
    wgmma_wait<1>();
    if (pend >= 0 && lane == 0) mbar_arrive(&empty[pend]);
    pend = st;
    if (tid == 0) produce(i + G::kStages);
    __syncwarp();
  }
  wgmma_wait<0>();

  const float inv = head ? 1.0f / __ldg(a.scale2) : 1.0f / __ldg(a.scale);
  if (do_bias) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = bs[j];
#pragma unroll
      for (int off = 8; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
      if ((tid & 15) == 0) atomicAdd(a.db + mb * 128 + (tid >> 4) * 8 + j, v * inv);
    }
  }
  // ---- epilogue: fragments -> scaled fp32 atomics
  if (head) {
    // features 4..7 of the hg cell are the fp16 residuals of features 0..3: row r + row r + 4 (lane + 16)
    if (wgi == 0 && wq == 0) {
#pragma unroll
      for (int j = 0; j < FB / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = acc[4 * j + e] + __shfl_down_sync(0xffffffffu, acc[4 * j + e], 16);
          const int k = 8 * j + 2 * tq + e;
          if (g < 4 && a.dH[g] != nullptr && k < a.K) atomicAdd(a.dH[g] + k, v * inv);
        }
    }
    return;
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int m = mb * 128 + wgi * 64 + wq * 16 + g + 8 * rr;
    float* dst = a.dW + (size_t)m * a.ldw + a.col_off;
#pragma unroll
    for (int j = 0; j < FB / 8; ++j) {
      const int k = 8 * j + 2 * tq;
      if (k < a.K) red_add_pair(dst + k, acc[4 * j + 2 * rr] * inv, acc[4 * j + 2 * rr + 1] * inv, k + 1 < a.K);
    }
  }
}

template <int NM, int FB, bool kHead>
int launch_wgrad16(W16Args a, cudaStream_t st) {
  using G = W16Geo<NM, FB, kHead>;
  static SmemOptIn optin;
  if (int rc = ensure_smem(wgrad16_kernel<NM, FB, kHead>, optin, G::kSmemBytes, "wgrad16")) return rc;
  const int blocks = NM + (kHead ? 1 : 0);
  long long ctas = (sm_count() + blocks - 1) / blocks;
  if (ctas > a.n_tiles) ctas = a.n_tiles;
  a.tiles_per_cta = (a.n_tiles + ctas - 1) / ctas;
  ctas = (a.n_tiles + a.tiles_per_cta - 1) / a.tiles_per_cta;
  wgrad16_kernel<NM, FB, kHead><<<dim3((unsigned)ctas, blocks), kW16Threads, G::kSmemBytes, st>>>(a);
  return check_launch("wgrad16_kernel");
}

}  // namespace

// dY: (Ppad, FA) T32 fp16 scaled by *scale, FA = 128 or 256 (0 with dY == nullptr: head rows only);
// X: (Ppad, FB) T32 fp16, FB in {256, 128, 64, 32}, first K columns valid;
// hg (nullable): (Ppad, 8) T32 fp16 scaled by *scale2 -> dH[r] (r < 8, nullable) += hg[:, r]^T X.
int run_wgrad16(const void* dY, int FA, const void* X, int FB, int K, float* dW, int ldw, int col_off, float* db,
                const float* scale, const void* hg, float* const* dH, const float* scale2, long long n_points_pad,
                cudaStream_t st) {
  if (n_points_pad == 0) return SNB_OK;
  W16Args a{};
  a.dY = reinterpret_cast<const unsigned char*>(dY);
  a.X = reinterpret_cast<const unsigned char*>(X);
  a.hg = reinterpret_cast<const unsigned char*>(hg);
  a.K = K; a.dW = dW; a.ldw = ldw; a.col_off = col_off; a.db = db; a.scale = scale; a.scale2 = scale2;
  for (int r = 0; r < 8; ++r) a.dH[r] = (hg != nullptr && dH != nullptr) ? dH[r] : nullptr;
  a.n_tiles = n_points_pad / kA16Tile;
  const bool head = hg != nullptr;
  if (FA == 256 && FB == 256 && !head) return launch_wgrad16<2, 256, false>(a, st);
  if (FA == 128 && FB == 256 && head) return launch_wgrad16<1, 256, true>(a, st);
  if (FA == 128 && FB == 256 && !head) return launch_wgrad16<1, 256, false>(a, st);
  if (FA == 256 && FB == 64 && !head) return launch_wgrad16<2, 64, false>(a, st);
  if (FA == 128 && FB == 32 && !head) return launch_wgrad16<1, 32, false>(a, st);
  if (FA == 0 && FB == 128 && head) return launch_wgrad16<0, 128, true>(a, st);
  if (FA == 0 && FB == 256 && head) return launch_wgrad16<0, 256, true>(a, st);    // sigma-only passes: dW_sigma
  return fail(SNB_ERR_INVALID, "run_wgrad16: unsupported shape FA=%d FB=%d head=%d", FA, FB, (int)head);
}

}  // namespace snb
