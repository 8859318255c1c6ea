// field_tc.cu -- the fused field pass on Hopper tensor cores (wgmma / bulk TMA / mbarrier).
//
// Same contract as field_simt.cu (points o+d*z, both positional encodings, the 12-layer MLP,
// [r,g,b,sigma] out; reference models/rendering.py:184-212,284-285 + models/nerf.py:24-41,
// 105-148), but every 256-wide layer is a chain of wgmma.mma_async instructions:
//
//   * persistent CTAs of two consumer warpgroups and one producer warpgroup; a CTA works on 128-point
//     tiles, each consumer warpgroup owns 64 of the rows (wgmma M = 64) and both share one weight stream,
//     so every weight byte a CTA ingests from L2 feeds 128 points; setmaxnreg moves the producer's
//     registers to the consumers (24 / 240 per thread);
//   * a layer's whole 64 x 256 fp32 accumulator lives in registers (two N = 128 halves, 128 registers
//     per thread); the epilogue adds the bias, applies ReLU, splits the value into a 16-bit hi part and
//     a 16-bit lo part and writes both into shared memory in the SWIZZLE_NONE K-major canonical layout,
//     where the next layer's wgmmas read them as the A operand.  The consumers' layer schedule is unrolled at
//     compile time: chunk sources, offsets and accumulators are constants, and the first wgmma of a (layer, half)
//     writes its accumulator without reading it (scale-d = 0).  The epilogue runs in 32-column blocks, each one
//     K chunk of the next layer's input, interleaved with the wgmmas still in flight (see trunk_layer);
//   * weights stream from L2 through a shared-memory ring of chunks (128 output rows x 32 K x {hi, lo};
//     4 stages in the split modes, 18 in the single-product modes) with cp.async.bulk (1-D TMA) + mbarrier
//     complete_tx, issued by one producer thread that runs ahead over all of the CTA's tiles; the consumers only wait on
//     `full` and release stages.  The packed image is laid out in exactly the order the warpgroups consume
//     it, in the same canonical layout, so a chunk is one contiguous copy;
//   * fp32 parity (SNB_PREC_F16X3 / BF16X3): x*w ~= xh*wh + xl*wh + xh*wl, three wgmmas per K step
//     with fp32 accumulation -- 22 (fp16) or 16 (bf16) significand bits per operand;
//     SNB_PREC_BF16 and SNB_PREC_F16 are the single product (fp16 operands saturate at +-65504);
//   * positional encodings (63->64, 27->32 columns) are computed into shared memory in the canonical
//     layout and consumed at layers 1, 5 (skip) and the direction layer, so neither concat exists; the
//     xyz encoding is written at the start of a tile, the direction encoding over it once the skip
//     layer's (l = 4) enc chunks have retired; two threads per row share a row's channels;
//   * biases and head weights are read from the image through L1, not staged in shared memory;
//   * sigma (256->1) and rgb (128->3) heads are fp32 dot products inside the epilogue (quad shuffles
//     combine the columns a thread's neighbours hold);
//   * the bottleneck layer (256->256, no activation, nerf.py:140) is folded into the direction layer at
//     pack time: Wd[:, :256] (Wf h + bf) = (Wd[:, :256] Wf) h + Wd[:, :256] bf -- one 256-wide layer
//     (11 % of the MMA work) less per point, same function up to fp32 rounding.
//
// kTrain (snb_field_forward_train / _train16): the same kernel also writes the embeddings and every
// layer's post-activation output for the backward -- fp32 row-major (kTrain = 1) or fp16 cells of the
// T32 layout + ReLU mask words (kTrain = 2, act16.cuh).
//
// Roofline: tensor pipe.  Executed MMA FLOPs are 3x the algorithmic 1 186 816 FLOP/point in the
// split modes.  HBM traffic: 4 B/point in (z) + 16 B/point out; weights (2.2 MB per tile pass)
// are L2 hits.
#include <stddef.h>
#include <stdlib.h>

#include <type_traits>
#include <utility>

#include "act16.cuh"
#include "common.cuh"
#include "wgmma.cuh"

namespace snb {
using namespace wg;

// ------------------------------------------------------------------ geometry
constexpr int kTile = 128;             // points per CTA tile
constexpr int kNh = 128;               // output columns per wgmma (N); a 256-wide layer is two halves
constexpr int kKc = 32;                // K per weight chunk
constexpr uint32_t kStepBytes = kNh * 16 * 2;   // one K16 step of one of {hi, lo} of a chunk
constexpr int kWgs = 2;                // consumer warpgroups, 64 tile rows each
constexpr int kThreads = (kWgs + 1) * 128;   // + one producer warpgroup
constexpr int kProducerRegs = 24, kConsumerRegs = 240;   // setmaxnreg: 128 x 24 + 256 x 240 <= 64 K registers
static_assert(128 * kProducerRegs + kWgs * 128 * kConsumerRegs <= 65536, "register file");
constexpr size_t kSmemOptIn = 232448;  // opt-in dynamic shared memory per block on sm_90

enum { SRC_ENC = 0, SRC_HID = 1, SRC_DIR = 2 };

struct alignas(16) Chunk {
  uint8_t layer;     // 0..9 (8 = bottleneck, 9 = direction layer)
  uint8_t half;      // output columns [128*half, +128)
  uint8_t src;       // SRC_*: where the A operand of this chunk lives
  uint8_t a16;       // K offset of the chunk inside that source, in K16 steps
  uint8_t w16;       // K offset in the layer's padded weight K space (gemm_k), in K16 steps
  uint8_t steps;     // K16 steps in this chunk
  uint8_t first;     // first chunk of this (layer, half): accumulate = 0
  uint8_t pad;
  uint16_t off;      // K16 steps of all earlier chunks: byte offset in the image = off * step bytes
  uint16_t pad2;
};
constexpr int kMaxChunks = 160;
struct ChunkTable {
  Chunk c[kMaxChunks];
  int n_total;       // chunks per tile, full head
  int n_sigma_only;  // chunks per tile through layer 8
  int steps_total;   // sum of steps
};

// order inside a layer: half a (enc, hid, dir segments in K order) | half b (same)
__host__ __device__ constexpr ChunkTable make_chunk_table() {
  ChunkTable t{};
  int n = 0, off = 0;
  for (int l = 0; l < kNumGemm; ++l) {
    if (l == 8) continue;   // bottleneck: folded into the direction layer's weights (pack_tc_kernel)
    const bool has_enc = (l == 0 || l == 4);
    const bool has_hid = (l != 0);
    const int n_halves = l == 9 ? 1 : 2;
    for (int half = 0; half < n_halves; ++half) {
      bool first = true;
      // segments of this (layer, half): [enc 64] [hid 256] [dir 32]
      for (int seg = 0; seg < 3; ++seg) {
        const int src = seg == 0 ? SRC_ENC : (seg == 1 ? SRC_HID : SRC_DIR);
        const int klen = seg == 0 ? (has_enc ? kXyzPad : 0) : (seg == 1 ? (has_hid ? kWidth : 0) : (l == 9 ? kDirPad : 0));
        const int wbase = seg == 0 ? 0 : (seg == 1 ? (has_enc ? kXyzPad : 0) : kWidth);   // padded weight K offset
        for (int k0 = 0; k0 < klen; k0 += kKc) {
          const int kc = klen - k0 < kKc ? klen - k0 : kKc;
          Chunk c{};
          c.layer = l; c.half = half; c.src = src; c.a16 = k0 / 16; c.w16 = (wbase + k0) / 16; c.steps = kc / 16;
          c.first = first; c.off = off;
          t.c[n++] = c;
          off += c.steps;
          first = false;
        }
      }
    }
    if (l == 7) t.n_sigma_only = n;
  }
  t.n_total = n;
  t.steps_total = off;
  return t;
}
__constant__ ChunkTable c_chunks = make_chunk_table();
static constexpr ChunkTable h_chunks = make_chunk_table();
static_assert(h_chunks.n_total == 129 && h_chunks.n_sigma_only == 120, "chunk schedule (K32)");
static_assert(h_chunks.steps_total == 258, "K16 steps per tile");
// first chunk and number of chunks of (layer, half) in the schedule
__host__ __device__ constexpr int chunk_index(int l, int half) {
  for (int i = 0; i < h_chunks.n_total; ++i)
    if (h_chunks.c[i].layer == l && h_chunks.c[i].half == half) return i;
  return -1;
}
__host__ __device__ constexpr int chunk_count(int l, int half) {
  int n = 0;
  for (int i = 0; i < h_chunks.n_total; ++i) n += h_chunks.c[i].layer == l && h_chunks.c[i].half == half;
  return n;
}
static_assert(chunk_count(4, 0) == 10 && chunk_count(9, 0) == 9 && chunk_count(9, 1) == 0, "chunk schedule");
// layers 1-3, 5 and 6 consume their chunks exactly like layer 1 (only the image offsets differ), so the consumers
// run them with one copy of layer 1's code
__host__ __device__ constexpr bool same_schedule_as_layer1(int l) {
  for (int h = 0; h < 2; ++h) {
    if (chunk_count(l, h) != chunk_count(1, h)) return false;
    for (int i = 0; i < chunk_count(1, h); ++i) {
      const Chunk a = h_chunks.c[chunk_index(1, h) + i], b = h_chunks.c[chunk_index(l, h) + i];
      if (a.half != b.half || a.src != b.src || a.a16 != b.a16 || a.steps != b.steps || a.first != b.first) return false;
    }
  }
  return true;
}
static_assert(same_schedule_as_layer1(2) && same_schedule_as_layer1(3) && same_schedule_as_layer1(5) &&
              same_schedule_as_layer1(6), "plain layers share layer 1's schedule");
// chunks of (l, 1) that read the xyz encoding; they come first
__host__ __device__ constexpr int enc_chunks(int l) {
  int n = 0;
  for (int i = 0; i < chunk_count(l, 1); ++i) n += h_chunks.c[chunk_index(l, 1) + i].src == SRC_ENC;
  return n;
}
// the consumers run each trunk layer's epilogue in four 32-column blocks under the wgmmas (field_tc_kernel): a
// layer's half-0 chunks 0-3 read only enc or hid blocks 0-3, and chunk e + b of its half 1 reads hid block b
__host__ __device__ constexpr bool epilogue_blocks_fit(int l, bool check_half1) {
  for (int b = 0; b < 4; ++b) {
    const Chunk a = h_chunks.c[chunk_index(l, 0) + b];
    if (a.src == SRC_DIR || (a.src == SRC_HID && a.a16 >= 8)) return false;
    if (!check_half1) continue;
    const Chunk c = h_chunks.c[chunk_index(l, 1) + enc_chunks(l) + b];
    if (c.src != SRC_HID || c.a16 != 2 * b) return false;
  }
  return true;
}
static_assert(kKc == 32 && epilogue_blocks_fit(1, true) && epilogue_blocks_fit(4, true) && epilogue_blocks_fit(7, true) &&
              epilogue_blocks_fit(9, false) && chunk_count(1, 0) >= 4 && chunk_count(1, 1) == enc_chunks(1) + 8 &&
              chunk_count(4, 1) == enc_chunks(4) + 8 && chunk_count(0, 1) == enc_chunks(0),
              "epilogue blocks of 32 columns interleave with the next layer's chunks");

// ------------------------------------------------------------------ packed image
// [PackedHeader 256 B][consts: biases + head weights, fp32][chunk 0][chunk 1]...
struct ConstLayout {
  int b[kNumGemm];
  int sigma_w, sigma_b, rgb_w, rgb_b, total;
};
__host__ __device__ constexpr ConstLayout make_const_layout() {
  ConstLayout L{};
  int off = 0;
  for (int l = 0; l < kNumGemm; ++l) { L.b[l] = off; off += gemm_n(l); }
  L.sigma_w = off; off += kWidth;
  L.sigma_b = off; off += 4;
  L.rgb_w = off; off += 3 * kHalf;
  L.rgb_b = off; off += 4;
  L.total = (off + 63) & ~63;
  return L;
}
constexpr int kConstFloats = make_const_layout().total;
__host__ __device__ constexpr bool trunk_biases_strided() {   // the trunk epilogue computes CL.b[l] as l * kWidth
  for (int l = 0; l < 8; ++l)
    if (make_const_layout().b[l] != l * kWidth) return false;
  return true;
}
static_assert(trunk_biases_strided(), "trunk layer l's bias starts at l * kWidth in the image's constants");
constexpr size_t kConstBytes = (size_t)kConstFloats * 4;

__host__ __device__ constexpr bool prec_split(int precision) {
  return precision != SNB_PREC_BF16 && precision != SNB_PREC_F16;
}
// image bytes of one K16 step of a chunk (hi and lo): 128 rows x 16 K x 2 B (x2)
__host__ __device__ constexpr uint32_t step_image_bytes(int precision) {
  return (uint32_t)(kNh * 16 * 2 * (prec_split(precision) ? 2 : 1));
}
// scratch at the end of the image: W' = Wd[:, :256] Wf (128 x 256) and b' = bd + Wd[:, :256] bf (128)
constexpr size_t kFusedFloats = (size_t)kHalf * kWidth + kHalf;
__host__ __device__ constexpr size_t chunks_bytes(int precision) {
  return (size_t)make_chunk_table().steps_total * step_image_bytes(precision);
}
size_t tc_packed_bytes(int precision) {
  return sizeof(PackedHeader) + kConstBytes + chunks_bytes(precision) + kFusedFloats * sizeof(float);
}

// lambdas of the unrolled consumer schedule must inline: an accumulator array passed to an out-of-line call would
// live in local memory
#define SNB_INLINE __attribute__((always_inline))

template <class F, int... I>
__device__ __forceinline__ void static_for_impl(F&& f, std::integer_sequence<int, I...>) {
  (f(std::integral_constant<int, I>{}), ...);
}
template <int N, class F>
__device__ __forceinline__ void static_for(F&& f) { static_for_impl(f, std::make_integer_sequence<int, N>{}); }
template <int N>
using Int = std::integral_constant<int, N>;

// A read-only float2 from global memory as a volatile load, so the front end does not hoist an epilogue's bias loads
// into the preceding MMA issue, where their registers push other values out to local memory.  (ptxas still moves
// some of them up; DESIGN.md §4.1 lists the spills that remain.)
__device__ __forceinline__ float2 ldg_f2_here(const float* p) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(p));
  return v;
}

// 16-bit conversions -------------------------------------------------------------------
template <bool kBf16>
__device__ __forceinline__ uint16_t cvt16(float x) {
  if (kBf16) return __bfloat16_as_ushort(__float2bfloat16_rn(x));
  return __half_as_ushort(__float2half_rn(x));
}
template <bool kBf16>
__device__ __forceinline__ float up16(uint16_t h) {
  if (kBf16) return __bfloat162float(__ushort_as_bfloat16(h));
  return __half2float(__ushort_as_half(h));
}
// x -> (hi, lo) with hi + lo ~= x.  fp16 saturates at +-65504 instead of overflowing to inf.
template <bool kBf16>
__device__ __forceinline__ void split16(float x, uint16_t& hi, uint16_t& lo) {
  if (!kBf16) x = fminf(fmaxf(x, -65504.f), 65504.f);
  hi = cvt16<kBf16>(x);
  lo = cvt16<kBf16>(x - up16<kBf16>(hi));
}

// Two values at once, with the packed converts (F2FP.*.PACK_AB, full-rate pipe) instead of four
// scalar F2F (quarter-rate MIO pipe): hi = pack(x0, x1); lo = pack(x0 - up(hi.x), x1 - up(hi.y)).
template <bool kBf16, bool kSplit, bool kNonNeg = false>
__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  if (kBf16) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    if (kSplit) {
      const float b0 = __uint_as_float(hi << 16), b1 = __uint_as_float(hi & 0xffff0000u);
      const __nv_bfloat162 l = __floats2bfloat162_rn(x0 - b0, x1 - b1);
      lo = *reinterpret_cast<const uint32_t*>(&l);
    } else {
      lo = 0;
    }
  } else {
    if (kNonNeg) { x0 = fminf(x0, 65504.f); x1 = fminf(x1, 65504.f); }   // ReLU output: one-sided
    else { x0 = fminf(fmaxf(x0, -65504.f), 65504.f); x1 = fminf(fmaxf(x1, -65504.f), 65504.f); }
    const __half2 h = __floats2half2_rn(x0, x1);
    hi = *reinterpret_cast<const uint32_t*>(&h);
    if (kSplit) {
      const float2 b = __half22float2(h);
      const __half2 l = __floats2half2_rn(x0 - b.x, x1 - b.y);
      lo = *reinterpret_cast<const uint32_t*>(&l);
    } else {
      lo = 0;
    }
  }
}

// ReLU + split of two PRE-activation values with no separate max / clamp instructions: the packed converts
// carry .relu and .satfinite themselves.  hi = relu(x) rounded TOWARD ZERO, so the residual x - hi is >= 0
// whenever x >= 0 and negative only when x < 0 (hi = 0) -- then lo = rn(relu(residual)) is 0, as it must be.
// (Truncation leaves a residual of up to one ulp of hi instead of half: hi + lo still carries 21 (fp16) /
// 15 (bf16) significand bits.)  4 + 2 instructions per pair instead of 8 + 2.
template <bool kBf16, bool kSplit>
__device__ __forceinline__ void split_pair_relu(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  if (kBf16) {
    if (kSplit) asm("cvt.rz.relu.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    else asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    if (kSplit) {
      const float r0 = x0 - __uint_as_float(hi << 16), r1 = x1 - __uint_as_float(hi & 0xffff0000u);
      asm("cvt.rn.relu.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
    } else {
      lo = 0;
    }
  } else {
    if (kSplit) asm("cvt.rz.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    else asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));
    if (kSplit) {
      const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&hi));
      const float r0 = x0 - b.x, r1 = x1 - b.y;
      asm("cvt.rn.relu.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
    } else {
      lo = 0;
    }
  }
}

// softplus(x - 1) with the hardware ex2 / lg2 approximations (abs error ~1e-7 on an O(1..200)
// value; the accurate expf/log1pf pair cost the dir-layer epilogue ~10k cycles per tile).
// `s` is already shifted (x - 1): 4 FP32 ops + 2 MUFU.
__device__ __forceinline__ float softplus_fast(float s) {
  float t;                                                             // exp(-|s|) in (0, 1]
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(-1.4426950408889634f * fabsf(s)));
  return fmaf(__log2f(1.0f + t), 0.6931471805599453f, fmaxf(s, 0.0f));   // max(s,0) + log1p(t)  (lg2.approx)
}

// sin / cos for the positional encoding of the single-product modes: two-constant Cody-Waite reduction to
// [-pi, pi] and the MUFU approximations (abs error ~1e-6 for |x| up to ~1e4 -- three orders below bf16's 2^-9 and
// two below fp16's 2^-11 rounding of the encoded value), ~8 instructions instead of sincosf's ~50; the encoding of a
// tile sits between two tiles' MMAs.  The fp32-parity modes keep the accurate sincosf.
__device__ __forceinline__ void sincos_fast(float x, float* sn, float* cs) {
  const float k = rintf(x * 0.15915494309189535f);
  float r = fmaf(k, -6.2831854820251465f, x);
  r = fmaf(k, 1.7484555e-7f, r);
  *sn = __sinf(r);
  *cs = __cosf(r);
}
// ------------------------------------------------------------------ pack kernel

// W'[n][k] = sum_j Wd[n][j] Wf[j][k],  b'[n] = bd[n] + sum_j Wd[n][j] bf[j]   (double accumulation)
__global__ void fuse_bottleneck_kernel(ParamPtrs pp, float* fused, const PackedHeader* hdr, int only_if_dirty) {
  if (only_if_dirty && !hdr->dirty) return;
  const float* Wd = pp.p[18];   // (128, 283)
  const float* Wf = pp.p[16];   // (256, 256)
  const float* bf = pp.p[17];
  const float* bd = pp.p[19];
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < kHalf * (kWidth + 1); e += gridDim.x * blockDim.x) {
    const int n = e / (kWidth + 1), k = e - n * (kWidth + 1);
    double acc = k == kWidth ? (double)bd[n] : 0.0;
    for (int j = 0; j < kWidth; ++j) acc += (double)Wd[n * 283 + j] * (double)(k == kWidth ? bf[j] : Wf[j * kWidth + k]);
    if (k == kWidth) fused[kHalf * kWidth + n] = (float)acc;
    else fused[n * kWidth + k] = (float)acc;
  }
}

template <bool kBf16, bool kSplit>
__global__ void pack_tc_kernel(ParamPtrs pp, int precision, int new_activation, unsigned char* image, int only_if_dirty) {
  constexpr ConstLayout CL = make_const_layout();
  const ChunkTable& tab = c_chunks;
  PackedHeader* hdr = reinterpret_cast<PackedHeader*>(image);
  if (only_if_dirty && !hdr->dirty) return;
  float* cst = reinterpret_cast<float*>(image + sizeof(PackedHeader));
  unsigned char* chunks = image + sizeof(PackedHeader) + kConstBytes;
  const float* fused = reinterpret_cast<const float*>(chunks + chunks_bytes(precision));   // fuse_bottleneck_kernel
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x, gsz = gridDim.x * blockDim.x;
  if (gtid == 0) {
    hdr->magic = kMagic;
    hdr->precision = precision;
    hdr->new_activation = new_activation;
    hdr->cta_group = 1;
  }
  for (int e = gtid; e < kConstFloats; e += gsz) {
    float v = 0.f;
    if (e < CL.sigma_w) {
      int l = 0;
      while (l + 1 < kNumGemm && e >= CL.b[l + 1]) ++l;
      v = l == 9 ? fused[kHalf * kWidth + (e - CL.b[l])] : pp.p[param_weight_index(l) + 1][e - CL.b[l]];
    } else if (e < CL.sigma_b) v = pp.p[kSigmaW][e - CL.sigma_w];
    else if (e == CL.sigma_b) v = pp.p[kSigmaB][0];
    else if (e >= CL.rgb_w && e < CL.rgb_b) v = pp.p[kRgbW][e - CL.rgb_w];
    else if (e >= CL.rgb_b && e < CL.rgb_b + 3) v = pp.p[kRgbB][e - CL.rgb_b];
    cst[e] = v;
  }
  // chunk image: [hi | lo]; each of hi / lo is the canonical (SWIZZLE_NONE, K-major) block
  // [k8][128 rows][8 elements] of the chunk's 16*steps K columns
  constexpr int kParts = kSplit ? 2 : 1;
  const int total = tab.steps_total * kNh * 16;
  for (int e = gtid; e < total; e += gsz) {
    const int gstep = e / (kNh * 16), rem = e - gstep * (kNh * 16);
    const int r = rem >> 4, k16 = rem & 15;
    int ci = 0;
    while (ci + 1 < tab.n_total && gstep >= tab.c[ci + 1].off) ++ci;
    const Chunk c = tab.c[ci];
    const int kk = (gstep - c.off) * 16 + k16;       // K index inside the chunk
    const int l = c.layer;
    const int n = c.half * kNh + r;
    const int kpad = c.w16 * 16 + kk;
    const int col = kpad < gemm_k(l) ? gemm_src_col(l, kpad) : -1;
    const int src_k = l == 0 ? 63 : (l == 4 ? 319 : (l == 9 ? 283 : 256));
    float w = col >= 0 ? pp.p[param_weight_index(l)][n * src_k + col] : 0.f;
    if (l == 9 && kpad < kWidth) w = fused[n * kWidth + kpad];     // direction layer sees h8 through W'
    const uint32_t part = kStepBytes * c.steps;                   // bytes of one of {hi, lo} of a chunk
    unsigned char* base = chunks + (size_t)c.off * (kStepBytes * kParts);
    const uint32_t off = (uint32_t)(kk >> 3) * (kNh * 16) + r * 16 + (kk & 7) * 2;
    if (kSplit) {
      uint16_t hi, lo;
      split16<kBf16>(w, hi, lo);
      *reinterpret_cast<uint16_t*>(base + off) = hi;
      *reinterpret_cast<uint16_t*>(base + part + off) = lo;
    } else {
      if (!kBf16) w = fminf(fmaxf(w, -65504.f), 65504.f);   // fp16 saturates instead of overflowing, as in split16
      *reinterpret_cast<uint16_t*>(base + off) = cvt16<kBf16>(w);
    }
  }
}

int launch_pack_tc(const float* const* params, int precision, int new_activation, void* image, int only_if_dirty,
                   cudaStream_t st) {
  ParamPtrs pp;
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) pp.p[i] = params[i];
  unsigned char* img = reinterpret_cast<unsigned char*>(image);
  if (precision < SNB_PREC_F16X3 || precision > SNB_PREC_F16)
    return fail(SNB_ERR_INVALID, "launch_pack_tc: precision %d is not a tensor-core mode", precision);
  float* fused = reinterpret_cast<float*>(img + sizeof(PackedHeader) + kConstBytes + chunks_bytes(precision));
  fuse_bottleneck_kernel<<<132, 256, 0, st>>>(pp, fused, reinterpret_cast<const PackedHeader*>(img), only_if_dirty);
  if (int rc = check_launch("fuse_bottleneck_kernel")) return rc;
  if (precision == SNB_PREC_F16X3) pack_tc_kernel<false, true><<<264, 256, 0, st>>>(pp, precision, new_activation, img, only_if_dirty);
  else if (precision == SNB_PREC_BF16X3) pack_tc_kernel<true, true><<<264, 256, 0, st>>>(pp, precision, new_activation, img, only_if_dirty);
  else if (precision == SNB_PREC_BF16) pack_tc_kernel<true, false><<<264, 256, 0, st>>>(pp, precision, new_activation, img, only_if_dirty);
  else pack_tc_kernel<false, false><<<264, 256, 0, st>>>(pp, precision, new_activation, img, only_if_dirty);
  return check_launch("pack_tc_kernel");
}

// ------------------------------------------------------------------ shared memory
// The direction encoding has no buffer of its own: it is written over the first kDirPad columns of `enc` once the
// layer-4 wgmmas (the last reader of the xyz encoding) have retired.  Biases and head weights are read from the
// image (__ldg), not staged.  The ring takes every stage that fits in what is left.
template <bool kSplit>
struct TcSmem {
  static constexpr int kParts = kSplit ? 2 : 1;
  static constexpr uint32_t kStageBytes = kStepBytes * (kKc / 16) * kParts;   // one full chunk
  static constexpr size_t kActBytes = (size_t)kParts * kTile * (kWidth + kXyzPad) * 2;
  static constexpr int kStages = (int)((kSmemOptIn - 128 - kActBytes) / (kStageBytes + 2 * sizeof(uint64_t)));
  alignas(128) unsigned char ring[kStages][kStageBytes];
  alignas(128) unsigned char hid[kParts][kTile * kWidth * 2];    // canonical [k8][row][8] hi (, lo)
  alignas(128) unsigned char enc[kParts][kTile * kXyzPad * 2];   // xyz encoding, then the direction encoding
  uint64_t full[kStages], empty[kStages];
};
static_assert(kDirPad <= kXyzPad, "the direction encoding fits in the xyz encoding's buffer");
static_assert(sizeof(TcSmem<true>) + 128 <= kSmemOptIn && sizeof(TcSmem<false>) + 128 <= kSmemOptIn, "shared memory");
static_assert(TcSmem<true>::kStages >= 4 && TcSmem<false>::kStages >= 6, "weight ring depth");

struct TcParams {
  const unsigned char* image;
  const float* rays;
  const float* z;
  int n_samples;
  const float* x;          // embedded input rows (standalone NeRF.forward)
  long long x_stride;
  long long n_points;
  int sigma_only;
  float* out;
  // training forward (kTrain): what the backward needs, row-major fp32 (snb_field_forward_train)
  float* save_enc;         // (P,64)
  float* save_dir;         // (P,32)
  float* save_h;           // (8,P,256)
  float* save_g;           // (P,128)
  // training forward, 16-bit storage (kTrain == 2): sections of the act16 buffer (act16.cuh)
  unsigned char* a_enc;    // (Ppad,64)  fp16 T32
  unsigned char* a_dir;    // (Ppad,32)
  unsigned char* a_h;      // 8 x (Ppad,256)
  unsigned char* a_g;      // (Ppad,128)
  uint32_t* a_mask;        // (8, 8, Ppad)
  long long ppad;
};

// kTrain: 0 = inference, 1 = training forward keeping fp32 row-major activations (snb_field_forward_train),
//         2 = training forward keeping fp16 activations in the T32 layout + ReLU mask words (act16.cuh)
template <bool kBf16, bool kSplit, bool kEmbedded, int kTrain = 0>
__global__ void __launch_bounds__(kThreads, 1) field_tc_kernel(TcParams p) {
  static_assert(!(kTrain != 0 && kEmbedded), "the training forward is the fused (rays, z) entry only");
  using Smem = TcSmem<kSplit>;
  extern __shared__ unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  constexpr ConstLayout CL = make_const_layout();
  constexpr int kStages = Smem::kStages;
  constexpr int kParts = Smem::kParts;
  const ChunkTable& tab = c_chunks;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const PackedHeader* hdr = reinterpret_cast<const PackedHeader*>(p.image);
  const int new_activation = hdr->new_activation;
  const float* g_cst = reinterpret_cast<const float*>(p.image + sizeof(PackedHeader));
  const unsigned char* g_chunks = p.image + sizeof(PackedHeader) + kConstBytes;
  const long long ntiles = (p.n_points + kTile - 1) / kTile;
  const int n_chunks = p.sigma_only ? tab.n_sigma_only : tab.n_total;

  if (tid == 0) {
    for (int i = 0; i < kStages; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], kWgs * 4); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kWgs * 4) {
    // ======================= producer warpgroup: one thread keeps the ring kStages chunks ahead of consumption
    // over all of the CTA's tiles; a stage is refilled once all eight consumer warps have released it.  No
    // consumer thread ever waits on `empty`.
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kWgs * 4 && elect_one()) {
      const long long my_tiles = ntiles > (long long)blockIdx.x ? (ntiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
      const long long n_loads = my_tiles * n_chunks;
      uint32_t st = 0, ph = 0;
      int ci = 0;
      for (long long i = 0; i < n_loads; ++i) {
        mbar_wait(&s.empty[st], ph ^ 1);
        const Chunk c = tab.c[ci];
        const uint32_t bytes = kStepBytes * kParts * c.steps;
        mbar_arrive_expect_tx(&s.full[st], bytes);
        bulk_g2s(s.ring[st], g_chunks + (size_t)c.off * (kStepBytes * kParts), bytes, &s.full[st]);
        if (++ci == n_chunks) ci = 0;
        if (++st == kStages) { st = 0; ph ^= 1; }
      }
    }
    return;
  }
  setmaxnreg_inc<kConsumerRegs>();

  // ======================= consumer warpgroups =======================
  // The layer schedule is unrolled at compile time: every chunk's A source, K offset, step count and accumulator
  // register set are constants, and a layer's first wgmma (scale-d = 0) is the only write of its accumulator.
  const int wgi = warp >> 2, wq = warp & 3, tq = lane & 3;
  const int r0 = wgi * 64 + wq * 16 + (lane >> 2);   // tile rows of this thread's accumulator fragments: r0, r0 + 8
  auto wg_sync = [&]() { named_bar_sync(1 + wgi, 128); };
  constexpr uint32_t kHidPart = kTile * kWidth * 2, kEncPart = kTile * kXyzPad * 2;   // bytes of one of {hi, lo}
  // shared-window addresses are one base plus compile-time offsets, so they cost few registers
  constexpr uint32_t kOffRing = offsetof(Smem, ring), kOffHid = offsetof(Smem, hid), kOffEnc = offsetof(Smem, enc);
  const uint32_t sbase = smem_u32(&s);
  const uint32_t a_wg = sbase + wgi * 64 * 16;              // this warpgroup's A rows (+ kOffHid / kOffEnc)
  // this thread's first epilogue word, (row r0, column 2 tq): the canonical [k8][row][8] layout puts (row, k) at byte
  // (k >> 3) * (kTile * 16) + row * 16 + (k & 7) * 2
  const uint32_t hid_thr = sbase + kOffHid + r0 * 16 + tq * 4;
  // encodings: the tile row and the half of its channels this thread computes (all 128 threads of a warpgroup)
  const int er = wgi * 64 + (tid & 63), epart = (tid >> 6) & 1;

  // 16-bit storage: 8 consecutive features of one point -> one 16-byte cell of a T32 tensor
  auto store_cell16 = [&](unsigned char* base, long long pt, int f8, int F, const float (&v)[8]) SNB_INLINE {
    if (pt >= p.ppad) return;
    const bool live = pt < p.n_points;
    uint4 c;
    c.x = live ? pack_half2_sat(v[0], v[1]) : 0u; c.y = live ? pack_half2_sat(v[2], v[3]) : 0u;
    c.z = live ? pack_half2_sat(v[4], v[5]) : 0u; c.w = live ? pack_half2_sat(v[6], v[7]) : 0u;
    *reinterpret_cast<uint4*>(base + a16_cell(pt, f8, F)) = c;
  };

  // the encoder thread's ray (o, d) and sample depth, loaded one tile ahead (before the direction layer of the
  // previous tile) so the HBM latency hides under that layer's MMAs
  struct RowIn { float4 q0, q1; float z; };
  RowIn in{};
  auto load_row = [&](long long tile) SNB_INLINE {
    const long long pt = tile * kTile + er;
    if (!kEmbedded && tile < ntiles && pt < p.n_points) {
      const long long ray = pt / p.n_samples;
      in.q0 = *reinterpret_cast<const float4*>(p.rays + ray * 8);
      in.q1 = *reinterpret_cast<const float4*>(p.rays + ray * 8 + 4);
      in.z = p.z[pt];
    }
  };
  // positional encoding of tile row er, channels [32 P, 32 P + 32) of the xyz encoding (Embedding(3, 10) of
  // o + d z) or [16 P, 16 P + 16) of the direction encoding (Embedding(3, 4) of d)
  auto encode = [&](auto ltag, auto ptag, long long tile) SNB_INLINE {
    constexpr int L = decltype(ltag)::value, P = decltype(ptag)::value;
    constexpr bool kXyz = L == SNB_XYZ_FREQS;
    constexpr int kCh = 3 * (2 * L + 1), kPad = (kCh + 7) / 8 * 8, kK8 = kPad / 16;   // k8 groups per thread
    constexpr int c_lo = 8 * kK8 * P, c_hi = 8 * kK8 * (P + 1);
    const long long pt = tile * kTile + er;
    const bool live = pt < p.n_points;
    float v[kPad];
#pragma unroll
    for (int j = 0; j < kPad; ++j) v[j] = 0.f;
    if (kEmbedded) {
      const float* xr = p.x + pt * p.x_stride;
      const int nin = p.sigma_only ? kXyzCh : kXyzCh + kDirCh;
#pragma unroll
      for (int j = c_lo; j < (c_hi < kCh ? c_hi : kCh); ++j) {
        const int col = kXyz ? j : kXyzCh + j;
        v[j] = (live && col < nin) ? xr[col] : 0.f;
      }
    } else {
      float x[3] = {0.f, 0.f, 0.f};
      if (live) {
        if (kXyz) {
          x[0] = __fadd_rn(in.q0.x, __fmul_rn(in.q0.w, in.z));   // rendering.py:284-285 rounding
          x[1] = __fadd_rn(in.q0.y, __fmul_rn(in.q1.x, in.z));
          x[2] = __fadd_rn(in.q0.z, __fmul_rn(in.q1.y, in.z));
        } else {
          x[0] = in.q0.w; x[1] = in.q1.x; x[2] = in.q1.y;      // ray direction (not normalised, rendering.py:261)
        }
      }
      v[0] = x[0]; v[1] = x[1]; v[2] = x[2];
#pragma unroll
      for (int f = 0; f < L; ++f)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int cs = 3 + 6 * f + c, cc = cs + 3;     // channels of sin and cos
          if ((cs >= c_lo && cs < c_hi) || (cc >= c_lo && cc < c_hi)) {
            float sn, cs_;
            if (kSplit) sincosf(x[c] * (float)(1 << f), &sn, &cs_);
            else sincos_fast(x[c] * (float)(1 << f), &sn, &cs_);
            v[cs] = sn;
            v[cc] = cs_;
          }
        }
    }
    static_for<kK8>([&](auto ktag) SNB_INLINE {
      constexpr int k8 = kK8 * P + decltype(ktag)::value;
      const float v8[8] = {v[8 * k8], v[8 * k8 + 1], v[8 * k8 + 2], v[8 * k8 + 3], v[8 * k8 + 4], v[8 * k8 + 5], v[8 * k8 + 6], v[8 * k8 + 7]};
      if (!kEmbedded) {
        if (kTrain == 1 && live) {
          float4* dst = reinterpret_cast<float4*>((kXyz ? p.save_enc + pt * kXyzPad : p.save_dir + pt * kDirPad) + k8 * 8);
          dst[0] = make_float4(v8[0], v8[1], v8[2], v8[3]); dst[1] = make_float4(v8[4], v8[5], v8[6], v8[7]);
        }
        if (kTrain == 2) store_cell16(kXyz ? p.a_enc : p.a_dir, pt, k8, kXyz ? kXyzPad : kDirPad, v8);
      }
      uint32_t h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split_pair<kBf16, kSplit>(v8[2 * j], v8[2 * j + 1], h[j], l[j]);
      const uint32_t a = sbase + kOffEnc + k8 * (kTile * 16) + er * 16;
      st_shared_v4(a, h[0], h[1], h[2], h[3]);
      if (kSplit) st_shared_v4(a + kEncPart, l[0], l[1], l[2], l[3]);
    });
  };
  auto encode_rows = [&](auto ltag, long long tile) SNB_INLINE {
    if (epart == 0) encode(ltag, std::integral_constant<int, 0>{}, tile);
    else encode(ltag, std::integral_constant<int, 1>{}, tile);
  };

  auto mma = [&](float (&d)[64], uint64_t a, uint64_t b, bool first) SNB_INLINE {
    if (first) {                 // accumulate = 0, D write-only
      if (kBf16) wgmma_m64n128_bf16_first(d, a, b);
      else wgmma_m64n128_f16_first(d, a, b);
    } else {
      if (kBf16) wgmma_m64n128_bf16(d, a, b, 1u);
      else wgmma_m64n128_f16(d, a, b, 1u);
    }
  };
  // K16 step of a chunk into accumulator d: hi*hi (+ lo*hi + hi*lo); `first` starts the (layer, half)
  auto issue_step = [&](float (&d)[64], uint32_t ah, uint32_t al, uint32_t bh, uint32_t bl, bool first) SNB_INLINE {
    const uint64_t da_h = make_smem_desc(ah, kTile * 16, 128), db_h = make_smem_desc(bh, kNh * 16, 128);
    mma(d, da_h, db_h, first);
    if (kSplit) {
      mma(d, make_smem_desc(al, kTile * 16, 128), db_h, false);
      mma(d, da_h, make_smem_desc(bl, kNh * 16, 128), false);
    }
  };

  constexpr bool kDrained = kTrain != 0;   // the training forward keeps the drained schedule (trunk_layer)
  float acc[2][64];              // a layer's two N = 128 halves
  float sig[2] = {0.f, 0.f};     // sigma of rows r0, r0 + 8 (layer 7's epilogue -> the direction layer's)

  // Ring position of the next chunk.  Chunks are consumed in exactly the producer's order; the stage of chunk i is
  // released once the wgmmas of chunk i + 1 are committed and chunk i's have retired (or at the tile's drain).
  uint32_t st = 0, ph = 0;
  auto prev_stage = [&]() { return st == 0 ? (uint32_t)kStages - 1 : st - 1; };
  // chunk ci of the schedule into the accumulator of its half; on return only its own wgmmas may still be in flight
  auto issue = [&](auto ctag) SNB_INLINE {
    constexpr int ci = decltype(ctag)::value;
    constexpr Chunk c = h_chunks.c[ci];
    float (&d)[64] = acc[c.half];
    mbar_wait(&s.full[st], ph);
    wgmma_fence();
    const uint32_t bh = sbase + kOffRing + st * Smem::kStageBytes, bl = bh + kStepBytes * c.steps;
    // the A base goes through an opaque move: otherwise the compiler computes the descriptors of every chunk once,
    // shares them between layers (they repeat) and keeps them live across the tile, out of the accumulators' registers
    uint32_t abase;
    asm volatile("mov.b32 %0, %1;" : "=r"(abase) : "r"(a_wg));
    const uint32_t ah = abase + (c.src == SRC_HID ? kOffHid : kOffEnc) + c.a16 * 2 * (kTile * 16);
    constexpr uint32_t part = c.src == SRC_HID ? kHidPart : kEncPart;
    static_for<c.steps>([&](auto ktag) SNB_INLINE {
      constexpr int ks = decltype(ktag)::value;
      issue_step(d, ah + ks * 2 * (kTile * 16), ah + ks * 2 * (kTile * 16) + part, bh + ks * kStepBytes,
                 bl + ks * kStepBytes, ks == 0 && c.first);
    });
    wgmma_commit();
    // a chunk that follows a drain has nothing to release: a tile's first chunk, and in the drained schedule
    // (kTrain != 0) every layer's first chunk
    if (kDrained ? !(c.first && c.half == 0) : ci != 0) {
      wgmma_wait<1>();                      // the previous chunk's wgmmas have retired
      if (lane == 0) mbar_arrive(&s.empty[prev_stage()]);
      __syncwarp();
    }
    if (++st == kStages) { st = 0; ph ^= 1; }
  };
  auto issue_range = [&](auto c0tag, auto ntag) SNB_INLINE {
    static_for<decltype(ntag)::value>([&](auto i) SNB_INLINE { issue(Int<decltype(c0tag)::value + decltype(i)::value>{}); });
  };
  auto drain = [&]() {                      // all of the tile's wgmmas have retired
    wgmma_wait<0>();
    if (lane == 0) mbar_arrive(&s.empty[prev_stage()]);
    __syncwarp();
  };

  // Epilogue block E(l, h, b) of trunk layer l (0..7): columns [128 h + 32 b, +32) of acc[h] -- bias, ReLU, hi/lo
  // split -> hid K-block 4 h + b, which is one 32-K chunk of the next layer's A operand.  The sigma layer (kSigma) also
  // accumulates the sigma head's partial sums, over its blocks in column order.  The training forward saves the
  // post-activation values: kTrain == 1 stores them as fp32 rows; for kTrain == 2 the block returns its fp16 words and
  // its ReLU mask word (one 32-column block is one word) for the caller to store after the epilogue's barrier.
  struct Block16 { uint32_t h16[4][2], mask[2]; };
  auto epi_block = [&](auto sigtag, auto htag, auto btag, int l, long long pt0) SNB_INLINE {
    constexpr bool kSigma = decltype(sigtag)::value;
    constexpr int h = decltype(htag)::value, b = decltype(btag)::value;
    const float* bias = g_cst + l * kWidth;            // CL.b[l]
    const float (&d)[64] = acc[h];
    Block16 k16{};
    if (kSigma && h == 0 && b == 0) { sig[0] = 0.f; sig[1] = 0.f; }
    static_for<4>([&](auto jtag) SNB_INLINE {
      constexpr int jj = decltype(jtag)::value, j = 4 * b + jj;
      const int col = h * kNh + 8 * j + 2 * tq;
      const float2 bb = ldg_f2_here(bias + col);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        float x0 = d[4 * j + 2 * rr] + bb.x, x1 = d[4 * j + 2 * rr + 1] + bb.y;
        uint32_t hi, lo;
        if (kTrain == 0 && !kSigma) {
          // nobody needs the fp32 post-activation value: ReLU and the fp16 range guard ride on the converts
          split_pair_relu<kBf16, kSplit>(x0, x1, hi, lo);
        } else {
          x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f);
          if (kSigma) {
            const float2 ww = ldg_f2_here(g_cst + CL.sigma_w + col);
            sig[rr] = fmaf(x0, ww.x, sig[rr]); sig[rr] = fmaf(x1, ww.y, sig[rr]);
          }
          split_pair<kBf16, kSplit, true>(x0, x1, hi, lo);
          const long long pt = pt0 + 8 * rr;
          if (kTrain == 1 && pt < p.n_points)
            *reinterpret_cast<float2*>(p.save_h + ((size_t)l * p.n_points + pt) * kWidth + col) = make_float2(x0, x1);
          if (kTrain == 2) {
            // fp16 modes: the hi word of the split IS rn_fp16(value) (saturated); bf16 modes convert separately
            k16.h16[jj][rr] = kBf16 ? pack_half2_sat(x0, x1) : hi;
            k16.mask[rr] |= ((x0 > 0.f ? 1u : 0u) << (col & 31)) | ((x1 > 0.f ? 1u : 0u) << ((col & 31) + 1));
          }
        }
        const uint32_t a = hid_thr + (h * 16 + j) * (kTile * 16) + rr * 128;   // (row r0 + 8 rr, column col)
        st_shared_u32(a, hi);
        if (kSplit) st_shared_u32(a + kHidPart, lo);
      }
    });
    if (kTrain == 2) {
      // the quad's four threads hold the block's 32 ReLU bits of each row
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        k16.mask[rr] |= __shfl_xor_sync(0xffffffffu, k16.mask[rr], 1);
        k16.mask[rr] |= __shfl_xor_sync(0xffffffffu, k16.mask[rr], 2);
      }
    }
    return k16;
  };
  // the end of an epilogue (half): its hid blocks become visible to the next layer's wgmmas
  auto epi_half_end = [&]() SNB_INLINE {
    fence_proxy_async_smem();     // generic-proxy smem writes -> visible to the async proxy
    wg_sync();
  };
  // sigma head (nerf.py:136) after the sigma layer's last epilogue block: the quad's four threads hold the row's columns
  auto sigma_head = [&](long long pt0) SNB_INLINE {
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      float v = sig[rr];
      v += __shfl_xor_sync(0xffffffffu, v, 1);
      v += __shfl_xor_sync(0xffffffffu, v, 2);
      sig[rr] = v + __ldg(g_cst + CL.sigma_b);
      const long long pt = pt0 + 8 * rr;
      if (p.sigma_only && tq == 0 && pt < p.n_points) p.out[pt] = sig[rr];
    }
  };

  // direction layer: shifted softplus / ReLU, rgb head (nerf.py:142-146), the [r, g, b, sigma] rows
  auto dir_epilogue = [&](const float (&d)[64], long long pt0) SNB_INLINE {
    const float sh = new_activation ? 1.0f : 0.0f;   // shifted softplus: fold the -1 into the bias
    float a[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = 8 * j + 2 * tq;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(g_cst + CL.b[9] + col));
      const float2 w0 = __ldg(reinterpret_cast<const float2*>(g_cst + CL.rgb_w + col));
      const float2 w1 = __ldg(reinterpret_cast<const float2*>(g_cst + CL.rgb_w + kHalf + col));
      const float2 w2 = __ldg(reinterpret_cast<const float2*>(g_cst + CL.rgb_w + 2 * kHalf + col));
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const long long pt = pt0 + 8 * rr;
        float x0 = d[4 * j + 2 * rr] + (bb.x - sh), x1 = d[4 * j + 2 * rr + 1] + (bb.y - sh);
        if (new_activation) { x0 = softplus_fast(x0); x1 = softplus_fast(x1); }
        else { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        if (kTrain == 1 && pt < p.n_points) *reinterpret_cast<float2*>(p.save_g + pt * kHalf + col) = make_float2(x0, x1);
        if (kTrain == 2 && pt < p.ppad)
          *reinterpret_cast<uint32_t*>(p.a_g + a16_cell(pt, col >> 3, kHalf) + (col & 7) * 2) =
              pt < p.n_points ? pack_half2_sat(x0, x1) : 0u;
        a[rr][0] = fmaf(x1, w0.y, fmaf(x0, w0.x, a[rr][0]));
        a[rr][1] = fmaf(x1, w1.y, fmaf(x0, w1.x, a[rr][1]));
        a[rr][2] = fmaf(x1, w2.y, fmaf(x0, w2.x, a[rr][2]));
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      float c[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        float v = a[rr][k];
        v += __shfl_xor_sync(0xffffffffu, v, 1);
        v += __shfl_xor_sync(0xffffffffu, v, 2);
        v += __ldg(g_cst + CL.rgb_b + k);
        c[k] = new_activation ? widened_sigmoid_f(v) : sigmoid_f(v);
      }
      const long long pt = pt0 + 8 * rr;
      if (tq == 0 && pt < p.n_points) reinterpret_cast<float4*>(p.out)[pt] = make_float4(c[0], c[1], c[2], sig[rr]);
    }
  };

  // The drained trunk epilogue of layer l: all eight blocks in drain order, the sigma head, the skip layer's direction
  // encoding and one barrier.  kTrain == 2 keeps the fp16 activation words and ReLU mask words in registers and stores
  // them to global memory after that barrier; stored inside it, they made the epilogue's `fence.proxy.async`
  // (MEMBAR.ALL.CTA) wait for their completion in every layer.
  auto trunk_epilogue = [&](auto ltag, int l, long long tile, long long pt0) SNB_INLINE {
    constexpr int L = decltype(ltag)::value;
    Block16 k16[2][4];
    static_for<2>([&](auto htag) SNB_INLINE {
      static_for<4>([&](auto btag) SNB_INLINE {
        k16[decltype(htag)::value][decltype(btag)::value] = epi_block(std::bool_constant<L == 7>{}, htag, btag, l, pt0);
      });
    });
    if (L == 7) sigma_head(pt0);
    if (L == 4 && !p.sigma_only) encode_rows(Int<SNB_DIR_FREQS>{}, tile);
    epi_half_end();
    if (kTrain == 2) {
      unsigned char* hb = p.a_h + (size_t)l * (size_t)p.ppad * (kWidth * 2);
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const long long pt = pt0 + 8 * rr;
        if (pt >= p.ppad) continue;
        const bool live = pt < p.n_points;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int col = h * kNh + 8 * j + 2 * tq;
            *reinterpret_cast<uint32_t*>(hb + a16_cell(pt, col >> 3, kWidth) + (col & 7) * 2) =
                live ? k16[h][j / 4].h16[j % 4][rr] : 0u;
          }
#pragma unroll
          for (int b = 0; b < 4; ++b)
            if (tq == 0) p.a_mask[a16_mask_index(l, h * 4 + b, pt, p.ppad)] = live ? k16[h][b].mask[rr] : 0u;
        }
      }
    }
  };

  // Two schedules, selected at compile time.  Inference (the render path and the embedded entry) runs the epilogues
  // under the wgmmas: each epilogue block follows a chunk's issue and the wait<1> that retires the chunk before it, so
  // one chunk stays queued on the tensor pipe while the block runs.  The training forward (kDrained) runs a layer's
  // wgmmas, drains them, then runs the layer's whole epilogue under one barrier: with the blocked schedule it was
  // slower (DESIGN.md §4.1), since the global stores of the saved activations end up in front of one of a layer's two
  // fences and the registers that hold them push values out to local memory.
  //
  // Blocked, per warpgroup (each reads and writes only its own rows of hid and enc):
  //   1. E(l, h, b) reads acc[h]: every chunk of (l, h) has retired;
  //   2. E(l, h, b) overwrites hid block 4 h + b: the chunk of (l, 1) that reads it has retired;
  //   3. chunk k of (l + 1, h) reads hid block k only after the epilogue half that writes it has been fenced
  //      (fence.proxy.async + warpgroup barrier);
  //   4. the first wgmma of (l + 1, h) (accumulate = 0, writes acc[h]) follows every E(l, h, .) in program order.
  //
  // trunk_layer(L, l): the wgmmas of trunk layer l, whose chunks follow layer L's schedule (layers 1-3, 5 and 6 share
  // layer 1's), and the epilogue blocks the schedule places under them.  Blocked, layer l > 0 interleaves them with
  // E(l - 1, 1, .) and E(l, 0, .).  On entry every chunk of layer l - 1 is issued and E(l - 1, 0, .) is fenced; on
  // return every chunk of layer l is issued and E(l, 0, .) is fenced.
  //   * E(l - 1, 1, b) follows (l, 0)'s chunk b: (l - 1, 1) has retired (rules 1, 2), and those chunks read only enc
  //     and hid blocks 0-3 (rule 3);
  //   * E(l, 0, b) follows (l, 1)'s chunk e + b + 1 (e = its enc chunks): (l, 0) and the (l, 1) chunk e + b that reads
  //     hid block b have retired (rules 1, 2);
  //   * layer 0 reads only enc and its half 1 holds only enc chunks, so its blocks have no hid hazard: E(0, 0, .)
  //     needs only (0, 0) retired.
  // No wgmma is in flight where a loop over layers is entered or repeats: with an accumulator in flight there, ptxas
  // serializes every wgmma of the kernel (C7514), since it may have to move the accumulator's registers at the merge.
  // So every blocked layer but 7 ends by waiting for its last chunk, which costs the tensor pipe one restart per layer.
  //
  // The skip layer (L = 4) writes the direction encoding over this warpgroup's rows of the xyz encoding once (4, 0)
  // and (4, 1)'s enc chunks, its last readers, have retired.
  auto trunk_layer = [&](auto ltag, int l, long long tile, long long pt0) SNB_INLINE {
    constexpr int L = decltype(ltag)::value;
    constexpr int c0 = chunk_index(L, 0), n0 = chunk_count(L, 0), c1 = chunk_index(L, 1), n1 = chunk_count(L, 1);
    constexpr int e = enc_chunks(L);
    if constexpr (kDrained) {
      issue_range(Int<c0>{}, Int<n0>{});
      issue_range(Int<c1>{}, Int<n1>{});
      drain();
      trunk_epilogue(ltag, l, tile, pt0);
    } else if constexpr (L == 0) {
      issue_range(Int<c0>{}, Int<n0>{});
      static_for<4>([&](auto btag) SNB_INLINE {
        constexpr int b = decltype(btag)::value;
        if constexpr (b < n1) issue(Int<c1 + b>{});
        epi_block(std::false_type{}, Int<0>{}, btag, 0, pt0);
      });
      epi_half_end();
      wgmma_wait<0>();
    } else {
      static_for<4>([&](auto btag) SNB_INLINE {
        issue(Int<c0 + decltype(btag)::value>{});
        epi_block(std::false_type{}, Int<1>{}, btag, l - 1, pt0);
      });
      epi_half_end();
      issue_range(Int<c0 + 4>{}, Int<n0 - 4>{});
      issue_range(Int<c1>{}, Int<e + 1>{});
      static_for<4>([&](auto btag) SNB_INLINE {
        issue(Int<c1 + e + 1 + decltype(btag)::value>{});
        epi_block(std::bool_constant<L == 7>{}, Int<0>{}, btag, l, pt0);
      });
      if (L == 4 && !p.sigma_only) encode_rows(Int<SNB_DIR_FREQS>{}, tile);
      epi_half_end();
      issue_range(Int<c1 + e + 5>{}, Int<n1 - e - 5>{});
      if constexpr (L != 7) wgmma_wait<0>();
    }
  };
  // The end of a tile: the direction layer 9 (the bottleneck, 8, is folded into it) and its epilogue.  Blocked,
  // E(7, 1, .) runs under the direction layer's chunks 0-3, which read hid blocks 0-3 only; sigma-only passes end with
  // layer 7, so there E(7, 1, .) runs after the drain.
  auto tile_end = [&](long long tile, long long pt0) SNB_INLINE {
    constexpr int c9 = chunk_index(9, 0), n9 = chunk_count(9, 0);
    load_row(tile + gridDim.x);   // the next tile's rays and depths, under this tile's last MMAs
    if (p.sigma_only) {
      if constexpr (!kDrained) {
        drain();
        static_for<4>([&](auto btag) SNB_INLINE { epi_block(std::true_type{}, Int<1>{}, btag, 7, pt0); });
        sigma_head(pt0);
        epi_half_end();
      }
      return;
    }
    if constexpr (kDrained) {
      issue_range(Int<c9>{}, Int<n9>{});
    } else {
      static_for<4>([&](auto btag) SNB_INLINE {
        issue(Int<c9 + decltype(btag)::value>{});
        epi_block(std::true_type{}, Int<1>{}, btag, 7, pt0);
      });
      sigma_head(pt0);
      epi_half_end();
      issue_range(Int<c9 + 4>{}, Int<n9 - 4>{});
    }
    drain();
    dir_epilogue(acc[0], pt0);
  };

  load_row(blockIdx.x);
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long pt0 = tile * kTile + r0;
    // ---- xyz encoding of this warpgroup's 64 rows (the direction encoding follows layer 4's enc chunks)
    encode_rows(Int<SNB_XYZ_FREQS>{}, tile);
    fence_proxy_async_smem();
    wg_sync();
    // the plain hidden layers run as loops over one copy of the code, which keeps the kernel's instruction footprint down
    trunk_layer(Int<0>{}, 0, tile, pt0);
#pragma unroll 1
    for (int l = 1; l < 4; ++l) trunk_layer(Int<1>{}, l, tile, pt0);
    trunk_layer(Int<4>{}, 4, tile, pt0);
#pragma unroll 1
    for (int l = 5; l < 7; ++l) trunk_layer(Int<1>{}, l, tile, pt0);
    trunk_layer(Int<7>{}, 7, tile, pt0);
    tile_end(tile, pt0);
  }
}

// ------------------------------------------------------------------ host
template <bool kBf16, bool kSplit, bool kEmbedded, int kTrain = 0>
static int launch_tc(const TcParams& p, cudaStream_t st) {
  static SmemOptIn optin;
  const long long ntiles = (p.n_points + kTile - 1) / kTile;
  if (ntiles == 0) return SNB_OK;       // an empty pass is a no-op: no CUDA call at all
  const size_t smem = sizeof(TcSmem<kSplit>) + 128;
  auto kern = field_tc_kernel<kBf16, kSplit, kEmbedded, kTrain>;
  if (int rc = ensure_smem(kern, optin, (int)smem, "field_tc")) return rc;
  long long ctas = sm_count();
  if (ctas > ntiles) ctas = ntiles;
  kern<<<(unsigned)ctas, kThreads, smem, st>>>(p);
  return check_launch("field_tc_kernel");
}

template <bool kEmbedded, int kTrain = 0>
static int dispatch_tc(int precision, const TcParams& p, cudaStream_t st) {
  switch (precision) {
    case SNB_PREC_F16X3: return launch_tc<false, true, kEmbedded, kTrain>(p, st);
    case SNB_PREC_BF16X3: return launch_tc<true, true, kEmbedded, kTrain>(p, st);
    case SNB_PREC_BF16: return launch_tc<true, false, kEmbedded, kTrain>(p, st);
    case SNB_PREC_F16: return launch_tc<false, false, kEmbedded, kTrain>(p, st);
  }
  return fail(SNB_ERR_INVALID, "precision %d is not a tensor-core mode", precision);
}

int field_forward_tc(const void* packed, int precision, const float* rays, const float* z, int64_t n_rays,
                     int n_samples, int sigma_only, float* raw, cudaStream_t st) {
  TcParams p{};
  p.image = reinterpret_cast<const unsigned char*>(packed);
  p.rays = rays; p.z = z; p.n_samples = n_samples;
  p.n_points = (long long)n_rays * n_samples;
  p.sigma_only = sigma_only;
  p.out = raw;
  return dispatch_tc<false>(precision, p, st);
}

// sigma_only (both training entries): layers 1-8 and the sigma head only; raw is (P,) sigma, the direction encoding
// and the direction layer's output are neither computed nor stored (save_dir / save_g may be NULL)
int field_forward_train_tc(const void* packed, int precision, const float* rays, const float* z, int64_t n_rays,
                           int n_samples, int sigma_only, float* raw, float* save_enc, float* save_dir, float* save_h,
                           float* save_g, cudaStream_t st) {
  TcParams p{};
  p.image = reinterpret_cast<const unsigned char*>(packed);
  p.rays = rays; p.z = z; p.n_samples = n_samples;
  p.n_points = (long long)n_rays * n_samples;
  p.sigma_only = sigma_only;
  p.out = raw;
  p.save_enc = save_enc; p.save_dir = save_dir; p.save_h = save_h; p.save_g = save_g;
  return dispatch_tc<false, 1>(precision, p, st);
}

// training forward with 16-bit activation storage (act16.cuh): `act16` = one buffer of make_act16_layout(P).total bytes
int field_forward_train16_tc(const void* packed, int precision, const float* rays, const float* z, int64_t n_rays,
                             int n_samples, int sigma_only, float* raw, void* act16, cudaStream_t st) {
  TcParams p{};
  p.image = reinterpret_cast<const unsigned char*>(packed);
  p.rays = rays; p.z = z; p.n_samples = n_samples;
  p.n_points = (long long)n_rays * n_samples;
  p.sigma_only = sigma_only;
  p.out = raw;
  const Act16Layout L = make_act16_layout(p.n_points);
  unsigned char* b = reinterpret_cast<unsigned char*>(act16);
  p.a_enc = b + L.enc; p.a_dir = b + L.dir; p.a_h = b + L.h[0]; p.a_g = b + L.g;
  p.a_mask = reinterpret_cast<uint32_t*>(b + L.mask);
  p.ppad = a16_pad(p.n_points);
  return dispatch_tc<false, 2>(precision, p, st);
}

int mlp_forward_tc(const void* packed, int precision, const float* x, int64_t x_stride, int64_t n_points,
                   int sigma_only, float* out, cudaStream_t st) {
  TcParams p{};
  p.image = reinterpret_cast<const unsigned char*>(packed);
  p.x = x; p.x_stride = x_stride;
  p.n_points = n_points;
  p.sigma_only = sigma_only;
  p.out = out;
  return dispatch_tc<true>(precision, p, st);
}

}  // namespace snb
