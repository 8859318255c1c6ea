// vit.cu -- DINO ViT-S/16 CLS feature (SinNeRF's semantic loss, models/sinnerf.py:162-169) and its gradient with
// respect to the input images, on Hopper tensor cores.
//
// One pass stacks the token rows of n images (M = 197 n).  Every matrix product -- the patch embedding, qkv, the
// attention scores and P.V, proj, fc1, fc2 and all of their input gradients -- goes through one wgmma GEMM kernel
// (64 x 64 output tile per warpgroup, 64-deep K chunks staged through shared memory, fp32 accumulate) whose
// operands are fp32 tensors read through strides, or the packed 16-bit weight planes.  The operand arithmetic is
// a template parameter: fp16 hi + lo with three products (fp32 parity), or one fp16 or one bf16 product.
// LayerNorm, softmax, GELU and the residual stream stay fp32.
//
// Block 11 is pruned: only its CLS row is consumed, so it computes K and V for every token but Q, proj, LN2 and the
// MLP for the CLS rows only.  The backward runs to the images only (no weight gradients): dgrad GEMMs against the
// same packed weights, the flash-attention backward recurrences (P recomputed from the saved row log-sum-exp,
// D = rowsum(dO o O)) over per-(image, head) 197 x 197 tiles kept in the workspace, LayerNorm and GELU backward,
// the patch-embedding dgrad, and a fold of the 224 x 224 gradient onto the source pixels that gathers over the
// inverse of the monotone nearest map.  No atomics and no split reductions: two identical calls give the same bits.
//
// The upstream gradient of each image is scaled by a power of two (its largest element to [1, 2)) before the chain
// and unscaled in the fold: the chain is linear in it, so this is exact, and it keeps fp16 operands clear of
// their subnormal range whatever the loss weight.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "tc_gemm.cuh"
#include "wgmma.cuh"

namespace snb {
using namespace wg;

namespace {

constexpr int kD = SNB_VIT_DIM, kHeads = 6, kHd = 64, kTok = 197, kPatches = 196, kGrid = 14, kMlp = 1536,
              kQkv = 3 * kD, kPatchK = 768, kBlocks = 12, kRes = 224;
constexpr int kLdS = 200;                       // row stride of the 197 x 197 score tiles (16-byte aligned rows)
constexpr long long kTileS = (long long)kTok * kLdS;
constexpr float kLnEps = 1e-6f;
__constant__ float kMean[3] = {0.485f, 0.456f, 0.406f};
__constant__ float kStd[3] = {0.229f, 0.224f, 0.225f};

// ------------------------------------------------------------------ weight image
// [fp32 vectors][16-bit planes]; every piece 256-byte aligned.  Matrices are row-major (out, in) like nn.Linear's
// weight (the patch embedding as (384, 768) = (out, c ky kx)); split mode stores the hi plane then the lo plane.
struct VitBlockW {
  long long n1w, n1b, qkv_b, proj_b, n2w, n2b, fc1_b, fc2_b;   // float offsets
  long long qkv, proj, fc1, fc2;                               // element offsets of plane 0 in the 16-bit region
};
struct VitLayout {
  long long cls, pos, pe_b, pe;
  VitBlockW blk[kBlocks];
  long long n_floats, n_halfs;
  int planes;
};
long long al64(long long x) { return (x + 63) & ~63ll; }
long long al128(long long x) { return (x + 127) & ~127ll; }
VitLayout vit_layout(int mode) {
  VitLayout L{};
  L.planes = mode == kSplit ? 2 : 1;
  long long f = 0, h = 0;
  auto vec = [&](long long n) { long long o = f; f = al64(f + n); return o; };
  auto mat = [&](long long n) { long long o = h; h = al128(h + (long long)L.planes * n); return o; };
  L.cls = vec(kD); L.pos = vec((long long)kTok * kD); L.pe_b = vec(kD);
  L.pe = mat((long long)kD * kPatchK);
  for (int b = 0; b < kBlocks; ++b) {
    VitBlockW& B = L.blk[b];
    B.n1w = vec(kD); B.n1b = vec(kD); B.qkv_b = vec(kQkv); B.proj_b = vec(kD);
    B.n2w = vec(kD); B.n2b = vec(kD); B.fc1_b = vec(kMlp); B.fc2_b = vec(kD);
    B.qkv = mat((long long)kQkv * kD); B.proj = mat((long long)kD * kD);
    B.fc1 = mat((long long)kMlp * kD); B.fc2 = mat((long long)kD * kMlp);
  }
  L.n_floats = f; L.n_halfs = h;
  return L;
}
size_t vit_image_bytes(int mode) {
  const VitLayout L = vit_layout(mode);
  return (size_t)L.n_floats * 4 + (size_t)L.n_halfs * 2;
}

// host view of a packed image
struct Mat {
  const uint16_t* hi; const uint16_t* lo; int rows, cols;   // lo: split mode only
};
struct VitW {
  const float* f;
  const uint16_t* h;
  VitLayout L;
  Mat mat(long long off, int rows, int cols) const {
    return Mat{h + off, L.planes == 2 ? h + off + (long long)rows * cols : nullptr, rows, cols};
  }
  const float* v(long long off) const { return f + off; }
};
VitW vit_view(const void* image, int mode) {
  VitW w;
  w.L = vit_layout(mode);
  w.f = static_cast<const float*>(image);
  w.h = reinterpret_cast<const uint16_t*>(w.f + w.L.n_floats);
  return w;
}

template <int kMode>
__global__ void vit_pack_kernel(const float* __restrict__ w, long long n, uint16_t* __restrict__ hi,
                                uint16_t* __restrict__ lo) {
  const long long i = 2 * ((long long)blockIdx.x * blockDim.x + threadIdx.x);
  if (i >= n) return;
  const float x0 = w[i], x1 = i + 1 < n ? w[i + 1] : 0.f;
  uint32_t h, l;
  cvt2<kMode>(x0, x1, h, l);
  hi[i] = (uint16_t)(h & 0xffffu);
  if (kMode == kSplit) lo[i] = (uint16_t)(l & 0xffffu);
  if (i + 1 < n) {
    hi[i + 1] = (uint16_t)(h >> 16);
    if (kMode == kSplit) lo[i + 1] = (uint16_t)(l >> 16);
  }
}

// B = W (y = x W^T: B(n, k) = W[n][k]) or, transposed, W^T (dx = dy W: B(n, k) = W[k][n]); rows r0.. of W
void set_w(Gemm& g, const Mat& w, bool transposed, int r0 = 0) {
  const long long off = (long long)r0 * w.cols;
  g.Bh = w.hi + off;
  g.Bl = w.lo != nullptr ? w.lo + off : nullptr;
  if (transposed) { g.b_n = 1; g.b_k = w.cols; }
  else { g.b_n = w.cols; g.b_k = 1; }
}

// ------------------------------------------------------------------ row kernels (one warp per row of 384)
constexpr int kRowThreads = 256;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void ln_stats(const float (&v)[12], float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 12; ++i) s += v[i];
  mean = warp_sum(s) * (1.f / kD);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 12; ++i) q += (v[i] - mean) * (v[i] - mean);
  rstd = 1.f / sqrtf(warp_sum(q) * (1.f / kD) + kLnEps);
}

__global__ void vit_ln_fwd_kernel(const float* __restrict__ x, long long x_m, const float* __restrict__ gam,
                                  const float* __restrict__ bet, float* __restrict__ y, long long y_m, int rows) {
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float v[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) v[i] = x[row * x_m + lane + 32 * i];
  float mean, rstd;
  ln_stats(v, mean, rstd);
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const int c = lane + 32 * i;
    y[row * y_m + c] = (v[i] - mean) * rstd * gam[c] + bet[c];
  }
}

// dx = LayerNorm backward (statistics recomputed from x) + residual.  res_cls: the residual is given for the CLS
// rows only, compactly (row i 197 -> res row i).
__global__ void vit_ln_bwd_kernel(const float* __restrict__ x, long long x_m, const float* __restrict__ gam,
                                  const float* __restrict__ dy, long long dy_m, const float* __restrict__ res,
                                  long long res_m, int res_cls, float* __restrict__ dx, long long dx_m, int rows) {
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= rows) return;
  float v[12], gd[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) v[i] = x[row * x_m + lane + 32 * i];
  float mean, rstd;
  ln_stats(v, mean, rstd);
  float a = 0.f, b = 0.f;
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const int c = lane + 32 * i;
    v[i] = (v[i] - mean) * rstd;
    gd[i] = dy[row * dy_m + c] * gam[c];
    a += gd[i];
    b += gd[i] * v[i];
  }
  a = warp_sum(a) * (1.f / kD);
  b = warp_sum(b) * (1.f / kD);
  const float* r = nullptr;
  if (res != nullptr) {
    if (!res_cls) r = res + row * res_m;
    else if (row % kTok == 0) r = res + (row / kTok) * res_m;
  }
#pragma unroll
  for (int i = 0; i < 12; ++i) {
    const int c = lane + 32 * i;
    const float g = rstd * (gd[i] - a - v[i] * b);
    dx[row * dx_m + c] = r != nullptr ? r[c] + g : g;
  }
}

// softmax over the 197 keys of each score row (rows_per_z rows per (image, head)), in place; saves the row lse
__global__ void vit_softmax_kernel(float* __restrict__ S, float* __restrict__ lse, int rows_per_z, int n_rows) {
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int z = row / rows_per_z, r = row % rows_per_z;
  float* s = S + z * kTileS + (long long)r * kLdS;
  float v[7];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const int j = lane + 32 * i;
    v[i] = j < kTok ? s[j] : -INFINITY;
    mx = fmaxf(mx, v[i]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    v[i] = expf(v[i] - mx);
    sum += v[i];
  }
  sum = warp_sum(sum);
  const float inv = 1.f / sum;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const int j = lane + 32 * i;
    if (j < kTok) s[j] = v[i] * inv;
  }
  if (lane == 0) lse[row] = mx + logf(sum);
}

// attention backward per score row: P = exp(S - lse), D = rowsum(dO o O), dS = scale P (dP - D).
// S holds the recomputed scaled logits and becomes P; dP becomes dS.  O / dO row r of (image i, head h) at
// base + i o_z1 + 64 h + r o_m.
__global__ void vit_softmax_bwd_kernel(float* __restrict__ S, float* __restrict__ dP, const float* __restrict__ lse,
                                       const float* __restrict__ O, long long o_z1, long long o_m,
                                       const float* __restrict__ dO, long long do_z1, long long do_m, int rows_per_z,
                                       int n_rows, float scale) {
  const int row = blockIdx.x * (kRowThreads / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= n_rows) return;
  const int z = row / rows_per_z, r = row % rows_per_z, img = z / kHeads, h = z % kHeads;
  const float* o = O + img * o_z1 + h * kHd + r * o_m;
  const float* d = dO + img * do_z1 + h * kHd + r * do_m;
  const float D = warp_sum(o[lane] * d[lane] + o[lane + 32] * d[lane + 32]);
  const float l = lse[row];
  float* s = S + z * kTileS + (long long)r * kLdS;
  float* p = dP + z * kTileS + (long long)r * kLdS;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const int j = lane + 32 * i;
    if (j < kTok) {
      const float pr = expf(s[j] - l);
      s[j] = pr;
      p[j] = scale * pr * (p[j] - D);
    }
  }
}

// ------------------------------------------------------------------ embedding, fold, gradient scale
struct ImgSet {
  const float* p[SNB_VIT_MAX_IMAGES];
  long long s[SNB_VIT_MAX_IMAGES][3];
  int h[SNB_VIT_MAX_IMAGES], w[SNB_VIT_MAX_IMAGES];
};

// F.interpolate(mode='nearest') source index: min(floor(dst * (float)in / out), in - 1), in fp32
__device__ __forceinline__ int nearest_src(int dst, int in) {
  const float scale = (float)in / (float)kRes;
  return min((int)floorf((float)dst * scale), in - 1);
}
// first destination index whose source is >= y (kRes if none): the map is monotone
__device__ __forceinline__ int nearest_first(int y, int in) {
  int lo = 0, hi = kRes;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (nearest_src(mid, in) >= y) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// im2col rows of the 224 x 224 normalised images: col[i][p][c 256 + ky 16 + kx]
__global__ void vit_embed_gather_kernel(ImgSet im, int n, float* __restrict__ col) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (long long)n * kPatches * kPatchK) return;
  const int k = (int)(t % kPatchK), p = (int)((t / kPatchK) % kPatches), i = (int)(t / ((long long)kPatchK * kPatches));
  const int ch = k >> 8, Y = (p / kGrid) * 16 + ((k >> 4) & 15), X = (p % kGrid) * 16 + (k & 15);
  const int sy = nearest_src(Y, im.h[i]), sx = nearest_src(X, im.w[i]);
  const float v = __ldg(im.p[i] + ch * im.s[i][0] + sy * im.s[i][1] + sx * im.s[i][2]);
  col[t] = (v - kMean[ch]) / kStd[ch];
}

__global__ void vit_cls_rows_kernel(const float* __restrict__ cls, const float* __restrict__ pos, float* __restrict__ x,
                                    long long x_z, int n) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * kD) return;
  x[(t / kD) * x_z + t % kD] = cls[t % kD] + pos[t % kD];
}

// the 224 x 224 gradient (patch-embedding dgrad, dcol) folded onto the source pixels: each pixel sums the
// destination rectangle that the nearest map sends to it, in a fixed order
__global__ void vit_fold_kernel(const float* __restrict__ dcol, const float* __restrict__ inv_scale, ImgSet im,
                                int i) {
  const int h = im.h[i], w = im.w[i];
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 3ll * h * w) return;
  const int x = (int)(t % w), y = (int)((t / w) % h), ch = (int)(t / ((long long)w * h));
  const int y0 = nearest_first(y, h), y1 = nearest_first(y + 1, h);
  const int x0 = nearest_first(x, w), x1 = nearest_first(x + 1, w);
  const float* d = dcol + (long long)i * kPatches * kPatchK + ch * 256;
  float acc = 0.f;
  for (int Y = y0; Y < y1; ++Y)
    for (int X = x0; X < x1; ++X) acc += d[((Y >> 4) * kGrid + (X >> 4)) * kPatchK + (Y & 15) * 16 + (X & 15)];
  float* out = const_cast<float*>(im.p[i]) + ch * im.s[i][0] + y * im.s[i][1] + x * im.s[i][2];
  *out = acc / kStd[ch] * inv_scale[i];
}

// per image: k with max |g| 2^k in [1, 2) (0 for an all-zero or non-finite row); dx = g 2^k, inv = 2^-k.  Both go
// through ldexpf, never through s = 2^k as a float: for a subnormal max |g|, k reaches 149 and 2^k overflows (inf,
// then inv = 0 and NaN gradients in the bf16 mode), while g 2^k < 2 and 2^-k >= 2^-149 are exact.
__global__ void vit_grad_scale_kernel(const float* __restrict__ g, float* __restrict__ dx, float* __restrict__ inv) {
  __shared__ float red[4];
  const int i = blockIdx.x, tid = threadIdx.x;
  float m = 0.f;
  for (int c = tid; c < kD; c += 128) m = fmaxf(m, fabsf(g[i * kD + c]));
  m = warp_max(m);
  if ((tid & 31) == 0) red[tid >> 5] = m;
  __syncthreads();
  m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  int k = 0;
  if (m > 0.f && isfinite(m)) {
    int e;
    frexpf(m, &e);               // m = f 2^e, f in [0.5, 1)
    k = 1 - e;
  }
  for (int c = tid; c < kD; c += 128) dx[i * kD + c] = ldexpf(g[i * kD + c], k);
  if (tid == 0) inv[i] = ldexpf(1.f, -k);
}

// ------------------------------------------------------------------ workspace
struct SavedBlock {
  float *x_in, *x_mid, *qkv, *O, *pre, *lse;
};
struct VitWs {
  float *col, *X0, *X1, *ln, *qkv, *O, *h, *S, *dP, *lse;
  float *xmid_c, *ln_c, *O_c, *h_c, *pre_c, *lse_c;         // block 11, CLS rows (saved for the backward)
  float *dx, *dx2, *dln, *dqkv, *dO, *dh, *c0, *c1, *c2, *ch, *inv;
  SavedBlock blk[kBlocks];
  size_t bytes;
};
VitWs vit_ws(void* base, int n, int save) {
  VitWs W{};
  const long long M = (long long)n * kTok;
  float* b = static_cast<float*>(base);
  long long off = 0;
  auto take = [&](long long floats) { float* p = b == nullptr ? nullptr : b + off; off = al64(off + floats); return p; };
  W.col = take((long long)n * kPatches * kPatchK);
  W.X0 = take(M * kD); W.X1 = take(M * kD); W.ln = take(M * kD); W.qkv = take(M * kQkv); W.O = take(M * kD);
  W.h = take(M * kMlp);
  W.S = take(n * kHeads * kTileS); W.dP = take(n * kHeads * kTileS); W.lse = take((long long)n * kHeads * kTok);
  W.xmid_c = take(n * kD); W.ln_c = take(n * kD); W.O_c = take(n * kD); W.h_c = take(n * kMlp);
  W.pre_c = take(n * kMlp); W.lse_c = take(n * kHeads);
  if (save) {
    W.dx = take(M * kD); W.dx2 = take(M * kD); W.dln = take(M * kD); W.dqkv = take(M * kQkv); W.dO = take(M * kD);
    W.dh = take(M * kMlp);
    W.c0 = take(n * kD); W.c1 = take(n * kD); W.c2 = take(n * kD); W.ch = take(n * kMlp); W.inv = take(n);
    for (int l = 0; l < kBlocks; ++l) {
      SavedBlock& s = W.blk[l];
      s.x_in = take(M * kD); s.x_mid = take(M * kD); s.qkv = take(M * kQkv); s.O = take(M * kD);
      s.pre = take(M * kMlp); s.lse = take((long long)n * kHeads * kTok);
    }
  }
  W.bytes = (size_t)off * 4;
  return W;
}

int row_grid(long long rows) { return (int)((rows + kRowThreads / 32 - 1) / (kRowThreads / 32)); }

int ln_fwd(const float* x, long long x_m, const float* gam, const float* bet, float* y, long long y_m, int rows,
           cudaStream_t st) {
  vit_ln_fwd_kernel<<<row_grid(rows), kRowThreads, 0, st>>>(x, x_m, gam, bet, y, y_m, rows);
  return check_launch("vit_ln_fwd_kernel");
}
int ln_bwd(const float* x, long long x_m, const float* gam, const float* dy, long long dy_m, const float* res,
           long long res_m, int res_cls, float* dx, long long dx_m, int rows, cudaStream_t st) {
  vit_ln_bwd_kernel<<<row_grid(rows), kRowThreads, 0, st>>>(x, x_m, gam, dy, dy_m, res, res_m, res_cls, dx, dx_m, rows);
  return check_launch("vit_ln_bwd_kernel");
}

#define VIT_TRY(x)            \
  do {                        \
    if (int rc_ = (x)) return rc_; \
  } while (0)

// the scores of every (image, head): S[z] (q_rows x 197) = 0.125 Q K^T; Q rows q_rows per image with row stride q_m
template <int kMode>
int scores(const float* qkv, int n, int q_rows, long long q_m, float* S, cudaStream_t st) {
  Gemm g = gemm(q_rows, kTok, kHd);
  g.A = qkv; g.a_z1 = (long long)kTok * kQkv; g.a_z2 = kHd; g.a_m = q_m; g.a_k = 1;
  g.Bf = qkv + kD; g.b_z1 = (long long)kTok * kQkv; g.b_z2 = kHd; g.b_n = kQkv; g.b_k = 1;
  g.C = S; g.c_z1 = kHeads * kTileS; g.c_z2 = kTileS; g.c_m = kLdS;
  g.nz2 = kHeads; g.alpha = 0.125f;
  return run_gemm<kMode>(g, n * kHeads, st);
}

// O[z] (q_rows x 64) = P V, written at column 64 h of rows with stride o_m, image stride o_z1
template <int kMode>
int attn_pv(const float* S, const float* qkv, int n, int q_rows, float* O, long long o_z1, long long o_m,
            cudaStream_t st) {
  Gemm g = gemm(q_rows, kHd, kTok);
  g.A = S; g.a_z1 = kHeads * kTileS; g.a_z2 = kTileS; g.a_m = kLdS; g.a_k = 1;
  g.Bf = qkv + 2 * kD; g.b_z1 = (long long)kTok * kQkv; g.b_z2 = kHd; g.b_n = 1; g.b_k = kQkv;
  g.C = O; g.c_z1 = o_z1; g.c_z2 = kHd; g.c_m = o_m;
  g.nz2 = kHeads;
  return run_gemm<kMode>(g, n * kHeads, st);
}

// y = x W^T + b with an epilogue, over `rows` rows
template <int kMode>
int linear(const float* x, long long x_m, const Mat& w, const float* bias, int rows, float* y, long long y_m, int epi,
           const float* aux, float* aux_out, long long aux_m, cudaStream_t st, int r0 = 0, int n_out = -1) {
  Gemm g = gemm(rows, n_out < 0 ? w.rows : n_out, w.cols);
  g.A = x; g.a_m = x_m; g.a_k = 1;
  set_w(g, w, false, r0);
  g.C = y; g.c_m = y_m;
  g.bias = bias; g.epi = epi; g.aux = aux; g.aux_out = aux_out; g.aux_m = aux_m;
  return run_gemm<kMode>(g, 1, st);
}

// dx = dy W (input gradient of a Linear), with an epilogue
template <int kMode>
int linear_dgrad(const float* dy, long long dy_m, const Mat& w, int rows, float* dx, long long dx_m, int epi,
                 const float* aux, long long aux_m, cudaStream_t st) {
  Gemm g = gemm(rows, w.cols, w.rows);
  g.A = dy; g.a_m = dy_m; g.a_k = 1;
  set_w(g, w, true);
  g.C = dx; g.c_m = dx_m;
  g.epi = epi; g.aux = aux; g.aux_m = aux_m;
  return run_gemm<kMode>(g, 1, st);
}

template <int kMode>
int vit_forward_impl(const VitW& P, const ImgSet& im, int n, int save, float* out, const VitWs& W, cudaStream_t st) {
  const int M = n * kTok;
  const long long tok_z = (long long)kTok * kD;
  // embedding: im2col gather, patch GEMM (+ bias + pos_embed) into token rows 1..196, cls_token + pos_embed[0]
  {
    const long long tot = (long long)n * kPatches * kPatchK;
    vit_embed_gather_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(im, n, W.col);
    VIT_TRY(check_launch("vit_embed_gather_kernel"));
    float* x0 = save ? W.blk[0].x_in : W.X0;
    Gemm g = gemm(kPatches, kD, kPatchK);
    g.A = W.col; g.a_z1 = (long long)kPatches * kPatchK; g.a_m = kPatchK; g.a_k = 1;
    set_w(g, P.mat(P.L.pe, kD, kPatchK), false);
    g.C = x0 + kD; g.c_z1 = tok_z; g.c_m = kD;
    g.bias = P.v(P.L.pe_b); g.epi = EPI_EMBED; g.pos = P.v(P.L.pos);
    VIT_TRY(run_gemm<kMode>(g, n, st));
    vit_cls_rows_kernel<<<(n * kD + 255) / 256, 256, 0, st>>>(P.v(P.L.cls), P.v(P.L.pos), x0, tok_z, n);
    VIT_TRY(check_launch("vit_cls_rows_kernel"));
  }
  for (int l = 0; l < kBlocks - 1; ++l) {
    const VitBlockW& B = P.L.blk[l];
    float* x_in = save ? W.blk[l].x_in : W.X0;
    float* x_mid = save ? W.blk[l].x_mid : W.X1;
    float* x_out = save ? W.blk[l + 1].x_in : W.X0;
    float* qkv = save ? W.blk[l].qkv : W.qkv;
    float* O = save ? W.blk[l].O : W.O;
    float* lse = save ? W.blk[l].lse : W.lse;
    VIT_TRY(ln_fwd(x_in, kD, P.v(B.n1w), P.v(B.n1b), W.ln, kD, M, st));
    VIT_TRY(linear<kMode>(W.ln, kD, P.mat(B.qkv, kQkv, kD), P.v(B.qkv_b), M, qkv, kQkv, EPI_STORE, nullptr, nullptr, 0, st));
    VIT_TRY(scores<kMode>(qkv, n, kTok, kQkv, W.S, st));
    vit_softmax_kernel<<<row_grid((long long)n * kHeads * kTok), kRowThreads, 0, st>>>(W.S, lse, kTok, n * kHeads * kTok);
    VIT_TRY(check_launch("vit_softmax_kernel"));
    VIT_TRY(attn_pv<kMode>(W.S, qkv, n, kTok, O, tok_z, kD, st));
    VIT_TRY(linear<kMode>(O, kD, P.mat(B.proj, kD, kD), P.v(B.proj_b), M, x_mid, kD, EPI_RESID, x_in, nullptr, kD, st));
    VIT_TRY(ln_fwd(x_mid, kD, P.v(B.n2w), P.v(B.n2b), W.ln, kD, M, st));
    VIT_TRY(linear<kMode>(W.ln, kD, P.mat(B.fc1, kMlp, kD), P.v(B.fc1_b), M, W.h, kMlp, EPI_GELU, nullptr,
                          save ? W.blk[l].pre : nullptr, kMlp, st));
    VIT_TRY(linear<kMode>(W.h, kMlp, P.mat(B.fc2, kD, kMlp), P.v(B.fc2_b), M, x_out, kD, EPI_RESID, x_mid, nullptr, kD, st));
  }
  // block 11, pruned to the CLS rows: K, V for every token, Q and the rest for row 0 of each image
  const VitBlockW& B = P.L.blk[kBlocks - 1];
  float* x_in = save ? W.blk[kBlocks - 1].x_in : W.X0;
  float* qkv = save ? W.blk[kBlocks - 1].qkv : W.qkv;
  const Mat wqkv = P.mat(B.qkv, kQkv, kD);
  VIT_TRY(ln_fwd(x_in, kD, P.v(B.n1w), P.v(B.n1b), W.ln, kD, M, st));
  VIT_TRY(linear<kMode>(W.ln, kD, wqkv, P.v(B.qkv_b) + kD, M, qkv + kD, kQkv, EPI_STORE, nullptr, nullptr, 0, st, kD, 2 * kD));
  VIT_TRY(linear<kMode>(W.ln, tok_z, wqkv, P.v(B.qkv_b), n, qkv, (long long)kTok * kQkv, EPI_STORE, nullptr, nullptr, 0,
                        st, 0, kD));
  VIT_TRY(scores<kMode>(qkv, n, 1, kQkv, W.S, st));
  vit_softmax_kernel<<<row_grid((long long)n * kHeads), kRowThreads, 0, st>>>(W.S, W.lse_c, 1, n * kHeads);
  VIT_TRY(check_launch("vit_softmax_kernel"));
  VIT_TRY(attn_pv<kMode>(W.S, qkv, n, 1, W.O_c, kD, kD, st));
  VIT_TRY(linear<kMode>(W.O_c, kD, P.mat(B.proj, kD, kD), P.v(B.proj_b), n, W.xmid_c, kD, EPI_RESID, x_in, nullptr, tok_z, st));
  VIT_TRY(ln_fwd(W.xmid_c, kD, P.v(B.n2w), P.v(B.n2b), W.ln_c, kD, n, st));
  VIT_TRY(linear<kMode>(W.ln_c, kD, P.mat(B.fc1, kMlp, kD), P.v(B.fc1_b), n, W.h_c, kMlp, EPI_GELU, nullptr, W.pre_c, kMlp, st));
  VIT_TRY(linear<kMode>(W.h_c, kMlp, P.mat(B.fc2, kD, kMlp), P.v(B.fc2_b), n, out, kD, EPI_RESID, W.xmid_c, nullptr, kD, st));
  return SNB_OK;
}

// gradient of one block's attention half: from dx_mid (rows q_rows per image, stride dxm_m) to dqkv
template <int kMode>
int attn_bwd(const VitW& P, const VitBlockW& B, const float* qkv, const float* O, long long o_z1, long long o_m,
             const float* lse, int n, int q_rows, long long q_m, const float* dxm, long long dxm_m, float* dO,
             long long do_z1, long long do_m, const VitWs& W, cudaStream_t st) {
  VIT_TRY(linear_dgrad<kMode>(dxm, dxm_m, P.mat(B.proj, kD, kD), n * q_rows, dO, kD, EPI_STORE, nullptr, 0, st));
  VIT_TRY(scores<kMode>(qkv, n, q_rows, q_m, W.S, st));
  {  // dP = dO V^T
    Gemm g = gemm(q_rows, kTok, kHd);
    g.A = dO; g.a_z1 = do_z1; g.a_z2 = kHd; g.a_m = do_m; g.a_k = 1;
    g.Bf = qkv + 2 * kD; g.b_z1 = (long long)kTok * kQkv; g.b_z2 = kHd; g.b_n = kQkv; g.b_k = 1;
    g.C = W.dP; g.c_z1 = kHeads * kTileS; g.c_z2 = kTileS; g.c_m = kLdS; g.nz2 = kHeads;
    VIT_TRY(run_gemm<kMode>(g, n * kHeads, st));
  }
  vit_softmax_bwd_kernel<<<row_grid((long long)n * kHeads * q_rows), kRowThreads, 0, st>>>(
      W.S, W.dP, lse, O, o_z1, o_m, dO, do_z1, do_m, q_rows, n * kHeads * q_rows, 0.125f);
  VIT_TRY(check_launch("vit_softmax_bwd_kernel"));
  const long long qkv_z = (long long)kTok * kQkv;
  {  // dQ = dS K  (query rows only)
    Gemm g = gemm(q_rows, kHd, kTok);
    g.A = W.dP; g.a_z1 = kHeads * kTileS; g.a_z2 = kTileS; g.a_m = kLdS; g.a_k = 1;
    g.Bf = qkv + kD; g.b_z1 = qkv_z; g.b_z2 = kHd; g.b_n = 1; g.b_k = kQkv;
    g.C = W.dqkv; g.c_z1 = qkv_z; g.c_z2 = kHd; g.c_m = q_m; g.nz2 = kHeads;
    VIT_TRY(run_gemm<kMode>(g, n * kHeads, st));
  }
  {  // dK = dS^T Q
    Gemm g = gemm(kTok, kHd, q_rows);
    g.A = W.dP; g.a_z1 = kHeads * kTileS; g.a_z2 = kTileS; g.a_m = 1; g.a_k = kLdS;
    g.Bf = qkv; g.b_z1 = qkv_z; g.b_z2 = kHd; g.b_n = 1; g.b_k = q_m;
    g.C = W.dqkv + kD; g.c_z1 = qkv_z; g.c_z2 = kHd; g.c_m = kQkv; g.nz2 = kHeads;
    VIT_TRY(run_gemm<kMode>(g, n * kHeads, st));
  }
  {  // dV = P^T dO
    Gemm g = gemm(kTok, kHd, q_rows);
    g.A = W.S; g.a_z1 = kHeads * kTileS; g.a_z2 = kTileS; g.a_m = 1; g.a_k = kLdS;
    g.Bf = dO; g.b_z1 = do_z1; g.b_z2 = kHd; g.b_n = 1; g.b_k = do_m;
    g.C = W.dqkv + 2 * kD; g.c_z1 = qkv_z; g.c_z2 = kHd; g.c_m = kQkv; g.nz2 = kHeads;
    VIT_TRY(run_gemm<kMode>(g, n * kHeads, st));
  }
  return linear_dgrad<kMode>(W.dqkv, kQkv, P.mat(B.qkv, kQkv, kD), n * kTok, W.dln, kD, EPI_STORE, nullptr, 0, st);
}

template <int kMode>
int vit_backward_impl(const VitW& P, const ImgSet& dim, int n, const float* d_out, const VitWs& W, cudaStream_t st) {
  const int M = n * kTok;
  const long long tok_z = (long long)kTok * kD;
  vit_grad_scale_kernel<<<n, 128, 0, st>>>(d_out, W.c0, W.inv);
  VIT_TRY(check_launch("vit_grad_scale_kernel"));
  {  // block 11 (CLS rows)
    const VitBlockW& B = P.L.blk[kBlocks - 1];
    const SavedBlock& S = W.blk[kBlocks - 1];
    VIT_TRY(linear_dgrad<kMode>(W.c0, kD, P.mat(B.fc2, kD, kMlp), n, W.ch, kMlp, EPI_GELU_BWD, W.pre_c, kMlp, st));
    VIT_TRY(linear_dgrad<kMode>(W.ch, kMlp, P.mat(B.fc1, kMlp, kD), n, W.c1, kD, EPI_STORE, nullptr, 0, st));
    VIT_TRY(ln_bwd(W.xmid_c, kD, P.v(B.n2w), W.c1, kD, W.c0, kD, 0, W.c2, kD, n, st));
    if (cudaMemsetAsync(W.dqkv, 0, sizeof(float) * M * kQkv, st) != cudaSuccess)
      return fail(SNB_ERR_CUDA, "snb_vit_backward: cudaMemsetAsync failed");
    VIT_TRY(attn_bwd<kMode>(P, B, S.qkv, W.O_c, kD, kD, W.lse_c, n, 1, kQkv, W.c2, kD, W.c1, kD, kD, W, st));
    VIT_TRY(ln_bwd(S.x_in, kD, P.v(B.n1w), W.dln, kD, W.c2, kD, 1, W.dx, kD, M, st));
  }
  for (int l = kBlocks - 2; l >= 0; --l) {
    const VitBlockW& B = P.L.blk[l];
    const SavedBlock& S = W.blk[l];
    VIT_TRY(linear_dgrad<kMode>(W.dx, kD, P.mat(B.fc2, kD, kMlp), M, W.dh, kMlp, EPI_GELU_BWD, S.pre, kMlp, st));
    VIT_TRY(linear_dgrad<kMode>(W.dh, kMlp, P.mat(B.fc1, kMlp, kD), M, W.dln, kD, EPI_STORE, nullptr, 0, st));
    VIT_TRY(ln_bwd(S.x_mid, kD, P.v(B.n2w), W.dln, kD, W.dx, kD, 0, W.dx2, kD, M, st));
    VIT_TRY(attn_bwd<kMode>(P, B, S.qkv, S.O, tok_z, kD, S.lse, n, kTok, kQkv, W.dx2, kD, W.dO, tok_z, kD, W, st));
    VIT_TRY(ln_bwd(S.x_in, kD, P.v(B.n1w), W.dln, kD, W.dx2, kD, 0, W.dx, kD, M, st));
  }
  {  // patch embedding dgrad into the im2col rows, then the fold onto each image's pixels
    Gemm g = gemm(kPatches, kPatchK, kD);
    g.A = W.dx + kD; g.a_z1 = tok_z; g.a_m = kD; g.a_k = 1;
    set_w(g, P.mat(P.L.pe, kD, kPatchK), true);
    g.C = W.col; g.c_z1 = (long long)kPatches * kPatchK; g.c_m = kPatchK;
    VIT_TRY(run_gemm<kMode>(g, n, st));
  }
  for (int i = 0; i < n; ++i) {
    const long long tot = 3ll * dim.h[i] * dim.w[i];
    vit_fold_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(W.col, W.inv, dim, i);
    VIT_TRY(check_launch("vit_fold_kernel"));
  }
  return SNB_OK;
}

template <int kMode>
int vit_pack_impl(const float* const* params, void* image, cudaStream_t st) {
  const VitLayout L = vit_layout(kMode);
  float* f = static_cast<float*>(image);
  uint16_t* h = reinterpret_cast<uint16_t*>(f + L.n_floats);
  auto vec = [&](int idx, long long off, long long numel) -> int {
    if (cudaMemcpyAsync(f + off, params[idx], numel * 4, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
      return fail(SNB_ERR_CUDA, "snb_vit_pack: cudaMemcpyAsync of tensor %d failed", idx);
    return SNB_OK;
  };
  auto mat = [&](int idx, long long off, long long numel) -> int {
    uint16_t* hi = h + off;
    vit_pack_kernel<kMode><<<(unsigned)((numel / 2 + 255) / 256), 256, 0, st>>>(params[idx], numel, hi, hi + numel);
    return check_launch("vit_pack_kernel");
  };
  VIT_TRY(vec(0, L.cls, kD));
  VIT_TRY(vec(1, L.pos, (long long)kTok * kD));
  VIT_TRY(mat(2, L.pe, (long long)kD * kPatchK));
  VIT_TRY(vec(3, L.pe_b, kD));
  for (int b = 0; b < kBlocks; ++b) {
    const VitBlockW& B = L.blk[b];
    const int p = 4 + 12 * b;
    VIT_TRY(vec(p + 0, B.n1w, kD));
    VIT_TRY(vec(p + 1, B.n1b, kD));
    VIT_TRY(mat(p + 2, B.qkv, (long long)kQkv * kD));
    VIT_TRY(vec(p + 3, B.qkv_b, kQkv));
    VIT_TRY(mat(p + 4, B.proj, (long long)kD * kD));
    VIT_TRY(vec(p + 5, B.proj_b, kD));
    VIT_TRY(vec(p + 6, B.n2w, kD));
    VIT_TRY(vec(p + 7, B.n2b, kD));
    VIT_TRY(mat(p + 8, B.fc1, (long long)kMlp * kD));
    VIT_TRY(vec(p + 9, B.fc1_b, kMlp));
    VIT_TRY(mat(p + 10, B.fc2, (long long)kD * kMlp));
    VIT_TRY(vec(p + 11, B.fc2_b, kD));
  }
  return SNB_OK;
}

int fill_images(const char* who, const float* const* images, const int64_t* strides, const int* sizes, int n,
                ImgSet& im) {
  SNB_REQUIRE(n >= 1 && n <= SNB_VIT_MAX_IMAGES, "%s: n_images must be in [1, %d] (got %d)", who, SNB_VIT_MAX_IMAGES, n);
  SNB_REQUIRE(images != nullptr && strides != nullptr && sizes != nullptr, "%s: null image / stride / size array", who);
  for (int i = 0; i < n; ++i) {
    SNB_REQUIRE(images[i] != nullptr, "%s: null image pointer %d", who, i);
    SNB_REQUIRE(sizes[2 * i] >= 1 && sizes[2 * i + 1] >= 1, "%s: image %d has size %d x %d", who, i, sizes[2 * i],
                sizes[2 * i + 1]);
    im.p[i] = images[i];
    im.h[i] = sizes[2 * i];
    im.w[i] = sizes[2 * i + 1];
    for (int j = 0; j < 3; ++j) im.s[i][j] = strides[3 * i + j];
  }
  return SNB_OK;
}

}  // namespace
}  // namespace snb

using namespace snb;

extern "C" {

size_t snb_vit_pack_bytes(int precision) {
  const int mode = mode_of(precision);
  return mode < 0 ? 0 : vit_image_bytes(mode);
}

int snb_vit_pack(const float* const* params, int precision, void* image, void* stream) {
  const int mode = mode_of(precision);
  if (mode < 0) return fail(SNB_ERR_UNSUPPORTED, "snb_vit_pack: unknown precision %d", precision);
  SNB_REQUIRE(params != nullptr && image != nullptr, "snb_vit_pack: null params or image");
  for (int i = 0; i < SNB_VIT_N_TENSORS; ++i) SNB_REQUIRE(params[i] != nullptr, "snb_vit_pack: null tensor %d", i);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == kSplit) return vit_pack_impl<kSplit>(params, image, st);
  if (mode == kF16) return vit_pack_impl<kF16>(params, image, st);
  return vit_pack_impl<kBf16>(params, image, st);
}

size_t snb_vit_workspace_bytes(int n_images, int save) {
  if (n_images < 1 || n_images > SNB_VIT_MAX_IMAGES) return 0;
  return vit_ws(nullptr, n_images, save ? 1 : 0).bytes;
}

int snb_vit_forward(const void* image, int precision, const float* const* images, const int64_t* strides,
                    const int* sizes, int n_images, int save, float* out, void* workspace, void* stream) {
  const char* who = "snb_vit_forward";
  const int mode = mode_of(precision);
  if (mode < 0) return fail(SNB_ERR_UNSUPPORTED, "%s: unknown precision %d", who, precision);
  ImgSet im{};
  VIT_TRY(fill_images(who, images, strides, sizes, n_images, im));
  SNB_REQUIRE(image != nullptr && out != nullptr && workspace != nullptr, "%s: null weight image, out or workspace", who);
  const VitW P = vit_view(image, mode);
  const VitWs W = vit_ws(workspace, n_images, save ? 1 : 0);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == kSplit) return vit_forward_impl<kSplit>(P, im, n_images, save ? 1 : 0, out, W, st);
  if (mode == kF16) return vit_forward_impl<kF16>(P, im, n_images, save ? 1 : 0, out, W, st);
  return vit_forward_impl<kBf16>(P, im, n_images, save ? 1 : 0, out, W, st);
}

int snb_vit_backward(const void* image, int precision, const int* sizes, int n_images, const float* d_out,
                     float* const* d_images, const int64_t* d_strides, void* workspace, void* stream) {
  const char* who = "snb_vit_backward";
  const int mode = mode_of(precision);
  if (mode < 0) return fail(SNB_ERR_UNSUPPORTED, "%s: unknown precision %d", who, precision);
  ImgSet im{};
  VIT_TRY(fill_images(who, const_cast<const float* const*>(d_images), d_strides, sizes, n_images, im));
  SNB_REQUIRE(image != nullptr && d_out != nullptr && workspace != nullptr, "%s: null weight image, d_out or workspace",
              who);
  const VitW P = vit_view(image, mode);
  const VitWs W = vit_ws(workspace, n_images, 1);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == kSplit) return vit_backward_impl<kSplit>(P, im, n_images, d_out, W, st);
  if (mode == kF16) return vit_backward_impl<kF16>(P, im, n_images, d_out, W, st);
  return vit_backward_impl<kBf16>(P, im, n_images, d_out, W, st);
}

}  // extern "C"
