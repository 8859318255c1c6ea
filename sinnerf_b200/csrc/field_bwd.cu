// field_bwd.cu -- backward of the field MLP (reference: autograd through models/nerf.py:105-148):
// the driver that walks the layers, the head kernel, the folded bottleneck, and the fp32 FFMA
// versions of the two GEMMs.  The GEMMs themselves run on tensor cores (wgrad_tc.cu, dgrad_tc.cu).
//
// Per render pass, given g_raw (P,4) = dL/d[r,g,b,sigma] from composite_bwd:
//   heads     : rgb head + its activation, direction-layer activation, sigma head  (head_bwd_kernel)
//   dir layer : W' = Wd[:, :256] Wf (fold_weights_kernel); dW', db' by one wgrad against h8; the chain
//               rule back to Wd, Wf, bf, bd is three P-independent products (unfold_grads_kernel)
//   per layer : dW_l += dY_l^T X_l, db_l += sum dY_l          (run_wgrad -> wgrad_tc_kernel | wgrad_kernel)
//               dX_l  = dY_l W_l  (x ReLU mask of the saved input, + sigma term at h8)
//                                                              (run_dgrad -> dgrad_tc_kernel | dgrad_kernel)
// walking dir layer -> layers 8..1.  Nothing flows into rays, z or across sample_pdf (the reference
// detaches it, models/rendering.py:311-313).
//
// Activations are plain (P, C) row-major fp32 tensors.  The FFMA kernels (SNB_BWD_SIMT=1) stream rows
// with 16-byte cp.async copies; wgrad_kernel accumulates a 128x128 block of dW per CTA in registers
// over a slice of P and finishes with atomics (split-P), dgrad_kernel is the forward tiling with W
// used untransposed.  Their roofline is the FP32 FFMA pipe; the tensor-core versions are HBM-bound.
#include <stdlib.h>

#include "common.cuh"

namespace snb {

constexpr int BT = 256;  // threads

__device__ __forceinline__ void cp16(void* smem, const void* gmem) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(a), "l"(gmem));
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// ------------------------------------------------------------------------------------------
// wgrad:  dW[n0+n][col_off + k] += sum_p dY[p][n0+n] * X[p][k0+k],  db[n0+n] += sum_p dY[p][n0+n]
// grid = (N/128, ceil(K/128), splits); each CTA walks rows [split*rows_per, +rows_per) in 32-row stages.
// ------------------------------------------------------------------------------------------
constexpr int WG_ROWS = 16;
struct WgradArgs {
  const float* dY; int ldy;        // (P, ldy)
  const float* X; int ldx;         // (P, ldx)
  int K;                           // valid columns of X
  float* dW; int ldw; int col_off; // dW (N, ldw): block lands at columns [col_off, col_off + K)
  float* db;                       // nullable; written by k-block 0 only
  long long P;
  long long rows_per_split;
};

__global__ void __launch_bounds__(BT) wgrad_kernel(WgradArgs a) {
  __shared__ __align__(16) float sY[2][WG_ROWS][128];
  __shared__ __align__(16) float sX[2][WG_ROWS][128];
  const int tid = threadIdx.x, tn = tid >> 4, tk = tid & 15;   // 16 x 16 threads, 8x8 outputs each
  const int n0 = blockIdx.x * 128, k0 = blockIdx.y * 128;
  const long long r_begin = (long long)blockIdx.z * a.rows_per_split;
  const long long r_end = r_begin + a.rows_per_split < a.P ? r_begin + a.rows_per_split : a.P;
  float acc[8][8];
  float accb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    accb[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  }
  const int kcols = a.K - k0 < 128 ? a.K - k0 : 128;   // valid X columns in this block (multiple of 4 by padding)
  auto load_stage = [&](int buf, long long r0) {
    // 32 rows x 128 floats from each operand = 1024 float4 each; 4 per thread per operand
#pragma unroll
    for (int v = tid; v < WG_ROWS * 32; v += BT) {
      const int r = v >> 5, c4 = (v & 31) * 4;
      const long long row = r0 + r;
      float* dy = &sY[buf][r][c4];
      float* dx = &sX[buf][r][c4];
      if (row < r_end) {
        cp16(dy, a.dY + row * a.ldy + n0 + c4);
        if (c4 < kcols) cp16(dx, a.X + row * a.ldx + k0 + c4);
        else *reinterpret_cast<float4*>(dx) = make_float4(0.f, 0.f, 0.f, 0.f);
      } else {
        *reinterpret_cast<float4*>(dy) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(dx) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  if (r_begin < r_end) {
    load_stage(0, r_begin);
    cp_commit();
    int buf = 0;
    for (long long r0 = r_begin; r0 < r_end; r0 += WG_ROWS, buf ^= 1) {
      if (r0 + WG_ROWS < r_end) {
        load_stage(buf ^ 1, r0 + WG_ROWS);
        cp_commit();
        cp_wait<1>();
      } else {
        cp_wait<0>();
      }
      __syncthreads();
#pragma unroll 4
      for (int r = 0; r < WG_ROWS; ++r) {
        const float4 y0 = *reinterpret_cast<const float4*>(&sY[buf][r][tn * 8]);
        const float4 y1 = *reinterpret_cast<const float4*>(&sY[buf][r][tn * 8 + 4]);
        const float4 x0 = *reinterpret_cast<const float4*>(&sX[buf][r][tk * 8]);
        const float4 x1 = *reinterpret_cast<const float4*>(&sX[buf][r][tk * 8 + 4]);
        const float y[8] = {y0.x, y0.y, y0.z, y0.w, y1.x, y1.y, y1.z, y1.w};
        const float x[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          if (tk == 0) accb[i] += y[i];
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(y[i], x[j], acc[i][j]);
        }
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int n = n0 + tn * 8 + i;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int k = k0 + tk * 8 + j;
      if (k < a.K) atomicAdd(a.dW + (size_t)n * a.ldw + a.col_off + k, acc[i][j]);
    }
    if (a.db != nullptr && blockIdx.y == 0 && tk == 0) atomicAdd(a.db + n, accb[i]);
  }
}

// ------------------------------------------------------------------------------------------
// dgrad:  dX[p][k] = ( sum_n dY[p][n] * W[n][col_off + k] + extra[p] * evec[k] ) * [mask[p][k] > 0]
// 128-row tile per CTA, K = 256 outputs, N = 256 or 128 reduction.
// ------------------------------------------------------------------------------------------
struct DgradArgs {
  const float* dY; int N;          // (P, N)
  const float* W; int ldw; int col_off;   // nn.Linear weight (N, ldw)
  const float* mask;               // (P,256) saved input activation (ReLU mask), nullable
  const float* extra; int extra_stride;   // nullable: per-row scalar (g_sigma = g_raw[:,3])
  const float* evec;               // (256) sigma head weight
  float* dX;                       // (P,256)
  long long P;
};

struct DgradSmem {
  float y[128][260];        // dY tile, row-major, padded
  float w[2][16][256];      // weight slices W[n..n+15][col_off..+255]
};

__global__ void __launch_bounds__(BT, 1) dgrad_kernel(DgradArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  DgradSmem& s = *reinterpret_cast<DgradSmem*>(smem_raw);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long ntiles = (a.P + 127) / 128;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long p0 = tile * 128;
    // stage the dY tile
    const int nvec = a.N / 4;
    for (int v = tid; v < 128 * nvec; v += BT) {
      const int r = v / nvec, c4 = (v - r * nvec) * 4;
      if (p0 + r < a.P) cp16(&s.y[r][c4], a.dY + (p0 + r) * a.N + c4);
      else *reinterpret_cast<float4*>(&s.y[r][c4]) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    auto load_w = [&](int buf, int n_base) {
      for (int v = tid; v < 16 * 64; v += BT) {
        const int r = v >> 6, c4 = (v & 63) * 4;
        // W rows are ldw floats apart and col_off may be odd (skip layer: 63): scalar-safe path
        const float* src = a.W + (size_t)(n_base + r) * a.ldw + a.col_off + c4;
        if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) cp16(&s.w[buf][r][c4], src);
        else {
          s.w[buf][r][c4] = src[0]; s.w[buf][r][c4 + 1] = src[1];
          s.w[buf][r][c4 + 2] = src[2]; s.w[buf][r][c4 + 3] = src[3];
        }
      }
    };
    load_w(0, 0);
    cp_commit();
    float acc[8][16];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[i][j] = 0.f;
    const int nslices = a.N / 16;
    for (int sl = 0; sl < nslices; ++sl) {
      if (sl + 1 < nslices) {
        load_w((sl + 1) & 1, (sl + 1) * 16);
        cp_commit();
        cp_wait<1>();
      } else {
        cp_wait<0>();
      }
      __syncthreads();
      const float(*wb)[256] = s.w[sl & 1];
#pragma unroll
      for (int n4 = 0; n4 < 16; n4 += 4) {
        float4 yv[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) yv[i] = *reinterpret_cast<const float4*>(&s.y[ty * 8 + i][sl * 16 + n4]);
#pragma unroll
        for (int nn = 0; nn < 4; ++nn) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float4 b = *reinterpret_cast<const float4*>(&wb[n4 + nn][j * 64 + tx * 4]);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float y = nn == 0 ? yv[i].x : (nn == 1 ? yv[i].y : (nn == 2 ? yv[i].z : yv[i].w));
              acc[i][j * 4 + 0] = fmaf(y, b.x, acc[i][j * 4 + 0]);
              acc[i][j * 4 + 1] = fmaf(y, b.y, acc[i][j * 4 + 1]);
              acc[i][j * 4 + 2] = fmaf(y, b.z, acc[i][j * 4 + 2]);
              acc[i][j * 4 + 3] = fmaf(y, b.w, acc[i][j * 4 + 3]);
            }
          }
        }
      }
      __syncthreads();
    }
    // epilogue: + g_sigma * w_sigma, ReLU mask of the saved activation, store
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long row = p0 + ty * 8 + i;
      if (row >= a.P) continue;
      const float ex = a.extra != nullptr ? a.extra[row * a.extra_stride] : 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = j * 64 + tx * 4;
        float4 v = make_float4(acc[i][j * 4], acc[i][j * 4 + 1], acc[i][j * 4 + 2], acc[i][j * 4 + 3]);
        if (a.extra != nullptr) {
          const float4 e = *reinterpret_cast<const float4*>(a.evec + c);
          v.x = fmaf(ex, e.x, v.x); v.y = fmaf(ex, e.y, v.y); v.z = fmaf(ex, e.z, v.z); v.w = fmaf(ex, e.w, v.w);
        }
        if (a.mask != nullptr) {
          const float4 m = *reinterpret_cast<const float4*>(a.mask + row * 256 + c);
          v.x = m.x > 0.f ? v.x : 0.f; v.y = m.y > 0.f ? v.y : 0.f;
          v.z = m.z > 0.f ? v.z : 0.f; v.w = m.w > 0.f ? v.w : 0.f;
        }
        *reinterpret_cast<float4*>(a.dX + row * 256 + c) = v;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------
// heads: one warp walks points; lanes own 4 of the 128 direction-layer units and 8 of the 256
// trunk units.  dS = (W_rgb^T g_pre_rgb) * act'(G);  dW_rgb, db_rgb, dW_sigma, db_sigma.
// ------------------------------------------------------------------------------------------
struct HeadArgs {
  const float* g_raw;   // (P,4)
  const float* raw;     // (P,4) forward output [rgb (post-activation), sigma]
  const float* G;       // (P,128) direction layer output
  const float* H8;      // (P,256)
  const float* Wr;      // (3,128)
  int new_activation;
  float* dS;            // (P,128)
  float* dWr; float* dbr; float* dWs; float* dbs;
  long long P;
};

__global__ void __launch_bounds__(256) head_bwd_kernel(HeadArgs a) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  float wr[3][4];
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int j = 0; j < 4; ++j) wr[c][j] = a.Wr[c * 128 + lane * 4 + j];
  float awr[3][4] = {}, abr[3] = {0.f, 0.f, 0.f}, aws[8] = {}, abs_ = 0.f;
  // 4 points per warp iteration: all their loads are issued before any is used (the kernel is a pure
  // HBM stream, 2 KB per point; one point at a time left it latency-bound)
  constexpr int kU = 4;
  for (long long pb = warp * kU; pb < a.P; pb += nwarps * kU) {
    float4 g[kU], o[kU], gv[kU], h0[kU], h1[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const long long p = pb + u < a.P ? pb + u : a.P - 1;      // tail: re-read the last point, contribute nothing
      g[u] = reinterpret_cast<const float4*>(a.g_raw)[p];
      o[u] = reinterpret_cast<const float4*>(a.raw)[p];
      gv[u] = *reinterpret_cast<const float4*>(a.G + p * 128 + lane * 4);
      h0[u] = *reinterpret_cast<const float4*>(a.H8 + p * 256 + lane * 8);
      h1[u] = *reinterpret_cast<const float4*>(a.H8 + p * 256 + lane * 8 + 4);
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      if (pb + u >= a.P) break;
      const long long p = pb + u;
      float gp[3];
      const float gin[3] = {g[u].x, g[u].y, g[u].z}, out[3] = {o[u].x, o[u].y, o[u].z};
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        if (a.new_activation) {
          // y = 0.5 (1 + 1.002 tanh(x/2))  ->  dy/dx = 0.2505 (1 - tanh^2)
          const float t = (2.0f * out[c] - 1.0f) * (1.0f / 1.002f);
          gp[c] = gin[c] * 0.2505f * (1.0f - t * t);
        } else {
          gp[c] = gin[c] * out[c] * (1.0f - out[c]);
        }
      }
      const float gg[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
      float ds[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float dg = wr[0][j] * gp[0] + wr[1][j] * gp[1] + wr[2][j] * gp[2];
        // softplus'(s) = sigmoid(s) = 1 - exp(-softplus(s));  ReLU' = [g > 0]
        const float der = a.new_activation ? (1.0f - expf(-gg[j])) : (gg[j] > 0.f ? 1.0f : 0.f);
        ds[j] = dg * der;
#pragma unroll
        for (int c = 0; c < 3; ++c) awr[c][j] = fmaf(gp[c], gg[j], awr[c][j]);
      }
      *reinterpret_cast<float4*>(a.dS + p * 128 + lane * 4) = make_float4(ds[0], ds[1], ds[2], ds[3]);
      const float hv[8] = {h0[u].x, h0[u].y, h0[u].z, h0[u].w, h1[u].x, h1[u].y, h1[u].z, h1[u].w};
#pragma unroll
      for (int j = 0; j < 8; ++j) aws[j] = fmaf(g[u].w, hv[j], aws[j]);
      if (lane == 0) { abr[0] += gp[0]; abr[1] += gp[1]; abr[2] += gp[2]; abs_ += g[u].w; }
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int j = 0; j < 4; ++j) atomicAdd(a.dWr + c * 128 + lane * 4 + j, awr[c][j]);
#pragma unroll
  for (int j = 0; j < 8; ++j) atomicAdd(a.dWs + lane * 8 + j, aws[j]);
  if (lane == 0) {
    atomicAdd(a.dbr + 0, abr[0]); atomicAdd(a.dbr + 1, abr[1]); atomicAdd(a.dbr + 2, abr[2]);
    atomicAdd(a.dbs, abs_);
  }
}

// ------------------------------------------------------------------------------------------
// host: the whole MLP backward of one render pass
// ------------------------------------------------------------------------------------------
static int dev_sms() { return sm_count(); }

// wgrad_tc.cu: the same contraction on tensor cores (wgmma, bf16 hi/lo split, fp32 accumulate in registers)
int run_wgrad_tc(const float* dY, int N, const float* X, int ldx, int K, float* dW, int ldw, int col_off, float* db,
                 uint32_t* x_pos_bits, long long P, cudaStream_t st);

// SNB_BWD_SIMT=1 keeps the FFMA kernels (debugging / A-B timing); the tensor-core kernels are the default
static bool bwd_simt() {
  static const bool simt = getenv("SNB_BWD_SIMT") && atoi(getenv("SNB_BWD_SIMT")) != 0;
  return simt;
}

// x_bits (nullable): where the tensor-core kernel leaves [X > 0] for the dgrad of the same layer
static int run_wgrad(const float* dY, int N, const float* X, int ldx, int K, float* dW, int ldw, int col_off,
                     float* db, uint32_t* x_bits, long long P, cudaStream_t st) {
  if (!bwd_simt()) return run_wgrad_tc(dY, N, X, ldx, K, dW, ldw, col_off, db, x_bits, P, st);
  WgradArgs a{dY, N, X, ldx, K, dW, ldw, col_off, db, P, 0};
  const int nb = N / 128, kb = (K + 127) / 128;
  int splits = (2 * dev_sms()) / (nb * kb);
  if (splits < 1) splits = 1;
  long long rows = (P + splits - 1) / splits;
  rows = (rows + WG_ROWS - 1) / WG_ROWS * WG_ROWS;
  splits = (int)((P + rows - 1) / rows);
  a.rows_per_split = rows;
  wgrad_kernel<<<dim3(nb, kb, splits), BT, 0, st>>>(a);
  return check_launch("wgrad_kernel");
}

// dgrad_tc.cu: the same product on tensor cores (CTA pairs, W^T resident in shared memory)
int run_dgrad_tc(const float* dY, int N, const float* W, int ldw, int col_off, const uint32_t* mask_bits,
                 const float* extra, int extra_stride, const float* evec, float* dX, long long P, cudaStream_t st);

// mask: the saved fp32 input of the layer (FFMA kernel); mask_bits: its sign bits (tensor-core kernel)
static int run_dgrad(const float* dY, int N, const float* W, int ldw, int col_off, const float* mask,
                     const uint32_t* mask_bits, const float* extra, int extra_stride, const float* evec, float* dX,
                     long long P, cudaStream_t st) {
  if (!bwd_simt()) return run_dgrad_tc(dY, N, W, ldw, col_off, mask_bits, extra, extra_stride, evec, dX, P, st);
  static SmemOptIn optin;
  if (int rc = ensure_smem(dgrad_kernel, optin, (int)sizeof(DgradSmem), "dgrad")) return rc;
  DgradArgs a{dY, N, W, ldw, col_off, mask, extra, extra_stride, evec, dX, P};
  const long long ntiles = (P + 127) / 128;
  const int grid = (int)(ntiles < dev_sms() ? ntiles : dev_sms());
  dgrad_kernel<<<grid, BT, sizeof(DgradSmem), st>>>(a);
  return check_launch("dgrad_kernel");
}

// params / grads: 24 device pointers in state-dict order (SNB_N_PARAM_TENSORS); grads are accumulated into.
// ------------------------------------------------------------------------------------------
// The bottleneck ("xyz_encoding_final", nerf.py:140) has no activation, so the direction layer sees
//   s = Wd[:, :256] (Wf h8 + bf) + Wd[:, 256:] dir + bd = W' h8 + Wd[:, 256:] dir + b',  W' = Wd[:, :256] Wf
// -- the forward kernels use exactly that (field_tc.cu folds W' at pack time), and so does the
// backward: one wgrad against h8 gives dW' (128 x 256) and db' (128), and the chain rule through the
// product is three tiny matrix products that do not depend on the number of points:
//   dWd[:, :256] += dW' Wf^T + db' (x) bf     dWf += Wd[:, :256]^T dW'     dbf += Wd[:, :256]^T db'     dbd += db'
// No per-point bottleneck activations, no P-sized wgrad / dgrad for that layer.
// ------------------------------------------------------------------------------------------
constexpr int kFoldW = 0, kFoldDW = kHalf * kWidth, kFoldDB = 2 * kHalf * kWidth;   // offsets into ws_w (floats)

__global__ void fold_weights_kernel(const float* __restrict__ Wd, const float* __restrict__ Wf, float* __restrict__ ws) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < kHalf * kWidth; e += gridDim.x * blockDim.x) {
    const int n = e / kWidth, k = e - n * kWidth;
    float acc = 0.f;
    for (int j = 0; j < kWidth; ++j) acc = fmaf(Wd[n * 283 + j], Wf[j * kWidth + k], acc);
    ws[kFoldW + e] = acc;
    ws[kFoldDW + e] = 0.f;
    if (e < kHalf) ws[kFoldDB + e] = 0.f;
  }
}

__global__ void unfold_grads_kernel(const float* __restrict__ Wd, const float* __restrict__ Wf, const float* __restrict__ bf,
                                    const float* __restrict__ ws, float* __restrict__ dWd, float* __restrict__ dbd,
                                    float* __restrict__ dWf, float* __restrict__ dbf) {
  const float* dWp = ws + kFoldDW;
  const float* dbp = ws + kFoldDB;
  const int n_a = kHalf * kWidth, n_b = kWidth * kWidth;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n_a + n_b + kWidth + kHalf; e += gridDim.x * blockDim.x) {
    if (e < n_a) {                       // dWd[n][j] += sum_k dW'[n][k] Wf[j][k] + db'[n] bf[j]
      const int n = e / kWidth, j = e - n * kWidth;
      float acc = dbp[n] * bf[j];
      for (int k = 0; k < kWidth; ++k) acc = fmaf(dWp[n * kWidth + k], Wf[j * kWidth + k], acc);
      dWd[n * 283 + j] += acc;
    } else if (e < n_a + n_b) {          // dWf[j][k] += sum_n Wd[n][j] dW'[n][k]
      const int f = e - n_a, j = f / kWidth, k = f - j * kWidth;
      float acc = 0.f;
      for (int n = 0; n < kHalf; ++n) acc = fmaf(Wd[n * 283 + j], dWp[n * kWidth + k], acc);
      dWf[f] += acc;
    } else if (e < n_a + n_b + kWidth) { // dbf[j] += sum_n Wd[n][j] db'[n]
      const int j = e - n_a - n_b;
      float acc = 0.f;
      for (int n = 0; n < kHalf; ++n) acc = fmaf(Wd[n * 283 + j], dbp[n], acc);
      dbf[j] += acc;
    } else {
      const int n = e - n_a - n_b - kWidth;
      dbd[n] += dbp[n];
    }
  }
}

// launch wrappers shared with the 16-bit backward (bwd16.cu)
int launch_fold_weights(const float* Wd, const float* Wf, float* ws, cudaStream_t st) {
  fold_weights_kernel<<<128, 256, 0, st>>>(Wd, Wf, ws);
  return check_launch("fold_weights_kernel");
}
int launch_unfold_grads(const float* Wd, const float* Wf, const float* bf, const float* ws, float* dWd, float* dbd,
                        float* dWf, float* dbf, cudaStream_t st) {
  unfold_grads_kernel<<<392, 256, 0, st>>>(Wd, Wf, bf, ws, dWd, dbd, dWf, dbf);
  return check_launch("unfold_grads_kernel");
}

int field_backward_fp32(const float* const* params, float* const* grads, int new_activation, const float* g_raw,
                        const float* raw, const float* save_enc, const float* save_dir, const float* save_h,
                        const float* save_g, int64_t n_points, float* ws_a, float* ws_b, float* ws_s, float* ws_w,
                        uint32_t* ws_m, cudaStream_t st) {
  const long long P = n_points;
  if (P == 0) return SNB_OK;
  auto H = [&](int l) { return save_h + (size_t)l * P * kWidth; };   // l = 0..7: h1..h8
  int rc;
  // heads
  {
    HeadArgs a{g_raw, raw, save_g, H(7), params[kRgbW], new_activation, ws_s,
               grads[kRgbW], grads[kRgbB], grads[kSigmaW], grads[kSigmaB], P};
    const int grid = dev_sms() * 4;
    head_bwd_kernel<<<grid, 256, 0, st>>>(a);
    if ((rc = check_launch("head_bwd_kernel"))) return rc;
  }
  // direction layer with the bottleneck folded in: X = [h8 (through W') | dir]
  fold_weights_kernel<<<128, 256, 0, st>>>(params[18], params[16], ws_w);
  if ((rc = check_launch("fold_weights_kernel"))) return rc;
  if ((rc = run_wgrad(ws_s, 128, H(7), 256, 256, ws_w + kFoldDW, 256, 0, ws_w + kFoldDB, ws_m, P, st))) return rc;
  if ((rc = run_wgrad(ws_s, 128, save_dir, kDirPad, kDirCh, grads[18], 283, 256, nullptr, nullptr, P, st))) return rc;
  unfold_grads_kernel<<<392, 256, 0, st>>>(params[18], params[16], params[17], ws_w, grads[18], grads[19], grads[16],
                                           grads[17]);
  if ((rc = check_launch("unfold_grads_kernel"))) return rc;
  // into h8: through W', plus the sigma head's term; ReLU mask of h8
  if ((rc = run_dgrad(ws_s, 128, ws_w + kFoldW, 256, 0, H(7), ws_m, g_raw + 3, 4, params[kSigmaW], ws_b, P, st))) return rc;
  // trunk layers 8..2 (index l = 7..1): dY lives in cur, dX goes to nxt
  float* cur = ws_b;
  float* nxt = ws_a;
  for (int l = 7; l >= 1; --l) {
    const int ldw = l == 4 ? 319 : 256;
    if (l == 4) {
      if ((rc = run_wgrad(cur, 256, save_enc, kXyzPad, kXyzCh, grads[2 * l], ldw, 0, grads[2 * l + 1], nullptr, P, st))) return rc;
      if ((rc = run_wgrad(cur, 256, H(l - 1), 256, 256, grads[2 * l], ldw, kXyzCh, nullptr, ws_m, P, st))) return rc;
      if ((rc = run_dgrad(cur, 256, params[2 * l], ldw, kXyzCh, H(l - 1), ws_m, nullptr, 0, nullptr, nxt, P, st))) return rc;
    } else {
      if ((rc = run_wgrad(cur, 256, H(l - 1), 256, 256, grads[2 * l], ldw, 0, grads[2 * l + 1], ws_m, P, st))) return rc;
      if ((rc = run_dgrad(cur, 256, params[2 * l], ldw, 0, H(l - 1), ws_m, nullptr, 0, nullptr, nxt, P, st))) return rc;
    }
    float* t = cur; cur = nxt; nxt = t;
  }
  // layer 1: weights only
  return run_wgrad(cur, 256, save_enc, kXyzPad, kXyzCh, grads[0], 63, 0, grads[1], nullptr, P, st);
}

}  // namespace snb
