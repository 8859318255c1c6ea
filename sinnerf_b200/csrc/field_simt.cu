// field_simt.cu -- exact-fp32 fused field pass (FFMA on CUDA cores).
//
// Replaces, per tile of 128 sample points, the reference's
//   xyz = o + d*z                      models/rendering.py:284-285
//   Embedding(3,10), Embedding(3,4)    models/nerf.py:24-41
//   repeat_interleave + cat            models/rendering.py:188-201
//   NeRF.forward (12 Linear layers)    models/nerf.py:105-148
// with ONE kernel whose activations never leave shared memory.  This is the SNB_PREC_FP32
// mode: plain fp32 FMA chains, so it matches the reference's fp32 GEMMs to round-off.  The
// tensor-core modes live in field_tc.cu.
//
// Roofline: FP32 FFMA pipe.  Per point 593 408 FMA.  HBM traffic is 20 B/point
// (z in, rgbsigma out) + 32 B/ray, i.e. nothing: weights (2.4 MB) stay L2-resident.
//
// Tiling: one CTA (256 threads) owns a 128-point tile; activations live K-major in smem
// (act[k][row]) so a thread's 8-row register tile is two LDS.128; weights stream from L2 in
// 16-deep K slices through a cp.async double buffer; each thread accumulates an 8x16 (8x8 for
// the 128-wide direction layer) fp32 register tile.
#include "common.cuh"

namespace snb {

constexpr int TM = 128;       // points per tile
constexpr int NTHREADS = 256;
constexpr int KS = 16;        // K slice depth per pipeline stage

struct __align__(16) FieldSmem {
  float act[kWidth * TM];     // hidden activations, K-major, 8-row groups XOR-swizzled by k
  float enc[kXyzPad * TM];    // xyz embedding (63 + zero pad)
  float dir[kDirPad * TM];    // dir embedding (27 + zero pad), replicated per point
  float wbuf[2][KS * kWidth]; // weight K-slices
  float red[8 * TM];          // head partial sums
  float sig[TM];
};

// swizzled index of element (k, row): the 8-row group index is XORed with bits of k so the
// transposing epilogue stores (16 different k per warp) spread over banks.
__device__ __forceinline__ int aidx(int k, int r) { return k * TM + (r ^ (((k >> 2) & 15) << 3)); }

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

template <int N>
__device__ __forceinline__ void load_slice(float* dst, const float* __restrict__ src, int tid) {
  // KS x N floats, contiguous in global
  constexpr int kVec = KS * N / 4;
#pragma unroll
  for (int v = tid; v < kVec; v += NTHREADS) cp_async16(dst + v * 4, src + v * 4);
}

enum { ACT_NONE = 0, ACT_RELU = 1, ACT_SOFTPLUS = 2 };

// out[c][r] = act( sum_k A[k][r] * Wt[k][c] + bias[c] ),  A = [A0 (K0 rows) | A1 (K1 rows)]
template <int N>
__device__ __forceinline__ void gemm_layer(FieldSmem& s, const float* __restrict__ Wt,
                                           const float* __restrict__ bias, const float* A0, int K0,
                                           const float* A1, int K1, int act, float* out,
                                           float* __restrict__ save = nullptr, long long p0 = 0,
                                           long long n_points = 0) {
  constexpr int NJ = N / 64;  // float4 column chunks per thread
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  float acc[8][NJ * 4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < NJ * 4; ++j) acc[i][j] = 0.f;

  const int nslices = (K0 + K1) / KS;
  load_slice<N>(s.wbuf[0], Wt, tid);
  cp_async_commit();
  for (int sl = 0; sl < nslices; ++sl) {
    if (sl + 1 < nslices) {
      load_slice<N>(s.wbuf[(sl + 1) & 1], Wt + (size_t)(sl + 1) * KS * N, tid);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* wb = s.wbuf[sl & 1];
    const int kbase = sl * KS;
    const float* A = kbase < K0 ? A0 : A1;
    const int ks = kbase < K0 ? kbase : kbase - K0;
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      const int k = ks + kk;
      const float* ap = A + k * TM + ((ty ^ ((k >> 2) & 15)) << 3);
      const float4 a0 = *reinterpret_cast<const float4*>(ap);
      const float4 a1 = *reinterpret_cast<const float4*>(ap + 4);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const float4 b = *reinterpret_cast<const float4*>(wb + kk * N + j * 64 + tx * 4);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i][j * 4 + 0] = fmaf(a[i], b.x, acc[i][j * 4 + 0]);
          acc[i][j * 4 + 1] = fmaf(a[i], b.y, acc[i][j * 4 + 1]);
          acc[i][j * 4 + 2] = fmaf(a[i], b.z, acc[i][j * 4 + 2]);
          acc[i][j * 4 + 3] = fmaf(a[i], b.w, acc[i][j * 4 + 3]);
        }
      }
    }
    __syncthreads();  // all reads of wbuf[sl&1] (and, on the last slice, of A) are done
  }
  // epilogue: bias + activation, transposed store into out[c][rows]
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int c = j * 64 + tx * 4 + jj;
      const float b = __ldg(bias + c);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float x = acc[i][j * 4 + jj] + b;
        if (act == ACT_RELU) x = fmaxf(x, 0.f);
        else if (act == ACT_SOFTPLUS) x = shifted_softplus_f(x);
        acc[i][j * 4 + jj] = x;
      }
      float* op = out + c * TM + ((ty ^ ((c >> 2) & 15)) << 3);
      *reinterpret_cast<float4*>(op) = make_float4(acc[0][j * 4 + jj], acc[1][j * 4 + jj], acc[2][j * 4 + jj], acc[3][j * 4 + jj]);
      *reinterpret_cast<float4*>(op + 4) = make_float4(acc[4][j * 4 + jj], acc[5][j * 4 + jj], acc[6][j * 4 + jj], acc[7][j * 4 + jj]);
    }
  }
  // training forward: keep the layer output, (P, N) row-major, for the backward kernels
  if (save != nullptr) {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long row = p0 + ty * 8 + i;
      if (row < n_points) {
#pragma unroll
        for (int j = 0; j < NJ; ++j)
          *reinterpret_cast<float4*>(save + row * N + j * 64 + tx * 4) =
              make_float4(acc[i][j * 4], acc[i][j * 4 + 1], acc[i][j * 4 + 2], acc[i][j * 4 + 3]);
      }
    }
  }
  __syncthreads();
}

struct FieldParams {
  const PackedHeader* hdr;  // packed image; fp32 payload follows the header
  // MODE_RAYS
  const float* rays;     // (N,8)
  const float* z;        // (N,S)
  int n_samples;
  // MODE_EMBEDDED
  const float* x;        // (P, x_stride): [xyz_enc(63) | dir_enc(27)]
  long long x_stride;
  long long n_points;
  int sigma_only;
  float* out;            // (P,4) or (P,)
  // training forward (all nullable together): activations kept for field_bwd.cu
  float* save_enc;       // (P,64)  xyz embedding, pad column zero
  float* save_dir;       // (P,32)  dir embedding, pad columns zero
  float* save_h;         // (8,P,256) h1..h8 (post-ReLU)
  float* save_g;         // (P,128) direction layer output (post-activation)
};

template <bool kEmbedded>
__global__ void __launch_bounds__(NTHREADS, 1) field_simt_kernel(FieldParams p) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FieldSmem& s = *reinterpret_cast<FieldSmem*>(smem_raw);
  constexpr Fp32Layout L = make_fp32_layout();
  const float* W = reinterpret_cast<const float*>(p.hdr + 1);
  const int new_activation = p.hdr->new_activation;
  const int tid = threadIdx.x;
  const long long ntiles = (p.n_points + TM - 1) / TM;

  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long p0 = tile * TM;
    // ---------------- prologue: fill enc / dir ----------------
    if (kEmbedded) {
      const int nin = p.sigma_only ? kXyzCh : kXyzCh + kDirCh;
      for (int e = tid; e < TM * 96; e += NTHREADS) {
        const int r = e / 96, k = e - r * 96;
        const long long pt = p0 + r;
        float v = 0.f;
        if (pt < p.n_points) {
          if (k < kXyzCh) v = p.x[pt * p.x_stride + k];
          else if (k >= kXyzPad && k - kXyzPad < kDirCh && kXyzCh + (k - kXyzPad) < nin)
            v = p.x[pt * p.x_stride + kXyzCh + (k - kXyzPad)];
        }
        if (k < kXyzPad) s.enc[aidx(k, r)] = v;
        else s.dir[aidx(k - kXyzPad, r)] = v;
      }
    } else {
      const int r = tid & (TM - 1), h = tid >> 7;
      const long long pt = p0 + r;
      float o[3] = {0.f, 0.f, 0.f}, d[3] = {0.f, 0.f, 0.f}, zz = 0.f;
      if (pt < p.n_points) {
        const long long ray = pt / p.n_samples;
        const float4 r0 = *reinterpret_cast<const float4*>(p.rays + ray * 8);
        const float4 r1 = *reinterpret_cast<const float4*>(p.rays + ray * 8 + 4);
        o[0] = r0.x; o[1] = r0.y; o[2] = r0.z;
        d[0] = r0.w; d[1] = r1.x; d[2] = r1.y;
        zz = p.z[pt];
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        // mul and add rounded separately, as torch does (no FMA contraction)
        const float x = __fadd_rn(o[c], __fmul_rn(d[c], zz));
        if (h == 0) { s.enc[aidx(c, r)] = x; s.dir[aidx(c, r)] = d[c]; }
#pragma unroll
        for (int f = 0; f < 5; ++f) {
          const int fr = h * 5 + f;
          float sn, cs;
          sincosf(x * (float)(1 << fr), &sn, &cs);
          s.enc[aidx(3 + fr * 6 + c, r)] = sn;
          s.enc[aidx(3 + fr * 6 + 3 + c, r)] = cs;
        }
#pragma unroll
        for (int f = 0; f < 2; ++f) {
          const int fr = h * 2 + f;
          float sn, cs;
          sincosf(d[c] * (float)(1 << fr), &sn, &cs);
          s.dir[aidx(3 + fr * 6 + c, r)] = sn;
          s.dir[aidx(3 + fr * 6 + 3 + c, r)] = cs;
        }
      }
      if (h == 1) {
        s.enc[aidx(kXyzCh, r)] = 0.f;
#pragma unroll
        for (int k = kDirCh; k < kDirPad; ++k) s.dir[aidx(k, r)] = 0.f;
      }
    }
    __syncthreads();
    const bool saving = p.save_h != nullptr;
    if (saving) {
      for (int e = tid; e < TM * 96; e += NTHREADS) {
        const int r = e / 96, k = e - r * 96;
        if (p0 + r < p.n_points) {
          if (k < kXyzPad) p.save_enc[(p0 + r) * kXyzPad + k] = s.enc[aidx(k, r)];
          else if (p.save_dir != nullptr) p.save_dir[(p0 + r) * kDirPad + (k - kXyzPad)] = s.dir[aidx(k - kXyzPad, r)];
        }
      }
    }
    auto save_ptr = [&](int l) { return saving ? p.save_h + (size_t)l * p.n_points * kWidth : nullptr; };

    // ---------------- trunk: 8 layers, skip at layer 5 (index 4) ----------------
    gemm_layer<256>(s, W + L.w[0], W + L.b[0], s.enc, 64, nullptr, 0, ACT_RELU, s.act, save_ptr(0), p0, p.n_points);
#pragma unroll 1
    for (int l = 1; l < 8; ++l) {
      if (l == 4)
        gemm_layer<256>(s, W + L.w[4], W + L.b[4], s.enc, 64, s.act, 256, ACT_RELU, s.act, save_ptr(4), p0, p.n_points);
      else
        gemm_layer<256>(s, W + L.w[l], W + L.b[l], s.act, 256, nullptr, 0, ACT_RELU, s.act, save_ptr(l), p0, p.n_points);
    }
    // ---------------- sigma head (no activation, nerf.py:136) ----------------
    {
      const int r = tid & (TM - 1), h = tid >> 7;
      const float* ws = W + L.sigma_w + h * 128;
      float acc = 0.f;
#pragma unroll 8
      for (int k = 0; k < 128; ++k) acc = fmaf(s.act[aidx(h * 128 + k, r)], __ldg(ws + k), acc);
      s.red[h * TM + r] = acc;
      __syncthreads();
      if (h == 0) {
        const float sg = s.red[r] + s.red[TM + r] + __ldg(W + L.sigma_b);
        s.sig[r] = sg;
        if (p.sigma_only && p0 + r < p.n_points) p.out[p0 + r] = sg;
      }
      __syncthreads();
    }
    if (p.sigma_only) continue;  // uniform across the CTA

    // ---------------- bottleneck (no activation) + direction layer ----------------
    gemm_layer<256>(s, W + L.w[8], W + L.b[8], s.act, 256, nullptr, 0, ACT_NONE, s.act, nullptr, p0, p.n_points);   // not kept: the backward folds this layer
    gemm_layer<128>(s, W + L.w[9], W + L.b[9], s.act, 256, s.dir, 32,
                    new_activation ? ACT_SOFTPLUS : ACT_RELU, s.act, saving ? p.save_g : nullptr, p0, p.n_points);
    // ---------------- rgb head ----------------
    {
      const int r = tid & (TM - 1), h = tid >> 7;
      const float* wr = W + L.rgb_w + h * 64;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll 8
      for (int k = 0; k < 64; ++k) {
        const float g = s.act[aidx(h * 64 + k, r)];
        a0 = fmaf(g, __ldg(wr + k), a0);
        a1 = fmaf(g, __ldg(wr + kHalf + k), a1);
        a2 = fmaf(g, __ldg(wr + 2 * kHalf + k), a2);
      }
      s.red[(h * 3 + 0) * TM + r] = a0;
      s.red[(h * 3 + 1) * TM + r] = a1;
      s.red[(h * 3 + 2) * TM + r] = a2;
      __syncthreads();
      if (h == 0 && p0 + r < p.n_points) {
        float c[3];
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) {
          const float x = s.red[ch * TM + r] + s.red[(3 + ch) * TM + r] + __ldg(W + L.rgb_b + ch);
          c[ch] = new_activation ? widened_sigmoid_f(x) : sigmoid_f(x);
        }
        reinterpret_cast<float4*>(p.out)[p0 + r] = make_float4(c[0], c[1], c[2], s.sig[r]);
      }
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------ host launchers
template <bool kEmbedded>
static int launch_field_simt(const FieldParams& p, cudaStream_t st) {
  static SmemOptIn optin;
  const size_t smem = sizeof(FieldSmem);
  if (int rc = ensure_smem(field_simt_kernel<kEmbedded>, optin, (int)smem, "field_simt")) return rc;
  const long long ntiles = (p.n_points + TM - 1) / TM;
  if (ntiles == 0) return SNB_OK;
  const int grid = (int)(ntiles < sm_count() ? ntiles : sm_count());
  field_simt_kernel<kEmbedded><<<grid, NTHREADS, smem, st>>>(p);
  return check_launch("field_simt_kernel");
}

// sigma_only: raw is (P,) sigma and save_dir / save_g are not written (may be NULL)
int field_forward_train_fp32(const void* packed, const float* rays, const float* z, int64_t n_rays, int n_samples,
                             int sigma_only, float* raw, float* save_enc, float* save_dir, float* save_h, float* save_g,
                             cudaStream_t st) {
  FieldParams p{};
  p.hdr = reinterpret_cast<const PackedHeader*>(packed);
  p.rays = rays;
  p.z = z;
  p.n_samples = n_samples;
  p.n_points = (long long)n_rays * n_samples;
  p.sigma_only = sigma_only;
  p.out = raw;
  p.save_enc = save_enc; p.save_dir = save_dir; p.save_h = save_h; p.save_g = save_g;
  return launch_field_simt<false>(p, st);
}

int field_forward_fp32(const void* packed, const float* rays, const float* z, int64_t n_rays,
                       int n_samples, int sigma_only, float* raw, cudaStream_t st) {
  FieldParams p{};
  p.hdr = reinterpret_cast<const PackedHeader*>(packed);
  p.rays = rays;
  p.z = z;
  p.n_samples = n_samples;
  p.n_points = (long long)n_rays * n_samples;
  p.sigma_only = sigma_only;
  p.out = raw;
  return launch_field_simt<false>(p, st);
}

int mlp_forward_fp32(const void* packed, const float* x, int64_t x_stride, int64_t n_points,
                     int sigma_only, float* out, cudaStream_t st) {
  FieldParams p{};
  p.hdr = reinterpret_cast<const PackedHeader*>(packed);
  p.x = x;
  p.x_stride = x_stride;
  p.n_points = n_points;
  p.sigma_only = sigma_only;
  p.out = out;
  return launch_field_simt<true>(p, st);
}

}  // namespace snb
