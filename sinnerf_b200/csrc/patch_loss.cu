// patch_loss.cu -- the image-space patch losses SinNeRF puts on render_rays' outputs, forward and backward:
//   kornia.losses.inverse_depth_smoothness_loss  (models/sinnerf.py:370-373, :395-398)
//   kornia.losses.ssim_loss, window 11           (losses.py:105, selected by --patch_loss l2_ssim)
// Every tensor is read and written through four element strides (N, C, H, W), so the '(b p q) c -> b c p q' views
// of the ray-major (N,3) / (N,) outputs are read where the compositing kernels wrote them, and gradients land in
// tensors of the inputs' own strides.  Loss means go through the deterministic ticket reduction of the compositing
// kernels (ray_kernels.cu) on the same SNB_LOSS_WS_FLOATS scratch; the backwards use no atomics.  Both backwards
// form the gradient for a unit upstream gradient and multiply by the device scalar g_loss last, so scaling the
// upstream gradient scales every gradient exactly and a zero upstream gradient gives exact zeros.
#include "common.cuh"

namespace snb {

namespace {

constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kThreads = 256;
// blocks whose partials fit in the loss scratch (ticket word + padding, then one float pair per block)
constexpr int kMaxLossBlocks = (SNB_LOSS_WS_FLOATS - 4) / 2;

struct Strides4 {
  long long n, c, h, w;
};
__device__ __forceinline__ long long at(const Strides4& s, long long b, long long c, long long i, long long j) {
  return b * s.n + c * s.c + i * s.h + j * s.w;
}

// Per-thread (a, b) -> block partials in loss_ws; the last block to arrive adds the block partials in index order and
// writes out[0] = sa * A + sb * B.  Same protocol and scratch layout as composite_fwd_kernel's reduction: the value is
// deterministic for a given grid, and the ticket word is reset for the next user of the scratch.
__device__ void ticket_reduce(float a, float b, float sa, float sb, float* out, float* loss_ws) {
  __shared__ float part[kThreads / 32][2];
  __shared__ bool last;
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    a += __shfl_xor_sync(kFullMask, a, off);
    b += __shfl_xor_sync(kFullMask, b, off);
  }
  if (lane == 0) { part[threadIdx.x >> 5][0] = a; part[threadIdx.x >> 5][1] = b; }
  __syncthreads();
  unsigned int* ticket = reinterpret_cast<unsigned int*>(loss_ws);
  float* partials = loss_ws + 4;
  if (threadIdx.x == 0) {
    float pa = 0.f, pb = 0.f;
    for (int i = 0; i < kThreads / 32; ++i) { pa += part[i][0]; pb += part[i][1]; }
    partials[2 * blockIdx.x] = pa; partials[2 * blockIdx.x + 1] = pb;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (last && threadIdx.x < 32) {
    __threadfence();
    float ta = 0.f, tb = 0.f;
    for (unsigned int i = lane; i < gridDim.x; i += 32) { ta += __ldcg(partials + 2 * i); tb += __ldcg(partials + 2 * i + 1); }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      ta += __shfl_xor_sync(kFullMask, ta, off);
      tb += __shfl_xor_sync(kFullMask, tb, off);
    }
    if (lane == 0) { out[0] = sa * ta + sb * tb; *ticket = 0u; }
  }
}

__device__ __forceinline__ float sgn(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }  // torch.sign

// ---------------------------------------------------------------------------------------------------------------
// inverse_depth_smoothness_loss(idepth (B,1,H,W), image (B,C,H,W)):
//   wx = exp(-mean_c |image[.., j] - image[.., j+1]|),   wy likewise along H
//   loss = mean |(d[.., j] - d[.., j+1]) wx|  +  mean |(d[i, ..] - d[i+1, ..]) wy|
// the two means over B*H*(W-1) and B*(H-1)*W edges.  One thread per pixel, owning its right and lower edge.
// ---------------------------------------------------------------------------------------------------------------
struct SmoothArgs {
  const float* d;
  const float* img;
  Strides4 sd, si;
  long long B;
  int C, H, W;
};

// 1 / C * sum_c |image(p) - image(q)|, in kornia's order (sum over channels, then the division)
__device__ __forceinline__ float channel_mean_absdiff(const SmoothArgs& a, long long b, int i, int j, int i2, int j2) {
  float m = 0.f;
  for (int c = 0; c < a.C; ++c) m += fabsf(a.img[at(a.si, b, c, i, j)] - a.img[at(a.si, b, c, i2, j2)]);
  return m / (float)a.C;
}

__global__ void __launch_bounds__(kThreads) depth_smooth_fwd_kernel(SmoothArgs a, float inv_nx, float inv_ny, float* loss,
                                                                    float* loss_ws) {
  const long long n = a.B * a.H * a.W;
  float sx = 0.f, sy = 0.f;
  for (long long p = (long long)blockIdx.x * kThreads + threadIdx.x; p < n; p += (long long)gridDim.x * kThreads) {
    const int j = (int)(p % a.W);
    const int i = (int)((p / a.W) % a.H);
    const long long b = p / ((long long)a.W * a.H);
    const float dp = a.d[at(a.sd, b, 0, i, j)];
    if (j + 1 < a.W) {
      const float w = expf(-channel_mean_absdiff(a, b, i, j, i, j + 1));
      sx += fabsf((dp - a.d[at(a.sd, b, 0, i, j + 1)]) * w);
    }
    if (i + 1 < a.H) {
      const float w = expf(-channel_mean_absdiff(a, b, i, j, i + 1, j));
      sy += fabsf((dp - a.d[at(a.sd, b, 0, i + 1, j)]) * w);
    }
  }
  ticket_reduce(sx, sy, inv_nx, inv_ny, loss, loss_ws);
}

// The edge p -> q (q = p + one pixel) for a unit upstream gradient: t = (d(p) - d(q)) w, w = exp(-m).
//   dL/dd(p) = -dL/dd(q) = sign(t) inv_n w =: gd
//   dL/dm = -sign(t) inv_n (d(p) - d(q)) w =: gm,   dL/dimage_c(p) = -dL/dimage_c(q) = gm sign(image_c(p) - image_c(q)) / C
__device__ __forceinline__ void smooth_edge(const SmoothArgs& a, long long b, int i, int j, int i2, int j2, float inv_n,
                                            float& gd, float& gm) {
  const float w = expf(-channel_mean_absdiff(a, b, i, j, i2, j2));
  const float dd = a.d[at(a.sd, b, 0, i, j)] - a.d[at(a.sd, b, 0, i2, j2)];
  const float gt = sgn(dd * w) * inv_n;
  gd = gt * w;
  gm = -(gt * dd) * w;
}

__global__ void __launch_bounds__(kThreads) depth_smooth_bwd_kernel(SmoothArgs a, float inv_nx, float inv_ny,
                                                                    const float* __restrict__ g_loss, float* g_d,
                                                                    Strides4 sgd, float* g_img, Strides4 sgi) {
  const long long n = a.B * a.H * a.W;
  const float g = *g_loss;
  const float inv_c = 1.0f / (float)a.C;
  for (long long p = (long long)blockIdx.x * kThreads + threadIdx.x; p < n; p += (long long)gridDim.x * kThreads) {
    const int j = (int)(p % a.W);
    const int i = (int)((p / a.W) % a.H);
    const long long b = p / ((long long)a.W * a.H);
    // the up to four incident edges, this pixel as the edge's first (right, down) or second (left, up) end
    float gd[4] = {0.f, 0.f, 0.f, 0.f}, gm[4] = {0.f, 0.f, 0.f, 0.f};
    if (j + 1 < a.W) smooth_edge(a, b, i, j, i, j + 1, inv_nx, gd[0], gm[0]);
    if (i + 1 < a.H) smooth_edge(a, b, i, j, i + 1, j, inv_ny, gd[1], gm[1]);
    if (j > 0) smooth_edge(a, b, i, j - 1, i, j, inv_nx, gd[2], gm[2]);
    if (i > 0) smooth_edge(a, b, i - 1, j, i, j, inv_ny, gd[3], gm[3]);
    if (g_d != nullptr) g_d[at(sgd, b, 0, i, j)] = ((gd[0] + gd[1]) - (gd[2] + gd[3])) * g;
    if (g_img != nullptr) {
      for (int c = 0; c < a.C; ++c) {
        const float v = a.img[at(a.si, b, c, i, j)];
        float acc = 0.f;
        if (j + 1 < a.W) acc += gm[0] * sgn(v - a.img[at(a.si, b, c, i, j + 1)]);
        if (i + 1 < a.H) acc += gm[1] * sgn(v - a.img[at(a.si, b, c, i + 1, j)]);
        if (j > 0) acc -= gm[2] * sgn(a.img[at(a.si, b, c, i, j - 1)] - v);
        if (i > 0) acc -= gm[3] * sgn(a.img[at(a.si, b, c, i - 1, j)] - v);
        g_img[at(sgi, b, c, i, j)] = acc * inv_c * g;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// ssim_loss(x, y, 11): kornia's filter2d (reflect padding of 5, depthwise correlation with the 11x11 Gaussian,
// sigma 1.5) of x, y, x^2, y^2, xy; ssim = (2 mu1 mu2 + C1)(2 s12 + C2) / ((mu1^2 + mu2^2 + C1)(s1 + s2 + C2) + eps)
// with s1 = f(x^2) - mu1^2, ...; loss = mean clamp((1 - ssim) / 2, 0, 1).
// The window sums and the SSIM expression are evaluated in fp64.  For depth-valued inputs (the depth patch loss, values
// 2..6 against max_val = 1) s1 = f(x^2) - mu1^2 cancels most of its digits: in fp32 the variance of a smooth depth
// patch is mostly rounding noise of f(x^2) and mu1^2, so the loss and its gradient would be only as good as that.  The
// problem is small (a patch of 64x64 pixels) and fp64 costs nothing measurable here.
// CTAs walk (plane, 16x32 output tile); the tile plus a 5-pixel halo is staged in shared memory with the reflection
// applied at load time, then two separable 11-tap passes.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kWin = 11, kPad = kWin / 2;
constexpr int kTH = 16, kTW = 32;                      // output tile
constexpr int kHH = kTH + 2 * kPad, kHW = kTW + 2 * kPad;   // tile + halo: 26 x 42
struct Taps {
  double g[kWin];
};

struct SsimArgs {
  const float* x;
  const float* y;
  Strides4 sx, sy;
  long long B;
  int C, H, W;
  double c1, c2, eps, inv_n;
};

__device__ __forceinline__ int reflect(int k, int n) {   // F.pad(mode='reflect') index for -kPad <= k < n + kPad
  k = k < 0 ? -k : (k >= n ? 2 * (n - 1) - k : k);
  return min(max(k, 0), n - 1);    // rows / columns past a ragged tile's edge: any valid index (results unused)
}

__device__ __forceinline__ void tile_coords(const SsimArgs& a, long long t, long long& plane, int& r0, int& c0) {
  const int tw = (a.W + kTW - 1) / kTW, th = (a.H + kTH - 1) / kTH;
  c0 = (int)(t % tw) * kTW;
  r0 = (int)((t / tw) % th) * kTH;
  plane = t / ((long long)tw * th);
}

// forward: loss mean (ticket reduction) and, when coef != nullptr, the per-pixel coefficient maps of the backward for a
// unit upstream gradient: coef[0] = dL/dmu1, coef[1] = dL/df(x^2), coef[2] = dL/df(xy), each (B,C,H,W) contiguous fp64.
__global__ void __launch_bounds__(kThreads) ssim_fwd_kernel(SsimArgs a, Taps taps, long long n_tiles, float* loss,
                                                            double* coef, float* loss_ws) {
  __shared__ float sxv[kHH][kHW], syv[kHH][kHW];
  __shared__ double hs[5][kHH][kTW];
  const long long plane_elems = (long long)a.H * a.W;
  const long long total = a.B * a.C * plane_elems;
  float lsum = 0.f;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    long long plane;
    int r0, c0;
    tile_coords(a, t, plane, r0, c0);
    const long long b = plane / a.C;
    const int ch = (int)(plane % a.C);
    for (int e = threadIdx.x; e < kHH * kHW; e += kThreads) {
      const int r = e / kHW, c = e % kHW;
      const int gi = reflect(r0 + r - kPad, a.H), gj = reflect(c0 + c - kPad, a.W);
      sxv[r][c] = a.x[at(a.sx, b, ch, gi, gj)];
      syv[r][c] = a.y[at(a.sy, b, ch, gi, gj)];
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kHH * kTW; e += kThreads) {   // along W
      const int r = e / kTW, c = e % kTW;
      double m0 = 0.0, m1 = 0.0, m2 = 0.0, m3 = 0.0, m4 = 0.0;
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const double xv = sxv[r][c + k], yv = syv[r][c + k], g = taps.g[k];
        m0 = fma(g, xv, m0);
        m1 = fma(g, yv, m1);
        m2 = fma(g, xv * xv, m2);   // products of two fp32 values are exact in fp64
        m3 = fma(g, yv * yv, m3);
        m4 = fma(g, xv * yv, m4);
      }
      hs[0][r][c] = m0; hs[1][r][c] = m1; hs[2][r][c] = m2; hs[3][r][c] = m3; hs[4][r][c] = m4;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kTH * kTW; e += kThreads) {   // along H, then the SSIM expression per pixel
      const int r = e / kTW, c = e % kTW;
      const int i = r0 + r, j = c0 + c;
      if (i >= a.H || j >= a.W) continue;
      double mu1 = 0.0, mu2 = 0.0, fxx = 0.0, fyy = 0.0, fxy = 0.0;
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const double g = taps.g[k];
        mu1 = fma(g, hs[0][r + k][c], mu1);
        mu2 = fma(g, hs[1][r + k][c], mu2);
        fxx = fma(g, hs[2][r + k][c], fxx);
        fyy = fma(g, hs[3][r + k][c], fyy);
        fxy = fma(g, hs[4][r + k][c], fxy);
      }
      const double s1 = fxx - mu1 * mu1, s2 = fyy - mu2 * mu2, s12 = fxy - mu1 * mu2;
      const double A1 = 2.0 * mu1 * mu2 + a.c1, A2 = 2.0 * s12 + a.c2;
      const double B1 = mu1 * mu1 + mu2 * mu2 + a.c1, B2 = s1 + s2 + a.c2;
      const double den = B1 * B2 + a.eps;
      const double ssim = A1 * A2 / den;
      const double u = (1.0 - ssim) * 0.5;
      // torch.clamp keeps a NaN, where fmax(NaN, 0) would return 0: a NaN in either image makes the loss NaN
      lsum += (float)(isnan(u) ? u : fmin(fmax(u, 0.0), 1.0));
      if (coef != nullptr) {
        // dL/dssim for the mean of clamp(u, 0, 1); torch.clamp passes the gradient for min <= u <= max
        const double gs = (u >= 0.0 && u <= 1.0) ? -0.5 * a.inv_n : 0.0;
        const double dA1 = gs * A2 / den, dA2 = gs * A1 / den;
        const double dB1 = -gs * ssim * B2 / den, dB2 = -gs * ssim * B1 / den;
        // d/dmu1 with f(x^2), f(xy) held: A1 -> 2 mu2, A2 -> -2 mu2, B1 -> 2 mu1, B2 -> -2 mu1
        const long long o = plane * plane_elems + (long long)i * a.W + j;
        coef[o] = 2.0 * mu2 * (dA1 - dA2) + 2.0 * mu1 * (dB1 - dB2);
        coef[total + o] = dB2;           // d/df(x^2): B2 -> 1
        coef[2 * total + o] = 2.0 * dA2; // d/df(xy):  A2 -> 2
      }
    }
    __syncthreads();
  }
  ticket_reduce(lsum, 0.f, (float)a.inv_n, 0.f, loss, loss_ws);
}

// The 1-D adjoint of "reflect-pad by 5, then correlate with g": the weight with which output position p reads input
// position q is  g(q - p)  plus, for q in [1, 5], the mirror image -q of q in the top / left pad, g(-q - p),  plus, for
// q in [n-6, n-2], the mirror image 2(n-1) - q in the bottom / right pad, g(2(n-1) - q - p).  Every p it is non-zero
// for lies in [q - 5, q + 5].  (n >= 6, so each padded position has exactly one source pixel.)
__device__ __forceinline__ double adj_weight(const double* g, int p, int q, int n) {   // g: the taps in shared memory
  auto tap = [&](int k) { return (k >= -kPad && k <= kPad) ? g[k + kPad] : 0.0; };
  double w = tap(q - p);
  if (q >= 1 && q <= kPad) w += tap(-q - p);
  if (q >= n - 1 - kPad && q <= n - 2) w += tap(2 * (n - 1) - q - p);
  return w;
}

// backward: g_x(q) = g_loss * sum_p W(p, q) [coef0(p) + 2 x(q) coef1(p) + y(q) coef2(p)], W the 2-D adjoint weight
// (separable: adj_weight along W, then along H).  The coefficient maps of the tile plus a 5-pixel halo (zero outside the
// image) are staged in shared memory.
__global__ void __launch_bounds__(kThreads) ssim_bwd_kernel(SsimArgs a, Taps taps, long long n_tiles,
                                                            const double* __restrict__ coef,
                                                            const float* __restrict__ g_loss, float* g_x, Strides4 sgx) {
  __shared__ double sv[3][kHH][kHW];
  __shared__ double su[3][kHH][kTW];
  __shared__ double sg[kWin];
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 0; k < kWin; ++k) sg[k] = taps.g[k];   // constant indices: the parameter is not copied to local memory
  }
  const long long plane_elems = (long long)a.H * a.W;
  const long long total = a.B * a.C * plane_elems;
  const float g = *g_loss;
  for (long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    long long plane;
    int r0, c0;
    tile_coords(a, t, plane, r0, c0);
    const long long b = plane / a.C;
    const int ch = (int)(plane % a.C);
    for (int e = threadIdx.x; e < kHH * kHW; e += kThreads) {
      const int r = e / kHW, c = e % kHW;
      const int pi = r0 + r - kPad, pj = c0 + c - kPad;
      const bool in = pi >= 0 && pi < a.H && pj >= 0 && pj < a.W;
      const long long o = plane * plane_elems + (long long)pi * a.W + pj;
#pragma unroll
      for (int m = 0; m < 3; ++m) sv[m][r][c] = in ? coef[m * total + o] : 0.0;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kHH * kTW; e += kThreads) {   // adjoint along W
      const int r = e / kTW, c = e % kTW;
      const int q = c0 + c;
      double u0 = 0.0, u1 = 0.0, u2 = 0.0;
      if (q < a.W) {
#pragma unroll
        for (int k = 0; k < kWin; ++k) {
          const double w = adj_weight(sg, q + k - kPad, q, a.W);
          u0 = fma(w, sv[0][r][c + k], u0);
          u1 = fma(w, sv[1][r][c + k], u1);
          u2 = fma(w, sv[2][r][c + k], u2);
        }
      }
      su[0][r][c] = u0; su[1][r][c] = u1; su[2][r][c] = u2;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < kTH * kTW; e += kThreads) {   // adjoint along H, then the chain through x^2 and xy
      const int r = e / kTW, c = e % kTW;
      const int q = r0 + r, j = c0 + c;
      if (q >= a.H || j >= a.W) continue;
      double s0 = 0.0, s1 = 0.0, s2 = 0.0;
#pragma unroll
      for (int k = 0; k < kWin; ++k) {
        const double w = adj_weight(sg, q + k - kPad, q, a.H);
        s0 = fma(w, su[0][r + k][c], s0);
        s1 = fma(w, su[1][r + k][c], s1);
        s2 = fma(w, su[2][r + k][c], s2);
      }
      const double xv = a.x[at(a.sx, b, ch, q, j)], yv = a.y[at(a.sy, b, ch, q, j)];
      g_x[at(sgx, b, ch, q, j)] = (float)(s0 + 2.0 * xv * s1 + yv * s2) * g;
    }
    __syncthreads();
  }
}

Strides4 to_strides(const int64_t* s) { return Strides4{s[0], s[1], s[2], s[3]}; }

int grid_for_elems(long long n, int cap) {
  const long long blocks = (n + kThreads - 1) / kThreads;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

Taps gaussian_taps() {   // kornia get_gaussian_kernel1d(11, 1.5): exp(-x^2 / (2 sigma^2)), x = -5..5, normalised to sum 1
  Taps t;
  double s = 0.0;
  for (int k = 0; k < kWin; ++k) {
    const double x = k - kPad;
    t.g[k] = exp(-x * x / (2.0 * 1.5 * 1.5));
    s += t.g[k];
  }
  for (int k = 0; k < kWin; ++k) t.g[k] /= s;
  return t;
}

SsimArgs ssim_args(const float* x, const int64_t* sx, const float* y, const int64_t* sy, long long B, int C, int H, int W,
                   float max_val, float eps) {
  SsimArgs a;
  a.x = x; a.y = y; a.sx = to_strides(sx); a.sy = to_strides(sy);
  a.B = B; a.C = C; a.H = H; a.W = W;
  // kornia forms C1 = (0.01 * max_val) ** 2 from the Python float max_val
  a.c1 = (0.01 * (double)max_val) * (0.01 * (double)max_val);
  a.c2 = (0.03 * (double)max_val) * (0.03 * (double)max_val);
  a.eps = eps;
  a.inv_n = 1.0 / (double)(B * C * (long long)H * W);
  return a;
}

long long ssim_tiles(long long B, int C, int H, int W) {
  return B * C * (long long)((H + kTH - 1) / kTH) * ((W + kTW - 1) / kTW);
}

}  // namespace

int launch_depth_smooth_fwd(const float* d, const int64_t* sd, const float* img, const int64_t* si, long long B, int C,
                            int H, int W, float* loss, float* loss_ws, cudaStream_t st) {
  const SmoothArgs a{d, img, to_strides(sd), to_strides(si), B, C, H, W};
  const float inv_nx = (float)(1.0 / (double)(B * H * (long long)(W - 1)));
  const float inv_ny = (float)(1.0 / (double)(B * (long long)(H - 1) * W));
  depth_smooth_fwd_kernel<<<grid_for_elems(B * H * (long long)W, kMaxLossBlocks), kThreads, 0, st>>>(a, inv_nx, inv_ny,
                                                                                                     loss, loss_ws);
  return check_launch("depth_smooth_fwd_kernel");
}

int launch_depth_smooth_bwd(const float* d, const int64_t* sd, const float* img, const int64_t* si, long long B, int C,
                            int H, int W, const float* g_loss, float* g_d, const int64_t* sgd, float* g_img,
                            const int64_t* sgi, cudaStream_t st) {
  if (g_d == nullptr && g_img == nullptr) return SNB_OK;
  const SmoothArgs a{d, img, to_strides(sd), to_strides(si), B, C, H, W};
  const float inv_nx = (float)(1.0 / (double)(B * H * (long long)(W - 1)));
  const float inv_ny = (float)(1.0 / (double)(B * (long long)(H - 1) * W));
  const Strides4 zero{0, 0, 0, 0};
  depth_smooth_bwd_kernel<<<grid_for_elems(B * H * (long long)W, sm_count() * 16), kThreads, 0, st>>>(
      a, inv_nx, inv_ny, g_loss, g_d, g_d ? to_strides(sgd) : zero, g_img, g_img ? to_strides(sgi) : zero);
  return check_launch("depth_smooth_bwd_kernel");
}

int launch_ssim_fwd(const float* x, const int64_t* sx, const float* y, const int64_t* sy, long long B, int C, int H,
                    int W, float max_val, float eps, float* loss, double* coef, float* loss_ws, cudaStream_t st) {
  const SsimArgs a = ssim_args(x, sx, y, sy, B, C, H, W, max_val, eps);
  const long long n_tiles = ssim_tiles(B, C, H, W);
  const int grid = (int)(n_tiles < kMaxLossBlocks ? n_tiles : kMaxLossBlocks);
  ssim_fwd_kernel<<<grid, kThreads, 0, st>>>(a, gaussian_taps(), n_tiles, loss, coef, loss_ws);
  return check_launch("ssim_fwd_kernel");
}

int launch_ssim_bwd(const float* x, const int64_t* sx, const float* y, const int64_t* sy, long long B, int C, int H,
                    int W, const double* coef, const float* g_loss, float* g_x, const int64_t* sgx, cudaStream_t st) {
  const SsimArgs a = ssim_args(x, sx, y, sy, B, C, H, W, 1.0f, 0.0f);   // constants unused: coef holds them
  const long long n_tiles = ssim_tiles(B, C, H, W);
  const long long cap = (long long)sm_count() * 8;
  const int grid = (int)(n_tiles < cap ? n_tiles : cap);
  ssim_bwd_kernel<<<grid, kThreads, 0, st>>>(a, gaussian_taps(), n_tiles, coef, g_loss, g_x, to_strides(sgx));
  return check_launch("ssim_bwd_kernel");
}

}  // namespace snb
