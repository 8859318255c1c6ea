// disc.cu -- SinNeRF's adversarial-loss discriminator (models/discriminator.py Discriminator(conditional=False,
// policy='color,cutout', ndf=64, imsize)) with DiffAugment (models/diff_aug.py) applied to its input: forward, the
// gradient with respect to the input and the gradients with respect to every spectral-norm weight_orig.
//
// Every convolution (4 x 4, no bias) is a GEMM on the wgmma kernel of tc_gemm.cuh over an im2col matrix:
//   forward  y[co][j]   = (1 / sigma) sum_k W[co][k] col[j][k]      j = (image, output pixel), k = (ci, ky, kx)
//   wgrad    dW[co][k]  = sum_j dy[co][j] col[j][k]
//   dgrad    dcol[j][k] = (1 / sigma) sum_co dy[co][j] W[co][k]
// Activations are kept channel-major, (C, n, P), so a layer's rows are one contiguous run per (channel, image) and
// the last layer's (1, n, P) output is the (n, 1, oh, ow) result.  Around the GEMMs:
//   - the gather that builds col applies the previous layer's InstanceNorm and LeakyReLU on load (layer 1: the
//     DiffAugment colour maps and the cutout mask);
//   - per-(channel, image) InstanceNorm statistics;
//   - the col2im fold of dcol, written as a gather (no atomics), fused with the LeakyReLU and InstanceNorm backward;
//   - the DiffAugment backward to the input, written through the input's strides;
//   - the spectral-norm power iteration (one step, in place on weight_u / weight_v in training mode) and the
//     weight-gradient correction dW_orig = dW / sigma - (<dW, W_orig> / sigma^2) u v^T.
// sigma, u and v never leave the device.  The upstream gradient is scaled by a power of two (its largest element to
// [2^14, 2^15)) before the chain, each layer's output gradient is rescaled the same way after its fold, the GEMMs
// read a copy of each weight scaled likewise, and normalised activations are scaled on their way into im2col; the
// exponents are undone in the GEMMs' alpha and in the final gradients.
// Every factor is a power of two, and it keeps the fp16 hi / lo operand words out of their subnormal range whatever
// the loss weight.  The gradient exponents are carried as integers and applied once, with ldexpf, as each final
// gradient is written: the scaling is exact wherever that gradient is a normal float, and below that it is rounded
// once (never flushed to zero by an intermediate factor).  Every reduction runs in a fixed order: two identical calls
// give the same bits.
// The gradient penalty of dloss='wgan_gp' (snb_disc_penalty_*, DESIGN §4.6) reuses this chain: g = grad_x sum(out)
// is the backward from an all-ones upstream, and the penalty's second-order gradients are a tangent forward along
// v = 2 d_reg g followed by a reverse pass over two adjoint streams, on the same GEMM and the same scaling rules.
#include "common.cuh"
#include "tc_gemm.cuh"

namespace snb {
namespace {

constexpr int kMaxLayers = SNB_DISC_MAX_LAYERS;
constexpr float kSnEps = 1e-12f, kInEps = 1e-5f, kSlope = 0.2f;
constexpr int kAugFloats = 16;   // per image: enabled, brightness shift, saturation, contrast, mean, cutout box

// ------------------------------------------------------------------ layer schedule
struct Layer {
  int cin, cout, stride, pad;
  int in_norm;   // InstanceNorm2d after this convolution
  int act;       // LeakyReLU(0.2) after it (every layer but the last)
  int hin, win, hout, wout;
  long long P() const { return (long long)hout * wout; }
  long long K() const { return 16ll * cin; }
};
struct Net {
  int n_layers, n, h, w;
  Layer l[kMaxLayers];
};

// the branches of Discriminator.__init__ (ndf = 64): imsize 128, 64, 32, anything else
int net_of(const char* who, int imsize, int n, int h, int w, Net& net) {
  static const int k128[][3] = {{3, 32, 0}, {32, 64, 1}, {64, 128, 1}, {128, 256, 1}, {256, 512, 1}, {512, 1, 0}};
  static const int k64[][3] = {{3, 64, 0}, {64, 128, 1}, {128, 256, 1}, {256, 512, 1}, {512, 1, 0}};
  static const int k32[][3] = {{3, 128, 1}, {128, 256, 1}, {256, 512, 1}, {512, 1, 0}};
  static const int kElse[][3] = {{3, 256, 1}, {256, 512, 1}, {512, 1, 0}};
  const int(*spec)[3] = imsize == 128 ? k128 : imsize == 64 ? k64 : imsize == 32 ? k32 : kElse;
  const int L = imsize == 128 ? 6 : imsize == 64 ? 5 : imsize == 32 ? 4 : 3;
  SNB_REQUIRE(n >= 1, "%s: batch size must be >= 1 (got %d)", who, n);
  SNB_REQUIRE(h >= 1 && w >= 1, "%s: image size %d x %d", who, h, w);
  net.n_layers = L; net.n = n; net.h = h; net.w = w;
  int H = h, W = w;
  for (int i = 0; i < L; ++i) {
    Layer& y = net.l[i];
    y.cin = spec[i][0]; y.cout = spec[i][1]; y.in_norm = spec[i][2];
    y.act = i + 1 < L;
    y.stride = i + 1 < L ? 2 : 1;
    y.pad = i + 1 < L ? 1 : 0;
    y.hin = H; y.win = W;
    y.hout = (H + 2 * y.pad - 4) / y.stride + 1;
    y.wout = (W + 2 * y.pad - 4) / y.stride + 1;
    SNB_REQUIRE(H + 2 * y.pad >= 4 && W + 2 * y.pad >= 4,
                "%s: a %d x %d image leaves layer %d's input %d x %d smaller than its 4 x 4 kernel", who, h, w, i, H, W);
    SNB_REQUIRE(!y.in_norm || y.P() > 1,
                "%s: a %d x %d image leaves one spatial element for layer %d's InstanceNorm", who, h, w, i);
    SNB_REQUIRE((long long)n * y.P() * y.K() < (1ll << 31), "%s: batch %d of %d x %d images is too large", who, n, h, w);
    // the dgrad GEMM tiles layer i's n P rows 64 to a block along grid.y
    SNB_REQUIRE((long long)n * y.P() <= kMaxGemmRows,
                "%s: batch %d of %d x %d images gives layer %d %lld rows (n x %d x %d output pixels), more than its input "
                "gradient GEMM's %lld", who, n, h, w, i, (long long)n * y.P(), y.hout, y.wout, kMaxGemmRows);
    H = y.hout; W = y.wout;
  }
  return SNB_OK;
}

// ------------------------------------------------------------------ workspace
long long al64(long long x) { return (x + 63) & ~63ll; }
struct DiscWs {
  float *sigma, *inv_sigma, *alpha, *wscale, *aug, *dot;
  int* gexp;                      // per layer: the exponent that undoes the scaling of its output gradient
  float *u[kMaxLayers], *v[kMaxLayers], *t[kMaxLayers], *s[kMaxLayers], *rmax[kMaxLayers], *part[kMaxLayers];
  float* ws[kMaxLayers];          // 2^e W_orig, its largest element in [2^14, 2^15)
  float *col[kMaxLayers], *y[kMaxLayers], *mean[kMaxLayers], *rstd[kMaxLayers];
  float *dy0, *dy1, *dcol, *dx;   // backward scratch
  // gradient penalty (pen = 1): g = grad_x sum(out) (n, 3, h, w), the tangent direction v, its DiffAugment
  // parameters, each layer's tangent im2col and pre-norm tangent output with its InstanceNorm statistics, the
  // primal-adjoint stream's scratch and both streams' raw weight gradients
  float *g, *ones, *vt, *taug, *dreg, *dp0, *dp1, *dcolp;   // dreg: d_reg 2^-ev[0] (see disc_pen_dir_kernel)
  float *tcol[kMaxLayers], *ty[kMaxLayers], *tmean[kMaxLayers], *tq[kMaxLayers], *dwt[kMaxLayers], *dwp[kMaxLayers];
  int *ev, *gt, *gp, *gu, *gw;    // per layer: exponents of the tangent col, of both adjoint streams, of a fold's
                                  // primal output and of the combined weight gradient
  size_t bytes;
};
DiscWs disc_ws(void* base, const Net& N, int save, int pen = 0) {
  DiscWs W{};
  float* b = static_cast<float*>(base);
  long long off = 0;
  auto take = [&](long long floats) { float* p = b == nullptr ? nullptr : b + off; off = al64(off + floats); return p; };
  W.sigma = take(kMaxLayers); W.inv_sigma = take(kMaxLayers); W.alpha = take(kMaxLayers); W.wscale = take(kMaxLayers);
  W.dot = take(kMaxLayers); W.gexp = reinterpret_cast<int*>(take(kMaxLayers));
  W.aug = take((long long)kAugFloats * N.n);
  long long dy_max = 0, dcol_max = 0;
  for (int i = 0; i < N.n_layers; ++i) {
    const Layer& y = N.l[i];
    const long long rows = (long long)N.n * y.P();
    W.u[i] = take(y.cout); W.v[i] = take(y.K()); W.t[i] = take(y.K()); W.s[i] = take(y.cout); W.part[i] = take(y.cout);
    W.rmax[i] = take(y.cout); W.ws[i] = take(y.cout * y.K());
    W.col[i] = take(rows * y.K());
    if (y.act) W.y[i] = take(rows * y.cout);
    if (y.in_norm) { W.mean[i] = take((long long)y.cout * N.n); W.rstd[i] = take((long long)y.cout * N.n); }
    dy_max = dy_max > rows * y.cout ? dy_max : rows * y.cout;
    dcol_max = dcol_max > rows * y.K() ? dcol_max : rows * y.K();
  }
  if (save) {
    W.dy0 = take(dy_max); W.dy1 = take(dy_max); W.dcol = take(dcol_max);
    W.dx = take(3ll * N.n * N.h * N.w);
  }
  if (pen) {
    const long long img = 3ll * N.n * N.h * N.w;
    W.g = take(img); W.vt = take(img); W.ones = take((long long)N.n * N.l[N.n_layers - 1].P());
    W.taug = take((long long)kAugFloats * N.n);
    W.dreg = take(N.n);
    W.dp0 = take(dy_max); W.dp1 = take(dy_max); W.dcolp = take(dcol_max);
    int* e = reinterpret_cast<int*>(take(5 * kMaxLayers));
    W.ev = e; W.gt = e + kMaxLayers; W.gp = e + 2 * kMaxLayers; W.gu = e + 3 * kMaxLayers; W.gw = e + 4 * kMaxLayers;
    for (int i = 0; i < N.n_layers; ++i) {
      const Layer& y = N.l[i];
      const long long rows = (long long)N.n * y.P();
      W.tcol[i] = take(rows * y.K());
      if (y.act) W.ty[i] = take(rows * y.cout);
      if (y.in_norm) { W.tmean[i] = take((long long)y.cout * N.n); W.tq[i] = take((long long)y.cout * N.n); }
      W.dwt[i] = take(y.cout * y.K()); W.dwp[i] = take(y.cout * y.K());
    }
  }
  W.bytes = (size_t)off * 4;
  return W;
}

// ------------------------------------------------------------------ reductions (fixed order)
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
// the block's sum, the same bits in every thread; red: blockDim.x / 32 floats of shared memory
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) r += red[i];
  __syncthreads();
  return r;
}

__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) r = fmaxf(r, red[i]);
  __syncthreads();
  return r;
}
// k with m 2^k in [2^14, 2^15); 0 for m = 0 or non-finite.  Operands scaled so sit high in fp16's range: an element
// down to 2^-11 of the largest still has a normal lo word (below 2^15 nothing reaches the +-65504 clamp)
__device__ __forceinline__ int pow2_exponent(float m) {
  if (!(m > 0.f) || !isfinite(m)) return 0;
  int e;
  frexpf(m, &e);   // m = f 2^e, f in [0.5, 1)
  return 15 - e;
}

__device__ __forceinline__ float lrelu(float x) { return x > 0.f ? x : x * kSlope; }

// ------------------------------------------------------------------ spectral norm
struct SnArgs {
  const float* W[kMaxLayers];
  float* u_mod[kMaxLayers];   // the module's weight_u / weight_v buffers
  float* v_mod[kMaxLayers];
  float *u[kMaxLayers], *v[kMaxLayers], *t[kMaxLayers], *s[kMaxLayers];   // this call's copies and scratch
  float *rmax[kMaxLayers], *ws[kMaxLayers];
  int rows[kMaxLayers], cols[kMaxLayers];
  float *sigma, *inv_sigma, *alpha, *wscale;
};

// t = W^T u_mod (one thread per column, rows in order)
__global__ void disc_sn_wtu_kernel(const SnArgs a) {
  const int l = blockIdx.y, k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.cols[l]) return;
  const float* W = a.W[l] + k;
  const float* u = a.u_mod[l];
  float acc = 0.f;
  for (int r = 0; r < a.rows[l]; ++r) acc += W[(long long)r * a.cols[l]] * u[r];
  a.t[l][k] = acc;
}

// training: v = t / max(|t|, eps), written to the call's copy and to weight_v; eval: v = weight_v
__global__ void disc_sn_v_kernel(const SnArgs a, int training) {
  __shared__ float red[32];
  const int l = blockIdx.x, K = a.cols[l];
  if (!training) {
    for (int k = threadIdx.x; k < K; k += blockDim.x) a.v[l][k] = a.v_mod[l][k];
    return;
  }
  float q = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) q += a.t[l][k] * a.t[l][k];
  const float nrm = fmaxf(sqrtf(block_sum(q, red)), kSnEps);
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float v = a.t[l][k] / nrm;
    a.v[l][k] = v;
    a.v_mod[l][k] = v;
  }
}

// s = W v and the row's largest |W| (one block per row)
__global__ void disc_sn_wv_kernel(const SnArgs a) {
  __shared__ float red[32];
  const int l = blockIdx.y, r = blockIdx.x;
  if (r >= a.rows[l]) return;
  const float* W = a.W[l] + (long long)r * a.cols[l];
  float acc = 0.f, mx = 0.f;
  for (int k = threadIdx.x; k < a.cols[l]; k += blockDim.x) {
    acc += W[k] * a.v[l][k];
    mx = fmaxf(mx, fabsf(W[k]));
  }
  acc = block_sum(acc, red);
  mx = block_max(mx, red);
  if (threadIdx.x == 0) {
    a.s[l][r] = acc;
    a.rmax[l][r] = mx;
  }
}

// training: u = s / max(|s|, eps) (call's copy and weight_u); eval: u = weight_u.  sigma = u . s
__global__ void disc_sn_u_kernel(const SnArgs a, int training) {
  __shared__ float red[32];
  const int l = blockIdx.x, R = a.rows[l];
  float nrm = 1.f;
  if (training) {
    float q = 0.f;
    for (int r = threadIdx.x; r < R; r += blockDim.x) q += a.s[l][r] * a.s[l][r];
    nrm = fmaxf(sqrtf(block_sum(q, red)), kSnEps);
  }
  float d = 0.f;
  for (int r = threadIdx.x; r < R; r += blockDim.x) {
    const float u = training ? a.s[l][r] / nrm : a.u_mod[l][r];
    a.u[l][r] = u;
    if (training) a.u_mod[l][r] = u;
    d += u * a.s[l][r];
  }
  d = block_sum(d, red);
  float mx = 0.f;
  for (int r = threadIdx.x; r < R; r += blockDim.x) mx = fmaxf(mx, a.rmax[l][r]);
  const int e = pow2_exponent(block_max(mx, red));
  if (threadIdx.x == 0) {
    a.sigma[l] = d;
    a.inv_sigma[l] = 1.f / d;
    a.alpha[l] = ldexpf(1.f / d, -e);
    a.wscale[l] = ldexpf(1.f, e);
  }
}

// the GEMMs' copy of W_orig, scaled by the power of two that puts its largest element in [2^14, 2^15) (exact): the
// fp16 lo words of weights of ~1e-2 would otherwise be subnormal; the GEMMs undo it in alpha = 2^-e / sigma
__global__ void disc_w_scale_kernel(const SnArgs a) {
  const int l = blockIdx.y;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)a.rows[l] * a.cols[l]) return;
  a.ws[l][i] = a.W[l][i] * a.wscale[l];
}

// ------------------------------------------------------------------ DiffAugment
// per image: [0] enabled, [1] brightness shift rand - 0.5, [2] saturation factor 2 rand, [3] contrast factor
// rand + 0.5, [4] the mean of the saturated image (rand_contrast's x_mean), [5..8] the zeroed rows y0..y1 and
// columns x0..x1 (inclusive; rand_cutout's clamped index range)
struct AugIn {
  const float *bright, *sat, *con;
  const int64_t *cut_y, *cut_x;
  int cut_h, cut_w;
};

__device__ __forceinline__ float aug_saturated(const float* x, long long s_c, int c, float shift, float sat) {
  const float x0 = x[0] + shift, x1 = x[s_c] + shift, x2 = x[2 * s_c] + shift;
  const float m = (x0 + x1 + x2) / 3.f;
  const float v = c == 0 ? x0 : c == 1 ? x1 : x2;
  return (v - m) * sat + m;
}

__global__ void disc_aug_params_kernel(const float* __restrict__ x, long long s_b, long long s_c, long long s_y,
                                       long long s_x, int h, int w, AugIn in, float* __restrict__ aug) {
  __shared__ float red[32];
  const int b = blockIdx.x;
  float* p = aug + (long long)kAugFloats * b;
  if (in.bright == nullptr) {
    if (threadIdx.x == 0) p[0] = 0.f;
    return;
  }
  const float shift = in.bright[b] - 0.5f, sat = in.sat[b] * 2.f;
  float acc = 0.f;
  for (int t = threadIdx.x; t < h * w; t += blockDim.x) {
    const float* px = x + b * s_b + (t / w) * s_y + (t % w) * s_x;
    for (int c = 0; c < 3; ++c) acc += aug_saturated(px, s_c, c, shift, sat);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) {
    const long long oy = in.cut_y[b] - in.cut_h / 2, ox = in.cut_x[b] - in.cut_w / 2;
    auto clampi = [](long long v, int hi) { return (float)(v < 0 ? 0 : v > hi ? hi : v); };
    p[0] = 1.f; p[1] = shift; p[2] = sat; p[3] = in.con[b] + 0.5f;
    p[4] = acc / (3.f * h * w);
    p[5] = clampi(oy, h - 1); p[6] = clampi(oy + in.cut_h - 1, h - 1);
    p[7] = clampi(ox, w - 1); p[8] = clampi(ox + in.cut_w - 1, w - 1);
  }
}

// DiffAugment is affine in its input; the parameters of its linear part for a tangent v (n, 3, h, w) contiguous:
// the call's own, without the brightness shift and with the contrast mean taken over the saturated tangent
__global__ void disc_aug_tangent_params_kernel(const float* __restrict__ v, int h, int w, const float* __restrict__ aug,
                                               float* __restrict__ taug) {
  __shared__ float red[32];
  const int b = blockIdx.x, P = h * w;
  const float* q = aug + (long long)kAugFloats * b;
  float* p = taug + (long long)kAugFloats * b;
  if (q[0] == 0.f) {
    if (threadIdx.x == 0) p[0] = 0.f;
    return;
  }
  float acc = 0.f;
  for (int t = threadIdx.x; t < P; t += blockDim.x)
    for (int c = 0; c < 3; ++c) acc += aug_saturated(v + 3ll * b * P + t, P, c, 0.f, q[2]);
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) {
    for (int k = 0; k < 9; ++k) p[k] = q[k];
    p[1] = 0.f;
    p[4] = acc / (3.f * P);
  }
}

__device__ __forceinline__ bool aug_cut(const float* p, int y, int x) {
  return (float)y >= p[5] && (float)y <= p[6] && (float)x >= p[7] && (float)x <= p[8];
}

// ------------------------------------------------------------------ im2col gather
struct GatherArgs {
  const float* src; long long s_b, s_c, s_y, s_x;
  const float *mean, *rstd;     // the source layer's InstanceNorm statistics, or null
  int act;                      // LeakyReLU on load (layers 2..)
  float scale;                  // power of two applied on load (col_scale)
  const float* aug;             // layer 1: DiffAugment parameters
  int n, hin, win, hout, wout, stride, pad, K;
  float* col;
  const float* prim;            // kTangent: the source layer's primal pre-norm output (LeakyReLU slope mask)
};

// kTangent (layers 2..): src holds the source layer's normalised tangent, which passes the LeakyReLU with the
// slope the primal input took
template <bool kTangent = false>
__global__ void disc_gather_kernel(const GatherArgs a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long P = (long long)a.hout * a.wout;
  if (t >= (long long)a.n * P * a.K) return;
  const int k = (int)(t % a.K);
  const long long j = t / a.K;
  const int b = (int)(j / P), p = (int)(j % P);
  const int ci = k >> 4, iy = (p / a.wout) * a.stride - a.pad + ((k >> 2) & 3),
            ix = (p % a.wout) * a.stride - a.pad + (k & 3);
  float v = 0.f;
  if (iy >= 0 && iy < a.hin && ix >= 0 && ix < a.win) {
    if (a.aug != nullptr) {
      const float* px = a.src + b * a.s_b + iy * a.s_y + ix * a.s_x;
      const float* q = a.aug + (long long)kAugFloats * b;
      if (q[0] != 0.f) {
        v = (aug_saturated(px, a.s_c, ci, q[1], q[2]) - q[4]) * q[3] + q[4];
        if (aug_cut(q, iy, ix)) v *= 0.f;
      } else {
        v = __ldg(px + ci * a.s_c);
      }
    } else if constexpr (kTangent) {
      const long long o = b * a.s_b + ci * a.s_c + iy * a.s_y + ix * a.s_x;
      v = __ldg(a.src + o);
      float nv = __ldg(a.prim + o);
      if (a.mean != nullptr) {
        const int r = ci * a.n + b;
        nv = (nv - a.mean[r]) * a.rstd[r];
      }
      if (!(nv > 0.f)) v *= kSlope;
    } else {
      v = __ldg(a.src + b * a.s_b + ci * a.s_c + iy * a.s_y + ix * a.s_x);
      if (a.mean != nullptr) {
        const int r = ci * a.n + b;
        v = (v - a.mean[r]) * a.rstd[r];
      }
      if (a.act) v = lrelu(v);
      v *= a.scale;
    }
  }
  a.col[t] = v;
}

// ------------------------------------------------------------------ InstanceNorm statistics (one block per row)
__global__ void disc_in_stats_kernel(const float* __restrict__ y, int P, float* __restrict__ mean,
                                     float* __restrict__ rstd) {
  __shared__ float red[32];
  const float* row = y + (long long)blockIdx.x * P;
  float s = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) s += row[p];
  const float m = block_sum(s, red) / (float)P;
  float q = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) q += (row[p] - m) * (row[p] - m);
  const float var = block_sum(q, red) / (float)P;
  if (threadIdx.x == 0) {
    mean[blockIdx.x] = m;
    rstd[blockIdx.x] = 1.f / sqrtf(var + kInEps);
  }
}

// ------------------------------------------------------------------ fold + activation backward
// One block per (channel, image) row of a layer's input: each pixel sums the dcol entries of the (up to 2 x 2)
// output positions whose window covers it, then (layers 2..) goes back through the previous layer's LeakyReLU and
// InstanceNorm: dy = rstd (g - mean(g) - n mean(g n)).
struct FoldArgs {
  const float* dcol;
  int n, cin, hin, win, hout, wout, stride, pad, K;
  const float* y;               // the previous layer's pre-norm output (null: layer 1, no activation)
  const float *mean, *rstd;
  float* out;                   // (cin, n, hin win)
};

// input pixel (y, x) of channel ci, image b: the sum of the dcol entries of the (up to 2 x 2) output positions whose
// window covers it
__device__ __forceinline__ float fold_at(const float* dcol, int b, int ci, int y, int x, int hout, int wout,
                                         int stride, int pad, int K) {
  float g = 0.f;
  for (int ky = 0; ky < 4; ++ky) {
    const int ty = y + pad - ky;
    if (ty < 0 || ty % stride != 0 || ty / stride >= hout) continue;
    for (int kx = 0; kx < 4; ++kx) {
      const int tx = x + pad - kx;
      if (tx < 0 || tx % stride != 0 || tx / stride >= wout) continue;
      const long long j = (long long)b * hout * wout + (ty / stride) * wout + tx / stride;
      g += dcol[j * K + ci * 16 + ky * 4 + kx];
    }
  }
  return g;
}

__global__ void disc_fold_kernel(const FoldArgs a) {
  __shared__ float red[32];
  const int r = blockIdx.x, ci = r / a.n, b = r % a.n;
  const int P = a.hin * a.win;
  const float* yr = a.y != nullptr ? a.y + (long long)r * P : nullptr;
  float* o = a.out + (long long)r * P;
  const float mu = a.mean != nullptr ? a.mean[r] : 0.f, rs = a.mean != nullptr ? a.rstd[r] : 1.f;
  float sg = 0.f, sgn = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const int y = p / a.win, x = p % a.win;
    float g = fold_at(a.dcol, b, ci, y, x, a.hout, a.wout, a.stride, a.pad, a.K);
    if (yr != nullptr) {
      const float nv = (yr[p] - mu) * rs;
      if (!(nv > 0.f)) g *= kSlope;
      sg += g;
      sgn += g * nv;
    }
    o[p] = g;
  }
  if (a.mean == nullptr) return;
  const float mg = block_sum(sg, red) / (float)P, mgn = block_sum(sgn, red) / (float)P;
  for (int p = threadIdx.x; p < P; p += blockDim.x) o[p] = rs * (o[p] - mg - (yr[p] - mu) * rs * mgn);
}

// ------------------------------------------------------------------ gradient penalty: tangent and second-order fold
// One block per (channel, image) row of a layer with InstanceNorm: the tangent of z = (y - mean) rstd along the
// tangent yd of y, zd = rstd (yd - mean(yd) - z q) with q = mean(z (yd - mean(yd))); mean(yd) and q are kept for the
// second-order fold.
__global__ void disc_in_tangent_kernel(const float* __restrict__ yd, const float* __restrict__ y,
                                       const float* __restrict__ mean, const float* __restrict__ rstd, int P,
                                       float* __restrict__ tmean, float* __restrict__ tq, float* __restrict__ zd) {
  __shared__ float red[32];
  const long long o = (long long)blockIdx.x * P;
  const float mu = mean[blockIdx.x], rs = rstd[blockIdx.x];
  float s = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) s += yd[o + p];
  const float m = block_sum(s, red) / (float)P;
  float q = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) q += (y[o + p] - mu) * rs * (yd[o + p] - m);
  q = block_sum(q, red) / (float)P;
  for (int p = threadIdx.x; p < P; p += blockDim.x) zd[o + p] = rs * (yd[o + p] - m - (y[o + p] - mu) * rs * q);
  if (threadIdx.x == 0) {
    tmean[blockIdx.x] = m;
    tq[blockIdx.x] = q;
  }
}

// The fold of both adjoint streams into layer i's input row (ci, b), then back through layer i - 1's LeakyReLU and
// InstanceNorm.  With gt / gp the folded, slope-masked tangent / primal adjoints, z the primal normalised value,
// yc = yd - mean(yd) the tangent, q = mean(z yc), a = mean(gt yc) and c = mean(gt z):
//   tangent  out_t = rstd (gt - mean(gt) - z c)                       (the first-order InstanceNorm backward)
//   primal   out_p = rstd (gp - mean(gp) - z mean(gp z))
//                  + rstd^2 (-a z + 3 q c z - c yc - q (gt - mean(gt)))   (zd's dependence on y through z and rstd)
// The two primal terms carry the exponents gp_in and gt_in + ev (the tangent's); the sum is written at the latter,
// stored to *e_out.  dcol_p null: a zero primal adjoint (the top layer).  mean null (no InstanceNorm): the masked
// folds pass through.
struct Fold2Args {
  const float *dcol_t, *dcol_p;
  int n, cin, hin, win, hout, wout, stride, pad, K;
  const float *y, *mean, *rstd, *yd, *tmean, *tq;
  const int *gt_in, *gp_in, *ev;
  int* e_out;
  float *out_t, *out_p;
};

__global__ void disc_fold2_kernel(const Fold2Args a) {
  __shared__ float red[32];
  const int r = blockIdx.x, ci = r / a.n, b = r % a.n;
  const int P = a.hin * a.win;
  const long long o = (long long)r * P;
  const bool in = a.mean != nullptr;
  const float mu = in ? a.mean[r] : 0.f, rs = in ? a.rstd[r] : 1.f;
  const float tm = in ? a.tmean[r] : 0.f, q = in ? a.tq[r] : 0.f;
  float st = 0.f, stz = 0.f, sp = 0.f, spz = 0.f, sa = 0.f;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const int y = p / a.win, x = p % a.win;
    float gt = fold_at(a.dcol_t, b, ci, y, x, a.hout, a.wout, a.stride, a.pad, a.K);
    float gp = a.dcol_p != nullptr ? fold_at(a.dcol_p, b, ci, y, x, a.hout, a.wout, a.stride, a.pad, a.K) : 0.f;
    const float z = (a.y[o + p] - mu) * rs;
    if (!(z > 0.f)) {
      gt *= kSlope;
      gp *= kSlope;
    }
    if (in) {
      st += gt; stz += gt * z; sp += gp; spz += gp * z;
      sa += gt * (a.yd[o + p] - tm);
    }
    a.out_t[o + p] = gt;
    a.out_p[o + p] = gp;
  }
  const int eg = a.gp_in != nullptr ? *a.gp_in : 0;
  if (!in) {
    if (blockIdx.x == 0 && threadIdx.x == 0) *a.e_out = eg;
    return;
  }
  const float mt = block_sum(st, red) / (float)P, c = block_sum(stz, red) / (float)P;
  const float mp = block_sum(sp, red) / (float)P, cp = block_sum(spz, red) / (float)P;
  const float am = block_sum(sa, red) / (float)P;
  const int ex = *a.gt_in + *a.ev;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const float z = (a.y[o + p] - mu) * rs, gt = a.out_t[o + p], gp = a.out_p[o + p];
    const float cross = rs * rs * (-am * z + 3.f * q * c * z - c * (a.yd[o + p] - tm) - q * (gt - mt));
    a.out_t[o + p] = rs * (gt - mt - z * c);
    a.out_p[o + p] = ldexpf(rs * (gp - mp - z * cp), eg - ex) + cross;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) *a.e_out = ex;
}

// v = 2 d_reg[b] g[b] (n, 3, h, w): the tangent direction whose Hessian-vector product is the penalty's gradient.
// dreg is d_reg scaled by the power of two that puts its largest element in [2^14, 2^15), the exponent carried in
// ev[0]: as a float factor, a small d_reg (2^-126 times integers below 2^10) made v subnormal or 0 before its own
// rescale, and a large one could overflow it
__global__ void disc_pen_dir_kernel(const float* __restrict__ g, const float* __restrict__ dreg, long long per_image,
                                    long long m, float* __restrict__ v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) v[i] = 2.f * dreg[i / per_image] * g[i];
}

__global__ void disc_fill_kernel(float* __restrict__ x, long long m, float v) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < m) x[i] = v;
}

// reg[b] = sum g[b]^2, one block per image
__global__ void disc_pen_reg_kernel(const float* __restrict__ g, long long per_image, float* __restrict__ reg) {
  __shared__ float red[32];
  const float* gb = g + blockIdx.x * per_image;
  float s = 0.f;
  for (long long i = threadIdx.x; i < per_image; i += blockDim.x) s += gb[i] * gb[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) reg[blockIdx.x] = s;
}

// the raw second-order weight gradient of each layer: dwt 2^(gt + ev) + dwp 2^gp, written to dwt at the larger
// exponent (stored to gw); dwp null: no primal part (the top layer)
struct CombArgs {
  float* dwt[kMaxLayers];
  const float* dwp[kMaxLayers];
  int numel[kMaxLayers];
  const int *gt, *gp, *ev;
  int* gw;
};

__global__ void disc_pen_combine_kernel(const CombArgs a) {
  const int l = blockIdx.y;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (a.dwt[l] == nullptr) return;
  const int et = a.gt[l] + a.ev[l];
  const int ep = a.dwp[l] != nullptr ? a.gp[l] : et;
  const int e = et > ep ? et : ep;
  if (i == 0) a.gw[l] = e;
  if (i >= a.numel[l]) return;
  float v = ldexpf(a.dwt[l][i], et - e);
  if (a.dwp[l] != nullptr) v += ldexpf(a.dwp[l][i], ep - e);
  a.dwt[l][i] = v;
}

// out[l] = src[l] (kAcc: out[l] += src[l])
struct AddArgs {
  float* out[kMaxLayers];
  const float* src[kMaxLayers];
  int numel[kMaxLayers];
};

template <bool kAcc>
__global__ void disc_pen_add_kernel(const AddArgs a) {
  const int l = blockIdx.y;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (a.out[l] == nullptr || i >= a.numel[l]) return;
  a.out[l][i] = kAcc ? a.out[l][i] + a.src[l][i] : a.src[l][i];
}

// ------------------------------------------------------------------ gradient scale and DiffAugment backward
// dy = g 2^k with the largest |dy| in [2^14, 2^15) (dy may be g); e_out = e_in - k (e_in null: 0).  Applied to the
// upstream gradient and again to each layer's output gradient, so that no GEMM operand drifts into fp16's
// subnormal range along the chain.  The exponent stays an integer: as a float factor 2^e_out it would underflow to 0
// for an upstream below 2^-135 or a chain that shrinks the gradients far enough.
__global__ void disc_grad_scale_kernel(const float* g, long long m, float* dy, const int* __restrict__ e_in,
                                       int* __restrict__ e_out) {
  __shared__ float red[32];
  float mx = 0.f;
  for (long long i = threadIdx.x; i < m; i += blockDim.x) mx = fmaxf(mx, fabsf(g[i]));
  const int k = pow2_exponent(block_max(mx, red));
  for (long long i = threadIdx.x; i < m; i += blockDim.x) dy[i] = ldexpf(g[i], k);
  if (threadIdx.x == 0) *e_out = (e_in != nullptr ? *e_in : 0) - k;
}

// one block per image: dx (3, n, h w) -> the input gradient through d_strides, unscaled (kAcc: added to it)
template <bool kAcc = false>
__global__ void disc_aug_bwd_kernel(const float* __restrict__ dx, const float* __restrict__ aug, int n, int h, int w,
                                    const int* __restrict__ gexp, float* __restrict__ out, long long s_b,
                                    long long s_c, long long s_y, long long s_x) {
  __shared__ float red[32];
  const int b = blockIdx.x, P = h * w;
  const float* q = aug + (long long)kAugFloats * b;
  const int e = *gexp;
  const bool on = q[0] != 0.f;
  float S = 0.f;
  if (on) {
    for (int p = threadIdx.x; p < P; p += blockDim.x)
      if (!aug_cut(q, p / w, p % w))
        for (int c = 0; c < 3; ++c) S += dx[((long long)c * n + b) * P + p];
    S = block_sum(S, red) / (3.f * P);
  }
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    const int y = p / w, x = p % w;
    float g[3];
    for (int c = 0; c < 3; ++c) g[c] = dx[((long long)c * n + b) * P + p];
    if (on) {
      const bool cut = aug_cut(q, y, x);
      const float sat = q[2], con = q[3];
      for (int c = 0; c < 3; ++c) g[c] = con * (cut ? g[c] * 0.f : g[c]) + (1.f - con) * S;
      const float m = (g[0] + g[1] + g[2]) / 3.f;
      for (int c = 0; c < 3; ++c) g[c] = sat * g[c] + (1.f - sat) * m;
    }
    for (int c = 0; c < 3; ++c) {
      float* o = out + b * s_b + c * s_c + y * s_y + x * s_x;
      *o = kAcc ? *o + ldexpf(g[c], e) : ldexpf(g[c], e);
    }
  }
}

// ------------------------------------------------------------------ spectral-norm weight-gradient correction
struct FixArgs {
  float* dW[kMaxLayers];        // null: no gradient for that layer
  const float* W[kMaxLayers];
  const float *u[kMaxLayers], *v[kMaxLayers];
  float* part[kMaxLayers];
  int rows[kMaxLayers], cols[kMaxLayers];
  const float* inv_sigma;
  const int* gexp;
};

// part[r] = <dW[r], W[r]>
__global__ void disc_sn_dot_kernel(const FixArgs a) {
  __shared__ float red[32];
  const int l = blockIdx.y, r = blockIdx.x;
  if (a.dW[l] == nullptr || r >= a.rows[l]) return;
  const long long o = (long long)r * a.cols[l];
  float acc = 0.f;
  for (int k = threadIdx.x; k < a.cols[l]; k += blockDim.x) acc += a.dW[l][o + k] * a.W[l][o + k];
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) a.part[l][r] = acc;
}

// dW = (dW / sigma - (<dW, W> / sigma^2) u v^T) 2^gexp; every block sums part[] in the same order
__global__ void disc_sn_fix_kernel(const FixArgs a) {
  __shared__ float red[32];
  const int l = blockIdx.y;
  if (a.dW[l] == nullptr) return;
  const long long n = (long long)a.rows[l] * a.cols[l];
  if ((long long)blockIdx.x * blockDim.x >= n) return;
  float d = 0.f;
  for (int r = threadIdx.x; r < a.rows[l]; r += blockDim.x) d += a.part[l][r];
  d = block_sum(d, red);
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float is = a.inv_sigma[l], c = d * is * is;
  const int r = (int)(i / a.cols[l]), k = (int)(i % a.cols[l]);
  a.dW[l][i] = ldexpf(a.dW[l][i] * is - c * a.u[l][r] * a.v[l][k], a.gexp[l]);
}

// ------------------------------------------------------------------ host
#define DISC_TRY(x)                \
  do {                             \
    if (int rc_ = (x)) return rc_; \
  } while (0)

unsigned blocks_of(long long n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// The power of two layer i's im2col values are scaled by (undone in the GEMMs' alpha), so that small activations
// keep normal fp16 lo words.  An InstanceNorm output over P elements is bounded by sqrt(P - 1), and LeakyReLU keeps
// that bound, so 2^s sqrt(P) <= 2^15 stays clear of the fp16 clamp; the image and a layer without InstanceNorm
// have no such bound and are not scaled.
float col_scale(const Net& N, int i) {
  if (i == 0 || !N.l[i - 1].in_norm) return 1.f;
  return ldexpf(1.f, (int)floor(log2(32768.0 / sqrt((double)N.l[i - 1].P()))));
}

SnArgs sn_args(const Net& N, const float* const* W, float* const* u_mod, float* const* v_mod, const DiscWs& ws) {
  SnArgs a{};
  for (int i = 0; i < N.n_layers; ++i) {
    a.W[i] = W[i]; a.u_mod[i] = u_mod[i]; a.v_mod[i] = v_mod[i];
    a.u[i] = ws.u[i]; a.v[i] = ws.v[i]; a.t[i] = ws.t[i]; a.s[i] = ws.s[i]; a.rmax[i] = ws.rmax[i]; a.ws[i] = ws.ws[i];
    a.rows[i] = N.l[i].cout; a.cols[i] = (int)N.l[i].K();
  }
  a.sigma = ws.sigma; a.inv_sigma = ws.inv_sigma; a.alpha = ws.alpha; a.wscale = ws.wscale;
  return a;
}

template <int kMode>
int disc_forward_impl(const Net& N, const float* const* W, float* const* u_mod, float* const* v_mod, const float* x,
                      const int64_t* xs, const AugIn& aug, int training, float* out, const DiscWs& ws, cudaStream_t st) {
  const int L = N.n_layers;
  {  // spectral norm: sigma, u, v of every layer
    const SnArgs a = sn_args(N, W, u_mod, v_mod, ws);
    if (training) {
      disc_sn_wtu_kernel<<<dim3(blocks_of(16 * 512, 256), L), 256, 0, st>>>(a);
      DISC_TRY(check_launch("disc_sn_wtu_kernel"));
    }
    disc_sn_v_kernel<<<L, 1024, 0, st>>>(a, training);
    DISC_TRY(check_launch("disc_sn_v_kernel"));
    disc_sn_wv_kernel<<<dim3(512, L), 256, 0, st>>>(a);
    DISC_TRY(check_launch("disc_sn_wv_kernel"));
    disc_sn_u_kernel<<<L, 512, 0, st>>>(a, training);
    DISC_TRY(check_launch("disc_sn_u_kernel"));
    disc_w_scale_kernel<<<dim3(blocks_of(512ll * 16 * 512, 256), L), 256, 0, st>>>(a);
    DISC_TRY(check_launch("disc_w_scale_kernel"));
  }
  disc_aug_params_kernel<<<N.n, 256, 0, st>>>(x, xs[0], xs[1], xs[2], xs[3], N.h, N.w, aug, ws.aug);
  DISC_TRY(check_launch("disc_aug_params_kernel"));
  for (int i = 0; i < L; ++i) {
    const Layer& y = N.l[i];
    const long long rows = (long long)N.n * y.P();
    GatherArgs g{};
    if (i == 0) {
      g.src = x; g.s_b = xs[0]; g.s_c = xs[1]; g.s_y = xs[2]; g.s_x = xs[3];
      g.aug = ws.aug;
    } else {
      const Layer& p = N.l[i - 1];
      g.src = ws.y[i - 1]; g.s_b = p.P(); g.s_c = N.n * p.P(); g.s_y = p.wout; g.s_x = 1;
      g.mean = ws.mean[i - 1]; g.rstd = ws.rstd[i - 1]; g.act = 1;
    }
    g.n = N.n; g.hin = y.hin; g.win = y.win; g.hout = y.hout; g.wout = y.wout; g.stride = y.stride; g.pad = y.pad;
    g.K = (int)y.K(); g.col = ws.col[i]; g.scale = col_scale(N, i);
    disc_gather_kernel<<<blocks_of(rows * y.K(), 256), 256, 0, st>>>(g);
    DISC_TRY(check_launch("disc_gather_kernel"));
    Gemm m = gemm(y.cout, (int)rows, (int)y.K());
    m.A = ws.ws[i]; m.a_m = y.K(); m.a_k = 1;
    m.Bf = ws.col[i]; m.b_n = y.K(); m.b_k = 1;
    m.C = y.act ? ws.y[i] : out; m.c_m = rows;
    m.alpha = 1.f / col_scale(N, i);
    m.alpha_dev = ws.alpha + i;
    DISC_TRY((run_gemm<kMode, true>(m, 1, st)));
    if (y.in_norm) {
      disc_in_stats_kernel<<<y.cout * N.n, 256, 0, st>>>(ws.y[i], (int)y.P(), ws.mean[i], ws.rstd[i]);
      DISC_TRY(check_launch("disc_in_stats_kernel"));
    }
  }
  return SNB_OK;
}

template <int kMode>
int disc_backward_impl(const Net& N, const float* const* W, const float* d_out, float* d_input, const int64_t* ds,
                       float* const* d_weights, const DiscWs& ws, cudaStream_t st) {
  const int L = N.n_layers;
  const Layer& last = N.l[L - 1];
  float* dy = ws.dy0;
  float* dy_next = ws.dy1;
  disc_grad_scale_kernel<<<1, 1024, 0, st>>>(d_out, (long long)N.n * last.P(), dy, nullptr, ws.gexp + L - 1);
  DISC_TRY(check_launch("disc_grad_scale_kernel"));
  // lowest layer whose input gradient is needed
  int stop = d_input != nullptr ? 0 : L;
  for (int i = 0; i < L && stop == L; ++i)
    if (d_weights[i] != nullptr) stop = i + 1;
  for (int i = L - 1; i >= 0; --i) {
    const Layer& y = N.l[i];
    const long long rows = (long long)N.n * y.P();
    if (d_weights[i] != nullptr) {  // dW[co][k] = sum_j dy[co][j] col[j][k]
      Gemm m = gemm(y.cout, (int)y.K(), (int)rows);
      m.A = dy; m.a_m = rows; m.a_k = 1;
      m.Bf = ws.col[i]; m.b_n = 1; m.b_k = y.K();
      m.C = d_weights[i]; m.c_m = y.K();
      m.alpha = 1.f / col_scale(N, i);
      DISC_TRY(run_gemm<kMode>(m, 1, st));
    }
    if (i < stop) break;
    {  // dcol[j][k] = (1 / sigma) sum_co dy[co][j] W[co][k]
      Gemm m = gemm((int)rows, (int)y.K(), y.cout);
      m.A = dy; m.a_m = 1; m.a_k = rows;
      m.Bf = ws.ws[i]; m.b_n = 1; m.b_k = y.K();
      m.C = ws.dcol; m.c_m = y.K();
      m.alpha_dev = ws.alpha + i;
      DISC_TRY((run_gemm<kMode, true>(m, 1, st)));
    }
    FoldArgs f{};
    f.dcol = ws.dcol; f.n = N.n; f.cin = y.cin; f.hin = y.hin; f.win = y.win; f.hout = y.hout; f.wout = y.wout;
    f.stride = y.stride; f.pad = y.pad; f.K = (int)y.K();
    if (i > 0) {
      f.y = ws.y[i - 1]; f.mean = ws.mean[i - 1]; f.rstd = ws.rstd[i - 1]; f.out = dy_next;
    } else {
      f.out = ws.dx;
    }
    disc_fold_kernel<<<y.cin * N.n, 256, 0, st>>>(f);
    DISC_TRY(check_launch("disc_fold_kernel"));
    if (i > 0) {
      disc_grad_scale_kernel<<<1, 1024, 0, st>>>(dy_next, (long long)y.cin * N.n * y.hin * y.win, dy_next, ws.gexp + i,
                                                 ws.gexp + i - 1);
      DISC_TRY(check_launch("disc_grad_scale_kernel"));
    }
    float* tmp = dy; dy = dy_next; dy_next = tmp;
  }
  if (d_input != nullptr) {
    disc_aug_bwd_kernel<<<N.n, 256, 0, st>>>(ws.dx, ws.aug, N.n, N.h, N.w, ws.gexp, d_input, ds[0], ds[1], ds[2], ds[3]);
    DISC_TRY(check_launch("disc_aug_bwd_kernel"));
  }
  FixArgs a{};
  long long most = 0;
  bool any = false;
  for (int i = 0; i < L; ++i) {
    a.dW[i] = d_weights[i]; a.W[i] = W[i]; a.u[i] = ws.u[i]; a.v[i] = ws.v[i]; a.part[i] = ws.part[i];
    a.rows[i] = N.l[i].cout; a.cols[i] = (int)N.l[i].K();
    if (d_weights[i] != nullptr) {
      any = true;
      most = most > N.l[i].cout * N.l[i].K() ? most : N.l[i].cout * N.l[i].K();
    }
  }
  a.inv_sigma = ws.inv_sigma; a.gexp = ws.gexp;
  if (any) {
    disc_sn_dot_kernel<<<dim3(512, L), 256, 0, st>>>(a);
    DISC_TRY(check_launch("disc_sn_dot_kernel"));
    disc_sn_fix_kernel<<<dim3(blocks_of(most, 256), L), 256, 0, st>>>(a);
    DISC_TRY(check_launch("disc_sn_fix_kernel"));
  }
  return SNB_OK;
}

// The forward, then g = grad_x sum(out) through the first-order chain (kept in the workspace) and reg[b] = |g[b]|^2.
template <int kMode>
int disc_penalty_forward_impl(const Net& N, const float* const* W, float* const* u_mod, float* const* v_mod,
                              const float* x, const int64_t* xs, const AugIn& aug, int training, float* out, float* reg,
                              const DiscWs& ws, cudaStream_t st) {
  DISC_TRY(disc_forward_impl<kMode>(N, W, u_mod, v_mod, x, xs, aug, training, out, ws, st));
  const long long n_out = (long long)N.n * N.l[N.n_layers - 1].P(), per_image = 3ll * N.h * N.w;
  disc_fill_kernel<<<blocks_of(n_out, 256), 256, 0, st>>>(ws.ones, n_out, 1.f);
  DISC_TRY(check_launch("disc_fill_kernel"));
  const int64_t gs[4] = {per_image, (int64_t)N.h * N.w, N.w, 1};
  float* none[kMaxLayers] = {};
  DISC_TRY(disc_backward_impl<kMode>(N, W, ws.ones, ws.g, gs, none, ws, st));
  disc_pen_reg_kernel<<<N.n, 256, 0, st>>>(ws.g, per_image, reg);
  return check_launch("disc_pen_reg_kernel");
}

// The first-order gradients from d_out (disc_backward_impl), then the penalty's: for v = 2 d_reg g, the gradients of
// sum(J_x out . v), by a tangent forward along v and a reverse pass over two adjoint streams (the tangent's, which
// starts at 1 on every output, and the primal's, which starts at 0 and is fed by the InstanceNorm cross terms).
template <int kMode>
int disc_penalty_backward_impl(const Net& N, const float* const* W, const float* d_out, const float* d_reg,
                               float* d_input, const int64_t* ds, float* const* d_weights, const DiscWs& ws,
                               cudaStream_t st) {
  const int L = N.n_layers;
  const bool first = d_out != nullptr;
  if (first) DISC_TRY(disc_backward_impl<kMode>(N, W, d_out, d_input, ds, d_weights, ws, st));
  if (d_reg == nullptr) return SNB_OK;
  // lowest layer whose input gradient is needed; stop = L with only the last weight wanted still runs that wgrad
  bool any = d_input != nullptr;
  int stop = d_input != nullptr ? 0 : L;
  for (int i = 0; i < L; ++i) {
    any = any || d_weights[i] != nullptr;
    if (d_weights[i] != nullptr && stop == L) stop = i + 1;
  }
  if (!any) return SNB_OK;
  const long long img = 3ll * N.n * N.h * N.w, P0 = (long long)N.h * N.w;
  // tangent forward along v, each layer's tangent col scaled to [2^14, 2^15) with its exponent in ev
  disc_grad_scale_kernel<<<1, 1024, 0, st>>>(d_reg, N.n, ws.dreg, nullptr, ws.ev);
  DISC_TRY(check_launch("disc_grad_scale_kernel"));
  disc_pen_dir_kernel<<<blocks_of(img, 256), 256, 0, st>>>(ws.g, ws.dreg, 3 * P0, img, ws.vt);
  DISC_TRY(check_launch("disc_pen_dir_kernel"));
  disc_grad_scale_kernel<<<1, 1024, 0, st>>>(ws.vt, img, ws.vt, ws.ev, ws.ev);
  DISC_TRY(check_launch("disc_grad_scale_kernel"));
  disc_aug_tangent_params_kernel<<<N.n, 256, 0, st>>>(ws.vt, N.h, N.w, ws.aug, ws.taug);
  DISC_TRY(check_launch("disc_aug_tangent_params_kernel"));
  float* zd = ws.dy0;
  for (int i = 0; i < L; ++i) {
    const Layer& y = N.l[i];
    const long long rows = (long long)N.n * y.P();
    GatherArgs g{};
    if (i == 0) {
      g.src = ws.vt; g.s_b = 3 * P0; g.s_c = P0; g.s_y = N.w; g.s_x = 1;
      g.aug = ws.taug;
    } else {
      const Layer& p = N.l[i - 1];
      g.src = zd; g.prim = ws.y[i - 1]; g.s_b = p.P(); g.s_c = N.n * p.P(); g.s_y = p.wout; g.s_x = 1;
      g.mean = ws.mean[i - 1]; g.rstd = ws.rstd[i - 1];
    }
    g.n = N.n; g.hin = y.hin; g.win = y.win; g.hout = y.hout; g.wout = y.wout; g.stride = y.stride; g.pad = y.pad;
    g.K = (int)y.K(); g.col = ws.tcol[i]; g.scale = 1.f;
    if (i == 0) disc_gather_kernel<<<blocks_of(rows * y.K(), 256), 256, 0, st>>>(g);
    else disc_gather_kernel<true><<<blocks_of(rows * y.K(), 256), 256, 0, st>>>(g);
    DISC_TRY(check_launch("disc_gather_kernel"));
    if (i == L - 1) break;   // the penalty needs only the adjoint of the last tangent output (1 everywhere)
    Gemm m = gemm(y.cout, (int)rows, (int)y.K());
    m.A = ws.ws[i]; m.a_m = y.K(); m.a_k = 1;
    m.Bf = ws.tcol[i]; m.b_n = y.K(); m.b_k = 1;
    m.C = ws.ty[i]; m.c_m = rows;
    m.alpha_dev = ws.alpha + i;
    DISC_TRY((run_gemm<kMode, true>(m, 1, st)));
    const float* zsrc = ws.ty[i];
    if (y.in_norm) {
      disc_in_tangent_kernel<<<y.cout * N.n, 256, 0, st>>>(ws.ty[i], ws.y[i], ws.mean[i], ws.rstd[i], (int)y.P(),
                                                            ws.tmean[i], ws.tq[i], zd);
      DISC_TRY(check_launch("disc_in_tangent_kernel"));
      zsrc = zd;
    }
    disc_grad_scale_kernel<<<1, 1024, 0, st>>>(zsrc, rows * y.cout, zd, ws.ev + i, ws.ev + i + 1);
    DISC_TRY(check_launch("disc_grad_scale_kernel"));
  }
  // reverse: t = the tangent stream's adjoint (exponents gt), p = the primal stream's (exponents gp)
  const Layer& last = N.l[L - 1];
  float *t = ws.dy0, *t_next = ws.dy1, *p = ws.dp0, *p_next = ws.dp1;
  disc_grad_scale_kernel<<<1, 1024, 0, st>>>(ws.ones, (long long)N.n * last.P(), t, nullptr, ws.gt + L - 1);
  DISC_TRY(check_launch("disc_grad_scale_kernel"));
  bool have_p = false;   // the primal adjoint of the top layer is zero
  for (int i = L - 1; i >= 0; --i) {
    const Layer& y = N.l[i];
    const long long rows = (long long)N.n * y.P();
    if (d_weights[i] != nullptr) {  // dW = t tcol^T (+ p col^T), each at its own exponent until combined
      Gemm m = gemm(y.cout, (int)y.K(), (int)rows);
      m.A = t; m.a_m = rows; m.a_k = 1;
      m.Bf = ws.tcol[i]; m.b_n = 1; m.b_k = y.K();
      m.C = ws.dwt[i]; m.c_m = y.K();
      DISC_TRY(run_gemm<kMode>(m, 1, st));
      if (have_p) {
        m.A = p; m.Bf = ws.col[i]; m.C = ws.dwp[i];
        m.alpha = 1.f / col_scale(N, i);
        DISC_TRY(run_gemm<kMode>(m, 1, st));
      }
    }
    if (i < stop) break;
    {  // dcol = (1 / sigma) W^T [t p]: both streams in one launch, as two matrices along z
      Gemm m = gemm((int)rows, (int)y.K(), y.cout);
      m.A = t; m.a_m = 1; m.a_k = rows; m.a_z1 = p - t;
      m.Bf = ws.ws[i]; m.b_n = 1; m.b_k = y.K();
      m.C = ws.dcol; m.c_m = y.K(); m.c_z1 = ws.dcolp - ws.dcol;
      m.alpha_dev = ws.alpha + i;
      if (i == 0) {   // only the primal stream reaches the input
        m.A = p; m.C = ws.dcolp;
      }
      DISC_TRY((run_gemm<kMode, true>(m, i > 0 && have_p ? 2 : 1, st)));
    }
    if (i > 0) {
      const int q = i - 1;
      Fold2Args f{};
      f.dcol_t = ws.dcol; f.dcol_p = have_p ? ws.dcolp : nullptr;
      f.n = N.n; f.cin = y.cin; f.hin = y.hin; f.win = y.win; f.hout = y.hout; f.wout = y.wout;
      f.stride = y.stride; f.pad = y.pad; f.K = (int)y.K();
      f.y = ws.y[q]; f.mean = ws.mean[q]; f.rstd = ws.rstd[q]; f.yd = ws.ty[q]; f.tmean = ws.tmean[q]; f.tq = ws.tq[q];
      f.gt_in = ws.gt + i; f.gp_in = have_p ? ws.gp + i : nullptr; f.ev = ws.ev + q; f.e_out = ws.gu + q;
      f.out_t = t_next; f.out_p = p_next;
      disc_fold2_kernel<<<y.cin * N.n, 256, 0, st>>>(f);
      DISC_TRY(check_launch("disc_fold2_kernel"));
      const long long m = (long long)y.cin * N.n * y.hin * y.win;
      disc_grad_scale_kernel<<<1, 1024, 0, st>>>(t_next, m, t_next, ws.gt + i, ws.gt + q);
      DISC_TRY(check_launch("disc_grad_scale_kernel"));
      disc_grad_scale_kernel<<<1, 1024, 0, st>>>(p_next, m, p_next, ws.gu + q, ws.gp + q);
      DISC_TRY(check_launch("disc_grad_scale_kernel"));
      float* tmp = t; t = t_next; t_next = tmp;
      tmp = p; p = p_next; p_next = tmp;
      have_p = true;
    } else {
      FoldArgs f{};
      f.dcol = ws.dcolp; f.n = N.n; f.cin = y.cin; f.hin = y.hin; f.win = y.win; f.hout = y.hout; f.wout = y.wout;
      f.stride = y.stride; f.pad = y.pad; f.K = (int)y.K(); f.out = ws.dx;
      disc_fold_kernel<<<y.cin * N.n, 256, 0, st>>>(f);
      DISC_TRY(check_launch("disc_fold_kernel"));
      if (first)
        disc_aug_bwd_kernel<true><<<N.n, 256, 0, st>>>(ws.dx, ws.aug, N.n, N.h, N.w, ws.gp, d_input, ds[0], ds[1],
                                                       ds[2], ds[3]);
      else
        disc_aug_bwd_kernel<<<N.n, 256, 0, st>>>(ws.dx, ws.aug, N.n, N.h, N.w, ws.gp, d_input, ds[0], ds[1], ds[2],
                                                 ds[3]);
      DISC_TRY(check_launch("disc_aug_bwd_kernel"));
    }
  }
  // the weight gradients: combine the two streams, the spectral-norm correction, then add to (or write) the output
  CombArgs c{};
  FixArgs a{};
  AddArgs d{};
  long long most = 0;
  for (int i = 0; i < L; ++i) {
    const long long numel = N.l[i].cout * N.l[i].K();
    const bool want = d_weights[i] != nullptr;
    c.dwt[i] = want ? ws.dwt[i] : nullptr; c.dwp[i] = want && i < L - 1 ? ws.dwp[i] : nullptr; c.numel[i] = (int)numel;
    a.dW[i] = c.dwt[i]; a.W[i] = W[i]; a.u[i] = ws.u[i]; a.v[i] = ws.v[i]; a.part[i] = ws.part[i];
    a.rows[i] = N.l[i].cout; a.cols[i] = (int)N.l[i].K();
    d.out[i] = d_weights[i]; d.src[i] = ws.dwt[i]; d.numel[i] = (int)numel;
    if (want) most = most > numel ? most : numel;
  }
  if (most == 0) return SNB_OK;
  c.gt = ws.gt; c.gp = ws.gp; c.ev = ws.ev; c.gw = ws.gw;
  a.inv_sigma = ws.inv_sigma; a.gexp = ws.gw;
  const dim3 grid(blocks_of(most, 256), L);
  disc_pen_combine_kernel<<<grid, 256, 0, st>>>(c);
  DISC_TRY(check_launch("disc_pen_combine_kernel"));
  disc_sn_dot_kernel<<<dim3(512, L), 256, 0, st>>>(a);
  DISC_TRY(check_launch("disc_sn_dot_kernel"));
  disc_sn_fix_kernel<<<grid, 256, 0, st>>>(a);
  DISC_TRY(check_launch("disc_sn_fix_kernel"));
  if (first) disc_pen_add_kernel<true><<<grid, 256, 0, st>>>(d);
  else disc_pen_add_kernel<false><<<grid, 256, 0, st>>>(d);
  return check_launch("disc_pen_add_kernel");
}

int check_ptrs(const char* who, const void* const* p, int n, const char* what, bool allow_null) {
  SNB_REQUIRE(p != nullptr, "%s: null %s array", who, what);
  for (int i = 0; i < n; ++i) SNB_REQUIRE(allow_null || p[i] != nullptr, "%s: null %s pointer %d", who, what, i);
  return SNB_OK;
}

// the checks of a forward call, shared by snb_disc_forward and snb_disc_penalty_forward
int forward_args(const char* who, int imsize, int precision, const float* const* weights, float* const* weight_u,
                 float* const* weight_v, const float* input, const int64_t* strides, int n, int height, int width,
                 const SnbDiscAug* aug, const float* out, const void* workspace, Net& N, AugIn& in, int& mode) {
  mode = mode_of(precision);
  if (mode < 0) return fail(SNB_ERR_UNSUPPORTED, "%s: unknown precision %d", who, precision);
  DISC_TRY(net_of(who, imsize, n, height, width, N));
  DISC_TRY(check_ptrs(who, reinterpret_cast<const void* const*>(weights), N.n_layers, "weight", false));
  DISC_TRY(check_ptrs(who, reinterpret_cast<const void* const*>(weight_u), N.n_layers, "weight_u", false));
  DISC_TRY(check_ptrs(who, reinterpret_cast<const void* const*>(weight_v), N.n_layers, "weight_v", false));
  SNB_REQUIRE(input != nullptr && strides != nullptr && out != nullptr && workspace != nullptr,
              "%s: null input, strides, out or workspace", who);
  in = AugIn{};
  if (aug != nullptr && aug->brightness != nullptr) {
    SNB_REQUIRE(aug->saturation != nullptr && aug->contrast != nullptr && aug->cutout_y != nullptr &&
                    aug->cutout_x != nullptr, "%s: DiffAugment draws must all be given or brightness NULL", who);
    in.bright = aug->brightness; in.sat = aug->saturation; in.con = aug->contrast;
    in.cut_y = aug->cutout_y; in.cut_x = aug->cutout_x;
    in.cut_h = (int)(height * 0.5 + 0.5); in.cut_w = (int)(width * 0.5 + 0.5);
  }
  return SNB_OK;
}

// ------------------------------------------------------------------ standalone DiffAugment (snb_diff_augment_*)
// Any policy, in its order, on (n, c, h, w) through strides.  Per image, 4 floats per op (the workspace):
//   color:       brightness shift rand - 0.5, saturation factor 2 rand, contrast factor rand + 0.5, and the forward's
//                contrast mean (rand_contrast's x_mean) or the backward's mean of the contrast's output gradient
//   translation: row and column shift (the input pixel an output pixel reads is its own plus the shift)
//   cutout:      the zeroed rows y0..y1 and columns x0..x1 (inclusive; rand_cutout's clamped index range)
// A pixel's value after ops [0, k) is a function of one input pixel (or of none: a translation moved in padding) and
// of per-pixel channel means, one per color op, which each thread recomputes for its own pixel: no pass stores an
// intermediate image.  The color arithmetic is the expressions of aug_saturated and disc_gather_kernel, channel sum
// in channel order, so 'color' followed by 'cutout' gives disc_gather_kernel's bits.
constexpr int kDaMaxOps = SNB_DIFF_AUG_MAX_OPS, kDaFloats = SNB_DIFF_AUG_WS_FLOATS;
static_assert(kDaFloats == 4 * kDaMaxOps, "4 workspace floats per op and image");

struct DaArgs {
  SnbDiffAugDraws d;
  int n_ops, op[kDaMaxOps], row[kDaMaxOps];   // row: the op's occurrence among the policy's ops of its kind
  int n, c, h, w, cut_h, cut_w;
  const float* src; long long s_b, s_c, s_y, s_x;   // forward: the input; backward: the output gradient
  float* dst; long long d_b, d_c, d_y, d_x;         // forward: the output; backward: the input gradient
  float* ws;
};

// image b's draws as op parameters, the means left zero
__device__ void da_params(const DaArgs& a, int b, float* q) {
  auto clampi = [](long long v, int hi) { return (float)(v < 0 ? 0 : v > hi ? hi : v); };
  for (int k = 0; k < a.n_ops; ++k) {
    const long long r = (long long)a.row[k] * a.n + b;
    float* p = q + 4 * k;
    if (a.op[k] == SNB_DIFF_AUG_COLOR) {
      p[0] = a.d.brightness[r] - 0.5f; p[1] = a.d.saturation[r] * 2.f; p[2] = a.d.contrast[r] + 0.5f; p[3] = 0.f;
    } else if (a.op[k] == SNB_DIFF_AUG_TRANSLATION) {
      p[0] = (float)a.d.translation_y[r]; p[1] = (float)a.d.translation_x[r]; p[2] = p[3] = 0.f;
    } else {
      const long long oy = a.d.cutout_y[r] - a.cut_h / 2, ox = a.d.cutout_x[r] - a.cut_w / 2;
      p[0] = clampi(oy, a.h - 1); p[1] = clampi(oy + a.cut_h - 1, a.h - 1);
      p[2] = clampi(ox, a.w - 1); p[3] = clampi(ox + a.cut_w - 1, a.w - 1);
    }
  }
}

__device__ __forceinline__ bool da_cut(const float* p, int y, int x) {
  return (float)y >= p[0] && (float)y <= p[1] && (float)x >= p[2] && (float)x <= p[3];
}

// forward: where pixel (y, x) of the image after ops [0, k) comes from.  start: the first op its value goes through
// (0: from the input at (y, x) as returned; j > 0: from the zero that op j - 1's translation read in the padding,
// (y, x) then being its position after op j - 1)
struct DaSrc { int start, y, x; };
__device__ DaSrc da_trace(const DaArgs& a, const float* q, int k, int y, int x) {
  for (int j = k - 1; j >= 0; --j) {
    if (a.op[j] != SNB_DIFF_AUG_TRANSLATION) continue;
    const int sy = y + (int)q[4 * j], sx = x + (int)q[4 * j + 1];
    if (sy < 0 || sy >= a.h || sx < 0 || sx >= a.w) return {j + 1, y, x};
    y = sy; x = sx;
  }
  return {0, y, x};
}

// channel c of that pixel after ops [s.start, k); m: its channel means of the color ops among them; px: its input
__device__ float da_value(const DaArgs& a, const float* q, const float* m, DaSrc s, int k, const float* px, int c) {
  float v = s.start == 0 ? px[c * a.s_c] : 0.f;
  int y = s.y, x = s.x;
  for (int j = s.start; j < k; ++j) {
    const float* p = q + 4 * j;
    if (a.op[j] == SNB_DIFF_AUG_COLOR) {
      const float t = (v + p[0] - m[j]) * p[1] + m[j];
      v = (t - p[3]) * p[2] + p[3];
    } else if (a.op[j] == SNB_DIFF_AUG_TRANSLATION) {
      y -= (int)p[0]; x -= (int)p[1];
    } else if (da_cut(p, y, x)) {
      v *= 0.f;
    }
  }
  return v;
}

// m[j] for every color op j in [s.start, k): the channel mean of its brightened input at this pixel
__device__ void da_means(const DaArgs& a, const float* q, DaSrc s, int k, const float* px, float* m) {
  for (int j = s.start; j < k; ++j) {
    if (a.op[j] != SNB_DIFF_AUG_COLOR) continue;
    float acc = da_value(a, q, m, s, j, px, 0) + q[4 * j];
    for (int c = 1; c < a.c; ++c) acc += da_value(a, q, m, s, j, px, c) + q[4 * j];
    m[j] = acc / (float)a.c;
  }
}

// backward: where the gradient with respect to pixel (y, x) of the image after ops [0, k) comes from.  end: the
// stage it starts at (n_ops: the output gradient at (y, x) as returned; j < n_ops: zero, op j's translation moving
// the pixel out, (y, x) then being its position before op j).  Color ops before that stage still pass it the
// gradient of their image-wide mean.
struct DaDst { int end, y, x; };
__device__ DaDst da_to_output(const DaArgs& a, const float* q, int k, int y, int x) {
  for (int j = k; j < a.n_ops; ++j) {
    if (a.op[j] != SNB_DIFF_AUG_TRANSLATION) continue;
    const int ny = y - (int)q[4 * j], nx = x - (int)q[4 * j + 1];
    if (ny < 0 || ny >= a.h || nx < 0 || nx >= a.w) return {j, y, x};
    y = ny; x = nx;
  }
  return {a.n_ops, y, x};
}

// channel c of the gradient with respect to the image after ops [0, k) at that pixel, through ops e.end - 1 .. k;
// gp: its output gradient; nm: its channel means of the gradient at each of those color ops' saturation output
__device__ float da_grad(const DaArgs& a, const float* q, const float* nm, int k, DaDst e, const float* gp, int c) {
  float g = e.end == a.n_ops ? gp[c * a.s_c] : 0.f;
  int y = e.y, x = e.x;
  for (int j = e.end - 1; j >= k; --j) {
    const float* p = q + 4 * j;
    if (a.op[j] == SNB_DIFF_AUG_COLOR) {
      g = p[2] * g + (1.f - p[2]) * p[3];
      g = p[1] * g + (1.f - p[1]) * nm[j];
    } else if (a.op[j] == SNB_DIFF_AUG_TRANSLATION) {
      y += (int)p[0]; x += (int)p[1];
    } else if (da_cut(p, y, x)) {
      g *= 0.f;
    }
  }
  return g;
}

__device__ void da_grad_means(const DaArgs& a, const float* q, int k, DaDst e, const float* gp, float* nm) {
  for (int j = e.end - 1; j >= k; --j) {
    if (a.op[j] != SNB_DIFF_AUG_COLOR) continue;
    const float con = q[4 * j + 2], S = q[4 * j + 3];
    float acc = con * da_grad(a, q, nm, j + 1, e, gp, 0) + (1.f - con) * S;
    for (int c = 1; c < a.c; ++c) acc += con * da_grad(a, q, nm, j + 1, e, gp, c) + (1.f - con) * S;
    nm[j] = acc / (float)a.c;
  }
}

// one block (256 threads) per image: the parameters, then each color op's image-wide mean in policy order (forward:
// of its saturated input, as disc_aug_params_kernel sums it) or in reverse order (backward: of its output gradient)
template <bool kBwd>
__global__ void __launch_bounds__(256) diff_aug_stats_kernel(const DaArgs a) {
  __shared__ float q[kDaFloats], red[32];
  const int b = blockIdx.x, P = a.h * a.w;
  if (threadIdx.x == 0) da_params(a, b, q);
  __syncthreads();
  for (int i = 0; i < a.n_ops; ++i) {
    const int k = kBwd ? a.n_ops - 1 - i : i;
    if (a.op[k] != SNB_DIFF_AUG_COLOR) continue;
    float acc = 0.f;
    for (int t = threadIdx.x; t < P; t += blockDim.x) {
      float m[kDaMaxOps];
      if constexpr (kBwd) {
        const DaDst e = da_to_output(a, q, k + 1, t / a.w, t % a.w);
        const float* gp = a.src + b * a.s_b + e.y * a.s_y + e.x * a.s_x;
        da_grad_means(a, q, k + 1, e, gp, m);
        for (int c = 0; c < a.c; ++c) acc += da_grad(a, q, m, k + 1, e, gp, c);
      } else {
        const DaSrc s = da_trace(a, q, k, t / a.w, t % a.w);
        const float* px = a.src + b * a.s_b + s.y * a.s_y + s.x * a.s_x;
        da_means(a, q, s, k + 1, px, m);
        for (int c = 0; c < a.c; ++c) acc += (da_value(a, q, m, s, k, px, c) + q[4 * k] - m[k]) * q[4 * k + 1] + m[k];
      }
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) q[4 * k + 3] = acc / ((float)a.c * a.h * a.w);
    __syncthreads();
  }
  if (threadIdx.x < kDaFloats) a.ws[(long long)kDaFloats * b + threadIdx.x] = q[threadIdx.x];
}

// one thread per pixel, all its channels.  Forward: output pixel (y, x); backward: input pixel (y, x)
template <bool kBwd>
__global__ void __launch_bounds__(256) diff_aug_map_kernel(const DaArgs a) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int P = a.h * a.w;
  if (t >= (long long)a.n * P) return;
  const int b = (int)(t / P), p = (int)(t % P), y = p / a.w, x = p % a.w;
  float q[kDaFloats], m[kDaMaxOps];
  for (int i = 0; i < 4 * a.n_ops; ++i) q[i] = a.ws[(long long)kDaFloats * b + i];
  float* o = a.dst + b * a.d_b + y * a.d_y + x * a.d_x;
  if constexpr (kBwd) {
    const DaDst e = da_to_output(a, q, 0, y, x);
    const float* gp = a.src + b * a.s_b + e.y * a.s_y + e.x * a.s_x;
    da_grad_means(a, q, 0, e, gp, m);
    for (int c = 0; c < a.c; ++c) o[c * a.d_c] = da_grad(a, q, m, 0, e, gp, c);
  } else {
    const DaSrc s = da_trace(a, q, a.n_ops, y, x);
    const float* px = a.src + b * a.s_b + s.y * a.s_y + s.x * a.s_x;
    da_means(a, q, s, a.n_ops, px, m);
    for (int c = 0; c < a.c; ++c) o[c * a.d_c] = da_value(a, q, m, s, a.n_ops, px, c);
  }
}

}  // namespace

// snb_diff_augment_forward / _backward after api.cu's checks: src -> dst through the strides (backward: the output
// gradient -> the input gradient)
int launch_diff_augment(bool backward, const int* ops, int n_ops, const SnbDiffAugDraws& draws, const float* src,
                        const int64_t* ss, int n, int c, int h, int w, float* dst, const int64_t* ds, float* ws,
                        cudaStream_t st) {
  DaArgs a{};
  a.d = draws;
  a.n_ops = n_ops;
  int seen[3] = {0, 0, 0};
  for (int k = 0; k < n_ops; ++k) { a.op[k] = ops[k]; a.row[k] = seen[ops[k]]++; }
  a.n = n; a.c = c; a.h = h; a.w = w;
  a.cut_h = (int)(h * 0.5 + 0.5); a.cut_w = (int)(w * 0.5 + 0.5);
  a.src = src; a.s_b = ss[0]; a.s_c = ss[1]; a.s_y = ss[2]; a.s_x = ss[3];
  a.dst = dst; a.d_b = ds[0]; a.d_c = ds[1]; a.d_y = ds[2]; a.d_x = ds[3];
  a.ws = ws;
  const unsigned blocks = (unsigned)(((long long)n * h * w + 255) / 256);
  if (backward) {
    diff_aug_stats_kernel<true><<<n, 256, 0, st>>>(a);
    DISC_TRY(check_launch("diff_aug_stats_kernel"));
    diff_aug_map_kernel<true><<<blocks, 256, 0, st>>>(a);
    return check_launch("diff_aug_map_kernel");
  }
  diff_aug_stats_kernel<false><<<n, 256, 0, st>>>(a);
  DISC_TRY(check_launch("diff_aug_stats_kernel"));
  diff_aug_map_kernel<false><<<blocks, 256, 0, st>>>(a);
  return check_launch("diff_aug_map_kernel");
}

}  // namespace snb

using namespace snb;

extern "C" {

size_t snb_disc_workspace_bytes(int imsize, int n, int height, int width, int save) {
  Net N;
  if (net_of("snb_disc_workspace_bytes", imsize, n, height, width, N) != SNB_OK) return 0;
  return disc_ws(nullptr, N, save ? 1 : 0).bytes;
}

int snb_disc_forward(int imsize, int precision, int training, const float* const* weights, float* const* weight_u,
                     float* const* weight_v, const float* input, const int64_t* strides, int n, int height, int width,
                     const SnbDiscAug* aug, float* out, void* workspace, void* stream) {
  const char* who = "snb_disc_forward";
  Net N;
  AugIn in{};
  int mode;
  DISC_TRY(forward_args(who, imsize, precision, weights, weight_u, weight_v, input, strides, n, height, width, aug,
                        out, workspace, N, in, mode));
  const DiscWs W = disc_ws(workspace, N, 0);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int tr = training ? 1 : 0;
  if (mode == kSplit) return disc_forward_impl<kSplit>(N, weights, weight_u, weight_v, input, strides, in, tr, out, W, st);
  if (mode == kF16) return disc_forward_impl<kF16>(N, weights, weight_u, weight_v, input, strides, in, tr, out, W, st);
  return disc_forward_impl<kBf16>(N, weights, weight_u, weight_v, input, strides, in, tr, out, W, st);
}

int snb_disc_backward(int imsize, int precision, const float* const* weights, int n, int height, int width,
                      const float* d_out, float* d_input, const int64_t* d_strides, float* const* d_weights,
                      void* workspace, void* stream) {
  const char* who = "snb_disc_backward";
  const int mode = mode_of(precision);
  if (mode < 0) return fail(SNB_ERR_UNSUPPORTED, "%s: unknown precision %d", who, precision);
  Net N;
  DISC_TRY(net_of(who, imsize, n, height, width, N));
  DISC_TRY(check_ptrs(who, reinterpret_cast<const void* const*>(weights), N.n_layers, "weight", false));
  DISC_TRY(check_ptrs(who, reinterpret_cast<const void* const*>(d_weights), N.n_layers, "d_weight", true));
  SNB_REQUIRE(d_out != nullptr && workspace != nullptr, "%s: null d_out or workspace", who);
  SNB_REQUIRE(d_input == nullptr || d_strides != nullptr, "%s: d_input without d_strides", who);
  const DiscWs W = disc_ws(workspace, N, 1);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == kSplit) return disc_backward_impl<kSplit>(N, weights, d_out, d_input, d_strides, d_weights, W, st);
  if (mode == kF16) return disc_backward_impl<kF16>(N, weights, d_out, d_input, d_strides, d_weights, W, st);
  return disc_backward_impl<kBf16>(N, weights, d_out, d_input, d_strides, d_weights, W, st);
}

size_t snb_disc_penalty_workspace_bytes(int imsize, int n, int height, int width) {
  Net N;
  if (net_of("snb_disc_penalty_workspace_bytes", imsize, n, height, width, N) != SNB_OK) return 0;
  return disc_ws(nullptr, N, 1, 1).bytes;
}

int snb_disc_penalty_forward(int imsize, int precision, int training, const float* const* weights,
                             float* const* weight_u, float* const* weight_v, const float* input, const int64_t* strides,
                             int n, int height, int width, const SnbDiscAug* aug, float* out, float* reg,
                             void* workspace, void* stream) {
  const char* who = "snb_disc_penalty_forward";
  Net N;
  AugIn in{};
  int mode;
  DISC_TRY(forward_args(who, imsize, precision, weights, weight_u, weight_v, input, strides, n, height, width, aug,
                        out, workspace, N, in, mode));
  SNB_REQUIRE(reg != nullptr, "%s: null reg", who);
  const DiscWs W = disc_ws(workspace, N, 1, 1);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int tr = training ? 1 : 0;
  if (mode == kSplit)
    return disc_penalty_forward_impl<kSplit>(N, weights, weight_u, weight_v, input, strides, in, tr, out, reg, W, st);
  if (mode == kF16)
    return disc_penalty_forward_impl<kF16>(N, weights, weight_u, weight_v, input, strides, in, tr, out, reg, W, st);
  return disc_penalty_forward_impl<kBf16>(N, weights, weight_u, weight_v, input, strides, in, tr, out, reg, W, st);
}

int snb_disc_penalty_backward(int imsize, int precision, const float* const* weights, int n, int height, int width,
                              const float* d_out, const float* d_reg, float* d_input, const int64_t* d_strides,
                              float* const* d_weights, void* workspace, void* stream) {
  const char* who = "snb_disc_penalty_backward";
  const int mode = mode_of(precision);
  if (mode < 0) return fail(SNB_ERR_UNSUPPORTED, "%s: unknown precision %d", who, precision);
  Net N;
  DISC_TRY(net_of(who, imsize, n, height, width, N));
  DISC_TRY(check_ptrs(who, reinterpret_cast<const void* const*>(weights), N.n_layers, "weight", false));
  DISC_TRY(check_ptrs(who, reinterpret_cast<const void* const*>(d_weights), N.n_layers, "d_weight", true));
  SNB_REQUIRE((d_out != nullptr || d_reg != nullptr) && workspace != nullptr, "%s: null d_out and d_reg, or null "
              "workspace", who);
  SNB_REQUIRE(d_input == nullptr || d_strides != nullptr, "%s: d_input without d_strides", who);
  const DiscWs W = disc_ws(workspace, N, 1, 1);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == kSplit)
    return disc_penalty_backward_impl<kSplit>(N, weights, d_out, d_reg, d_input, d_strides, d_weights, W, st);
  if (mode == kF16)
    return disc_penalty_backward_impl<kF16>(N, weights, d_out, d_reg, d_input, d_strides, d_weights, W, st);
  return disc_penalty_backward_impl<kBf16>(N, weights, d_out, d_reg, d_input, d_strides, d_weights, W, st);
}

}  // extern "C"
