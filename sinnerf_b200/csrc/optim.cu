// optim.cu -- fused optimiser step (Adam; SGD / RAdam / Ranger further down) over the 24 parameter tensors of one
// NeRF + refresh of its packed image (SURVEY.md 8f-4).  Reference: get_optimizer -> torch.optim.Adam(lr, eps=1e-8, weight_decay)
// (utils/__init__.py:19-21), stepped once per training iteration by Lightning (train.py:51-52 under DDP,
// i.e. after the gradient all-reduce).
//
// One launch updates all 595 844 parameters (torch runs ~10 multi-tensor launches over 24 tensors per
// model), accumulates the parameter checksum the packed image is stamped with (so the next
// snb_refresh_weights sees a clean image), and is followed on the same stream by the two pack kernels
// (bottleneck fold + chunk image) -- the image the forward streams is ready when step() returns, no
// per-step host-side re-pack decision.
//
// Arithmetic = torch.optim.Adam's single-tensor path (torch/optim/adam.py, amsgrad = False, maximize =
// False), operation for operation, every elementwise op rounded to fp32 like the separate ATen kernels:
//   g   = grad + weight_decay * p                         (add, alpha)
//   m   = m + (1 - beta1) * (g - m)                       (lerp, weight < 0.5)
//   v   = v * beta2;  v = v + (1 - beta2) * (g * g)       (mul_, addcmul_: ATen rounds the product g * g first)
//   den = sqrt(v) / sqrt(1 - beta2^t) + eps               (division by a python float: * (1 / scalar), the reciprocal
//                                                          formed in double and rounded to fp32 once)
//   p   = p + (-lr / (1 - beta1^t)) * (m / den)           (addcdiv_)
// Roofline: HBM/L2, 16 B read + 12 B written per parameter (17 MB per model) -- a few microseconds.
#include "common.cuh"

namespace snb {

struct AdamPtrs {
  float* p[SNB_N_PARAM_TENSORS];
  const float* g[SNB_N_PARAM_TENSORS];   // nullable per tensor: no gradient -> tensor skipped (as torch does)
};

// Block-reduces each thread's checksum sum and, in the last block to finish, stamps the image header with the
// checksum of the NEW values (the same sum params_check_kernel computes).
__device__ __forceinline__ void stamp_checksum(unsigned long long h, PackedHeader* hdr) {
  if (hdr == nullptr) return;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) h += __shfl_xor_sync(0xffffffffu, h, off);
  __shared__ unsigned long long part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = h;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long b = 0;
    for (int i = 0; i < 8; ++i) b += part[i];
    atomicAdd(&hdr->partial, b);
    __threadfence();
    if (atomicAdd(&hdr->blocks_done, 1u) == gridDim.x - 1) {
      __threadfence();
      hdr->checksum = atomicAdd(&hdr->partial, 0ull);
      hdr->dirty = 1;                  // the pack kernels that follow run unconditionally; keep the flag truthful
      hdr->partial = 0ull;
      hdr->blocks_done = 0u;
    }
  }
}

// One element of torch.optim.Adam's single-tensor step (the arithmetic listed above): m and v in, updated m, v and
// the new parameter out.  Shared by the NeRF kernel and the table walker (optim_tensors_kernel).
__device__ __forceinline__ float adam_update(float w, float gr, float& m, float& v, float lr_neg_step, float beta1_w,
                                             float beta2, float beta2_w, float eps, float weight_decay,
                                             float inv_bc2_sqrt) {
  if (weight_decay != 0.f) gr = fmaf(weight_decay, w, gr);
  m = fmaf(beta1_w, gr - m, m);
  v = __fmul_rn(v, beta2);
  v = fmaf(beta2_w, __fmul_rn(gr, gr), v);
  const float den = __fadd_rn(__fmul_rn(__fsqrt_rn(v), inv_bc2_sqrt), eps);
  return fmaf(lr_neg_step, __fdiv_rn(m, den), w);
}

__global__ void __launch_bounds__(256) adam_step_kernel(AdamPtrs a, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq,
                                                        float lr_neg_step, float beta1_w, float beta2, float beta2_w, float eps,
                                                        float weight_decay, float inv_bc2_sqrt, int precision, int new_activation,
                                                        PackedHeader* hdr) {
  unsigned long long h = 0;
  unsigned long long base = 0;
  for (int t = 0; t < SNB_N_PARAM_TENSORS; ++t) {
    const int n = param_numel(t);
    float* p = a.p[t];
    const float* g = a.g[t];
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
      float w = p[e];
      if (g != nullptr) {
        float m = exp_avg[base + e], v = exp_avg_sq[base + e];
        w = adam_update(w, g[e], m, v, lr_neg_step, beta1_w, beta2, beta2_w, eps, weight_decay, inv_bc2_sqrt);
        exp_avg[base + e] = m;
        exp_avg_sq[base + e] = v;
        p[e] = w;
      }
      h += param_checksum_term(base + e, __float_as_uint(w));
    }
    base += n;
  }
  stamp_checksum(h, hdr);
}

// The image the forward streams, re-packed on the step's stream from the updated parameters (packed == NULL: none).
static int repack(float* const* params, int precision, int new_activation, void* packed, cudaStream_t st) {
  if (packed == nullptr) return SNB_OK;
  const float* cp[SNB_N_PARAM_TENSORS];
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) cp[i] = params[i];
  if (precision == SNB_PREC_FP32) return launch_pack_fp32(cp, new_activation ? 1 : 0, packed, 0, st);
  return launch_pack_tc(cp, precision, new_activation ? 1 : 0, packed, 0, st);
}

// Adam's step-dependent scalars exactly as torch forms them: python doubles, cast to float where the kernels consume
// them.  -lr / (1 - beta1^t), and 1 / (1 - beta2^t) ** 0.5 with the reciprocal taken in double: a float reciprocal of
// the float cast rounds twice and differs from torch's by an ulp at most counts (at t = 1: 31.622778 vs 31.622776).
static void adam_bias_scalars(double lr, double beta1, double beta2, int step, float* lr_neg_step, float* inv_bc2_sqrt) {
  const double bc1 = 1.0 - pow(beta1, (double)step);
  const double bc2 = 1.0 - pow(beta2, (double)step);
  *lr_neg_step = (float)(-(lr / bc1));
  *inv_bc2_sqrt = (float)(1.0 / pow(bc2, 0.5));
}

int adam_step_pack(float* const* params, const float* const* grads, float* exp_avg, float* exp_avg_sq,
                   const SnbAdamArgs& o, int precision, int new_activation, void* packed, cudaStream_t st) {
  AdamPtrs a;
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) { a.p[i] = params[i]; a.g[i] = grads[i]; }
  float lr_neg_step, inv_bc2_sqrt;
  adam_bias_scalars(o.lr, o.beta1, o.beta2, o.step, &lr_neg_step, &inv_bc2_sqrt);
  const float beta1_w = (float)(1.0 - o.beta1), beta2_w = (float)(1.0 - o.beta2);
  adam_step_kernel<<<sm_count() * 2, 256, 0, st>>>(a, exp_avg, exp_avg_sq, lr_neg_step, beta1_w, (float)o.beta2, beta2_w,
                                                  (float)o.eps, (float)o.weight_decay, inv_bc2_sqrt, precision, new_activation,
                                                  reinterpret_cast<PackedHeader*>(packed));
  if (int rc = check_launch("adam_step_kernel")) return rc;
  return repack(params, precision, new_activation, packed, st);
}

// ---------------------------------------------------------------- SGD / RAdam / Ranger (snb_optim_step)
// Each line is one ATen elementwise kernel of the reference's step, rounded to fp32 as that kernel rounds it
// (ATen's CUDA add / addcmul / addcdiv contract `a + alpha * b` into one FMA, with b = t1 * t2 or t1 / t2 rounded on
// its own for addcmul / addcdiv; mul, sqrt, div round on their own):
//   SGD (torch/optim/sgd.py _multi_tensor_sgd, dampening 0, no Nesterov):
//     g = g + wd * p                 (_foreach_add, alpha)
//     b = g (first step)  |  b = b * momentum;  b = b + g         (_foreach_mul_, _foreach_add_)
//     p = p + (-lr) * b              (_foreach_add_, alpha)
//   RAdam / Ranger (utils/optimizers.py:65-66,90-104 / :393-425):
//     v = v * beta2;  v = v + (1 - beta2) * (g * g)               (mul_, addcmul_)
//     m = m * beta1;  m = m + (1 - beta1) * g                     (mul_, add_)
//     p = p + (-wd * lr) * p                                      (add_, when wd != 0)
//     p = p + (-step_size * lr) * (m / (sqrt(v) + eps))  if N_sma passes the threshold,   (sqrt, add_, addcdiv_)
//     p = p + (-step_size * lr) * m                       otherwise                        (add_)
//   Ranger, every k-th step of the tensor (:431-437): slow = slow + alpha * (p - slow);  p = slow    (sub, add_, copy_)
//   with slow = p (before the update) on the tensor's first step.
enum : unsigned { kFirst = 1u, kAdaptive = 2u, kSync = 4u };

struct RuleConsts {
  float lr_neg;         // SGD: -lr
  float decay;          // SGD / Adam: weight_decay;  RAdam / Ranger: -weight_decay * lr
  float momentum;       // SGD
  float beta1, beta1_w, beta2, beta2_w, eps, alpha;
};

struct RuleScalars {
  RuleConsts c;
  float step_lr[SNB_N_PARAM_TENSORS];           // RAdam / Ranger: -step_size * lr at the tensor's own step
  unsigned char flags[SNB_N_PARAM_TENSORS];     // kFirst | kAdaptive | kSync
};

// One element of SGD / RAdam / Ranger (the arithmetic listed above) at flat state index i: reads and writes the state
// buffers the rule keeps and returns the new parameter.  Shared by optim_step_kernel and optim_tensors_kernel.
template <int RULE>
__device__ __forceinline__ float rule_update(float w, float gr, unsigned long long i, float* __restrict__ exp_avg,
                                             float* __restrict__ exp_avg_sq, float* __restrict__ slow_buffer,
                                             const RuleConsts& s, unsigned f, float step_lr) {
  if (RULE == SNB_OPTIM_SGD) {
    if (s.decay != 0.f) gr = fmaf(s.decay, w, gr);
    if (s.momentum != 0.f) {
      if (!(f & kFirst)) gr = __fadd_rn(__fmul_rn(exp_avg[i], s.momentum), gr);
      exp_avg[i] = gr;
    }
    return fmaf(s.lr_neg, gr, w);
  }
  float v = __fmul_rn(exp_avg_sq[i], s.beta2);
  v = fmaf(s.beta2_w, __fmul_rn(gr, gr), v);
  float m = __fmul_rn(exp_avg[i], s.beta1);
  m = fmaf(s.beta1_w, gr, m);
  exp_avg[i] = m;
  exp_avg_sq[i] = v;
  float slow = 0.f;
  if (RULE == SNB_OPTIM_RANGER) slow = (f & kFirst) ? w : slow_buffer[i];
  if (s.decay != 0.f) w = fmaf(s.decay, w, w);
  if (f & kAdaptive)
    w = fmaf(step_lr, __fdiv_rn(m, __fadd_rn(__fsqrt_rn(v), s.eps)), w);
  else
    w = fmaf(step_lr, m, w);
  if (RULE == SNB_OPTIM_RANGER) {
    if (f & kSync) {
      slow = fmaf(s.alpha, __fsub_rn(w, slow), slow);
      w = slow;
    }
    if (f & (kFirst | kSync)) slow_buffer[i] = slow;
  }
  return w;
}

template <int RULE>
__global__ void __launch_bounds__(256) optim_step_kernel(AdamPtrs a, float* __restrict__ exp_avg,
                                                         float* __restrict__ exp_avg_sq, float* __restrict__ slow_buffer,
                                                         RuleScalars s, PackedHeader* hdr) {
  unsigned long long h = 0;
  unsigned long long base = 0;
  for (int t = 0; t < SNB_N_PARAM_TENSORS; ++t) {
    const int n = param_numel(t);
    float* p = a.p[t];
    const float* g = a.g[t];
    const unsigned f = s.flags[t];
    const float step_lr = s.step_lr[t];
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
      float w = p[e];
      if (g != nullptr) {
        w = rule_update<RULE>(w, g[e], base + e, exp_avg, exp_avg_sq, slow_buffer, s.c, f, step_lr);
        p[e] = w;
      }
      h += param_checksum_term(base + e, __float_as_uint(w));
    }
    base += n;
  }
  stamp_checksum(h, hdr);
}

static RuleConsts rule_consts(const SnbOptimArgs& o) {
  RuleConsts c = {};
  if (o.rule == SNB_OPTIM_SGD) {
    c.lr_neg = (float)(-o.lr);
    c.decay = (float)o.weight_decay;
    c.momentum = (float)o.momentum;
    return c;
  }
  c.beta1 = (float)o.beta1;
  c.beta1_w = (float)(1.0 - o.beta1);
  c.beta2 = (float)o.beta2;
  c.beta2_w = (float)(1.0 - o.beta2);
  c.eps = (float)o.eps;
  c.alpha = (float)o.alpha;
  c.decay = o.rule == SNB_OPTIM_ADAM ? (float)o.weight_decay : (float)(-o.weight_decay * o.lr);
  return c;
}

// SGD / RAdam / Ranger: the flags and -step_size * lr of a tensor at its own step count (its update count including
// this one).  RAdam / Ranger: utils/optimizers.py:68-86 / :397-411 in python doubles, the reference's expression order.
static void rule_tensor_scalars(const SnbOptimArgs& o, int step, float* step_lr, unsigned* flags) {
  if (o.rule == SNB_OPTIM_SGD) {
    *step_lr = 0.f;
    *flags = step == 1 ? kFirst : 0u;
    return;
  }
  const double beta2_t = pow(o.beta2, (double)step);
  const double n_sma_max = 2 / (1 - o.beta2) - 1;
  const double n_sma = n_sma_max - 2 * step * beta2_t / (1 - beta2_t);
  const bool adaptive = o.rule == SNB_OPTIM_RADAM ? n_sma >= 5 : n_sma > o.n_sma_threshold;
  const double step_size =
      adaptive ? sqrt((1 - beta2_t) * (n_sma - 4) / (n_sma_max - 4) * (n_sma - 2) / n_sma * n_sma_max /
                      (n_sma_max - 2)) / (1 - pow(o.beta1, (double)step))
               : 1.0 / (1 - pow(o.beta1, (double)step));
  *step_lr = (float)(-step_size * o.lr);
  *flags = (adaptive ? kAdaptive : 0u) | (step == 1 ? kFirst : 0u) |
           (o.rule == SNB_OPTIM_RANGER && step % o.k == 0 ? kSync : 0u);
}

int optim_step_pack(float* const* params, const float* const* grads, float* exp_avg, float* exp_avg_sq,
                    float* slow_buffer, const SnbOptimArgs& o, int precision, int new_activation, void* packed,
                    cudaStream_t st) {
  AdamPtrs a;
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) { a.p[i] = params[i]; a.g[i] = grads[i]; }
  RuleScalars s = {};
  s.c = rule_consts(o);
  for (int t = 0; t < SNB_N_PARAM_TENSORS; ++t) {
    if (o.rule != SNB_OPTIM_SGD && grads[t] == nullptr) continue;
    unsigned f;
    rule_tensor_scalars(o, o.step[t], &s.step_lr[t], &f);
    s.flags[t] = (unsigned char)f;
  }
  PackedHeader* hdr = reinterpret_cast<PackedHeader*>(packed);
  const int grid = sm_count() * 2;
  if (o.rule == SNB_OPTIM_SGD)
    optim_step_kernel<SNB_OPTIM_SGD><<<grid, 256, 0, st>>>(a, exp_avg, exp_avg_sq, slow_buffer, s, hdr);
  else if (o.rule == SNB_OPTIM_RADAM)
    optim_step_kernel<SNB_OPTIM_RADAM><<<grid, 256, 0, st>>>(a, exp_avg, exp_avg_sq, slow_buffer, s, hdr);
  else
    optim_step_kernel<SNB_OPTIM_RANGER><<<grid, 256, 0, st>>>(a, exp_avg, exp_avg_sq, slow_buffer, s, hdr);
  if (int rc = check_launch("optim_step_kernel")) return rc;
  return repack(params, precision, new_activation, packed, st);
}

// ---------------------------------------------------------------- any tensors (snb_optim_step_tensors)
// The four rules over a caller-given table of plain fp32 tensors (the discriminator's weight_orig): no checksum and no
// re-pack.  Tensor t's state sits at offset sum(numel[0..t)) of each flat buffer.  Tensors without a gradient are
// left out of the table on the host, so every entry is updated.
struct TensorEntry {
  float* p;
  const float* g;
  long long n;
  unsigned long long off;   // the tensor's offset in the flat state buffers
  float step_lr;            // Adam: -lr / (1 - beta1^t);  RAdam / Ranger: -step_size * lr
  float inv_bc2_sqrt;       // Adam: 1 / sqrt(1 - beta2^t)
  unsigned flags;           // SGD / RAdam / Ranger: kFirst | kAdaptive | kSync
};

struct TensorTable {
  TensorEntry t[SNB_OPTIM_MAX_TENSORS];
  int n;
};

template <int RULE>
__global__ void __launch_bounds__(256) optim_tensors_kernel(TensorTable tab, float* __restrict__ exp_avg,
                                                            float* __restrict__ exp_avg_sq,
                                                            float* __restrict__ slow_buffer, RuleConsts c) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (int t = 0; t < tab.n; ++t) {
    float* p = tab.t[t].p;
    const float* g = tab.t[t].g;
    const long long n = tab.t[t].n;
    const unsigned long long off = tab.t[t].off;
    const float step_lr = tab.t[t].step_lr;
    const float inv_bc2_sqrt = tab.t[t].inv_bc2_sqrt;
    const unsigned f = tab.t[t].flags;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
      const unsigned long long i = off + e;
      if (RULE == SNB_OPTIM_ADAM) {
        float m = exp_avg[i], v = exp_avg_sq[i];
        p[e] = adam_update(p[e], g[e], m, v, step_lr, c.beta1_w, c.beta2, c.beta2_w, c.eps, c.decay, inv_bc2_sqrt);
        exp_avg[i] = m;
        exp_avg_sq[i] = v;
      } else {
        p[e] = rule_update<RULE>(p[e], g[e], i, exp_avg, exp_avg_sq, slow_buffer, c, f, step_lr);
      }
    }
  }
}

int optim_step_tensors(int n, float* const* params, const float* const* grads, const int64_t* numel, const int* step,
                       float* exp_avg, float* exp_avg_sq, float* slow_buffer, const SnbOptimArgs& o, cudaStream_t st) {
  TensorTable tab = {};
  unsigned long long off = 0;
  for (int t = 0; t < n; off += (unsigned long long)numel[t], ++t) {
    if (grads[t] == nullptr) continue;
    TensorEntry& te = tab.t[tab.n++];
    te.p = params[t];
    te.g = grads[t];
    te.n = numel[t];
    te.off = off;
    if (o.rule == SNB_OPTIM_ADAM)
      adam_bias_scalars(o.lr, o.beta1, o.beta2, step[t], &te.step_lr, &te.inv_bc2_sqrt);
    else
      rule_tensor_scalars(o, step[t], &te.step_lr, &te.flags);
  }
  if (tab.n == 0) return SNB_OK;
  const RuleConsts c = rule_consts(o);
  const int grid = sm_count() * 4;
  if (o.rule == SNB_OPTIM_ADAM)
    optim_tensors_kernel<SNB_OPTIM_ADAM><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c);
  else if (o.rule == SNB_OPTIM_SGD)
    optim_tensors_kernel<SNB_OPTIM_SGD><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c);
  else if (o.rule == SNB_OPTIM_RADAM)
    optim_tensors_kernel<SNB_OPTIM_RADAM><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c);
  else
    optim_tensors_kernel<SNB_OPTIM_RANGER><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c);
  return check_launch("optim_tensors_kernel");
}

// ---------------------------------------------------------------- GradScaler-native steps (snb_*_amp)
// The three steps above as torch's GradScaler drives an optimiser that sets _step_supports_amp_scaling: the gradients
// arrive scaled, with GradScaler's scale and found_inf on the device, and the host does not wait for either.
//   * Every gradient element is unscaled as GradScaler.unscale_ does it -- inv = (float)(1 / (double)scale), then
//     g * inv unless inv == 1 (torch's _amp_foreach_non_finite_check_and_unscale_) -- and written back to the
//     gradient, taken step or not, so .grad ends as GradScaler's own unscale leaves it.  __fmul_rn keeps the product
//     out of any FMA, so the update sees the value it would read back from memory.
//   * *found_inf != 0: parameters, state, update counts, checksum and image stay as they are (GradScaler never calls
//     step() then).  The grid reads the same flag, so the branch is uniform.
//   * The update counts live on the device: the kernel reads count_in and block 0 writes count_out (a second buffer,
//     so no block can see a count advanced under it).  The step-dependent scalars are formed on the host, in doubles as
//     above, for the kOptimWindow counts base .. base + kOptimWindow - 1 a tensor can have reached, and each tensor
//     picks its entry by count_in + 1 - base.  The caller keeps that index in range (SnbAmpStep in the header).
constexpr int kOptimWindow = SNB_OPTIM_WINDOW;

struct AmpCtl {
  const float* scale;        // nullable: the gradients carry no scale
  const float* found_inf;    // nullable: never skip
  const int* count_in;
  int* count_out;
};

__device__ __forceinline__ float amp_inv_scale(const float* scale) {
  return scale == nullptr ? 1.f : (float)(1.0 / (double)*scale);
}
__device__ __forceinline__ bool amp_skip(const float* found_inf) { return found_inf != nullptr && *found_inf != 0.f; }
// The unscaled gradient element, written back when the scale changes it.
__device__ __forceinline__ float amp_unscale(float* g, long long e, float inv) {
  float gr = g[e];
  if (inv != 1.f) {
    gr = __fmul_rn(gr, inv);
    g[e] = gr;
  }
  return gr;
}

struct AdamWindow {
  int base;
  float lr_neg_step[kOptimWindow];
  float inv_bc2_sqrt[kOptimWindow];
};

// A skipped step clears header.dirty instead of stamping, so the pack kernels that follow (only_if_dirty) return at
// once and the image keeps the bytes and checksum it had.  The flag is the pack kernels' scratch: every refresh
// recomputes it from the checksum before it is read.
__global__ void __launch_bounds__(256) adam_step_amp_kernel(AdamPtrs a, float* __restrict__ exp_avg,
                                                            float* __restrict__ exp_avg_sq, float beta1_w, float beta2,
                                                            float beta2_w, float eps, float weight_decay, AdamWindow win,
                                                            AmpCtl amp, PackedHeader* hdr) {
  const bool skip = amp_skip(amp.found_inf);
  const float inv = amp_inv_scale(amp.scale);
  const int count = amp.count_in[0];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    amp.count_out[0] = skip ? count : count + 1;
    if (skip && hdr != nullptr) hdr->dirty = 0;
  }
  float lr_neg_step = 0.f, inv_bc2_sqrt = 0.f;
  if (!skip) {
    lr_neg_step = win.lr_neg_step[count + 1 - win.base];
    inv_bc2_sqrt = win.inv_bc2_sqrt[count + 1 - win.base];
  }
  unsigned long long h = 0;
  unsigned long long base = 0;
  for (int t = 0; t < SNB_N_PARAM_TENSORS; ++t) {
    const int n = param_numel(t);
    float* p = a.p[t];
    float* g = const_cast<float*>(a.g[t]);
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
      const float gr = g != nullptr ? amp_unscale(g, e, inv) : 0.f;
      if (skip) continue;
      float w = p[e];
      if (g != nullptr) {
        float m = exp_avg[base + e], v = exp_avg_sq[base + e];
        w = adam_update(w, gr, m, v, lr_neg_step, beta1_w, beta2, beta2_w, eps, weight_decay, inv_bc2_sqrt);
        exp_avg[base + e] = m;
        exp_avg_sq[base + e] = v;
        p[e] = w;
      }
      h += param_checksum_term(base + e, __float_as_uint(w));
    }
    base += n;
  }
  if (!skip) stamp_checksum(h, hdr);
}

static int repack_if_dirty(float* const* params, int precision, int new_activation, void* packed, cudaStream_t st) {
  if (packed == nullptr) return SNB_OK;
  const float* cp[SNB_N_PARAM_TENSORS];
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) cp[i] = params[i];
  if (precision == SNB_PREC_FP32) return launch_pack_fp32(cp, new_activation ? 1 : 0, packed, 1, st);
  return launch_pack_tc(cp, precision, new_activation ? 1 : 0, packed, 1, st);
}

static AmpCtl amp_ctl(const SnbAmpStep& amp) { return AmpCtl{amp.scale, amp.found_inf, amp.count_in, amp.count_out}; }

int adam_step_pack_amp(float* const* params, float* const* grads, float* exp_avg, float* exp_avg_sq,
                       const SnbAdamArgs& o, const SnbAmpStep& amp, int precision, int new_activation, void* packed,
                       cudaStream_t st) {
  AdamPtrs a;
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) { a.p[i] = params[i]; a.g[i] = grads[i]; }
  AdamWindow win;
  win.base = amp.base[0];
  for (int j = 0; j < kOptimWindow; ++j)
    adam_bias_scalars(o.lr, o.beta1, o.beta2, win.base + j, &win.lr_neg_step[j], &win.inv_bc2_sqrt[j]);
  const float beta1_w = (float)(1.0 - o.beta1), beta2_w = (float)(1.0 - o.beta2);
  adam_step_amp_kernel<<<sm_count() * 2, 256, 0, st>>>(a, exp_avg, exp_avg_sq, beta1_w, (float)o.beta2, beta2_w,
                                                      (float)o.eps, (float)o.weight_decay, win, amp_ctl(amp),
                                                      reinterpret_cast<PackedHeader*>(packed));
  if (int rc = check_launch("adam_step_amp_kernel")) return rc;
  return repack_if_dirty(params, precision, new_activation, packed, st);
}

// The window of one tensor: -step_size * lr and the flags at counts base .. base + kOptimWindow - 1.  Tensors at the
// same base (all of them, unless some lacked a gradient on some steps) share the host arithmetic.
static void rule_window(const SnbOptimArgs& o, int base, int* cached_base, float* step_lr, unsigned char* flags,
                        const float* cached_lr, const unsigned char* cached_flags) {
  if (*cached_base == base && cached_lr != nullptr) {
    for (int j = 0; j < kOptimWindow; ++j) { step_lr[j] = cached_lr[j]; flags[j] = cached_flags[j]; }
    return;
  }
  for (int j = 0; j < kOptimWindow; ++j) {
    unsigned f;
    rule_tensor_scalars(o, base + j, &step_lr[j], &f);
    flags[j] = (unsigned char)f;
  }
  *cached_base = base;
}

// Whether tensor t's count advances on a taken step: it has a gradient, and the rule keeps a count (SGD only with
// momentum, where the count says whether the momentum buffer exists yet).
static bool rule_advances(const SnbOptimArgs& o, const void* grad) {
  return grad != nullptr && (o.rule != SNB_OPTIM_SGD || o.momentum != 0.);
}

struct RuleWindow {
  RuleConsts c;
  unsigned adv;                                            // bit t: tensor t advances its count on a taken step
  int base[SNB_N_PARAM_TENSORS];
  float step_lr[SNB_N_PARAM_TENSORS][kOptimWindow];
  unsigned char flags[SNB_N_PARAM_TENSORS][kOptimWindow];
};

template <int RULE>
__global__ void __launch_bounds__(256) optim_step_amp_kernel(AdamPtrs a, float* __restrict__ exp_avg,
                                                             float* __restrict__ exp_avg_sq,
                                                             float* __restrict__ slow_buffer, RuleWindow s, AmpCtl amp,
                                                             PackedHeader* hdr) {
  const bool skip = amp_skip(amp.found_inf);
  const float inv = amp_inv_scale(amp.scale);
  if (blockIdx.x == 0) {
    if (threadIdx.x < SNB_N_PARAM_TENSORS)
      amp.count_out[threadIdx.x] = amp.count_in[threadIdx.x] + ((!skip && (s.adv >> threadIdx.x) & 1u) ? 1 : 0);
    if (threadIdx.x == 0 && skip && hdr != nullptr) hdr->dirty = 0;
  }
  unsigned long long h = 0;
  unsigned long long base = 0;
  for (int t = 0; t < SNB_N_PARAM_TENSORS; ++t) {
    const int n = param_numel(t);
    float* p = a.p[t];
    float* g = const_cast<float*>(a.g[t]);
    unsigned f = 0;
    float step_lr = 0.f;
    if (!skip && ((s.adv >> t) & 1u)) {
      const int j = amp.count_in[t] + 1 - s.base[t];
      f = s.flags[t][j];
      step_lr = s.step_lr[t][j];
    }
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
      const float gr = g != nullptr ? amp_unscale(g, e, inv) : 0.f;
      if (skip) continue;
      float w = p[e];
      if (g != nullptr) {
        w = rule_update<RULE>(w, gr, base + e, exp_avg, exp_avg_sq, slow_buffer, s.c, f, step_lr);
        p[e] = w;
      }
      h += param_checksum_term(base + e, __float_as_uint(w));
    }
    base += n;
  }
  if (!skip) stamp_checksum(h, hdr);
}

int optim_step_pack_amp(float* const* params, float* const* grads, float* exp_avg, float* exp_avg_sq,
                        float* slow_buffer, const SnbOptimArgs& o, const SnbAmpStep& amp, int precision,
                        int new_activation, void* packed, cudaStream_t st) {
  AdamPtrs a;
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) { a.p[i] = params[i]; a.g[i] = grads[i]; }
  RuleWindow s = {};
  s.c = rule_consts(o);
  int cached = -1, prev = -1;
  for (int t = 0; t < SNB_N_PARAM_TENSORS; ++t) {
    s.base[t] = amp.base[t];
    if (!rule_advances(o, grads[t])) continue;
    s.adv |= 1u << t;
    rule_window(o, amp.base[t], &cached, s.step_lr[t], s.flags[t], prev < 0 ? nullptr : s.step_lr[prev],
                prev < 0 ? nullptr : s.flags[prev]);
    prev = t;
  }
  PackedHeader* hdr = reinterpret_cast<PackedHeader*>(packed);
  const AmpCtl ctl = amp_ctl(amp);
  const int grid = sm_count() * 2;
  if (o.rule == SNB_OPTIM_SGD)
    optim_step_amp_kernel<SNB_OPTIM_SGD><<<grid, 256, 0, st>>>(a, exp_avg, exp_avg_sq, slow_buffer, s, ctl, hdr);
  else if (o.rule == SNB_OPTIM_RADAM)
    optim_step_amp_kernel<SNB_OPTIM_RADAM><<<grid, 256, 0, st>>>(a, exp_avg, exp_avg_sq, slow_buffer, s, ctl, hdr);
  else
    optim_step_amp_kernel<SNB_OPTIM_RANGER><<<grid, 256, 0, st>>>(a, exp_avg, exp_avg_sq, slow_buffer, s, ctl, hdr);
  if (int rc = check_launch("optim_step_amp_kernel")) return rc;
  return repack_if_dirty(params, precision, new_activation, packed, st);
}

// The table of snb_optim_step_tensors_amp: as TensorTable, with each entry's scalars over its window and the index of
// its count (entries are only the tensors with a gradient; counts cover all n_all tensors).
struct TensorEntryAmp {
  float* p;
  float* g;
  long long n;
  unsigned long long off;
  int slot;                            // index into the count arrays
  int base;
  float step_lr[kOptimWindow];         // Adam: -lr / (1 - beta1^t);  RAdam / Ranger: -step_size * lr
  float inv_bc2_sqrt[kOptimWindow];    // Adam: 1 / sqrt(1 - beta2^t)
  unsigned char flags[kOptimWindow];   // SGD / RAdam / Ranger: kFirst | kAdaptive | kSync
};

struct TensorTableAmp {
  TensorEntryAmp t[SNB_OPTIM_MAX_TENSORS];
  int n;
  int n_all;
  unsigned adv;                        // bit i: tensor i advances its count on a taken step
};

template <int RULE>
__global__ void __launch_bounds__(256) optim_tensors_amp_kernel(TensorTableAmp tab, float* __restrict__ exp_avg,
                                                                float* __restrict__ exp_avg_sq,
                                                                float* __restrict__ slow_buffer, RuleConsts c,
                                                                AmpCtl amp) {
  const bool skip = amp_skip(amp.found_inf);
  const float inv = amp_inv_scale(amp.scale);
  if (blockIdx.x == 0 && threadIdx.x < tab.n_all)
    amp.count_out[threadIdx.x] = amp.count_in[threadIdx.x] + ((!skip && (tab.adv >> threadIdx.x) & 1u) ? 1 : 0);
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (int t = 0; t < tab.n; ++t) {
    float* p = tab.t[t].p;
    float* g = tab.t[t].g;
    const long long n = tab.t[t].n;
    const unsigned long long off = tab.t[t].off;
    float step_lr = 0.f, inv_bc2_sqrt = 0.f;
    unsigned f = 0;
    if (!skip && ((tab.adv >> tab.t[t].slot) & 1u)) {
      const int j = amp.count_in[tab.t[t].slot] + 1 - tab.t[t].base;
      step_lr = tab.t[t].step_lr[j];
      inv_bc2_sqrt = tab.t[t].inv_bc2_sqrt[j];
      f = tab.t[t].flags[j];
    }
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
      const float gr = amp_unscale(g, e, inv);
      if (skip) continue;
      const unsigned long long i = off + e;
      if (RULE == SNB_OPTIM_ADAM) {
        float m = exp_avg[i], v = exp_avg_sq[i];
        p[e] = adam_update(p[e], gr, m, v, step_lr, c.beta1_w, c.beta2, c.beta2_w, c.eps, c.decay, inv_bc2_sqrt);
        exp_avg[i] = m;
        exp_avg_sq[i] = v;
      } else {
        p[e] = rule_update<RULE>(p[e], gr, i, exp_avg, exp_avg_sq, slow_buffer, c, f, step_lr);
      }
    }
  }
}

int optim_step_tensors_amp(int n, float* const* params, float* const* grads, const int64_t* numel, float* exp_avg,
                           float* exp_avg_sq, float* slow_buffer, const SnbOptimArgs& o, const SnbAmpStep& amp,
                           cudaStream_t st) {
  TensorTableAmp tab = {};
  tab.n_all = n;
  unsigned long long off = 0;
  int cached = -1;
  const TensorEntryAmp* prev = nullptr;
  for (int t = 0; t < n; off += (unsigned long long)numel[t], ++t) {
    if (grads[t] == nullptr) continue;
    TensorEntryAmp& te = tab.t[tab.n++];
    te.p = params[t];
    te.g = grads[t];
    te.n = numel[t];
    te.off = off;
    te.slot = t;
    te.base = amp.base[t];
    if (!rule_advances(o, grads[t])) continue;
    tab.adv |= 1u << t;
    if (o.rule == SNB_OPTIM_ADAM) {
      for (int j = 0; j < kOptimWindow; ++j)
        adam_bias_scalars(o.lr, o.beta1, o.beta2, te.base + j, &te.step_lr[j], &te.inv_bc2_sqrt[j]);
    } else {
      rule_window(o, te.base, &cached, te.step_lr, te.flags, prev ? prev->step_lr : nullptr,
                  prev ? prev->flags : nullptr);
      prev = &te;
    }
  }
  const RuleConsts c = rule_consts(o);
  const AmpCtl ctl = amp_ctl(amp);
  const int grid = tab.n == 0 ? 1 : sm_count() * 4;   // with no gradient at all, one block still copies the counts
  if (o.rule == SNB_OPTIM_ADAM)
    optim_tensors_amp_kernel<SNB_OPTIM_ADAM><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  else if (o.rule == SNB_OPTIM_SGD)
    optim_tensors_amp_kernel<SNB_OPTIM_SGD><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  else if (o.rule == SNB_OPTIM_RADAM)
    optim_tensors_amp_kernel<SNB_OPTIM_RADAM><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  else
    optim_tensors_amp_kernel<SNB_OPTIM_RANGER><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  return check_launch("optim_tensors_amp_kernel");
}

}  // namespace snb
