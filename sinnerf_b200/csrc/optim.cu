// optim.cu -- fused optimiser steps (Adam, SGD, RAdam, Ranger) over the 24 parameter tensors of one NeRF + refresh of
// its packed image (SURVEY.md 8f-4), or over a table of plain fp32 tensors.  Reference: get_optimizer ->
// torch.optim.Adam(lr, eps=1e-8, weight_decay) (utils/__init__.py:19-21), stepped once per training iteration by
// Lightning (train.py:51-52 under DDP, i.e. after the gradient all-reduce).
//
// All six entry points launch one walker, step_kernel<RULE>, over a table of tensors.  One launch updates all 595 844
// parameters of a NeRF (torch runs ~10 multi-tensor launches over 24 tensors per model), accumulates the parameter
// checksum the packed image is stamped with (so the next snb_refresh_weights sees a clean image), and is followed on
// the same stream by the two pack kernels (bottleneck fold + chunk image) -- the image the forward streams is ready
// when step() returns, no per-step host-side re-pack decision.
//
// Adam's arithmetic = torch.optim.Adam's single-tensor path (torch/optim/adam.py, amsgrad = False, maximize = False),
// operation for operation, every elementwise op rounded to fp32 like the separate ATen kernels:
//   g   = grad + weight_decay * p                         (add, alpha)
//   m   = m + (1 - beta1) * (g - m)                       (lerp, weight < 0.5)
//   v   = v * beta2;  v = v + (1 - beta2) * (g * g)       (mul_, addcmul_: ATen rounds the product g * g first)
//   den = sqrt(v) / sqrt(1 - beta2^t) + eps               (division by a python float: * (1 / scalar), the reciprocal
//                                                          formed in double and rounded to fp32 once)
//   p   = p + (-lr / (1 - beta1^t)) * (m / den)           (addcdiv_)
// Roofline: HBM/L2, 16 B read + 12 B written per parameter (17 MB per model) -- a few microseconds.
#include "common.cuh"

namespace snb {

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
// the new parameter out.
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

// ---------------------------------------------------------------- SGD / RAdam / Ranger
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

// One element of SGD / RAdam / Ranger (the arithmetic listed above) at flat state index i: reads and writes the state
// buffers the rule keeps and returns the new parameter.
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

// ---------------------------------------------------------------- the walker
// The GradScaler-native forms (snb_*_amp) step as torch's GradScaler drives an optimiser that sets
// _step_supports_amp_scaling: the gradients arrive scaled, with GradScaler's scale and found_inf on the device, and
// the host does not wait for either.
//   * Every gradient element is unscaled as GradScaler.unscale_ does it -- inv = (float)(1 / (double)scale), then
//     g * inv unless inv == 1 (torch's _amp_foreach_non_finite_check_and_unscale_) -- and written back to the
//     gradient, taken step or not, so .grad ends as GradScaler's own unscale leaves it.  __fmul_rn keeps the product
//     out of any FMA, so the update sees the value it would read back from memory.
//   * *found_inf != 0: parameters, state, update counts, checksum and image stay as they are (GradScaler never calls
//     step() then).  The grid reads the same flag, so the branch is uniform.  A skipped step clears header.dirty
//     instead of stamping, so the pack kernels that follow (only_if_dirty) return at once and the image keeps the
//     bytes and checksum it had.  The flag is the pack kernels' scratch: every refresh recomputes it from the checksum
//     before it is read.
//   * The update counts live on the device: the kernel reads count_in and block 0 writes count_out (a second buffer,
//     so no block can see a count advanced under it).  The step-dependent scalars are formed on the host, in doubles,
//     for the kOptimWindow counts base .. base + kOptimWindow - 1 a tensor can have reached, and each entry picks its
//     slot by count_in + 1 - base.  The caller keeps that index in range (SnbAmpStep in the header).
// The plain forms pass no scale, found_inf or counts: the gradients are read as they are, no step is skipped, and
// every entry reads window slot 0, which the host filled for the count it knows.
constexpr int kOptimWindow = SNB_OPTIM_WINDOW;

// One tensor of a launch.  Tensor t's state sits at offset sum(numel[0..t)) of each flat buffer, which is also the
// index its first element has in the NeRF checksum.
struct StepEntry {
  float* p;
  float* g;                              // NULL: no gradient; the entry only adds its values to the checksum
  long long n;
  unsigned long long off;
  int count;                             // index into the count arrays
  int base;                              // the count window slot 0 holds
  float step_lr[kOptimWindow];           // Adam: -lr / (1 - beta1^t);  RAdam / Ranger: -step_size * lr
  union {
    float inv_bc2_sqrt[kOptimWindow];    // Adam: 1 / sqrt(1 - beta2^t)
    unsigned char flags[kOptimWindow];   // SGD / RAdam / Ranger: kFirst | kAdaptive | kSync
  };
};

struct StepTable {
  StepEntry t[SNB_OPTIM_MAX_TENSORS];
  int n;
  int n_counts;
  unsigned adv;                          // bit c: count c advances on a taken step
};

struct StepCtl {
  const float* scale;        // nullable: the gradients carry no scale
  const float* found_inf;    // nullable: never skip
  const int* count_in;       // nullable (with count_out): window slot 0, no counts written
  int* count_out;
  PackedHeader* hdr;         // nullable: no checksum stamp
};

// The unscaled gradient element, written back when the scale changes it.
__device__ __forceinline__ float amp_unscale(float* g, long long e, float inv) {
  float gr = g[e];
  if (inv != 1.f) {
    gr = __fmul_rn(gr, inv);
    g[e] = gr;
  }
  return gr;
}

template <int RULE>
__global__ void __launch_bounds__(256) step_kernel(StepTable tab, float* __restrict__ exp_avg,
                                                   float* __restrict__ exp_avg_sq, float* __restrict__ slow_buffer,
                                                   RuleConsts c, StepCtl ctl) {
  const bool skip = ctl.found_inf != nullptr && *ctl.found_inf != 0.f;
  const float inv = ctl.scale == nullptr ? 1.f : (float)(1.0 / (double)*ctl.scale);
  if (blockIdx.x == 0) {
    if (ctl.count_out != nullptr && threadIdx.x < tab.n_counts)
      ctl.count_out[threadIdx.x] = ctl.count_in[threadIdx.x] + ((!skip && (tab.adv >> threadIdx.x) & 1u) ? 1 : 0);
    if (threadIdx.x == 0 && skip && ctl.hdr != nullptr) ctl.hdr->dirty = 0;
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  unsigned long long h = 0;
  for (int t = 0; t < tab.n; ++t) {
    float* p = tab.t[t].p;
    float* g = tab.t[t].g;
    const long long n = tab.t[t].n;
    const unsigned long long off = tab.t[t].off;
    float step_lr = 0.f, inv_bc2_sqrt = 0.f;
    unsigned f = 0;
    if (g != nullptr && !skip && ((tab.adv >> tab.t[t].count) & 1u)) {
      const int j = ctl.count_in == nullptr ? 0 : ctl.count_in[tab.t[t].count] + 1 - tab.t[t].base;
      step_lr = tab.t[t].step_lr[j];
      if (RULE == SNB_OPTIM_ADAM)
        inv_bc2_sqrt = tab.t[t].inv_bc2_sqrt[j];
      else
        f = tab.t[t].flags[j];
    }
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += stride) {
      const float gr = g != nullptr ? amp_unscale(g, e, inv) : 0.f;
      if (skip) continue;
      const unsigned long long i = off + e;
      float w = p[e];
      if (g != nullptr) {
        if (RULE == SNB_OPTIM_ADAM) {
          float m = exp_avg[i], v = exp_avg_sq[i];
          w = adam_update(w, gr, m, v, step_lr, c.beta1_w, c.beta2, c.beta2_w, c.eps, c.decay, inv_bc2_sqrt);
          exp_avg[i] = m;
          exp_avg_sq[i] = v;
        } else {
          w = rule_update<RULE>(w, gr, i, exp_avg, exp_avg_sq, slow_buffer, c, f, step_lr);
        }
        p[e] = w;
      }
      if (ctl.hdr != nullptr) h += param_checksum_term(i, __float_as_uint(w));
    }
  }
  if (!skip) stamp_checksum(h, ctl.hdr);
}

// ---------------------------------------------------------------- host
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

// Slot j of an entry's window: the scalars of o.rule at update count `step` (including this update), in python
// doubles as the replaced optimiser forms them, cast to float where the kernel consumes them.
//   Adam: -lr / (1 - beta1^t), and 1 / (1 - beta2^t) ** 0.5 with the reciprocal taken in double: a float reciprocal
//     of the float cast rounds twice and differs from torch's by an ulp at most counts (at t = 1: 31.622778 vs
//     31.622776).
//   RAdam / Ranger: utils/optimizers.py:68-86 / :397-411, in the reference's expression order.
static void rule_scalars(const SnbOptimArgs& o, int step, StepEntry& te, int j) {
  if (o.rule == SNB_OPTIM_ADAM) {
    const double bc1 = 1.0 - pow(o.beta1, (double)step);
    const double bc2 = 1.0 - pow(o.beta2, (double)step);
    te.step_lr[j] = (float)(-(o.lr / bc1));
    te.inv_bc2_sqrt[j] = (float)(1.0 / pow(bc2, 0.5));
    return;
  }
  if (o.rule == SNB_OPTIM_SGD) {
    te.step_lr[j] = 0.f;
    te.flags[j] = step == 1 ? kFirst : 0u;
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
  te.step_lr[j] = (float)(-step_size * o.lr);
  te.flags[j] = (adaptive ? kAdaptive : 0u) | (step == 1 ? kFirst : 0u) |
                (o.rule == SNB_OPTIM_RANGER && step % o.k == 0 ? kSync : 0u);
}

// Slots 0 .. width - 1 of te's window.  Entries at the same base (all of them, unless some lacked a gradient on some
// steps) share the host arithmetic: `prev` is the last entry filled.
static void fill_window(const SnbOptimArgs& o, int width, StepEntry& te, const StepEntry* prev) {
  if (prev != nullptr && prev->base == te.base) {
    for (int j = 0; j < kOptimWindow; ++j) {
      te.step_lr[j] = prev->step_lr[j];
      te.inv_bc2_sqrt[j] = prev->inv_bc2_sqrt[j];
    }
    return;
  }
  for (int j = 0; j < width; ++j) rule_scalars(o, te.base + j, te, j);
}

// Whether tensor t's count advances on a taken step: it has a gradient, and the rule keeps a count (SGD only with
// momentum, where the count says whether the momentum buffer exists yet).
static bool rule_advances(const SnbOptimArgs& o, const void* grad) {
  return grad != nullptr && (o.rule != SNB_OPTIM_SGD || o.momentum != 0.);
}

// The body of the six snb_*step* entry points, after their argument checks: one step of o.rule over n tensors.
//   numel: per tensor, or NULL for the NeRF's 24 parameter tensors (grid 2 x SMs instead of 4 x SMs).
//   one_count: every tensor steps by count 0, which every taken step advances (snb_adam_step*); otherwise tensor t
//     steps by count t, which advances where rule_advances says.
//   base: per count, the count of window slot 0: the plain forms' own count, or SnbAmpStep.base.
//   amp: NULL for the plain forms.  packed: the NeRF image to stamp and re-pack, or NULL.
int fused_step(int n, const int64_t* numel, float* const* params, const float* const* grads, bool one_count,
               const int* base, const SnbAmpStep* amp, float* exp_avg, float* exp_avg_sq, float* slow_buffer,
               const SnbOptimArgs& o, int precision, int new_activation, void* packed, cudaStream_t st) {
  PackedHeader* hdr = reinterpret_cast<PackedHeader*>(packed);
  const int width = amp != nullptr ? kOptimWindow : 1;
  StepTable tab = {};
  tab.n_counts = one_count ? 1 : n;
  tab.adv = one_count ? 1u : 0u;
  const StepEntry* prev = nullptr;
  unsigned long long off = 0;
  for (int t = 0; t < n; off += (unsigned long long)(numel ? numel[t] : param_numel(t)), ++t) {
    // Without a checksum to stamp, a tensor without a gradient has nothing to do.
    if (grads[t] == nullptr && hdr == nullptr) continue;
    StepEntry& te = tab.t[tab.n++];
    te.p = params[t];
    te.g = const_cast<float*>(grads[t]);   // written only when amp gives a scale
    te.n = numel ? numel[t] : param_numel(t);
    te.off = off;
    te.count = one_count ? 0 : t;
    te.base = base[te.count];
    if (!one_count && rule_advances(o, grads[t])) tab.adv |= 1u << t;
    if (grads[t] == nullptr || !((tab.adv >> te.count) & 1u)) continue;
    fill_window(o, width, te, prev);
    prev = &te;
  }
  if (tab.n == 0 && amp == nullptr) return SNB_OK;
  const RuleConsts c = rule_consts(o);
  const StepCtl ctl = amp != nullptr ? StepCtl{amp->scale, amp->found_inf, amp->count_in, amp->count_out, hdr}
                                     : StepCtl{nullptr, nullptr, nullptr, nullptr, hdr};
  // With no tensor to step, one block still copies the counts.
  const int grid = tab.n == 0 ? 1 : sm_count() * (numel ? 4 : 2);
  if (o.rule == SNB_OPTIM_ADAM)
    step_kernel<SNB_OPTIM_ADAM><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  else if (o.rule == SNB_OPTIM_SGD)
    step_kernel<SNB_OPTIM_SGD><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  else if (o.rule == SNB_OPTIM_RADAM)
    step_kernel<SNB_OPTIM_RADAM><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  else
    step_kernel<SNB_OPTIM_RANGER><<<grid, 256, 0, st>>>(tab, exp_avg, exp_avg_sq, slow_buffer, c, ctl);
  if (int rc = check_launch("step_kernel")) return rc;
  // The image the forward streams, re-packed on the step's stream from the updated parameters.  A taken step set
  // header.dirty; a skipped one cleared it.
  if (packed == nullptr) return SNB_OK;
  const float* cp[SNB_N_PARAM_TENSORS];
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) cp[i] = params[i];
  if (precision == SNB_PREC_FP32) return launch_pack_fp32(cp, new_activation ? 1 : 0, packed, 1, st);
  return launch_pack_tc(cp, precision, new_activation ? 1 : 0, packed, 1, st);
}

}  // namespace snb
