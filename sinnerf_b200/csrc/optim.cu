// optim.cu -- fused Adam step over the 24 parameter tensors of one NeRF + refresh of its packed image
// (SURVEY.md 8f-4).  Reference: get_optimizer -> torch.optim.Adam(lr, eps=1e-8, weight_decay)
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
//   v   = v * beta2;  v = v + (1 - beta2) * g * g         (mul_, addcmul_)
//   den = sqrt(v) / sqrt(1 - beta2^t) + eps               (ATen divides by a CPU scalar as * (1 / scalar))
//   p   = p + (-lr / (1 - beta1^t)) * (m / den)           (addcdiv_)
// Roofline: HBM/L2, 16 B read + 12 B written per parameter (17 MB per model) -- a few microseconds.
#include "common.cuh"

namespace snb {

struct AdamPtrs {
  float* p[SNB_N_PARAM_TENSORS];
  const float* g[SNB_N_PARAM_TENSORS];   // nullable per tensor: no gradient -> tensor skipped (as torch does)
};

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
        float gr = g[e];
        if (weight_decay != 0.f) gr = fmaf(weight_decay, w, gr);
        float m = exp_avg[base + e], v = exp_avg_sq[base + e];
        m = fmaf(beta1_w, gr - m, m);
        v = __fmul_rn(v, beta2);
        v = fmaf(__fmul_rn(beta2_w, gr), gr, v);
        const float den = __fadd_rn(__fmul_rn(__fsqrt_rn(v), inv_bc2_sqrt), eps);
        w = fmaf(lr_neg_step, __fdiv_rn(m, den), w);
        exp_avg[base + e] = m;
        exp_avg_sq[base + e] = v;
        p[e] = w;
      }
      h += param_checksum_term(base + e, __float_as_uint(w));
    }
    base += n;
  }
  if (hdr == nullptr) return;
  // stamp the image header with the checksum of the NEW values (same sum params_check_kernel computes)
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

int adam_step_pack(float* const* params, const float* const* grads, float* exp_avg, float* exp_avg_sq,
                   const SnbAdamArgs& o, int precision, int new_activation, void* packed, cudaStream_t st) {
  AdamPtrs a;
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) { a.p[i] = params[i]; a.g[i] = grads[i]; }
  // scalars exactly as torch forms them: python doubles, cast to float where the kernels consume them
  const double bc1 = 1.0 - pow(o.beta1, (double)o.step);
  const double bc2 = 1.0 - pow(o.beta2, (double)o.step);
  const float lr_neg_step = (float)(-(o.lr / bc1));
  const float inv_bc2_sqrt = 1.0f / (float)sqrt(bc2);
  const float beta1_w = (float)(1.0 - o.beta1), beta2_w = (float)(1.0 - o.beta2);
  adam_step_kernel<<<sm_count() * 2, 256, 0, st>>>(a, exp_avg, exp_avg_sq, lr_neg_step, beta1_w, (float)o.beta2, beta2_w,
                                                  (float)o.eps, (float)o.weight_decay, inv_bc2_sqrt, precision, new_activation,
                                                  reinterpret_cast<PackedHeader*>(packed));
  if (int rc = check_launch("adam_step_kernel")) return rc;
  if (packed == nullptr) return SNB_OK;
  const float* cp[SNB_N_PARAM_TENSORS];
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) cp[i] = params[i];
  if (precision == SNB_PREC_FP32) return launch_pack_fp32(cp, new_activation ? 1 : 0, packed, 0, st);
  return launch_pack_tc(cp, precision, new_activation ? 1 : 0, packed, 0, st);
}

}  // namespace snb
