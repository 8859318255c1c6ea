/* sinnerf_b200.h -- C ABI of libsinnerf_b200.so
 *
 * Drop-in boundary for the SinNeRF volumetric-rendering hot path.  The reference
 * (VITA-Group/SinNeRF @ bf147e4) is pure Python/PyTorch and has no FFI of its own; the
 * "operator interface" this library sits behind is
 *     models/rendering.py:126-139   render_rays(models, embeddings, rays, ...)
 *     models/rendering.py:15-61     sample_pdf(bins, weights, N_importance, det, eps)
 *     models/nerf.py:24-41          Embedding.forward
 *     models/nerf.py:105-148        NeRF.forward(x, sigma_only)
 * Each entry point below names the reference lines it replaces.  The Python mirror of
 * that interface (sinnerf_b200/rendering.py, sinnerf_b200/nerf.py) binds these symbols
 * with ctypes; INTEGRATION.md shows the two import lines a maintainer changes.
 *
 * Conventions
 *  - every pointer is a DEVICE pointer to caller-owned memory unless marked "host";
 *    the library never allocates, frees or retains device memory;
 *  - tensors are dense row-major fp32 unless a stride argument is given;
 *  - `stream` is a cudaStream_t / CUstream passed as void*; all work is enqueued on it,
 *    nothing synchronises the host;
 *  - functions return SNB_OK (0) or a negative SNB_ERR_* code; snb_last_error() returns
 *    a thread-local message for the last failing call on this thread;
 *  - the library is sm_90a (H100) only; snb_device_check() reports anything else as an error.
 */
#ifndef SINNERF_B200_H
#define SINNERF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SNB_VERSION 100 /* 0.1.0 */

#define SNB_OK 0
#define SNB_ERR_INVALID (-1)     /* bad argument (shape, null pointer, alignment)       */
#define SNB_ERR_CUDA (-2)        /* a CUDA runtime call or launch failed                */
#define SNB_ERR_UNSUPPORTED (-3) /* architecture / field shape / precision not built    */

/* Arithmetic used for the field MLP (every other stage is always fp32).
 *  FP32     : FFMA on CUDA cores, fp32 accumulate            -- exact-fp32 mode
 *  F16X3    : wgmma f16, operands split hi+lo (fp16), 3 products, fp32 accumulate
 *             in registers -- meets the <=1e-4 fp32 parity bar on tensor cores
 *  BF16X3   : same with bf16 halves (wider range, ~2e-5)
 *  BF16     : single-pass bf16 operands, fp32 accumulate (BASELINE.json configs[2])
 *  F16      : fp16 operands, one product, fp32 accumulate: the reference under `precision=16`
 *             (Lightning's native AMP: nn.Linear in fp16, everything else fp32); operands
 *             saturate at +-65504
 */
#define SNB_PREC_FP32 0
#define SNB_PREC_F16X3 1
#define SNB_PREC_BF16X3 2
#define SNB_PREC_BF16 3
#define SNB_PREC_F16 4

/* Field MLP shape: NeRF(D=8, W=256, in_channels_xyz=63, in_channels_dir=27, skips=[4])
 * (models/nerf.py:47-50), the only shape SinNeRF instantiates (models/sinnerf.py:137,140).
 * Parameter pointer order for snb_pack_weights = the module's state_dict order:
 *   xyz_encoding_{1..8}.0.{weight,bias}, xyz_encoding_final.{weight,bias},
 *   dir_encoding.0.{weight,bias}, sigma.{weight,bias}, rgb.0.{weight,bias}    (24 tensors)
 * weights are nn.Linear layout (out, in) row-major fp32. */
#define SNB_N_PARAM_TENSORS 24
#define SNB_XYZ_FREQS 10
#define SNB_DIR_FREQS 4
#define SNB_XYZ_CH 63
#define SNB_DIR_CH 27

int snb_version(void);
const char* snb_last_error(void);
/* SNB_OK iff the current CUDA device is compute capability 10.x; fills SM count. */
int snb_device_check(int* sm_count, int* cc_major, int* cc_minor);

/* ---- weights --------------------------------------------------------------------- */
/* Bytes of the packed weight image for a precision mode (device buffer the caller owns). */
size_t snb_packed_weights_bytes(int precision);
/* Re-layout the 24 nn.Linear tensors into the image the field kernels stream
 * (K-major, padded 63->64 / 27->32, skip and dir concatenations split; hi/lo halves for
 * the split modes).  `params` is a HOST array of 24 device pointers.
 * new_activation: 1 = ShiftedSoftplus/WidenedSigmoid (models/activations.py:8-35),
 *                 0 = ReLU/Sigmoid (models/nerf.py:92-103); stored in the image header. */
int snb_pack_weights(const float* const* params, int precision, int new_activation, void* packed,
                     void* stream);
/* Same, but packs only if `packed` does not already hold an image of exactly these parameter VALUES in this
 * mode: a check kernel recomputes a 64-bit checksum of the 24 tensors on the device and compares it with
 * the one in the image header; the pack kernels return at once when it matches.  No host synchronisation.
 * This is what NeRF.packed_weights() calls before every pass: optimizers that update weights through
 * `p.data` (reference utils/optimizers.py:98,104,180,187,268: RAdam / PlainRAdam / AdamW / Ranger) do not
 * bump autograd's version counter, so no host-side key can tell that the image is stale.
 * `packed` must start out zero-filled (or hold an earlier image). */
int snb_refresh_weights(const float* const* params, int precision, int new_activation, void* packed,
                        void* stream);

/* ---- stages (each maps to one oracle function) ------------------------------------- */

/* models/rendering.py:264-282.  rays (N,8) [o,d,near,far]; z_steps (S,) = torch.linspace(0,1,S);
 * perturb_u (N,S) U[0,1) or NULL when perturb == 0.  -> z_vals (N,S). */
int snb_sample_coarse(const float* rays, const float* z_steps, const float* perturb_u, float perturb,
                      int use_disp, int64_t n_rays, int n_samples, float* z_vals, void* stream);

/* Embedding.forward, models/nerf.py:24-41 (logscale bands 2^k).  x (B,C) -> out (B, C*(2L+1)). */
int snb_embed(const float* x, int64_t n, int in_channels, int n_freqs, float* out, void* stream);

/* NeRF.forward, models/nerf.py:105-148, on already-embedded rows.
 * x (P, 63+27) (or (P,63) with row stride x_stride when sigma_only) -> out (P,4) [r,g,b,sigma]
 * or (P,1). */
int snb_mlp_forward(const void* packed, int precision, const float* x, int64_t x_stride, int64_t n_points,
                    int sigma_only, float* out, void* stream);

/* The fused field pass, models/rendering.py:184-212 + :284-285: points o+d*z, xyz and dir
 * embeddings, MLP -- no (P,63)/(P,27)/(P,256) tensor ever reaches HBM.
 * -> raw (N,S,4), or sigma (N,S) when sigma_only. */
int snb_field_forward(const void* packed, int precision, const float* rays, const float* z_vals,
                      int64_t n_rays, int n_samples, int sigma_only, float* raw, void* stream);

/* models/rendering.py:215-248.  raw (N,S,4) (raw_channels=4) or sigma (N,S) (raw_channels=1);
 * noise (N,S) standard-normal draws or NULL (treated as 0; the reference scales by noise_std).
 * rgb (N,3) / depth (N,) may be NULL with raw_channels==1 (weights_only branch :237-238). */
int snb_composite_forward(const float* raw, int raw_channels, const float* z_vals, const float* rays,
                          const float* noise, float noise_std, int white_back, int64_t n_rays,
                          int n_samples, float* rgb, float* depth, float* weights, void* stream);

/* Pixel scatter (multi-GPU inference, SURVEY.md 8e "optional fusion"; the reference has no multi-GPU inference,
 * eval.py:141-142 -- this replaces the all-gather of rendered pixels that sharding its ray-chunk loop eval.py:92-115
 * over GPUs needs).  The compositing kernel also stores every ray's [r, g, b, depth] as ONE 16-byte row into up to
 * SNB_MAX_PIXEL_DST frame buffers at row (row_offset + ray): buffers of peer GPUs mapped into this process (NVLink
 * P2P / CUDA symmetric memory) or a single NVSwitch multicast address that reaches all of them -- the collective
 * happens in the kernel's epilogue, no staging copy, no collective kernel.  Visibility on the peers is the caller's
 * (a cross-device barrier after the kernel; sinnerf_b200/distributed.py: PeerPixels). */
#define SNB_MAX_PIXEL_DST 8
typedef struct SnbPixelScatter {
  void* dst[SNB_MAX_PIXEL_DST];  /* (rows,4) fp32 frame buffers, 16-byte aligned device-accessible addresses */
  int n_dst;                     /* 1..SNB_MAX_PIXEL_DST                                                       */
  int64_t row_offset;            /* row of this call's ray 0                                                   */
} SnbPixelScatter;
/* snb_composite_forward (raw_channels = 4) + the scatter above. */
int snb_composite_forward_scatter(const float* raw, const float* z_vals, const float* rays, const float* noise,
                                  float noise_std, int white_back, int64_t n_rays, int n_samples, float* rgb,
                                  float* depth, float* weights, const SnbPixelScatter* scatter, void* stream);

/* sample_pdf, models/rendering.py:15-61.  bins (N,M+1) row stride bins_stride; weights (N,M) row
 * stride w_stride; u: det -> (n_importance,) = torch.linspace(0,1,n_importance) with u_stride 0,
 * else (N,n_importance) with u_stride n_importance.  -> samples (N,n_importance). */
int snb_sample_pdf(const float* bins, int64_t bins_stride, const float* weights, int64_t w_stride,
                   const float* u, int64_t u_stride, int64_t n_rays, int m, int n_importance, float eps,
                   float* samples, void* stream);

/* models/rendering.py:310-315 in one kernel: z_mid, sample_pdf over weights[:,1:-1], then the
 * sorted union with the coarse depths.  -> z_fine (N,S+Ni); z_new (N,Ni) optional (may be NULL). */
int snb_importance_merge(const float* z_coarse, const float* weights_coarse, const float* u,
                         int64_t u_stride, int64_t n_rays, int n_samples, int n_importance, float eps,
                         float* z_fine, float* z_new, void* stream);

/* ---- ray generation (the step before the path; SURVEY.md 8f-1) ------------------------ */
/* Pinhole-camera rays of a strided pixel window, written directly in the (N,8) layout:
 * get_ray_directions (datasets/ray_utils.py:73-91; opencv=0: d = [(i-cx)/fx, -(j-cy)/fy, -1]) or
 * get_ray_directions_dtu (datasets/dtu_proj.py:17-34; opencv=1: d = [(i-cx)/fx, (j-cy)/fy, 1]),
 * get_rays (datasets/ray_utils.py:94-120: d @ c2w[:, :3].T, o = c2w[:, 3]) and the [o, d, near, far]
 * concatenation.  c2w: HOST pointer to 12 floats, row-major (3,4).  Pixel (row0 + r*stride,
 * col0 + c*stride) -> ray r*cols + c.  rays: device (rows*cols, 8), 16-byte aligned. */
int snb_generate_rays(const float* c2w, float fx, float fy, float cx, float cy, float near, float far, int opencv,
                      int row0, int col0, int rows, int cols, int stride, float* rays, void* stream);

/* ---- training: forward that keeps activations, and the backward ------------------------ */

/* The fused field pass of snb_field_forward (same `packed` image / `precision` pairing), additionally
 * keeping what the backward needs (the reference keeps the same tensors inside autograd): the two
 * embeddings and every ReLU / direction layer's post-activation output, as plain row-major fp32
 * tensors.  P = n_rays * n_samples.  The activation-free bottleneck (nerf.py:140) is not kept: the
 * backward differentiates through the folded product Wd[:, :256] Wf instead.
 *   save_enc (P,64)  save_dir (P,32)  save_h (8,P,256) [h1..h8]  save_g (P,128) */
int snb_field_forward_train(const void* packed, int precision, const float* rays, const float* z_vals,
                            int64_t n_rays, int n_samples, float* raw, float* save_enc, float* save_dir,
                            float* save_h, float* save_g, void* stream);

/* Backward of models/rendering.py:215-248 (closed form, SURVEY.md 8a-7).  g_rgb (N,3), g_depth (N,),
 * g_weights (N,S) are dL/d(outputs), any may be NULL (= 0).  -> g_raw (N,S,4) = dL/d[rgb, sigma]. */
int snb_composite_backward(const float* raw, const float* z_vals, const float* rays, const float* noise,
                           float noise_std, int white_back, const float* g_rgb, const float* g_depth,
                           const float* g_weights, int64_t n_rays, int n_samples, float* g_raw, void* stream);

/* ---- training with 16-bit activation storage (round 2) ------------------------------------------------
 * Same mathematics as snb_field_forward_train / snb_field_backward, but everything the backward streams
 * per point is stored once, as fp16, in the layout the tensor-core kernels consume directly (32-point tiles
 * of 16-byte cells, sinnerf_b200/csrc/act16.cuh): 4.5 KB of saved activations per point instead of 8.9 KB,
 * ~2.5 KB of HBM traffic per point and 256-wide layer in the backward instead of ~5 KB, no conversion /
 * transposition warps.  Gradients between layers are fp16 x a per-tensor power-of-two scale the kernels
 * choose on the device from a rigorous growth bound (nothing overflows, no host synchronisation); the
 * parameter gradients are accumulated in fp32.  Tensor-core precision modes only.
 *   act16     : one device buffer of snb_act16_bytes(P) bytes, 256-byte aligned (opaque; forward -> backward)
 *   workspace : one device buffer of snb_bwd16_workspace_bytes(P) bytes, 256-byte aligned
 *   g_amax    : device word holding the bit pattern of max |g_raw| as snb_composite_backward_loss leaves it,
 *               or NULL (the library then reduces g_raw itself)                                              */
size_t snb_act16_bytes(int64_t n_points);
size_t snb_bwd16_workspace_bytes(int64_t n_points);
int snb_field_forward_train16(const void* packed, int precision, const float* rays, const float* z_vals,
                              int64_t n_rays, int n_samples, float* raw, void* act16, void* stream);
int snb_field_backward16(const float* const* params, float* const* grads, int new_activation, const float* g_raw,
                         const float* raw, const void* act16, int64_t n_points, void* workspace,
                         const float* g_amax, void* stream);

/* ---- per-ray losses folded into the compositing (SURVEY.md 8f-3) ------------------------------------
 * The two losses SinNeRF puts directly on render_rays' outputs (models/sinnerf.py:310-319):
 *   MSELoss  (losses.py:12-22, nn.MSELoss 'mean' on rgb_coarse / rgb_fine)
 *   SL1Loss  (models/sinnerf.py:32-42, nn.SmoothL1Loss 'mean', beta = 1, on depth_coarse / depth_fine)
 * as weighted per-ray sums, so several ray sets with their own normalisation can share one pass:
 *   loss[0] = sum_ray rgb_weight[ray]   * sum_c (rgb[ray][c] - target_rgb[ray][c])^2     (1/(3N): 'mean')
 *   loss[1] = sum_ray depth_weight[ray] * smooth_l1(depth[ray] - target_depth[ray])       (1/N: 'mean')
 * A NULL target drops that term; NULL per-ray weights mean the scalar *_weight0 for every ray. */
typedef struct SnbLossSpec {
  const float* target_rgb;    /* (N,3) or NULL */
  const float* target_depth;  /* (N,)  or NULL */
  const float* rgb_weight;    /* (N,)  or NULL */
  const float* depth_weight;  /* (N,)  or NULL */
  float rgb_weight0, depth_weight0;
} SnbLossSpec;
/* floats of zero-initialised scratch for the deterministic loss reduction (reusable across calls on one stream) */
#define SNB_LOSS_WS_FLOATS 4096
/* snb_composite_forward with raw_channels = 4 that also writes loss (2,) = [loss[0], loss[1]] above. */
int snb_composite_forward_loss(const float* raw, const float* z_vals, const float* rays, const float* noise,
                               float noise_std, int white_back, int64_t n_rays, int n_samples,
                               const SnbLossSpec* loss, float* rgb, float* depth, float* weights, float* loss_out,
                               float* loss_ws, void* stream);
/* snb_composite_backward where dL/d(rgb, depth) = the given g_rgb / g_depth (either may be NULL) PLUS the
 * derivative of g_loss[0] loss[0] + g_loss[1] loss[1] (g_loss: device (2,), NULL = ones; `loss` may be NULL),
 * formed per ray in registers from the forward's rgb / depth outputs -- no (N,3)/(N,) gradient tensors and
 * no elementwise loss kernels.  g_amax (nullable): one 32-bit word, atomically raised to the bit pattern of
 * max |g_raw| (zero it first) -- the scale statistic of the 16-bit field backward. */
int snb_composite_backward_loss(const float* raw, const float* z_vals, const float* rays, const float* noise,
                                float noise_std, int white_back, const float* g_rgb, const float* g_depth,
                                const float* g_weights, const SnbLossSpec* loss, const float* rgb, const float* depth,
                                const float* g_loss, int64_t n_rays, int n_samples, float* g_raw, float* g_amax,
                                void* stream);

/* Backward of NeRF.forward (autograd through models/nerf.py:105-148) for one field pass.
 * params / grads: HOST arrays of 24 device pointers in state-dict order; grads are ACCUMULATED into
 * (zero them first).  Scratch: ws_a, ws_b (P,256), ws_s (P,128), ws_w (SNB_BWD_WS_FLOATS floats),
 * ws_m (P,8) 32-bit words (ReLU masks as bit rows, 16-byte aligned).  No gradient reaches rays or z. */
#define SNB_BWD_WS_FLOATS (2 * 128 * 256 + 128)
int snb_field_backward(const float* const* params, float* const* grads, int new_activation,
                       const float* g_raw, const float* raw, const float* save_enc, const float* save_dir,
                       const float* save_h, const float* save_g, int64_t n_points, float* ws_a, float* ws_b,
                       float* ws_s, float* ws_w, uint32_t* ws_m, void* stream);

/* ---- sigma-only training passes ----------------------------------------------------------------------
 * The field pass of render_rays(test_time=True)'s coarse model (models/rendering.py:287-292, weights_only=True)
 * and of eval_points (models/rendering.py:64-123) under autograd: layers 1-8 and the sigma head, no direction
 * layer, no rgb head (models/nerf.py:105-136 with sigma_only=True).
 *
 * snb_field_forward_train_sigma / snb_field_forward_train16_sigma: the sigma-only field pass keeping what the
 * sigma-only backward reads; sigma (N,S) = (P,).  The fp32-storage form keeps save_enc (P,64) and
 * save_h (8,P,256) as snb_field_forward_train does; the 16-bit form fills the enc, h1..h8 and ReLU-mask
 * sections of an snb_act16_bytes(P) buffer (the direction sections are left unwritten). */
int snb_field_forward_train_sigma(const void* packed, int precision, const float* rays, const float* z_vals,
                                  int64_t n_rays, int n_samples, float* sigma, float* save_enc, float* save_h,
                                  void* stream);
int snb_field_forward_train16_sigma(const void* packed, int precision, const float* rays, const float* z_vals,
                                    int64_t n_rays, int n_samples, float* sigma, void* act16, void* stream);
/* Backward of models/rendering.py:215-238 with weights_only (closed form, SURVEY.md 8a-7 with g_rgb = g_depth = 0):
 * g_weights (N,S) -> g_sigma (N,S).  sigma: what the sigma-only forward wrote.  g_amax (nullable): as in
 * snb_composite_backward_loss, raised to the bit pattern of max |g_sigma| (zero it first). */
int snb_composite_backward_weights(const float* sigma, const float* z_vals, const float* rays, const float* noise,
                                   float noise_std, const float* g_weights, int64_t n_rays, int n_samples,
                                   float* g_sigma, float* g_amax, void* stream);
/* Backward of a sigma-only field pass (autograd through models/nerf.py:105-136): g_sigma (P,) -> gradients of
 * xyz_encoding_1..8 and sigma (grads 0..15, 20, 21, ACCUMULATED into).  The entries for xyz_encoding_final,
 * dir_encoding and rgb (16..19, 22, 23) are neither read nor written and may be NULL in both arrays.
 * fp32 storage: scratch ws_a, ws_b (P,256) fp32 and ws_m (P,8) 32-bit words, all 16-byte aligned.
 * 16-bit storage: workspace of snb_bwd16_workspace_bytes(P) bytes; g_amax as snb_composite_backward_weights
 * leaves it, or NULL (the library then reduces g_sigma itself). */
int snb_field_backward_sigma(const float* const* params, float* const* grads, const float* g_sigma,
                             const float* save_enc, const float* save_h, int64_t n_points, float* ws_a, float* ws_b,
                             uint32_t* ws_m, void* stream);
int snb_field_backward16_sigma(const float* const* params, float* const* grads, const float* g_sigma,
                               const void* act16, int64_t n_points, void* workspace, const float* g_amax,
                               void* stream);

/* ---- image-space patch losses on render_rays' outputs ------------------------------------------------
 * The two kornia 0.6.3 losses the training step puts on (B,C,H,W) patches of rendered pixels:
 *   inverse_depth_smoothness_loss  models/sinnerf.py:370-373, :395-398 (kornia.losses, imported at :23)
 *   ssim_loss, window_size 11      losses.py:105 (kornia.losses, imported at :2)
 * Every tensor argument comes with `*_strides`: a HOST array of four int64 ELEMENT strides (N, C, H, W), so
 * permuted views such as '(b p q) c -> b c p q' of a ray-major (N,3) output are read in place, and gradients are
 * written with whatever strides the caller chose.  Losses are fp32 scalars; their means use the deterministic
 * reduction of snb_composite_forward_loss on the same zero-initialised SNB_LOSS_WS_FLOATS scratch.  The backwards
 * read the upstream gradient g_loss (device, one float) on the device and use no atomics: the result is the same
 * bits on every run, and scaling g_loss scales every gradient exactly. */

/* inverse_depth_smoothness_loss(idepth (B,1,H,W), image (B,C,H,W)), H, W >= 2:
 *   mean |dx(idepth) exp(-mean_c |dx(image)|)| + mean |dy(idepth) exp(-mean_c |dy(image)|)|,
 *   dx(t) = t[..., :, :-1] - t[..., :, 1:], dy likewise along H.  -> loss (1 float) */
int snb_depth_smooth_forward(const float* idepth, const int64_t* idepth_strides, const float* image,
                             const int64_t* image_strides, int64_t batch, int channels, int height, int width,
                             float* loss, float* loss_ws, void* stream);
/* Its backward: g_idepth (B,1,H,W) and g_image (B,C,H,W) = g_loss * dloss/d(input); either may be NULL (not formed,
 * its strides may then be NULL too).  |.| differentiates as torch.abs, with sign(0) = 0. */
int snb_depth_smooth_backward(const float* idepth, const int64_t* idepth_strides, const float* image,
                              const int64_t* image_strides, int64_t batch, int channels, int height, int width,
                              const float* g_loss, float* g_idepth, const int64_t* g_idepth_strides, float* g_image,
                              const int64_t* g_image_strides, void* stream);

/* ssim_loss(img1, img2, window_size, max_val, eps, reduction='mean') on (B,C,H,W) images, H, W >= 6: reflect padding
 * of 5, depthwise correlation with the 11x11 Gaussian window (sigma 1.5) of img1, img2, img1^2, img2^2, img1 img2, and
 * mean clamp((1 - ssim) / 2, 0, 1), C1 = (0.01 max_val)^2, C2 = (0.03 max_val)^2.  window_size other than 11:
 * SNB_ERR_UNSUPPORTED.  The window sums and the SSIM expression are evaluated in fp64 (see DESIGN.md section 4).
 * coef: NULL (no backward), or a device buffer of 3 B C H W doubles the forward fills with the per-pixel
 * coefficient maps snb_ssim_loss_backward reads.  -> loss (1 float) */
int snb_ssim_loss_forward(const float* img1, const int64_t* img1_strides, const float* img2,
                          const int64_t* img2_strides, int64_t batch, int channels, int height, int width,
                          int window_size, float max_val, float eps, float* loss, double* coef, float* loss_ws,
                          void* stream);
/* Its backward with respect to img1 only (the reference's img2 is always a target):
 * g_img1 (B,C,H,W) = g_loss * dloss/dimg1, from the coef maps of the forward on the same img1, img2. */
int snb_ssim_loss_backward(const float* img1, const int64_t* img1_strides, const float* img2,
                           const int64_t* img2_strides, int64_t batch, int channels, int height, int width,
                           const double* coef, const float* g_loss, float* g_img1, const int64_t* g_img1_strides,
                           void* stream);

/* ---- forward warp: the datasets' depth-warped pseudo-view labels --------------------------------------
 * The reference view splatted into P source views through its depth, as the datasets build their geometry
 * pseudo-labels:
 *   SNB_WARP_ZBUFFER  painter's algorithm, nearest depth wins: datasets/llff_ray_patch_1image_proj.py:144-166,
 *                     datasets/dtu_proj.py:236-273
 *   SNB_WARP_LAST     numpy scatter, the last source in raster order wins: datasets/blender_ray_patch_1image_rot3d.py
 *                     :130-150, datasets/blender_ray_patch_1image_proj.py:120-138 (whose depth_mask is `hit`)
 * image (H,W,3) and depth (H,W): the reference view, fp32.  mats: P row-major 3x4 fp64 matrices, the top three rows of
 * src_proj @ inv(ref_proj) (sinnerf_b200.warp composes them as I + (src_proj - ref_proj) inv(ref_proj)) for full
 * 4x4 projections [[K,0],[0,1]] @ E.  Source pixel (r, c) with d = depth[r,c] goes
 * to X = ((M00 (c d) + M01 (r d)) + M02 d) + M03 (Y, Z alike), every product and sum rounded on its own (no FMA),
 * x' = X / Z, y' = Y / Z in fp64 (divided by 1e-9 where Z == 0); target (clamp(floor(y'), 0, H-1), clamp(floor(x'), 0, W-1)),
 * depth zf = (float)Z.  A source with a non-finite d or a NaN coordinate is skipped.  The occlusion rule and why it
 * equals the painter loop: DESIGN.md section 4.4.  Outputs (P,H,W,3) rgb, (P,H,W) depth, (P,H,W) hit (bytes 0 / 1);
 * a pixel nothing landed on is 0.  The result is the same bits on every run.  H*W < 2^31.  workspace: a device
 * buffer of snb_forward_warp_workspace_bytes(P, H, W, occlusion) bytes, any content (the call initialises it). */
#define SNB_WARP_ZBUFFER 0
#define SNB_WARP_LAST 1
size_t snb_forward_warp_workspace_bytes(int64_t n_poses, int height, int width, int occlusion);
int snb_forward_warp(const float* image, const float* depth, int height, int width, const double* mats,
                     int64_t n_poses, int occlusion, float* out_rgb, float* out_depth, uint8_t* out_hit,
                     void* workspace, void* stream);

/* ---- semantic loss: DINO ViT-S/16 CLS feature -------------------------------------------------------
 * models/sinnerf.py:162-169 get_vit_feature(x): F.interpolate(x, (224, 224)) (nearest), (x - mean) / std with the
 * ImageNet constants, DINO vit_small/16 (12 pre-norm blocks, width 384, 6 heads of 64, MLP 1536 with exact GELU,
 * LayerNorm eps 1e-6), and the output of block 11 (before the final norm) at token 0 of image 0.
 * params: HOST array of SNB_VIT_N_TENSORS device pointers to the fp32 tensors of DINO's state dict in its order,
 * without the final norm: cls_token, pos_embed, patch_embed.proj.{weight,bias}, then for each of the 12 blocks
 * norm1.{weight,bias}, attn.qkv.{weight,bias}, attn.proj.{weight,bias}, norm2.{weight,bias}, mlp.fc1.{weight,bias},
 * mlp.fc2.{weight,bias}.  snb_vit_pack copies them into `image` (snb_vit_pack_bytes(precision) bytes): fp32 vectors
 * and the GEMM weights as fp16 hi + lo planes (SNB_PREC_FP32, _F16X3, _BF16X3: three products per GEMM) or one
 * fp16 (SNB_PREC_F16) or bf16 (SNB_PREC_BF16) plane.  Forward and backward must be called with the precision the
 * image was packed in.  Every GEMM runs on wgmma; LayerNorm, softmax, GELU and the residual stream are fp32. */
#define SNB_VIT_N_TENSORS 148
#define SNB_VIT_DIM 384
#define SNB_VIT_MAX_IMAGES 8
size_t snb_vit_pack_bytes(int precision);
int snb_vit_pack(const float* const* params, int precision, void* image, void* stream);
/* device workspace of a pass over n_images images; save = 1 keeps what snb_vit_backward reads */
size_t snb_vit_workspace_bytes(int n_images, int save);
/* CLS features of n_images (1..SNB_VIT_MAX_IMAGES) images in one batched pass.  images: HOST array of device
 * pointers to (3, h, w) fp32 images read through element strides (HOST, n x 3: channel, row, column); sizes: HOST,
 * n x 2 (h, w), each >= 1.  -> out (n, 384), row-major.  save = 1: the workspace keeps the activations of the
 * backward and must be handed to it unchanged. */
int snb_vit_forward(const void* image, int precision, const float* const* images, const int64_t* strides,
                    const int* sizes, int n_images, int save, float* out, void* workspace, void* stream);
/* Gradient of the n features with respect to the n images of the save = 1 forward whose workspace this is:
 * d_out (n, 384) -> d_images[i] (3, h_i, w_i) written through d_strides (HOST, n x 3).  Every element of each
 * d_images[i] is written; nothing is accumulated. */
int snb_vit_backward(const void* image, int precision, const int* sizes, int n_images, const float* d_out,
                     float* const* d_images, const int64_t* d_strides, void* workspace, void* stream);

/* ---- optimiser step (SURVEY.md 8f-4) --------------------------------------------------------------
 * torch.optim.Adam as the reference configures it (utils/__init__.py:19-21: lr, eps = 1e-8, weight_decay;
 * betas default (0.9, 0.999), amsgrad off), fused over the 24 parameter tensors of one NeRF, followed on the
 * same stream by the re-pack of `packed` (may be NULL: no re-pack) so that the image the field kernels
 * stream is up to date -- and stamped clean for snb_refresh_weights -- when the call returns.
 * params: HOST array of 24 device pointers (updated in place); grads: HOST array of 24 device pointers, a
 * NULL entry = no gradient for that tensor (skipped, as torch does); exp_avg / exp_avg_sq: device buffers
 * of SNB_PARAM_FLOATS floats (the tensors' flat concatenation in state-dict order), zero before step 1.
 * step = 1 for the first update. */
#define SNB_PARAM_FLOATS 595844
typedef struct SnbAdamArgs {
  double lr, beta1, beta2, eps, weight_decay;   /* doubles: torch forms its scalars from python floats */
  int step;
} SnbAdamArgs;
int snb_adam_step(float* const* params, const float* const* grads, float* exp_avg, float* exp_avg_sq,
                  const SnbAdamArgs* args, int precision, int new_activation, void* packed, void* stream);

/* The reference's other get_optimizer choices (utils/__init__.py:15-27), same launch shape, checksum stamp and
 * re-pack as snb_adam_step:
 *   SNB_OPTIM_SGD     torch.optim.SGD(lr, momentum, weight_decay), dampening 0, no Nesterov.  exp_avg = the
 *                     momentum buffer; exp_avg_sq / slow_buffer unused (may be NULL).
 *   SNB_OPTIM_RADAM   utils/optimizers.py:7-106 (degenerated_to_sgd = True); slow_buffer unused (may be NULL).
 *   SNB_OPTIM_RANGER  utils/optimizers.py:292-439: RAdam moments + lookahead every k-th step into slow_buffer.
 * step[i] is tensor i's update count INCLUDING this one (the reference's state['step'] after its increment; for
 * SGD: the momentum-buffer update count, 1 = the buffer is a copy of the gradient).  Each tensor is stepped by its
 * own count, so one that had no gradient on earlier steps gets the same scalars the reference gives it; step[i] is
 * ignored where grads[i] is NULL.  RAdam / Ranger: N_sma and step_size are formed per tensor on the host in double,
 * in the reference's expression order.  Buffers are SNB_PARAM_FLOATS floats, like snb_adam_step's. */
#define SNB_OPTIM_SGD 0
#define SNB_OPTIM_RADAM 1
#define SNB_OPTIM_RANGER 2
typedef struct SnbOptimArgs {
  int rule;                          /* SNB_OPTIM_*                                                      */
  double lr, weight_decay;
  double momentum;                   /* SGD                                                              */
  double beta1, beta2, eps;          /* RAdam / Ranger                                                   */
  double n_sma_threshold;            /* Ranger: adaptive step iff N_sma > threshold (RAdam: N_sma >= 5)   */
  double alpha;                      /* Ranger: slow += alpha * (p - slow) ...                           */
  int k;                             /* ... every k-th step of the tensor, then p = slow                 */
  int step[SNB_N_PARAM_TENSORS];
} SnbOptimArgs;
int snb_optim_step(float* const* params, const float* const* grads, float* exp_avg, float* exp_avg_sq,
                   float* slow_buffer, const SnbOptimArgs* args, int precision, int new_activation, void* packed,
                   void* stream);

/* ---- whole path -------------------------------------------------------------------- */
typedef struct SnbRenderArgs {
  const float* rays;        /* (N,8)                                                    */
  int64_t n_rays;
  int n_samples;            /* N_samples                                                */
  int n_importance;         /* N_importance (0 = coarse only)                           */
  int use_disp;
  float perturb;
  float noise_std;
  int white_back;
  int test_time;            /* coarse pass sigma-only (rendering.py:287-292)            */
  int precision;            /* SNB_PREC_*                                               */
  const void* packed_coarse;
  const void* packed_fine;  /* NULL iff n_importance == 0                               */
  const float* z_steps;     /* (S,)  torch.linspace(0,1,S)                              */
  const float* u_steps;     /* (Ni,) torch.linspace(0,1,Ni), used when perturb == 0     */
  /* random draws in the reference's order (SURVEY.md 8a); NULL = not used             */
  const float* perturb_u;   /* (N,S)   rand,  needed iff perturb > 0                    */
  const float* noise_coarse;/* (N,S)   randn, read iff noise_std != 0                   */
  const float* pdf_u;       /* (N,Ni)  rand,  needed iff perturb > 0 and Ni > 0         */
  const float* noise_fine;  /* (N,S+Ni) randn                                           */
  /* outputs                                                                            */
  float* z_coarse;          /* (N,S)      workspace + output                            */
  float* raw_coarse;        /* (N,S,4) or (N,S) when test_time -- workspace             */
  float* rgb_coarse;        /* (N,3)   NULL when test_time                              */
  float* depth_coarse;      /* (N,)    NULL when test_time                              */
  float* weights_coarse;    /* (N,S)                                                    */
  float* z_fine;            /* (N,S+Ni)                                                 */
  float* raw_fine;          /* (N,S+Ni,4) workspace                                     */
  float* rgb_fine;          /* (N,3)                                                    */
  float* depth_fine;        /* (N,)                                                     */
  float* weights_fine;      /* (N,S+Ni)                                                 */
  const SnbPixelScatter* pixel_scatter; /* NULL, or: the last pass's compositing also scatters [rgb, depth] rows */
} SnbRenderArgs;

/* render_rays forward, models/rendering.py:126-335, as one call: every stage above enqueued
 * back to back on `stream`. */
int snb_render_forward(const SnbRenderArgs* args, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SINNERF_B200_H */
