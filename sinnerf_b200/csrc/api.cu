// api.cu -- the extern "C" surface of libsinnerf_b200.so (include/sinnerf_b200.h).
// Host-side argument checking and stage sequencing only; kernels live in the other .cu files.
#include <stdarg.h>

#include "common.cuh"

namespace snb {

static thread_local std::string g_last_error;

void set_error(const std::string& msg) { g_last_error = msg; }

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_last_error = buf;
  return code;
}

int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(SNB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  return SNB_OK;
}

int current_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  return dev;
}

int sm_count() {
  static int sms[kMaxDevices];
  const int dev = current_device() & (kMaxDevices - 1);
  if (!sms[dev]) cudaDeviceGetAttribute(&sms[dev], cudaDevAttrMultiProcessorCount, dev);
  return sms[dev];
}

// launchers defined in ray_kernels.cu / field_simt.cu / field_tc.cu
int launch_sample_coarse(const float*, const float*, const float*, float, int, int64_t, int, float*, cudaStream_t);
int launch_embed(const float*, int64_t, int, int, float*, cudaStream_t);
int launch_composite(const float*, int, const float*, const float*, const float*, float, int, int64_t, int,
                     float*, float*, float*, const SnbLossSpec*, float*, float*, const SnbPixelScatter*, cudaStream_t);
int launch_sample_pdf(const float*, int64_t, const float*, int64_t, const float*, int64_t, int64_t, int, int,
                      float, float*, cudaStream_t);
int launch_importance_merge(const float*, const float*, const float*, int64_t, int64_t, int, int, float, float*,
                            float*, cudaStream_t);
int field_forward_fp32(const void*, const float*, const float*, int64_t, int, int, float*, cudaStream_t);
int mlp_forward_fp32(const void*, const float*, int64_t, int64_t, int, float*, cudaStream_t);
int field_forward_train_fp32(const void*, const float*, const float*, int64_t, int, int, float*, float*, float*, float*,
                             float*, cudaStream_t);
int launch_composite_bwd(const float*, int, const float*, const float*, const float*, float, int, const float*,
                         const float*, const float*, int64_t, int, float*, const SnbLossSpec*, const float*,
                         const float*, const float*, float*, cudaStream_t);
int field_backward_fp32(const float* const*, float* const*, int, const float*, const float*, const float*,
                        const float*, const float*, const float*, int64_t, float*, float*, float*, float*,
                        uint32_t*, cudaStream_t);
int field_backward_sigma_fp32(const float* const*, float* const*, const float*, const float*, const float*, int64_t, float*,
                              float*, uint32_t*, cudaStream_t);
int launch_generate_rays(const float*, float, float, float, float, float, float, int, int, int, int, int, int, float*,
                         cudaStream_t);
int field_forward_train16_tc(const void*, int, const float*, const float*, int64_t, int, int, float*, void*, cudaStream_t);
size_t act16_bytes(long long);
size_t bwd16_workspace_bytes(long long);
int field_backward16(const float* const*, float* const*, int, const float*, const float*, const void*, long long, void*,
                     const float*, cudaStream_t);
int field_backward16_sigma(const float* const*, float* const*, const float*, const void*, long long, void*, const float*,
                           cudaStream_t);
int fused_step(int, const int64_t*, float* const*, const float* const*, bool, const int*, const SnbAmpStep*, float*,
               float*, float*, const SnbOptimArgs&, int, int, void*, cudaStream_t);
// tensor-core modes (field_tc.cu)
size_t tc_packed_bytes(int precision);
int field_forward_tc(const void*, int, const float*, const float*, int64_t, int, int, float*, cudaStream_t);
int mlp_forward_tc(const void*, int, const float*, int64_t, int64_t, int, float*, cudaStream_t);
int field_forward_train_tc(const void*, int, const float*, const float*, int64_t, int, int, float*, float*, float*, float*,
                           float*, cudaStream_t);

// image-space patch losses (patch_loss.cu)
int launch_depth_smooth_fwd(const float*, const int64_t*, const float*, const int64_t*, long long, int, int, int, float*,
                            float*, cudaStream_t);
int launch_depth_smooth_bwd(const float*, const int64_t*, const float*, const int64_t*, long long, int, int, int,
                            const float*, float*, const int64_t*, float*, const int64_t*, cudaStream_t);
int launch_ssim_fwd(const float*, const int64_t*, const float*, const int64_t*, long long, int, int, int, float, float,
                    float*, double*, float*, cudaStream_t);
int launch_ssim_bwd(const float*, const int64_t*, const float*, const int64_t*, long long, int, int, int, const double*,
                    const float*, float*, const int64_t*, cudaStream_t);

// forward warp (warp.cu)
size_t forward_warp_workspace_bytes(long long, long long, int);
int launch_forward_warp(const float*, const float*, int, int, const double*, long long, int, float*, float*,
                        unsigned char*, void*, cudaStream_t);

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// a (B,C,H,W) patch-loss operand: data and its four element strides, both non-null, strides non-negative
static int check_nchw(const char* who, const char* name, const void* data, const int64_t* strides) {
  SNB_REQUIRE(data != nullptr && strides != nullptr, "%s: null pointer (%s or its strides)", who, name);
  for (int k = 0; k < 4; ++k) SNB_REQUIRE(strides[k] >= 0, "%s: negative stride in %s", who, name);
  return SNB_OK;
}

static int check_patch_extents(const char* who, int64_t batch, int channels, int height, int width, int min_hw) {
  SNB_REQUIRE(batch >= 1 && channels >= 1, "%s: needs batch >= 1 and channels >= 1 (got %lld, %d)", who,
              (long long)batch, channels);
  SNB_REQUIRE(height >= min_hw && width >= min_hw, "%s: needs H, W >= %d (got %d x %d)", who, min_hw, height, width);
  return SNB_OK;
}

static int check_precision(int precision) {
  if (precision < SNB_PREC_FP32 || precision > SNB_PREC_F16)
    return fail(SNB_ERR_INVALID, "unknown precision mode %d", precision);
  return SNB_OK;
}

// standalone DiffAugment (disc.cu)
int launch_diff_augment(bool, const int*, int, const SnbDiffAugDraws&, const float*, const int64_t*, int, int, int, int,
                        float*, const int64_t*, float*, cudaStream_t);

// the checks of snb_diff_augment_forward / _backward
static int check_diff_augment(const char* who, const int* ops, int n_ops, const SnbDiffAugDraws* d, const void* src,
                              const int64_t* ss, int n, int channels, int height, int width, const void* dst,
                              const int64_t* ds, const void* workspace) {
  SNB_REQUIRE(n_ops >= 0 && n_ops <= SNB_DIFF_AUG_MAX_OPS, "%s: n_ops %d outside 0..%d", who, n_ops,
              SNB_DIFF_AUG_MAX_OPS);
  SNB_REQUIRE(n_ops == 0 || (ops != nullptr && d != nullptr), "%s: null ops or draws", who);
  for (int k = 0; k < n_ops; ++k) {
    const int op = ops[k];
    SNB_REQUIRE(op == SNB_DIFF_AUG_COLOR || op == SNB_DIFF_AUG_TRANSLATION || op == SNB_DIFF_AUG_CUTOUT,
                "%s: unknown op code %d at %d", who, op, k);
    SNB_REQUIRE(op != SNB_DIFF_AUG_COLOR || (d->brightness && d->saturation && d->contrast),
                "%s: the policy lists color but a color draw is NULL", who);
    SNB_REQUIRE(op != SNB_DIFF_AUG_TRANSLATION || (d->translation_y && d->translation_x),
                "%s: the policy lists translation but a translation draw is NULL", who);
    SNB_REQUIRE(op != SNB_DIFF_AUG_CUTOUT || (d->cutout_y && d->cutout_x),
                "%s: the policy lists cutout but a cutout draw is NULL", who);
  }
  if (int rc = check_patch_extents(who, n, channels, height, width, 1)) return rc;
  SNB_REQUIRE((int64_t)n * height * width < (int64_t(1) << 31), "%s: %d images of %d x %d are too many pixels", who,
              n, height, width);
  if (int rc = check_nchw(who, "the source", src, ss)) return rc;
  if (int rc = check_nchw(who, "the destination", dst, ds)) return rc;
  SNB_REQUIRE(workspace != nullptr, "%s: null workspace", who);
  return SNB_OK;
}

}  // namespace snb

using namespace snb;

extern "C" {

int snb_version(void) { return SNB_VERSION; }

const char* snb_last_error(void) { return g_last_error.c_str(); }

int snb_device_check(int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return fail(SNB_ERR_CUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  int major = 0, minor = 0, sms = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (sm_count) *sm_count = sms;
  if (cc_major) *cc_major = major;
  if (cc_minor) *cc_minor = minor;
  if (major != 9 || minor != 0)   // sm_90a code (wgmma) loads on compute capability 9.0 only
    return fail(SNB_ERR_UNSUPPORTED, "libsinnerf_b200 is built for sm_90a only; device %d is sm_%d%d", dev, major,
                minor);
  return SNB_OK;
}

size_t snb_packed_weights_bytes(int precision) {
  if (precision == SNB_PREC_FP32) return sizeof(PackedHeader) + sizeof(float) * (size_t)make_fp32_layout().total;
  if (precision >= SNB_PREC_F16X3 && precision <= SNB_PREC_F16) return tc_packed_bytes(precision);
  return 0;
}

static int pack_weights_impl(const char* who, const float* const* params, int precision, int new_activation,
                             void* packed, int only_if_dirty, void* stream) {
  SNB_REQUIRE(params != nullptr && packed != nullptr, "%s: null pointer", who);
  SNB_REQUIRE(aligned16(packed), "%s: packed image must be 16-byte aligned", who);
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i)
    SNB_REQUIRE(params[i] != nullptr, "%s: parameter tensor %d is null", who, i);
  if (int rc = check_precision(precision)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the check kernel always runs: it also stamps the header with the checksum of what is being packed
  ParamPtrs pp;
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) pp.p[i] = params[i];
  if (int rc = launch_params_check(pp, precision, new_activation ? 1 : 0, packed, st)) return rc;
  if (precision == SNB_PREC_FP32) return launch_pack_fp32(params, new_activation ? 1 : 0, packed, only_if_dirty, st);
  return launch_pack_tc(params, precision, new_activation ? 1 : 0, packed, only_if_dirty, st);
}

int snb_pack_weights(const float* const* params, int precision, int new_activation, void* packed, void* stream) {
  return pack_weights_impl("snb_pack_weights", params, precision, new_activation, packed, 0, stream);
}

int snb_refresh_weights(const float* const* params, int precision, int new_activation, void* packed, void* stream) {
  return pack_weights_impl("snb_refresh_weights", params, precision, new_activation, packed, 1, stream);
}

int snb_sample_coarse(const float* rays, const float* z_steps, const float* perturb_u, float perturb, int use_disp,
                      int64_t n_rays, int n_samples, float* z_vals, void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_sample_coarse: bad extents (%lld rays, %d samples)",
              (long long)n_rays, n_samples);
  SNB_REQUIRE(n_rays == 0 || (rays && z_steps && z_vals), "snb_sample_coarse: null pointer");
  SNB_REQUIRE(!(perturb > 0.f) || perturb_u != nullptr, "snb_sample_coarse: perturb > 0 needs perturb_u");
  return launch_sample_coarse(rays, z_steps, perturb_u, perturb, use_disp, n_rays, n_samples, z_vals,
                              reinterpret_cast<cudaStream_t>(stream));
}

int snb_embed(const float* x, int64_t n, int in_channels, int n_freqs, float* out, void* stream) {
  SNB_REQUIRE(n >= 0 && in_channels >= 1 && n_freqs >= 0 && n_freqs <= 24, "snb_embed: bad extents");
  SNB_REQUIRE(n == 0 || (x && out), "snb_embed: null pointer");
  return launch_embed(x, n, in_channels, n_freqs, out, reinterpret_cast<cudaStream_t>(stream));
}

int snb_mlp_forward(const void* packed, int precision, const float* x, int64_t x_stride, int64_t n_points,
                    int sigma_only, float* out, void* stream) {
  SNB_REQUIRE(n_points >= 0, "snb_mlp_forward: negative point count");
  SNB_REQUIRE(n_points == 0 || (packed && x && out), "snb_mlp_forward: null pointer");
  SNB_REQUIRE(x_stride >= (sigma_only ? SNB_XYZ_CH : SNB_XYZ_CH + SNB_DIR_CH),
              "snb_mlp_forward: row stride %lld shorter than the embedded row", (long long)x_stride);
  SNB_REQUIRE(sigma_only || aligned16(out), "snb_mlp_forward: (P,4) output must be 16-byte aligned");
  if (int rc = check_precision(precision)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (precision == SNB_PREC_FP32) return mlp_forward_fp32(packed, x, x_stride, n_points, sigma_only, out, st);
  return mlp_forward_tc(packed, precision, x, x_stride, n_points, sigma_only, out, st);
}

int snb_field_forward(const void* packed, int precision, const float* rays, const float* z_vals, int64_t n_rays,
                      int n_samples, int sigma_only, float* raw, void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_field_forward: bad extents");
  SNB_REQUIRE(n_rays == 0 || (packed && rays && z_vals && raw), "snb_field_forward: null pointer");
  SNB_REQUIRE(aligned16(rays), "snb_field_forward: rays must be 16-byte aligned");
  SNB_REQUIRE(sigma_only || aligned16(raw), "snb_field_forward: (N,S,4) output must be 16-byte aligned");
  if (int rc = check_precision(precision)) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (precision == SNB_PREC_FP32) return field_forward_fp32(packed, rays, z_vals, n_rays, n_samples, sigma_only, raw, st);
  return field_forward_tc(packed, precision, rays, z_vals, n_rays, n_samples, sigma_only, raw, st);
}

int snb_composite_forward(const float* raw, int raw_channels, const float* z_vals, const float* rays,
                          const float* noise, float noise_std, int white_back, int64_t n_rays, int n_samples,
                          float* rgb, float* depth, float* weights, void* stream) {
  SNB_REQUIRE(raw_channels == 4 || raw_channels == 1, "snb_composite_forward: raw_channels must be 4 or 1");
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_composite_forward: bad extents");
  SNB_REQUIRE(n_rays == 0 || (raw && z_vals && rays && weights), "snb_composite_forward: null pointer");
  SNB_REQUIRE(n_rays == 0 || raw_channels == 1 || (rgb && depth), "snb_composite_forward: rgb/depth outputs required");
  SNB_REQUIRE(raw_channels == 1 || aligned16(raw), "snb_composite_forward: raw must be 16-byte aligned");
  const float* nz = (noise_std != 0.f) ? noise : nullptr;
  return launch_composite(raw, raw_channels, z_vals, rays, nz, noise_std, white_back, n_rays, n_samples, rgb,
                          depth, weights, nullptr, nullptr, nullptr, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int snb_composite_forward_scatter(const float* raw, const float* z_vals, const float* rays, const float* noise,
                                  float noise_std, int white_back, int64_t n_rays, int n_samples, float* rgb,
                                  float* depth, float* weights, const SnbPixelScatter* scatter, void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_composite_forward_scatter: bad extents");
  SNB_REQUIRE(n_rays == 0 || (raw && z_vals && rays && weights && rgb && depth), "snb_composite_forward_scatter: null pointer");
  SNB_REQUIRE(aligned16(raw), "snb_composite_forward_scatter: raw must be 16-byte aligned");
  SNB_REQUIRE(scatter != nullptr && scatter->n_dst >= 1 && scatter->n_dst <= SNB_MAX_PIXEL_DST && scatter->row_offset >= 0,
              "snb_composite_forward_scatter: scatter needs 1..%d destinations and a non-negative row offset", SNB_MAX_PIXEL_DST);
  for (int i = 0; i < scatter->n_dst; ++i)
    SNB_REQUIRE(scatter->dst[i] != nullptr && aligned16(scatter->dst[i]),
                "snb_composite_forward_scatter: destination %d is null or not 16-byte aligned", i);
  const float* nz = (noise_std != 0.f) ? noise : nullptr;
  return launch_composite(raw, 4, z_vals, rays, nz, noise_std, white_back, n_rays, n_samples, rgb, depth, weights,
                          nullptr, nullptr, nullptr, scatter, reinterpret_cast<cudaStream_t>(stream));
}

static int check_loss_spec(const char* who, const SnbLossSpec* loss) {
  SNB_REQUIRE(loss != nullptr, "%s: null loss spec", who);
  SNB_REQUIRE(loss->target_rgb != nullptr || loss->target_depth != nullptr, "%s: the loss spec has no target", who);
  return SNB_OK;
}

int snb_composite_forward_loss(const float* raw, const float* z_vals, const float* rays, const float* noise,
                               float noise_std, int white_back, int64_t n_rays, int n_samples,
                               const SnbLossSpec* loss, float* rgb, float* depth, float* weights, float* loss_out,
                               float* loss_ws, void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_composite_forward_loss: bad extents");
  if (int rc = check_loss_spec("snb_composite_forward_loss", loss)) return rc;
  SNB_REQUIRE(loss_out != nullptr && loss_ws != nullptr, "snb_composite_forward_loss: null loss output / workspace");
  SNB_REQUIRE(n_rays == 0 || (raw && z_vals && rays && weights && rgb && depth), "snb_composite_forward_loss: null pointer");
  SNB_REQUIRE(aligned16(raw), "snb_composite_forward_loss: raw must be 16-byte aligned");
  const float* nz = (noise_std != 0.f) ? noise : nullptr;
  return launch_composite(raw, 4, z_vals, rays, nz, noise_std, white_back, n_rays, n_samples, rgb, depth, weights,
                          loss, loss_out, loss_ws, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int snb_sample_pdf(const float* bins, int64_t bins_stride, const float* weights, int64_t w_stride, const float* u,
                   int64_t u_stride, int64_t n_rays, int m, int n_importance, float eps, float* samples,
                   void* stream) {
  SNB_REQUIRE(n_rays >= 0 && m >= 1 && n_importance >= 1, "snb_sample_pdf: bad extents");
  SNB_REQUIRE(n_rays == 0 || (bins && weights && u && samples), "snb_sample_pdf: null pointer");
  SNB_REQUIRE(bins_stride >= m + 1 && w_stride >= m, "snb_sample_pdf: row strides shorter than rows");
  SNB_REQUIRE(u_stride == 0 || u_stride >= n_importance, "snb_sample_pdf: bad u stride");
  return launch_sample_pdf(bins, bins_stride, weights, w_stride, u, u_stride, n_rays, m, n_importance, eps,
                           samples, reinterpret_cast<cudaStream_t>(stream));
}

int snb_importance_merge(const float* z_coarse, const float* weights_coarse, const float* u, int64_t u_stride,
                         int64_t n_rays, int n_samples, int n_importance, float eps, float* z_fine, float* z_new,
                         void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 3 && n_importance >= 1,
              "snb_importance_merge: needs N_samples >= 3 and N_importance >= 1");
  SNB_REQUIRE(n_rays == 0 || (z_coarse && weights_coarse && u && z_fine), "snb_importance_merge: null pointer");
  SNB_REQUIRE(u_stride == 0 || u_stride >= n_importance, "snb_importance_merge: bad u stride");
  return launch_importance_merge(z_coarse, weights_coarse, u, u_stride, n_rays, n_samples, n_importance, eps,
                                 z_fine, z_new, reinterpret_cast<cudaStream_t>(stream));
}

int snb_generate_rays(const float* c2w, float fx, float fy, float cx, float cy, float near, float far, int opencv,
                      int row0, int col0, int rows, int cols, int stride, float* rays, void* stream) {
  SNB_REQUIRE(c2w != nullptr, "snb_generate_rays: null camera matrix");
  SNB_REQUIRE(rows >= 0 && cols >= 0 && stride >= 1 && row0 >= 0 && col0 >= 0, "snb_generate_rays: bad window");
  SNB_REQUIRE(fx != 0.f && fy != 0.f, "snb_generate_rays: zero focal length");
  SNB_REQUIRE((long long)rows * cols == 0 || (rays != nullptr && aligned16(rays)),
              "snb_generate_rays: rays must be a 16-byte aligned device buffer");
  return launch_generate_rays(c2w, fx, fy, cx, cy, near, far, opencv, row0, col0, rows, cols, stride, rays,
                              reinterpret_cast<cudaStream_t>(stream));
}

int snb_field_forward_train(const void* packed, int precision, const float* rays, const float* z_vals,
                            int64_t n_rays, int n_samples, float* raw, float* save_enc, float* save_dir,
                            float* save_h, float* save_g, void* stream) {
  if (int rc = check_precision(precision)) return rc;
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_field_forward_train: bad extents");
  SNB_REQUIRE(n_rays == 0 || (packed && rays && z_vals && raw && save_enc && save_dir && save_h && save_g),
              "snb_field_forward_train: null pointer");
  SNB_REQUIRE(aligned16(rays) && aligned16(raw) && aligned16(save_enc) && aligned16(save_dir) && aligned16(save_h) &&
                  aligned16(save_g),
              "snb_field_forward_train: buffers must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (precision == SNB_PREC_FP32)
    return field_forward_train_fp32(packed, rays, z_vals, n_rays, n_samples, 0, raw, save_enc, save_dir, save_h, save_g, st);
  return field_forward_train_tc(packed, precision, rays, z_vals, n_rays, n_samples, 0, raw, save_enc, save_dir, save_h,
                                save_g, st);
}

int snb_field_forward_train_sigma(const void* packed, int precision, const float* rays, const float* z_vals,
                                  int64_t n_rays, int n_samples, float* sigma, float* save_enc, float* save_h,
                                  void* stream) {
  if (int rc = check_precision(precision)) return rc;
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_field_forward_train_sigma: bad extents");
  SNB_REQUIRE(n_rays == 0 || (packed && rays && z_vals && sigma && save_enc && save_h),
              "snb_field_forward_train_sigma: null pointer");
  SNB_REQUIRE(aligned16(rays) && aligned16(save_enc) && aligned16(save_h),
              "snb_field_forward_train_sigma: rays / save_enc / save_h must be 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (precision == SNB_PREC_FP32)
    return field_forward_train_fp32(packed, rays, z_vals, n_rays, n_samples, 1, sigma, save_enc, nullptr, save_h, nullptr, st);
  return field_forward_train_tc(packed, precision, rays, z_vals, n_rays, n_samples, 1, sigma, save_enc, nullptr, save_h,
                                nullptr, st);
}

int snb_composite_backward(const float* raw, const float* z_vals, const float* rays, const float* noise,
                           float noise_std, int white_back, const float* g_rgb, const float* g_depth,
                           const float* g_weights, int64_t n_rays, int n_samples, float* g_raw, void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_composite_backward: bad extents");
  SNB_REQUIRE(n_rays == 0 || (raw && z_vals && rays && g_raw), "snb_composite_backward: null pointer");
  SNB_REQUIRE(aligned16(raw) && aligned16(g_raw), "snb_composite_backward: raw / g_raw must be 16-byte aligned");
  const float* nz = (noise_std != 0.f) ? noise : nullptr;
  return launch_composite_bwd(raw, 4, z_vals, rays, nz, noise_std, white_back, g_rgb, g_depth, g_weights, n_rays,
                              n_samples, g_raw, nullptr, nullptr, nullptr, nullptr, nullptr,
                              reinterpret_cast<cudaStream_t>(stream));
}

int snb_composite_backward_weights(const float* sigma, const float* z_vals, const float* rays, const float* noise,
                                   float noise_std, const float* g_weights, int64_t n_rays, int n_samples,
                                   float* g_sigma, float* g_amax, void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_composite_backward_weights: bad extents");
  SNB_REQUIRE(n_rays == 0 || (sigma && z_vals && rays && g_weights && g_sigma), "snb_composite_backward_weights: null pointer");
  const float* nz = (noise_std != 0.f) ? noise : nullptr;
  return launch_composite_bwd(sigma, 1, z_vals, rays, nz, noise_std, 0, nullptr, nullptr, g_weights, n_rays, n_samples,
                              g_sigma, nullptr, nullptr, nullptr, nullptr, g_amax, reinterpret_cast<cudaStream_t>(stream));
}

int snb_composite_backward_loss(const float* raw, const float* z_vals, const float* rays, const float* noise,
                                float noise_std, int white_back, const float* g_rgb, const float* g_depth,
                                const float* g_weights, const SnbLossSpec* loss, const float* rgb, const float* depth,
                                const float* g_loss, int64_t n_rays, int n_samples, float* g_raw, float* g_amax,
                                void* stream) {
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_composite_backward_loss: bad extents");
  SNB_REQUIRE(n_rays == 0 || (raw && z_vals && rays && g_raw), "snb_composite_backward_loss: null pointer");
  SNB_REQUIRE(aligned16(raw) && aligned16(g_raw), "snb_composite_backward_loss: raw / g_raw must be 16-byte aligned");
  if (loss != nullptr) {
    if (int rc = check_loss_spec("snb_composite_backward_loss", loss)) return rc;
    SNB_REQUIRE(n_rays == 0 || ((loss->target_rgb == nullptr || rgb) && (loss->target_depth == nullptr || depth)),
                "snb_composite_backward_loss: the forward's rgb / depth outputs are required with a loss spec");
  }
  const float* nz = (noise_std != 0.f) ? noise : nullptr;
  return launch_composite_bwd(raw, 4, z_vals, rays, nz, noise_std, white_back, g_rgb, g_depth, g_weights, n_rays,
                              n_samples, g_raw, loss, rgb, depth, g_loss, g_amax, reinterpret_cast<cudaStream_t>(stream));
}

int snb_field_backward(const float* const* params, float* const* grads, int new_activation, const float* g_raw,
                       const float* raw, const float* save_enc, const float* save_dir, const float* save_h,
                       const float* save_g, int64_t n_points, float* ws_a, float* ws_b, float* ws_s,
                       float* ws_w, uint32_t* ws_m, void* stream) {
  SNB_REQUIRE(n_points >= 0, "snb_field_backward: negative point count");
  SNB_REQUIRE(params && grads, "snb_field_backward: null parameter arrays");
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i)
    SNB_REQUIRE(params[i] && grads[i], "snb_field_backward: parameter / gradient tensor %d is null", i);
  SNB_REQUIRE(n_points == 0 || (g_raw && raw && save_enc && save_dir && save_h && save_g && ws_a && ws_b && ws_s && ws_w && ws_m),
              "snb_field_backward: null pointer");
  return field_backward_fp32(params, grads, new_activation, g_raw, raw, save_enc, save_dir, save_h, save_g,
                             n_points, ws_a, ws_b, ws_s, ws_w, ws_m, reinterpret_cast<cudaStream_t>(stream));
}

// the tensors a sigma-only pass reads: layers 1-8 and the sigma head
static bool sigma_pass_tensor(int i) { return i < 16 || i == 20 || i == 21; }

int snb_field_backward_sigma(const float* const* params, float* const* grads, const float* g_sigma,
                             const float* save_enc, const float* save_h, int64_t n_points, float* ws_a, float* ws_b,
                             uint32_t* ws_m, void* stream) {
  SNB_REQUIRE(n_points >= 0, "snb_field_backward_sigma: negative point count");
  SNB_REQUIRE(params && grads, "snb_field_backward_sigma: null parameter arrays");
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i)
    SNB_REQUIRE(!sigma_pass_tensor(i) || (params[i] && grads[i]), "snb_field_backward_sigma: parameter / gradient tensor %d is null", i);
  SNB_REQUIRE(n_points == 0 || (g_sigma && save_enc && save_h && ws_a && ws_b && ws_m), "snb_field_backward_sigma: null pointer");
  SNB_REQUIRE(aligned16(save_enc) && aligned16(save_h) && aligned16(ws_a) && aligned16(ws_b) && aligned16(ws_m),
              "snb_field_backward_sigma: save_enc / save_h / scratch must be 16-byte aligned");
  return field_backward_sigma_fp32(params, grads, g_sigma, save_enc, save_h, n_points, ws_a, ws_b, ws_m,
                                   reinterpret_cast<cudaStream_t>(stream));
}

size_t snb_act16_bytes(int64_t n_points) { return n_points < 0 ? 0 : act16_bytes(n_points); }
size_t snb_bwd16_workspace_bytes(int64_t n_points) { return n_points < 0 ? 0 : bwd16_workspace_bytes(n_points); }

int snb_field_forward_train16(const void* packed, int precision, const float* rays, const float* z_vals, int64_t n_rays,
                              int n_samples, float* raw, void* act16, void* stream) {
  if (int rc = check_precision(precision)) return rc;
  if (precision == SNB_PREC_FP32)
    return fail(SNB_ERR_UNSUPPORTED, "snb_field_forward_train16: 16-bit activation storage needs a tensor-core precision mode");
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_field_forward_train16: bad extents");
  SNB_REQUIRE(n_rays == 0 || (packed && rays && z_vals && raw && act16), "snb_field_forward_train16: null pointer");
  SNB_REQUIRE(aligned16(rays) && aligned16(raw) && (reinterpret_cast<uintptr_t>(act16) & 255u) == 0,
              "snb_field_forward_train16: rays / raw must be 16-byte and act16 256-byte aligned");
  return field_forward_train16_tc(packed, precision, rays, z_vals, n_rays, n_samples, 0, raw, act16,
                                  reinterpret_cast<cudaStream_t>(stream));
}

int snb_field_forward_train16_sigma(const void* packed, int precision, const float* rays, const float* z_vals,
                                    int64_t n_rays, int n_samples, float* sigma, void* act16, void* stream) {
  if (int rc = check_precision(precision)) return rc;
  if (precision == SNB_PREC_FP32)
    return fail(SNB_ERR_UNSUPPORTED, "snb_field_forward_train16_sigma: 16-bit activation storage needs a tensor-core precision mode");
  SNB_REQUIRE(n_rays >= 0 && n_samples >= 1, "snb_field_forward_train16_sigma: bad extents");
  SNB_REQUIRE(n_rays == 0 || (packed && rays && z_vals && sigma && act16), "snb_field_forward_train16_sigma: null pointer");
  SNB_REQUIRE(aligned16(rays) && (reinterpret_cast<uintptr_t>(act16) & 255u) == 0,
              "snb_field_forward_train16_sigma: rays must be 16-byte and act16 256-byte aligned");
  return field_forward_train16_tc(packed, precision, rays, z_vals, n_rays, n_samples, 1, sigma, act16,
                                  reinterpret_cast<cudaStream_t>(stream));
}

int snb_field_backward16(const float* const* params, float* const* grads, int new_activation, const float* g_raw,
                         const float* raw, const void* act16, int64_t n_points, void* workspace, const float* g_amax,
                         void* stream) {
  SNB_REQUIRE(n_points >= 0, "snb_field_backward16: negative point count");
  SNB_REQUIRE(params && grads, "snb_field_backward16: null parameter arrays");
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i)
    SNB_REQUIRE(params[i] && grads[i], "snb_field_backward16: parameter / gradient tensor %d is null", i);
  SNB_REQUIRE(n_points == 0 || (g_raw && raw && act16 && workspace), "snb_field_backward16: null pointer");
  SNB_REQUIRE(aligned16(g_raw) && aligned16(raw) && (reinterpret_cast<uintptr_t>(act16) & 255u) == 0 &&
                  (reinterpret_cast<uintptr_t>(workspace) & 255u) == 0,
              "snb_field_backward16: g_raw / raw must be 16-byte, act16 / workspace 256-byte aligned");
  return field_backward16(params, grads, new_activation, g_raw, raw, act16, n_points, workspace, g_amax,
                          reinterpret_cast<cudaStream_t>(stream));
}

int snb_field_backward16_sigma(const float* const* params, float* const* grads, const float* g_sigma, const void* act16,
                               int64_t n_points, void* workspace, const float* g_amax, void* stream) {
  SNB_REQUIRE(n_points >= 0, "snb_field_backward16_sigma: negative point count");
  SNB_REQUIRE(params && grads, "snb_field_backward16_sigma: null parameter arrays");
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i)
    SNB_REQUIRE(!sigma_pass_tensor(i) || (params[i] && grads[i]), "snb_field_backward16_sigma: parameter / gradient tensor %d is null", i);
  SNB_REQUIRE(n_points == 0 || (g_sigma && act16 && workspace), "snb_field_backward16_sigma: null pointer");
  SNB_REQUIRE((reinterpret_cast<uintptr_t>(act16) & 255u) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 255u) == 0,
              "snb_field_backward16_sigma: act16 / workspace must be 256-byte aligned");
  return field_backward16_sigma(params, grads, g_sigma, act16, n_points, workspace, g_amax,
                                reinterpret_cast<cudaStream_t>(stream));
}

// Argument checks shared by the plain and GradScaler-native (_amp) forms of the three optimiser steps.  `step` is the
// plain form's count (snb_adam_step: one; the others: per tensor), or the _amp form's `base`, which the same rules bound.
static int check_adam_step(const char* who, float* const* params, const void* grads, const float* exp_avg,
                           const float* exp_avg_sq, const SnbAdamArgs* args, const int* step, int precision,
                           const void* packed) {
  SNB_REQUIRE(params && grads && exp_avg && exp_avg_sq && args && step, "%s: null pointer", who);
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) SNB_REQUIRE(params[i] != nullptr, "%s: parameter tensor %d is null", who, i);
  SNB_REQUIRE(*step >= 1, "%s: step counts from 1 (got %d)", who, *step);
  SNB_REQUIRE(args->lr >= 0. && args->eps >= 0. && args->beta1 >= 0. && args->beta1 < 1. && args->beta2 >= 0. &&
                  args->beta2 < 1. && args->weight_decay >= 0.,
              "%s: invalid hyper-parameters", who);
  SNB_REQUIRE(packed == nullptr || aligned16(packed), "%s: packed image must be 16-byte aligned", who);
  if (packed != nullptr)
    if (int rc = check_precision(precision)) return rc;
  static_assert(SNB_PARAM_FLOATS == 593408 + 2436, "parameter count");
  return SNB_OK;
}

static int check_optim_step(const char* who, float* const* params, const void* const* grads, const float* exp_avg,
                            const float* exp_avg_sq, const float* slow_buffer, const SnbOptimArgs* args,
                            const int* step, int precision, const void* packed) {
  SNB_REQUIRE(params && grads && args, "%s: null pointer", who);
  const int rule = args->rule;
  SNB_REQUIRE(rule == SNB_OPTIM_SGD || rule == SNB_OPTIM_RADAM || rule == SNB_OPTIM_RANGER,
              "%s: unknown rule %d", who, rule);
  SNB_REQUIRE(exp_avg != nullptr && (rule == SNB_OPTIM_SGD || exp_avg_sq != nullptr) &&
                  (rule != SNB_OPTIM_RANGER || slow_buffer != nullptr),
              "%s: null state buffer", who);
  for (int i = 0; i < SNB_N_PARAM_TENSORS; ++i) {
    SNB_REQUIRE(params[i] != nullptr, "%s: parameter tensor %d is null", who, i);
    SNB_REQUIRE(grads[i] == nullptr || step[i] >= 1 || (rule == SNB_OPTIM_SGD && args->momentum == 0.),
                "%s: step of tensor %d counts from 1 (got %d)", who, i, step[i]);
  }
  SNB_REQUIRE(args->lr >= 0. && args->weight_decay >= 0. && args->momentum >= 0. && args->eps >= 0. &&
                  args->beta1 >= 0. && args->beta1 < 1. && args->beta2 >= 0. && args->beta2 < 1. &&
                  args->alpha >= 0. && args->alpha <= 1. && args->k >= 1,
              "%s: invalid hyper-parameters", who);
  SNB_REQUIRE(packed == nullptr || aligned16(packed), "%s: packed image must be 16-byte aligned", who);
  if (packed != nullptr)
    if (int rc = check_precision(precision)) return rc;
  return SNB_OK;
}

static int check_optim_tensors(const char* who, int n, float* const* params, const void* const* grads,
                               const int64_t* numel, const int* step, const float* exp_avg, const float* exp_avg_sq,
                               const float* slow_buffer, const SnbOptimArgs* args) {
  SNB_REQUIRE(params && grads && numel && step && args, "%s: null table or args", who);
  SNB_REQUIRE(n >= 1 && n <= SNB_OPTIM_MAX_TENSORS, "%s: needs 1 <= n <= %d tensors (got %d)", who,
              SNB_OPTIM_MAX_TENSORS, n);
  const int rule = args->rule;
  SNB_REQUIRE(rule == SNB_OPTIM_SGD || rule == SNB_OPTIM_RADAM || rule == SNB_OPTIM_RANGER || rule == SNB_OPTIM_ADAM,
              "%s: unknown rule %d", who, rule);
  const bool sgd = rule == SNB_OPTIM_SGD;
  SNB_REQUIRE((exp_avg != nullptr || (sgd && args->momentum == 0.)) && (sgd || exp_avg_sq != nullptr) &&
                  (rule != SNB_OPTIM_RANGER || slow_buffer != nullptr),
              "%s: null state buffer (rule %d)", who, rule);
  for (int i = 0; i < n; ++i) {
    SNB_REQUIRE(params[i] != nullptr, "%s: parameter tensor %d is null", who, i);
    SNB_REQUIRE(numel[i] >= 1, "%s: numel of tensor %d must be >= 1 (got %lld)", who, i, (long long)numel[i]);
    SNB_REQUIRE(grads[i] == nullptr || step[i] >= 1 || (sgd && args->momentum == 0.),
                "%s: step of tensor %d counts from 1 (got %d)", who, i, step[i]);
  }
  SNB_REQUIRE(args->lr >= 0. && args->weight_decay >= 0. && args->momentum >= 0. && args->eps >= 0. &&
                  args->beta1 >= 0. && args->beta1 < 1. && args->beta2 >= 0. && args->beta2 < 1. &&
                  args->alpha >= 0. && args->alpha <= 1. && args->k >= 1,
              "%s: invalid hyper-parameters", who);
  return SNB_OK;
}

// The _amp forms' own arguments: n counts in each of two device arrays that must not overlap.
static int check_amp(const char* who, const SnbAmpStep* amp, int n) {
  SNB_REQUIRE(amp != nullptr && amp->count_in != nullptr && amp->count_out != nullptr, "%s: null amp or count array", who);
  SNB_REQUIRE(amp->count_in + n <= amp->count_out || amp->count_out + n <= amp->count_in,
              "%s: count_in and count_out overlap", who);
  return SNB_OK;
}

// snb_adam_step's hyper-parameters as the Adam rule of the shared step.
static SnbOptimArgs adam_rule(const SnbAdamArgs& a) {
  SnbOptimArgs o = {};
  o.rule = SNB_OPTIM_ADAM;
  o.lr = a.lr;
  o.beta1 = a.beta1;
  o.beta2 = a.beta2;
  o.eps = a.eps;
  o.weight_decay = a.weight_decay;
  return o;
}

int snb_adam_step(float* const* params, const float* const* grads, float* exp_avg, float* exp_avg_sq,
                  const SnbAdamArgs* args, int precision, int new_activation, void* packed, void* stream) {
  if (int rc = check_adam_step("snb_adam_step", params, grads, exp_avg, exp_avg_sq, args, args ? &args->step : nullptr,
                               precision, packed))
    return rc;
  return fused_step(SNB_N_PARAM_TENSORS, nullptr, params, grads, true, &args->step, nullptr, exp_avg, exp_avg_sq,
                    nullptr, adam_rule(*args), precision, new_activation, packed,
                    reinterpret_cast<cudaStream_t>(stream));
}

int snb_adam_step_amp(float* const* params, float* const* grads, float* exp_avg, float* exp_avg_sq,
                      const SnbAdamArgs* args, const SnbAmpStep* amp, int precision, int new_activation, void* packed,
                      void* stream) {
  const char* who = "snb_adam_step_amp";
  if (int rc = check_amp(who, amp, 1)) return rc;
  if (int rc = check_adam_step(who, params, grads, exp_avg, exp_avg_sq, args, amp->base, precision, packed)) return rc;
  return fused_step(SNB_N_PARAM_TENSORS, nullptr, params, grads, true, amp->base, amp, exp_avg, exp_avg_sq, nullptr,
                    adam_rule(*args), precision, new_activation, packed, reinterpret_cast<cudaStream_t>(stream));
}

int snb_optim_step(float* const* params, const float* const* grads, float* exp_avg, float* exp_avg_sq,
                   float* slow_buffer, const SnbOptimArgs* args, int precision, int new_activation, void* packed,
                   void* stream) {
  if (int rc = check_optim_step("snb_optim_step", params, reinterpret_cast<const void* const*>(grads), exp_avg,
                                exp_avg_sq, slow_buffer, args, args ? args->step : nullptr, precision, packed))
    return rc;
  return fused_step(SNB_N_PARAM_TENSORS, nullptr, params, grads, false, args->step, nullptr, exp_avg, exp_avg_sq,
                    slow_buffer, *args, precision, new_activation, packed, reinterpret_cast<cudaStream_t>(stream));
}

int snb_optim_step_amp(float* const* params, float* const* grads, float* exp_avg, float* exp_avg_sq,
                       float* slow_buffer, const SnbOptimArgs* args, const SnbAmpStep* amp, int precision,
                       int new_activation, void* packed, void* stream) {
  const char* who = "snb_optim_step_amp";
  if (int rc = check_amp(who, amp, SNB_N_PARAM_TENSORS)) return rc;
  if (int rc = check_optim_step(who, params, reinterpret_cast<const void* const*>(grads), exp_avg, exp_avg_sq,
                                slow_buffer, args, amp->base, precision, packed))
    return rc;
  return fused_step(SNB_N_PARAM_TENSORS, nullptr, params, grads, false, amp->base, amp, exp_avg, exp_avg_sq,
                    slow_buffer, *args, precision, new_activation, packed, reinterpret_cast<cudaStream_t>(stream));
}

int snb_optim_step_tensors(int n, float* const* params, const float* const* grads, const int64_t* numel,
                           const int* step, float* exp_avg, float* exp_avg_sq, float* slow_buffer,
                           const SnbOptimArgs* args, void* stream) {
  if (int rc = check_optim_tensors("snb_optim_step_tensors", n, params, reinterpret_cast<const void* const*>(grads),
                                   numel, step, exp_avg, exp_avg_sq, slow_buffer, args))
    return rc;
  return fused_step(n, numel, params, grads, false, step, nullptr, exp_avg, exp_avg_sq, slow_buffer, *args, 0, 0,
                    nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int snb_optim_step_tensors_amp(int n, float* const* params, float* const* grads, const int64_t* numel,
                               float* exp_avg, float* exp_avg_sq, float* slow_buffer, const SnbOptimArgs* args,
                               const SnbAmpStep* amp, void* stream) {
  const char* who = "snb_optim_step_tensors_amp";
  if (int rc = check_amp(who, amp, n < 1 ? 1 : (n > SNB_OPTIM_MAX_TENSORS ? SNB_OPTIM_MAX_TENSORS : n))) return rc;
  if (int rc = check_optim_tensors(who, n, params, reinterpret_cast<const void* const*>(grads), numel, amp->base,
                                   exp_avg, exp_avg_sq, slow_buffer, args))
    return rc;
  return fused_step(n, numel, params, grads, false, amp->base, amp, exp_avg, exp_avg_sq, slow_buffer, *args, 0, 0,
                    nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int snb_depth_smooth_forward(const float* idepth, const int64_t* idepth_strides, const float* image,
                             const int64_t* image_strides, int64_t batch, int channels, int height, int width,
                             float* loss, float* loss_ws, void* stream) {
  const char* who = "snb_depth_smooth_forward";
  if (int rc = check_patch_extents(who, batch, channels, height, width, 2)) return rc;
  if (int rc = check_nchw(who, "idepth", idepth, idepth_strides)) return rc;
  if (int rc = check_nchw(who, "image", image, image_strides)) return rc;
  SNB_REQUIRE(loss != nullptr && loss_ws != nullptr, "%s: null loss output / workspace", who);
  return launch_depth_smooth_fwd(idepth, idepth_strides, image, image_strides, batch, channels, height, width, loss,
                                 loss_ws, reinterpret_cast<cudaStream_t>(stream));
}

int snb_depth_smooth_backward(const float* idepth, const int64_t* idepth_strides, const float* image,
                              const int64_t* image_strides, int64_t batch, int channels, int height, int width,
                              const float* g_loss, float* g_idepth, const int64_t* g_idepth_strides, float* g_image,
                              const int64_t* g_image_strides, void* stream) {
  const char* who = "snb_depth_smooth_backward";
  if (int rc = check_patch_extents(who, batch, channels, height, width, 2)) return rc;
  if (int rc = check_nchw(who, "idepth", idepth, idepth_strides)) return rc;
  if (int rc = check_nchw(who, "image", image, image_strides)) return rc;
  SNB_REQUIRE(g_loss != nullptr, "%s: null pointer (g_loss)", who);
  if (g_idepth != nullptr)
    if (int rc = check_nchw(who, "g_idepth", g_idepth, g_idepth_strides)) return rc;
  if (g_image != nullptr)
    if (int rc = check_nchw(who, "g_image", g_image, g_image_strides)) return rc;
  return launch_depth_smooth_bwd(idepth, idepth_strides, image, image_strides, batch, channels, height, width, g_loss,
                                 g_idepth, g_idepth_strides, g_image, g_image_strides,
                                 reinterpret_cast<cudaStream_t>(stream));
}

int snb_ssim_loss_forward(const float* img1, const int64_t* img1_strides, const float* img2,
                          const int64_t* img2_strides, int64_t batch, int channels, int height, int width,
                          int window_size, float max_val, float eps, float* loss, double* coef, float* loss_ws,
                          void* stream) {
  const char* who = "snb_ssim_loss_forward";
  if (window_size != 11) return fail(SNB_ERR_UNSUPPORTED, "%s: only window_size 11 is built (got %d)", who, window_size);
  if (int rc = check_patch_extents(who, batch, channels, height, width, 6)) return rc;
  if (int rc = check_nchw(who, "img1", img1, img1_strides)) return rc;
  if (int rc = check_nchw(who, "img2", img2, img2_strides)) return rc;
  SNB_REQUIRE(loss != nullptr && loss_ws != nullptr, "%s: null loss output / workspace", who);
  return launch_ssim_fwd(img1, img1_strides, img2, img2_strides, batch, channels, height, width, max_val, eps, loss,
                         coef, loss_ws, reinterpret_cast<cudaStream_t>(stream));
}

int snb_ssim_loss_backward(const float* img1, const int64_t* img1_strides, const float* img2,
                           const int64_t* img2_strides, int64_t batch, int channels, int height, int width,
                           const double* coef, const float* g_loss, float* g_img1, const int64_t* g_img1_strides,
                           void* stream) {
  const char* who = "snb_ssim_loss_backward";
  if (int rc = check_patch_extents(who, batch, channels, height, width, 6)) return rc;
  if (int rc = check_nchw(who, "img1", img1, img1_strides)) return rc;
  if (int rc = check_nchw(who, "img2", img2, img2_strides)) return rc;
  if (int rc = check_nchw(who, "g_img1", g_img1, g_img1_strides)) return rc;
  SNB_REQUIRE(coef != nullptr && g_loss != nullptr, "%s: null pointer (coef or g_loss)", who);
  return launch_ssim_bwd(img1, img1_strides, img2, img2_strides, batch, channels, height, width, coef, g_loss, g_img1,
                         g_img1_strides, reinterpret_cast<cudaStream_t>(stream));
}

static int check_warp_extents(const char* who, int64_t n_poses, int height, int width, int occlusion) {
  SNB_REQUIRE(occlusion == SNB_WARP_ZBUFFER || occlusion == SNB_WARP_LAST, "%s: unknown occlusion mode %d", who,
              occlusion);
  SNB_REQUIRE(n_poses >= 1, "%s: needs n_poses >= 1 (got %lld)", who, (long long)n_poses);
  SNB_REQUIRE(height >= 1 && width >= 1 && (int64_t)height * width < (int64_t(1) << 31),
              "%s: needs H, W >= 1 and H*W < 2^31 (got %d x %d)", who, height, width);
  return SNB_OK;
}

size_t snb_forward_warp_workspace_bytes(int64_t n_poses, int height, int width, int occlusion) {
  if (check_warp_extents("snb_forward_warp_workspace_bytes", n_poses, height, width, occlusion)) return 0;
  return forward_warp_workspace_bytes(n_poses, (long long)height * width, occlusion);
}

int snb_forward_warp(const float* image, const float* depth, int height, int width, const double* mats,
                     int64_t n_poses, int occlusion, float* out_rgb, float* out_depth, uint8_t* out_hit,
                     void* workspace, void* stream) {
  const char* who = "snb_forward_warp";
  if (int rc = check_warp_extents(who, n_poses, height, width, occlusion)) return rc;
  SNB_REQUIRE(image != nullptr && depth != nullptr && mats != nullptr, "%s: null pointer (image, depth or mats)", who);
  SNB_REQUIRE(out_rgb != nullptr && out_depth != nullptr && out_hit != nullptr && workspace != nullptr,
              "%s: null pointer (an output or the workspace)", who);
  return launch_forward_warp(image, depth, height, width, mats, n_poses, occlusion, out_rgb, out_depth, out_hit,
                             workspace, reinterpret_cast<cudaStream_t>(stream));
}

int snb_render_forward(const SnbRenderArgs* a, void* stream) {
  SNB_REQUIRE(a != nullptr, "snb_render_forward: null args");
  SNB_REQUIRE(a->n_rays >= 0 && a->n_samples >= 1 && a->n_importance >= 0, "snb_render_forward: bad extents");
  if (a->n_rays == 0) return SNB_OK;
  SNB_REQUIRE(a->rays && a->packed_coarse && a->z_steps && a->z_coarse && a->raw_coarse && a->weights_coarse,
              "snb_render_forward: null coarse-pass pointer");
  SNB_REQUIRE(a->test_time || (a->rgb_coarse && a->depth_coarse), "snb_render_forward: coarse outputs required");
  // rendering.py:330-333 dereferences rgb_coarse, which test_time never defines
  SNB_REQUIRE(!(a->test_time && a->n_importance == 0),
              "snb_render_forward: test_time requires N_importance > 0 (the reference raises UnboundLocalError)");
  const int S = a->n_samples, Ni = a->n_importance;
  int rc;
  if ((rc = snb_sample_coarse(a->rays, a->z_steps, a->perturb_u, a->perturb, a->use_disp, a->n_rays, S,
                              a->z_coarse, stream)))
    return rc;
  if ((rc = snb_field_forward(a->packed_coarse, a->precision, a->rays, a->z_coarse, a->n_rays, S, a->test_time,
                              a->raw_coarse, stream)))
    return rc;
  if (Ni == 0 && a->pixel_scatter != nullptr)     // the coarse pass is the last one: its pixels are the frame's
    return snb_composite_forward_scatter(a->raw_coarse, a->z_coarse, a->rays, a->noise_coarse, a->noise_std, a->white_back,
                                         a->n_rays, S, a->rgb_coarse, a->depth_coarse, a->weights_coarse, a->pixel_scatter,
                                         stream);
  if ((rc = snb_composite_forward(a->raw_coarse, a->test_time ? 1 : 4, a->z_coarse, a->rays, a->noise_coarse,
                                  a->noise_std, a->white_back, a->n_rays, S, a->rgb_coarse, a->depth_coarse,
                                  a->weights_coarse, stream)))
    return rc;
  if (Ni == 0) return SNB_OK;
  SNB_REQUIRE(a->packed_fine && a->z_fine && a->raw_fine && a->rgb_fine && a->depth_fine && a->weights_fine,
              "snb_render_forward: null fine-pass pointer");
  const bool det = !(a->perturb > 0.f);
  const float* u = det ? a->u_steps : a->pdf_u;
  SNB_REQUIRE(u != nullptr, "snb_render_forward: %s required", det ? "u_steps" : "pdf_u");
  if ((rc = snb_importance_merge(a->z_coarse, a->weights_coarse, u, det ? 0 : Ni, a->n_rays, S, Ni, 1e-5f,
                                 a->z_fine, nullptr, stream)))
    return rc;
  if ((rc = snb_field_forward(a->packed_fine, a->precision, a->rays, a->z_fine, a->n_rays, S + Ni, 0, a->raw_fine,
                              stream)))
    return rc;
  if (a->pixel_scatter != nullptr)
    return snb_composite_forward_scatter(a->raw_fine, a->z_fine, a->rays, a->noise_fine, a->noise_std, a->white_back,
                                         a->n_rays, S + Ni, a->rgb_fine, a->depth_fine, a->weights_fine, a->pixel_scatter,
                                         stream);
  return snb_composite_forward(a->raw_fine, 4, a->z_fine, a->rays, a->noise_fine, a->noise_std, a->white_back,
                               a->n_rays, S + Ni, a->rgb_fine, a->depth_fine, a->weights_fine, stream);
}

int snb_diff_augment_forward(const int* ops, int n_ops, const SnbDiffAugDraws* draws, const float* input,
                             const int64_t* in_strides, int n, int channels, int height, int width, float* out,
                             const int64_t* out_strides, float* workspace, void* stream) {
  const char* who = "snb_diff_augment_forward";
  if (int rc = check_diff_augment(who, ops, n_ops, draws, input, in_strides, n, channels, height, width, out,
                                  out_strides, workspace))
    return rc;
  const SnbDiffAugDraws none{};
  return launch_diff_augment(false, ops, n_ops, draws ? *draws : none, input, in_strides, n, channels, height, width,
                             out, out_strides, workspace, reinterpret_cast<cudaStream_t>(stream));
}

int snb_diff_augment_backward(const int* ops, int n_ops, const SnbDiffAugDraws* draws, const float* d_out,
                              const int64_t* d_out_strides, int n, int channels, int height, int width, float* d_input,
                              const int64_t* d_in_strides, float* workspace, void* stream) {
  const char* who = "snb_diff_augment_backward";
  if (int rc = check_diff_augment(who, ops, n_ops, draws, d_out, d_out_strides, n, channels, height, width, d_input,
                                  d_in_strides, workspace))
    return rc;
  const SnbDiffAugDraws none{};
  return launch_diff_augment(true, ops, n_ops, draws ? *draws : none, d_out, d_out_strides, n, channels, height,
                             width, d_input, d_in_strides, workspace, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
