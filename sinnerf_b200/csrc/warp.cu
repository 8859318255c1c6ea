// warp.cu -- SinNeRF's depth-warped pseudo-view labels: the reference view splatted into P source views through its
// depth, nearest-depth-wins ("zbuffer", the LLFF / DTU datasets' painter loop) or last-writer-wins ("last", the
// blender datasets' numpy scatter).  DESIGN.md section 4.4 states the arithmetic and the occlusion rule.
//
// Three launches per call, every pose of the chunk in each (blockIdx.y = pose):
//   zero pass  (zbuffer only)  L[t]   = max index of the sources with zf == 0 that land on t
//   splat pass                 key[t] = min over the sources with (index > L[t] or zf < 0) of ordered(zf) << 32 | index
//                              (zbuffer), or the max source index (last)
//   resolve pass               one thread per target pixel: winner -> rgb, depth, hit
// Min and max do not depend on arrival order, so the result is the same bits on every run.  Sources that land on
// the same target within a warp are combined with __match_any_sync + __reduce_{min,max}_sync before the one atomic
// of their group: every hole pixel (depth 0) projects to the reference camera's centre, and that group can be more
// than half of a frame.
#include "common.cuh"

namespace snb {

namespace {

constexpr unsigned kFullMask = 0xffffffffu;
constexpr int kThreads = 256;
constexpr int kMaxGridY = 65535;
constexpr unsigned long long kNoKey = ~0ull;

struct WarpArgs {
  const float* image;    // (H*W, 3)
  const float* depth;    // (H*W)
  const double* mats;    // (P, 3, 4), this chunk's first pose at index 0
  int H, W;
  long long hw;
  float* rgb;            // (P, H*W, 3)
  float* zout;           // (P, H*W)
  unsigned char* hit;    // (P, H*W)
  unsigned long long* key;   // (P, H*W): zbuffer keys
  int* slot;                 // (P, H*W): zbuffer L, or the last mode's winning index
};

// The contract's projection of source pixel `s` through M (3x4, fp64): every product and sum rounded on its own
// (no FMA contraction), then x' = X / Z, y' likewise (Z == 0: divided by 1e-9), floor, clamp to the frame.  Returns
// false for a source the warp skips: depth not finite, or a NaN coordinate.
__device__ __forceinline__ bool project(const double* __restrict__ M, const float* __restrict__ depth, int W, int H,
                                        long long s, int* target, float* zf) {
  const double d = (double)__ldg(depth + s);
  if (!isfinite(d)) return false;
  const int r = (int)(s / W), c = (int)(s - (long long)r * W);
  const double u = __dmul_rn((double)c, d), v = __dmul_rn((double)r, d);
  double P[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double* m = M + 4 * k;
    P[k] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[0], u), __dmul_rn(m[1], v)), __dmul_rn(m[2], d)), m[3]);
  }
  // divide by Z, and by 1e-9 only where Z == 0: the reference's fp32 `Z + 1e-9` leaves every |Z| >= 2^-5 unchanged,
  // while an fp64 `Z + 1e-9` would pull every exact-integer coordinate (any pose that keeps a row or column, the
  // identity included) just below the integer, and floor would shift it by a pixel
  const double zd = P[2] != 0.0 ? P[2] : 1e-9;
  const double x = __ddiv_rn(P[0], zd), y = __ddiv_rn(P[1], zd);
  if (isnan(x) || isnan(y)) return false;
  // clamp in floating point, so +-inf lands on the border before the conversion to int
  const int col = (int)fmin(fmax(floor(x), 0.0), (double)(W - 1));
  const int row = (int)fmin(fmax(floor(y), 0.0), (double)(H - 1));
  *target = row * W + col;
  *zf = __double2float_rn(P[2]);
  return true;
}

// float -> uint32 whose unsigned order is the float order (for non-NaN; -0 sorts below +0, but zeros never compete)
__device__ __forceinline__ unsigned ordered_bits(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float from_ordered_bits(unsigned o) {
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7fffffffu) : ~o);
}

// Each lane names a target (or -1: nothing to contribute); returns the lanes of the warp that name the same target,
// and whether this lane is the group's leader (its lowest lane).  Every lane of the warp must call it.
__device__ __forceinline__ unsigned target_group(int target, bool* leader) {
  const unsigned grp = __match_any_sync(kFullMask, target);
  *leader = (int)(threadIdx.x & 31) == __ffs(grp) - 1;
  return grp;
}

__global__ void __launch_bounds__(kThreads) warp_zero_kernel(WarpArgs a) {
  const long long s = (long long)blockIdx.x * kThreads + threadIdx.x;
  const int p = blockIdx.y;
  int t = -1;
  float zf = 1.0f;
  if (s < a.hw && !project(a.mats + 12 * p, a.depth, a.W, a.H, s, &t, &zf)) t = -1;
  if (zf != 0.0f) t = -1;
  bool leader;
  const unsigned grp = target_group(t, &leader);
  const unsigned last = __reduce_max_sync(grp, (unsigned)s);
  if (t >= 0 && leader) atomicMax(a.slot + p * a.hw + t, (int)last);
}

template <bool kZbuffer>
__global__ void __launch_bounds__(kThreads) warp_splat_kernel(WarpArgs a) {
  const long long s = (long long)blockIdx.x * kThreads + threadIdx.x;
  const int p = blockIdx.y;
  int t = -1;
  float zf = 0.0f;
  if (s < a.hw && !project(a.mats + 12 * p, a.depth, a.W, a.H, s, &t, &zf)) t = -1;
  if (kZbuffer && t >= 0) {
    // the painter loop's empty test (`s == 0`) restarts at the last zero-depth source L: only later sources and
    // negative depths can still win; zeros themselves are excluded because no zero comes after L
    const int L = __ldcg(a.slot + p * a.hw + t);
    if (!(s > L || zf < 0.0f)) t = -1;
  }
  bool leader;
  const unsigned grp = target_group(t, &leader);
  if (kZbuffer) {
    const unsigned zb = t >= 0 ? ordered_bits(zf) : ~0u;
    const unsigned zmin = __reduce_min_sync(grp, zb);
    const unsigned imin = __reduce_min_sync(grp, zb == zmin ? (unsigned)s : ~0u);
    if (t >= 0 && leader) {
      unsigned long long* k = a.key + p * a.hw + t;
      const unsigned long long want = (unsigned long long)zmin << 32 | imin;
      // keys only decrease, so a stale read can only be larger: skipping on it is safe
      if (want < __ldcg(k)) atomicMin(k, want);
    }
  } else {
    const unsigned last = __reduce_max_sync(grp, (unsigned)s);
    if (t >= 0 && leader) atomicMax(a.slot + p * a.hw + t, (int)last);
  }
}

template <bool kZbuffer>
__global__ void __launch_bounds__(kThreads) warp_resolve_kernel(WarpArgs a) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (t >= a.hw) return;
  const int p = blockIdx.y;
  const long long o = p * a.hw + t;
  long long win = -1;
  float zf = 0.0f;
  bool have_z = false;
  if (kZbuffer) {
    const unsigned long long k = a.key[o];
    if (k != kNoKey) {
      win = (long long)(k & 0xffffffffu);
      zf = from_ordered_bits((unsigned)(k >> 32));
      have_z = true;
    } else {
      win = a.slot[o];   // the last zero-depth source, or -1
    }
  } else {
    win = a.slot[o];
  }
  float r = 0.0f, g = 0.0f, b = 0.0f;
  if (win >= 0) {
    if (!have_z) {     // recompute the winner's depth (keeps the sign of a zero)
      int tt;
      project(a.mats + 12 * p, a.depth, a.W, a.H, win, &tt, &zf);
    }
    r = __ldg(a.image + 3 * win);
    g = __ldg(a.image + 3 * win + 1);
    b = __ldg(a.image + 3 * win + 2);
  }
  float* out = a.rgb + 3 * o;
  out[0] = r;
  out[1] = g;
  out[2] = b;
  a.zout[o] = win >= 0 ? zf : 0.0f;
  a.hit[o] = win >= 0 ? 1 : 0;
}

}  // namespace

size_t forward_warp_workspace_bytes(long long n_poses, long long hw, int occlusion) {
  return (size_t)n_poses * (size_t)hw * (occlusion == SNB_WARP_ZBUFFER ? sizeof(unsigned long long) + sizeof(int)
                                                                       : sizeof(int));
}

int launch_forward_warp(const float* image, const float* depth, int H, int W, const double* mats, long long n_poses,
                        int occlusion, float* rgb, float* zout, unsigned char* hit, void* workspace, cudaStream_t st) {
  const long long hw = (long long)H * W;
  const bool zbuf = occlusion == SNB_WARP_ZBUFFER;
  // workspace: keys (zbuffer only), then one int slot per target; all-ones = no key / slot -1
  cudaError_t e = cudaMemsetAsync(workspace, 0xff, forward_warp_workspace_bytes(n_poses, hw, occlusion), st);
  if (e != cudaSuccess) return fail(SNB_ERR_CUDA, "snb_forward_warp: cudaMemsetAsync: %s", cudaGetErrorString(e));
  unsigned long long* keys = zbuf ? static_cast<unsigned long long*>(workspace) : nullptr;
  int* slots = zbuf ? reinterpret_cast<int*>(keys + n_poses * hw) : static_cast<int*>(workspace);
  const unsigned gx = (unsigned)((hw + kThreads - 1) / kThreads);
  for (long long p0 = 0; p0 < n_poses; p0 += kMaxGridY) {
    const int np = (int)(n_poses - p0 < kMaxGridY ? n_poses - p0 : kMaxGridY);
    const WarpArgs a{image, depth, mats + 12 * p0, H, W, hw, rgb + 3 * p0 * hw, zout + p0 * hw, hit + p0 * hw,
                     keys ? keys + p0 * hw : nullptr, slots + p0 * hw};
    const dim3 grid(gx, (unsigned)np);
    if (zbuf) {
      warp_zero_kernel<<<grid, kThreads, 0, st>>>(a);
      if (int rc = check_launch("warp_zero_kernel")) return rc;
      warp_splat_kernel<true><<<grid, kThreads, 0, st>>>(a);
      if (int rc = check_launch("warp_splat_kernel<zbuffer>")) return rc;
      warp_resolve_kernel<true><<<grid, kThreads, 0, st>>>(a);
      if (int rc = check_launch("warp_resolve_kernel<zbuffer>")) return rc;
    } else {
      warp_splat_kernel<false><<<grid, kThreads, 0, st>>>(a);
      if (int rc = check_launch("warp_splat_kernel<last>")) return rc;
      warp_resolve_kernel<false><<<grid, kThreads, 0, st>>>(a);
      if (int rc = check_launch("warp_resolve_kernel<last>")) return rc;
    }
  }
  return SNB_OK;
}

}  // namespace snb
