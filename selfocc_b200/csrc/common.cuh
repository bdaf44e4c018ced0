// Shared device/host helpers of libselfocc_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include "../../include/selfocc_b200.h"

namespace so {

extern thread_local int g_last_cuda_error;
void note_launch(int n = 1);

inline int check_cuda(cudaError_t e) {
  if (e != cudaSuccess) {
    g_last_cuda_error = (int)e;
    return SO_ERR_CUDA;
  }
  return SO_OK;
}
// Launch-error check without synchronising.
inline int check_launch() { return check_cuda(cudaGetLastError()); }

// SM count of the current device (cached per device ordinal): sizes the persistent grids of the GEMM and the decode and
// caps the grid-stride kernels, so a 132-SM H100 SXM, a 114-SM H100 PCIe or a partitioned device each get one wave.
int num_sms();

// cudaFuncSetAttribute is PER DEVICE: a process-wide `static bool` would leave the second GPU of a multi-device process
// without its opt-in shared-memory size.  One bit per device ordinal; setting the attribute twice is harmless, so the
// check-then-set race between host threads is benign.
struct PerDeviceOnce {
  std::atomic<uint64_t> done{0};
  template <typename F>
  int run(F&& set_attr) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return SO_ERR_CUDA;
    const uint64_t bit = 1ull << (dev & 63);
    if (done.load(std::memory_order_acquire) & bit) return SO_OK;
    int rc = set_attr();
    if (rc) return rc;
    done.fetch_or(bit, std::memory_order_release);
    return SO_OK;
  }
};

// Device-time bracket around the dominant kernel of an entry point (no-op unless so_profile_enable(1)).
void prof_begin(int tag, cudaStream_t st);
void prof_end(int tag, cudaStream_t st);
struct ProfScope {
  int tag; cudaStream_t st;
  ProfScope(int t, cudaStream_t s) : tag(t), st(s) { prof_begin(tag, st); }
  ~ProfScope() { prof_end(tag, st); }
};

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// ---- metre -> grid, one axis (mappings.py:97-150).  Device copy of so_axis_map with the two slopes
// precomputed on the host.
struct AxisMap {
  float start, range0, size0, offset, k0, k1;  // k0 = size0/range0, k1 = size1/range1 (0: no outer ring)
};

inline AxisMap make_axis(const so_axis_map& a) {
  AxisMap m;
  m.start = a.start;
  m.range0 = a.range0;
  m.size0 = a.size0;
  m.offset = a.offset;
  m.k0 = a.size0 / a.range0;
  m.k1 = (a.size1 > 0.f && a.range1 > 0.f) ? a.size1 / a.range1 : 0.f;
  return m;
}

// grid coordinate and d(grid)/d(metre) of one axis
__device__ __forceinline__ float axis_m2g(const AxisMap& a, float m, float& slope) {
  float c = m - a.start;
  float v = fabsf(c);
  float g;
  if (a.k1 > 0.f && v > a.range0) {
    g = a.size0 + (v - a.range0) * a.k1;
    slope = a.k1;
  } else {
    g = v * a.k0;
    slope = a.k0;
  }
  return copysignf(g, c) + a.offset;
}

struct VolumeDev {
  const float* sdf;   // [H][W][zpitch]
  const float* feat;  // [H][W][Z][feat_pitch] or nullptr
  int H, W, Z, zpitch, n_feat, feat_pitch;
  AxisMap ax[3];      // h (metre y), w (metre x), d (metre z)
};

inline VolumeDev make_volume(const so_volume_desc& d, const float* sdf, const float* feat) {
  VolumeDev v;
  v.sdf = sdf;
  v.feat = feat;
  v.H = d.H; v.W = d.W; v.Z = d.Z; v.zpitch = d.zpitch;
  v.n_feat = d.n_feat; v.feat_pitch = d.feat_pitch;
  for (int i = 0; i < 3; ++i) v.ax[i] = make_axis(d.axis[i]);
  return v;
}

inline int validate_volume(const so_volume_desc* d) {
  if (!d) return SO_ERR_INVALID_ARG;
  if (d->H < 1 || d->W < 1 || d->Z < 1 || d->zpitch < d->Z) return SO_ERR_INVALID_ARG;
  // the gather kernels index the sdf volume with 32-bit offsets
  if ((int64_t)d->H * d->W * d->zpitch >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;
  if (d->n_feat < 0 || (d->n_feat > 0 && (d->feat_pitch < d->n_feat || d->feat_pitch % 4))) return SO_ERR_INVALID_ARG;
  for (int i = 0; i < 3; ++i)
    if (!(d->axis[i].range0 > 0.f) || !(d->axis[i].size0 > 0.f)) return SO_ERR_INVALID_ARG;
  return SO_OK;
}

// Trilinear tap set of one sample: cell base indices, fractions and in-range flags, zero padding
// outside [0, size-1] exactly like F.grid_sample(padding_mode='zeros', align_corners=True).
struct Taps {
  int h0, w0, z0;
  float fh, fw, fz;
  float mh0, mh1, mw0, mw1, mz0, mz1;  // 1 if the corner index is inside the volume else 0
};

__device__ __forceinline__ Taps make_taps(const VolumeDev& v, float gh, float gw, float gd) {
  Taps t;
  float fl_h = floorf(gh), fl_w = floorf(gw), fl_z = floorf(gd);
  t.fh = gh - fl_h; t.fw = gw - fl_w; t.fz = gd - fl_z;
  // clamp before the int conversion so far-out samples cannot overflow
  int h0 = (int)fminf(fmaxf(fl_h, -2.f), (float)v.H);
  int w0 = (int)fminf(fmaxf(fl_w, -2.f), (float)v.W);
  int z0 = (int)fminf(fmaxf(fl_z, -2.f), (float)v.Z);
  t.mh0 = (h0 >= 0 && h0 < v.H) ? 1.f : 0.f;
  t.mh1 = (h0 + 1 >= 0 && h0 + 1 < v.H) ? 1.f : 0.f;
  t.mw0 = (w0 >= 0 && w0 < v.W) ? 1.f : 0.f;
  t.mw1 = (w0 + 1 >= 0 && w0 + 1 < v.W) ? 1.f : 0.f;
  t.mz0 = (z0 >= 0 && z0 < v.Z) ? 1.f : 0.f;
  t.mz1 = (z0 + 1 >= 0 && z0 + 1 < v.Z) ? 1.f : 0.f;
  t.h0 = h0; t.w0 = w0; t.z0 = z0;
  return t;
}

}  // namespace so
