// Occupancy evaluation (eval_iou.py:196-270, eval_iou_kitti.py:160-190) straight from the decoded volume:
//   so_occ_lattice_labels  occ / sem labels on the uniform lattice of NeuSHead.get_uniform_sdf (neus_head.py:265-293)
//   so_occ_sample_labels   the Occ3D branch: that lattice resampled by F.grid_sample at arbitrary points, the lattice values
//                          evaluated on the fly (the lattice itself is never stored)
//   so_occ_confusion       the confusion matrix every counter of MeanIoU / SSCMetrics is derived from
// Lattice values are the field query of so_field_query (same device functions, same operands, same rounding), so the
// labels equal thresholding / arg-maxing forward_occ's outputs without materialising them.
#include "render_common.cuh"
#include <math.h>

namespace so {

struct LatticeDev {
  const float *xs, *ys, *zs;  // lattice axes in metres: W = nx (x), H = ny (y), D = nz (z)
  int nx, ny, nz;
};

__device__ __forceinline__ Taps lattice_taps(const VolumeDev& V, const LatticeDev& L, int iy, int ix, int iz) {
  float kh, kw, kd;
  float gh = axis_m2g(V.ax[0], __ldg(L.ys + iy), kh);
  float gw = axis_m2g(V.ax[1], __ldg(L.xs + ix), kw);
  float gd = axis_m2g(V.ax[2], __ldg(L.zs + iz), kd);
  return make_taps(V, gh, gw, gd);
}

__device__ __forceinline__ float tap_sdf(const VolumeDev& V, const Taps& t) {
  float s, dgh, dgw, dgd;
  gather_sdf(V, t, s, dgh, dgw, dgd);
  return s;
}

// running first-maximum, NaN counting as the maximum (torch.argmax)
__device__ __forceinline__ void argmax_update(float v, int c, float& best, int& arg) {
  if (v > best || (isnan(v) && !isnan(best))) { best = v; arg = c; }
}

__device__ __forceinline__ uint8_t sem_label(int arg, const uint8_t* __restrict__ lut) {
  return lut ? __ldg(lut + arg) : (uint8_t)arg;
}

// argmax over feature channels [c0, c0 + n) of one lattice point
__device__ __forceinline__ int lattice_argmax(const VolumeDev& V, const Taps& t, int c0, int n) {
  float best = -INFINITY;
  int arg = 0, c = 0;
  for (; c + 4 <= n; c += 4) {
    float v[4];
    gather_feat<4>(V, t, c0 + c, v);
#pragma unroll
    for (int i = 0; i < 4; ++i) argmax_update(v[i], c + i, best, arg);
  }
  for (; c < n; ++c) {
    float v[1];
    gather_feat<1>(V, t, c0 + c, v);
    argmax_update(v[0], c, best, arg);
  }
  return arg;
}

__global__ void __launch_bounds__(256) occ_lattice_kernel(VolumeDev V, LatticeDev L, float thresh, int c0, int n_sem,
                                                          const uint8_t* __restrict__ lut, uint8_t* __restrict__ occ,
                                                          uint8_t* __restrict__ sem) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= L.ny * L.nx * L.nz) return;
  int iz = i % L.nz, r = i / L.nz;
  int ix = r % L.nx, iy = r / L.nx;
  Taps t = lattice_taps(V, L, iy, ix, iz);
  bool o = tap_sdf(V, t) <= thresh;
  occ[i] = o;
  if (sem) sem[i] = o ? sem_label(lattice_argmax(V, t, c0, n_sem), lut) : 0;   // logits gathered only where occupied
}

// One resampled point: F.grid_sample(lattice[None, None], u[[2, 0, 1]] * 2 - 1, bilinear, zeros, align_corners=True) with
// ATen's arithmetic (grid_sampler_3d: unnormalise ((g + 1) / 2) * (size - 1), corner weights as products of the three
// distances).  Grid x / y / z index the lattice's z / x / y, so ATen's corner order tnw, tne, tsw, tse, bnw, bne, bsw, bse
// is k = (dy << 2) | (dx << 1) | dz below.
struct SampleCell {
  int y0, x0, z0;           // lattice corner (y, x, z) of tnw
  unsigned inside;          // bit k: corner k lies inside the lattice (zero padding drops the others)
  float wz[2], wx[2], wy[2];  // distances to the far corner along each axis
  // ATen's weight of corner k: (z distance * x distance) * y distance (grid x, y, z order)
  __device__ __forceinline__ float w(int k) const {
    return __fmul_rn(__fmul_rn((k & 1) ? wz[1] : wz[0], ((k >> 1) & 1) ? wx[1] : wx[0]), (k >> 2) ? wy[1] : wy[0]);
  }
};

__device__ __forceinline__ float unnormalise(float u, int size) {
  float g = __fsub_rn(__fmul_rn(u, 2.f), 1.f);
  return __fmul_rn(__fdiv_rn(__fadd_rn(g, 1.f), 2.f), (float)(size - 1));
}

__device__ __forceinline__ SampleCell sample_cell(const LatticeDev& L, float u0, float u1, float u2) {
  float fz = unnormalise(u2, L.nz), fx = unnormalise(u0, L.nx), fy = unnormalise(u1, L.ny);
  float z0f = floorf(fz), x0f = floorf(fx), y0f = floorf(fy);
  SampleCell c;
  // clamp before the int conversion so far-out points cannot overflow (their taps are all outside anyway)
  c.z0 = (int)fminf(fmaxf(z0f, -2.f), (float)L.nz);
  c.x0 = (int)fminf(fmaxf(x0f, -2.f), (float)L.nx);
  c.y0 = (int)fminf(fmaxf(y0f, -2.f), (float)L.ny);
  c.wz[0] = __fsub_rn(__fadd_rn(z0f, 1.f), fz); c.wz[1] = __fsub_rn(fz, z0f);
  c.wx[0] = __fsub_rn(__fadd_rn(x0f, 1.f), fx); c.wx[1] = __fsub_rn(fx, x0f);
  c.wy[0] = __fsub_rn(__fadd_rn(y0f, 1.f), fy); c.wy[1] = __fsub_rn(fy, y0f);
  c.inside = 0u;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int dy = k >> 2, dx = (k >> 1) & 1, dz = k & 1;
    int y = c.y0 + dy, x = c.x0 + dx, z = c.z0 + dz;
    if (y >= 0 && y < L.ny && x >= 0 && x < L.nx && z >= 0 && z < L.nz) c.inside |= 1u << k;
  }
  return c;
}

// interpolated feature channels [c0, c0 + CH) of one resampled point; the 8 lattice corners are field queries
template <int CH>
__device__ __forceinline__ void sample_feat(const VolumeDev& V, const LatticeDev& L, const SampleCell& c, int c0, float out[CH]) {
#pragma unroll
  for (int i = 0; i < CH; ++i) out[i] = 0.f;
#pragma unroll 1
  for (int k = 0; k < 8; ++k) {
    if (!((c.inside >> k) & 1u)) continue;
    Taps t = lattice_taps(V, L, c.y0 + (k >> 2), c.x0 + ((k >> 1) & 1), c.z0 + (k & 1));
    float v[CH];
    gather_feat<CH>(V, t, c0, v);
    const float wk = c.w(k);
#pragma unroll
    for (int i = 0; i < CH; ++i) out[i] = fmaf(v[i], wk, out[i]);
  }
}

__global__ void __launch_bounds__(256) occ_sample_kernel(VolumeDev V, LatticeDev L, const float* __restrict__ pts, long long m,
                                                         float thresh, int c0, int n_sem, const uint8_t* __restrict__ lut,
                                                         uint8_t* __restrict__ occ, uint8_t* __restrict__ sem) {
  long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (p >= m) return;
  SampleCell c = sample_cell(L, pts[3 * p], pts[3 * p + 1], pts[3 * p + 2]);
  float s = 0.f;
#pragma unroll 1
  for (int k = 0; k < 8; ++k) {
    if (!((c.inside >> k) & 1u)) continue;
    s = fmaf(tap_sdf(V, lattice_taps(V, L, c.y0 + (k >> 2), c.x0 + ((k >> 1) & 1), c.z0 + (k & 1))), c.w(k), s);
  }
  const bool o = s <= thresh;
  occ[p] = o;
  if (!sem) return;
  uint8_t label = 0;
  if (o) {                                    // logits interpolated only where occupied
    float best = -INFINITY;
    int arg = 0, ch = 0;
    for (; ch + 4 <= n_sem; ch += 4) {
      float v[4];
      sample_feat<4>(V, L, c, c0 + ch, v);
#pragma unroll
      for (int i = 0; i < 4; ++i) argmax_update(v[i], ch + i, best, arg);
    }
    for (; ch < n_sem; ++ch) {
      float v[1];
      sample_feat<1>(V, L, c, c0 + ch, v);
      argmax_update(v[0], ch, best, arg);
    }
    label = sem_label(arg, lut);
  }
  sem[p] = label;
}

// Confusion matrix counts[(n_cls + 1) * g + p] over the elements with mask != 0 and gt != ignore; labels >= n_cls land in
// bin n_cls.  Up to 109 classes the bins live in per-warp shared-memory histograms (32-bit: a block sees < 2^32 elements)
// flushed with 64-bit integer atomics; above that they are counted with global atomics.  Integer additions commute, so
// the result does not depend on their order.
constexpr int kConfBlock = 256;
constexpr int kConfSmemBytes = 48 * 1024;

template <typename T>
__device__ __forceinline__ void conf_add(T* h, unsigned g, unsigned p, int n_cls, int ignore, unsigned mk) {
  if (!mk || (int)g == ignore) return;
  atomicAdd(h + min((int)g, n_cls) * (n_cls + 1) + min((int)p, n_cls), (T)1);
}

template <bool SHARED>
__global__ void __launch_bounds__(kConfBlock) occ_confusion_kernel(const uint8_t* __restrict__ pred, const uint8_t* __restrict__ gt,
                                                                   const uint8_t* __restrict__ mask, long long n, int n_cls,
                                                                   int ignore, int copies, bool vec4,
                                                                   unsigned long long* __restrict__ counts) {
  extern __shared__ unsigned hist[];
  const int nb = (n_cls + 1) * (n_cls + 1);
  if (SHARED) {
    for (int i = threadIdx.x; i < nb * copies; i += blockDim.x) hist[i] = 0u;
    __syncthreads();
  }
  auto* h = SHARED ? (void*)(hist + ((threadIdx.x >> 5) % copies) * nb) : (void*)counts;
  auto add = [&](unsigned g, unsigned p, unsigned mk) {
    if (SHARED) conf_add((unsigned*)h, g, p, n_cls, ignore, mk);
    else conf_add((unsigned long long*)h, g, p, n_cls, ignore, mk);
  };
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long done = 0;
  if (vec4) {
    const long long n4 = n >> 2;
    for (long long q = tid; q < n4; q += stride) {
      uchar4 pv = __ldg(reinterpret_cast<const uchar4*>(pred) + q), gv = __ldg(reinterpret_cast<const uchar4*>(gt) + q);
      uchar4 mv = mask ? __ldg(reinterpret_cast<const uchar4*>(mask) + q) : make_uchar4(1, 1, 1, 1);
      add(gv.x, pv.x, mv.x); add(gv.y, pv.y, mv.y); add(gv.z, pv.z, mv.z); add(gv.w, pv.w, mv.w);
    }
    done = n4 << 2;
  }
  for (long long i = done + tid; i < n; i += stride) add(__ldg(gt + i), __ldg(pred + i), mask ? __ldg(mask + i) : 1u);
  if (SHARED) {
    __syncthreads();
    for (int b = threadIdx.x; b < nb; b += blockDim.x) {
      unsigned long long s = 0;
      for (int c = 0; c < copies; ++c) s += hist[c * nb + b];
      if (s) atomicAdd(counts + b, s);
    }
  }
}

int check_lattice(const so_volume_desc* vol_host, const float* vol_sdf, const float* vol_feat, const float* xs, int32_t nx,
                  const float* ys, int32_t ny, const float* zs, int32_t nz, int32_t sem_begin, int32_t n_sem, const uint8_t* occ,
                  const uint8_t* sem) {
  if (!vol_sdf || !xs || !ys || !zs || !occ || nx < 1 || ny < 1 || nz < 1) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(vol_host);
  if (rc) return rc;
  if ((int64_t)nx * ny * nz >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;   // 32-bit lattice indices
  if (sem && (!vol_feat || n_sem < 1 || sem_begin < 0 || (int64_t)sem_begin + n_sem > vol_host->n_feat))
    return SO_ERR_INVALID_ARG;
  return SO_OK;
}

}  // namespace so

using namespace so;

extern "C" int so_occ_lattice_labels(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* xs,
                                     int32_t nx, const float* ys, int32_t ny, const float* zs, int32_t nz, float thresh,
                                     int32_t sem_begin, int32_t n_sem, const uint8_t* lut, uint8_t* occ, uint8_t* sem,
                                     void* stream) {
  int rc = check_lattice(vol_host, vol_sdf, vol_feat, xs, nx, ys, ny, zs, nz, sem_begin, n_sem, occ, sem);
  if (rc) return rc;
  VolumeDev V = make_volume(*vol_host, vol_sdf, vol_feat);
  LatticeDev L{xs, ys, zs, nx, ny, nz};
  const int64_t total = (int64_t)nx * ny * nz;
  occ_lattice_kernel<<<(unsigned)ceil_div64(total, 256), 256, 0, (cudaStream_t)stream>>>(V, L, thresh, sem_begin, n_sem, lut, occ, sem);
  note_launch(1);
  return check_launch();
}

extern "C" int so_occ_sample_labels(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* xs,
                                    int32_t nx, const float* ys, int32_t ny, const float* zs, int32_t nz, const float* points,
                                    int64_t m, float thresh, int32_t sem_begin, int32_t n_sem, const uint8_t* lut, uint8_t* occ,
                                    uint8_t* sem, void* stream) {
  if (!points || m < 1) return SO_ERR_INVALID_ARG;
  int rc = check_lattice(vol_host, vol_sdf, vol_feat, xs, nx, ys, ny, zs, nz, sem_begin, n_sem, occ, sem);
  if (rc) return rc;
  VolumeDev V = make_volume(*vol_host, vol_sdf, vol_feat);
  LatticeDev L{xs, ys, zs, nx, ny, nz};
  occ_sample_kernel<<<(unsigned)ceil_div64(m, 256), 256, 0, (cudaStream_t)stream>>>(V, L, points, m, thresh, sem_begin, n_sem, lut,
                                                                                    occ, sem);
  note_launch(1);
  return check_launch();
}

extern "C" int so_occ_confusion(const uint8_t* pred, const uint8_t* gt, const uint8_t* mask, int64_t n, int32_t n_cls,
                                int32_t ignore, int64_t* counts, void* stream) {
  if (!pred || !gt || !counts || n < 1 || n_cls < 1 || n_cls > 255 || ignore < -1 || ignore > 255) return SO_ERR_INVALID_ARG;
  const int nb = (n_cls + 1) * (n_cls + 1);
  const int max_copies = kConfSmemBytes / (int)(nb * sizeof(unsigned));
  const int copies = max_copies < kConfBlock / 32 ? max_copies : kConfBlock / 32;
  const bool vec4 = ((uintptr_t)pred | (uintptr_t)gt | (uintptr_t)mask) % 4 == 0;
  int64_t grid = ceil_div64(n, (int64_t)kConfBlock * 16);
  if (grid > 4 * (int64_t)num_sms()) grid = 4 * (int64_t)num_sms();
  const int64_t min_grid = ceil_div64(n, (int64_t)1 << 31);        // 32-bit per-block bins
  if (grid < min_grid) grid = min_grid;
  unsigned long long* cnt = reinterpret_cast<unsigned long long*>(counts);
  cudaStream_t st = (cudaStream_t)stream;
  if (copies >= 1)
    occ_confusion_kernel<true><<<(unsigned)grid, kConfBlock, copies * nb * sizeof(unsigned), st>>>(pred, gt, mask, n, n_cls, ignore,
                                                                                                 copies, vec4, cnt);
  else
    occ_confusion_kernel<false><<<(unsigned)grid, kConfBlock, 0, st>>>(pred, gt, mask, n, n_cls, ignore, 0, vec4, cnt);
  note_launch(1);
  return check_launch();
}
