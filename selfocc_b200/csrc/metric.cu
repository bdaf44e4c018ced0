// Device-side depth evaluation (SURVEY.md 8f-3): the DepthMetric step (utils/metric_util.py:247-279,311-349) and the
// per-source loop body of eval_novel_depth.py:159-208.  Rendered depth maps are sampled at the LiDAR pixel locations with
// F.grid_sample(bilinear, padding_mode='border', align_corners=True) and reduced to the seven error sums per camera,
// without the boolean-mask indexing (a host sync per camera) of the reference.
#include "common.cuh"
#include <math.h>

namespace so {

// F.grid_sample(pred[None, None], loc * 2 - 1, bilinear, padding_mode='border', align_corners=True) of one depth map
// p [h, w] at one location (lx, ly) in [0, 1]; metric_util.py:319-324 and eval_novel_depth.py:176-182 both sample this way.
// grid = loc * 2 - 1; ATen unnormalise (align_corners): ((g + 1) / 2) * (size - 1); border clip.
__device__ __forceinline__ float depth_sample_border(const float* __restrict__ p, int h, int w, float lx, float ly) {
  float gx = __fsub_rn(__fmul_rn(lx, 2.f), 1.f), gy = __fsub_rn(__fmul_rn(ly, 2.f), 1.f);
  float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.f), 2.f), (float)(w - 1));
  float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.f), 2.f), (float)(h - 1));
  ix = fminf((float)(w - 1), fmaxf(ix, 0.f));
  iy = fminf((float)(h - 1), fmaxf(iy, 0.f));
  float x0f = floorf(ix), y0f = floorf(iy);
  int x0 = (int)x0f, y0 = (int)y0f;
  float tx = __fsub_rn(ix, x0f), ty = __fsub_rn(iy, y0f);               // ix - ix_nw
  float ux = __fsub_rn(__fadd_rn(x0f, 1.f), ix), uy = __fsub_rn(__fadd_rn(y0f, 1.f), iy);   // ix_se - ix
  bool xb = x0 + 1 < w, yb = y0 + 1 < h;
  float nw = p[y0 * w + x0], ne = xb ? p[y0 * w + x0 + 1] : 0.f;
  float sw = yb ? p[(y0 + 1) * w + x0] : 0.f, se = (xb && yb) ? p[(y0 + 1) * w + x0 + 1] : 0.f;
  float r = __fmul_rn(nw, __fmul_rn(ux, uy));
  r = __fadd_rn(r, __fmul_rn(ne, __fmul_rn(tx, uy)));
  r = __fadd_rn(r, __fmul_rn(sw, __fmul_rn(ux, ty)));
  r = __fadd_rn(r, __fmul_rn(se, __fmul_rn(tx, ty)));
  return r;
}

// depth_pred [N, h, w], loc [N, n, 2] in [0, 1] (x, y) -> sampled [N, n]
__global__ void __launch_bounds__(256) depth_sample_kernel(const float* __restrict__ pred, const float* __restrict__ loc, int N, int n,
                                                           int h, int w, float* __restrict__ out) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= (long long)N * n) return;
  int cam = (int)(t / n);
  out[t] = depth_sample_border(pred + (long long)cam * h * w, h, w, loc[2 * t], loc[2 * t + 1]);
}

// The per-point terms of cal_depth_metric / compute_depth_errors_torch (metric_util.py:247-279,424-445) at the clamped
// prediction p, accumulated into a = (abs_rel, sq_rel, squared error, squared log error, a1, a2, a3, count) sums.
__device__ __forceinline__ void depth_error_terms(float g, float p, double (&a)[8]) {
  float th = fmaxf(g / p, p / g);
  float d = g - p, l = logf(g) - logf(p);
  a[0] += fabsf(d) / g; a[1] += d * d / g; a[2] += d * d; a[3] += l * l;
  a[4] += th < 1.25f ? 1.0 : 0.0; a[5] += th < 1.25f * 1.25f ? 1.0 : 0.0; a[6] += th < 1.25f * 1.25f * 1.25f ? 1.0 : 0.0;
  a[7] += 1.0;
}

// Block sum of the eight accumulators in a fixed order (warp butterflies, then the warps in index order), so the result
// does not depend on scheduling: tot[j] = sum over the block's threads of a[j], visible to every thread on return.
// blockDim.x is a multiple of 32 and at most 512.
__device__ __forceinline__ void block_sum8(const double (&a)[8], double (&tot)[8]) {
  __shared__ double sm[8][16];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    double v = a[j];
    for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
    if (lane == 0) sm[j][warp] = v;
  }
  __syncthreads();
  __shared__ double t[8];
  if (threadIdx.x < 8) {
    double v = 0;
    for (int wv = 0; wv < (int)(blockDim.x >> 5); ++wv) v += sm[threadIdx.x][wv];
    t[threadIdx.x] = v;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 8; ++j) tot[j] = t[j];
}

// One CTA per camera (a camera sees a few thousand LiDAR points): deterministic tree reduction of the error sums of
// cal_depth_metric (metric_util.py:247-279) over the masked points.  sums [N, 8] =
// (abs_rel, sq_rel, squared error, squared log error, a1, a2, a3, count); pred' = clamp(scale[cam] * pred, 1e-3, 80).
__global__ void __launch_bounds__(512) depth_metric_kernel(const float* __restrict__ sampled, const float* __restrict__ gt,
                                                           const unsigned char* __restrict__ mask, const float* __restrict__ scale,
                                                           int n, float* __restrict__ sums) {
  const int cam = blockIdx.x;
  const float sc = scale ? scale[cam] : 1.f;
  double a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    long long k = (long long)cam * n + i;
    if (!mask[k]) continue;
    depth_error_terms(gt[k], fminf(fmaxf(sc * sampled[k], 1e-3f), 80.f), a);
  }
  double tot[8];
  block_sum8(a, tot);
  if (threadIdx.x < 8) sums[cam * 8 + threadIdx.x] = (float)tot[threadIdx.x];
}

// Novel-view depth (eval_novel_depth.py:159-208, eval_novel_depth_kitti.py): one CTA per (pose, camera) segment
// [offsets[seg], offsets[seg + 1]) of a ragged LiDAR set.  Each masked point samples depth map seg at its location, and
// the segment's seven compute_depth_errors_torch metrics are finished from the fp64 sums: means over the segment's
// masked points, rmse / rmse_log as square roots of means.  A segment without a masked point gives NaN (the reference's
// mean of an empty tensor).
__global__ void __launch_bounds__(512) novel_depth_errors_kernel(const float* __restrict__ maps, int h, int w,
                                                                 const int64_t* __restrict__ offsets, const float* __restrict__ loc,
                                                                 const float* __restrict__ gt, const unsigned char* __restrict__ mask,
                                                                 float* __restrict__ errors) {
  const int seg = blockIdx.x;
  const long long b = offsets[seg], e = offsets[seg + 1];
  const float* p = maps + (long long)seg * h * w;
  double a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (long long i = b + threadIdx.x; i < e; i += blockDim.x) {
    if (!mask[i]) continue;
    float v = depth_sample_border(p, h, w, loc[2 * i], loc[2 * i + 1]);
    depth_error_terms(gt[i], fminf(fmaxf(v, 1e-3f), 80.f), a);
  }
  double tot[8];
  block_sum8(a, tot);
  if (threadIdx.x < 7) {
    const double c = tot[7];
    double m = tot[threadIdx.x] / c;
    if (threadIdx.x == 2 || threadIdx.x == 3) m = sqrt(m);
    errors[seg * 7 + threadIdx.x] = c > 0 ? (float)m : __int_as_float(0x7fc00000);
  }
}

}  // namespace so

using namespace so;

extern "C" int so_depth_metric_sample(const float* depth_pred, const float* loc, int32_t N, int32_t n, int32_t h, int32_t w,
                                      float* sampled, void* stream) {
  if (!depth_pred || !loc || !sampled || N < 1 || n < 0 || h < 1 || w < 1) return SO_ERR_INVALID_ARG;
  if (n == 0) return SO_OK;
  depth_sample_kernel<<<(unsigned)ceil_div64((int64_t)N * n, 256), 256, 0, (cudaStream_t)stream>>>(depth_pred, loc, N, n, h, w, sampled);
  note_launch(1);
  return check_launch();
}

extern "C" int so_depth_metric_sums(const float* sampled, const float* depth_gt, const uint8_t* mask, const float* scale, int32_t N,
                                    int32_t n, float* sums, void* stream) {
  if (!sampled || !depth_gt || !mask || !sums || N < 1 || n < 0) return SO_ERR_INVALID_ARG;
  depth_metric_kernel<<<N, 512, 0, (cudaStream_t)stream>>>(sampled, depth_gt, mask, scale, n, sums);
  note_launch(1);
  return check_launch();
}

extern "C" int so_novel_depth_errors(const float* depth_maps, int32_t n_seg, int32_t h, int32_t w, const int64_t* offsets,
                                     const int64_t* offsets_host, int64_t T, const float* loc, const float* depth_gt,
                                     const uint8_t* mask, float* errors, void* stream) {
  if (!depth_maps || !offsets || !offsets_host || !errors || n_seg < 1 || h < 1 || w < 1 || T < 0) return SO_ERR_INVALID_ARG;
  if (T > 0 && (!loc || !depth_gt || !mask)) return SO_ERR_INVALID_ARG;
  if (offsets_host[0] != 0 || offsets_host[n_seg] != T) return SO_ERR_INVALID_ARG;
  for (int32_t s = 0; s < n_seg; ++s)
    if (offsets_host[s + 1] < offsets_host[s]) return SO_ERR_INVALID_ARG;
  if ((int64_t)h * w > INT32_MAX) return SO_ERR_UNSUPPORTED;     // in-map indices are 32-bit
  novel_depth_errors_kernel<<<n_seg, 512, 0, (cudaStream_t)stream>>>(depth_maps, h, w, offsets, loc, depth_gt, mask, errors);
  note_launch(1);
  return check_launch();
}
