// `second_grad` training output (neus_head.py:177,703-706; consumer loss/second_grad_loss.py:19-20: |second_grad|.mean()).
// DECLARED ASSUMPTION -- the quantity is defined inside the un-vendored sdfstudio fork (cuda_gridsample_grad2); what is
// restated here is the standard double-backward idiom  second_grad = d( sum_j d sdf / d x_j ) / d x  of the trilinear field,
// i.e. the ROW SUMS of the Hessian of the interpolant in metres.  Inside a cell the pure second derivatives vanish and
//     d2 s / dh dw = sum_k wz_k (a11k - a10k - a01k + a00k)          (and cyclic),
// so  second_grad = (Hxy + Hxz, Hxy + Hyz, Hxz + Hyz),  Hxy = kw kh d2s/dw dh, ...  (x <-> w, y <-> h, z <-> d).
// Zero padding outside the volume like F.grid_sample(padding_mode='zeros', align_corners=True).  Opt-in (return_second_grad).
#include "hess_terms.cuh"

namespace so {

__global__ void __launch_bounds__(256) field_hess_kernel(VolumeDev V, const float* __restrict__ pts, long long n,
                                                         float* __restrict__ out) {
  long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (p >= n) return;
  float x = pts[3 * p], y = pts[3 * p + 1], z = pts[3 * p + 2];
  float kh, kw, kd;
  float gh = axis_m2g(V.ax[0], y, kh), gw = axis_m2g(V.ax[1], x, kw), gd = axis_m2g(V.ax[2], z, kd);
  Taps t = make_taps(V, gh, gw, gd);
  float o[3];
  second_grad_at(V, t, kh, kw, kd, o);
  out[3 * p] = o[0];
  out[3 * p + 1] = o[1];
  out[3 * p + 2] = o[2];
}

__global__ void __launch_bounds__(256) field_hess_bwd_kernel(VolumeDev V, const float* __restrict__ pts, long long n,
                                                             const float* __restrict__ g, float* __restrict__ gvs) {
  long long p = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (p >= n) return;
  float x = pts[3 * p], y = pts[3 * p + 1], z = pts[3 * p + 2];
  float kh, kw, kd;
  float gh = axis_m2g(V.ax[0], y, kh), gw = axis_m2g(V.ax[1], x, kw), gd = axis_m2g(V.ax[2], z, kd);
  Taps t = make_taps(V, gh, gw, gd);
  float g0 = g[3 * p], g1 = g[3 * p + 1], g2 = g[3 * p + 2];
  float c[2][2][2];
  second_grad_weights(t, kh, kw, kd, g0, g1, g2, c);
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int k = 0; k < 2; ++k)
        if (c[i][j][k] != 0.f) atomicAdd(gvs + corner_index(V, t, i, j, k), c[i][j][k]);
}

}  // namespace so

using namespace so;

extern "C" int so_field_second_grad(const float* vol_sdf, const so_volume_desc* vol_host, const float* points, int64_t n,
                                    float* second_grad, void* stream) {
  if (!vol_sdf || !points || !second_grad || n < 0) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(vol_host);
  if (rc) return rc;
  if (n == 0) return SO_OK;
  VolumeDev V = make_volume(*vol_host, vol_sdf, nullptr);
  field_hess_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(V, points, n, second_grad);
  note_launch(1);
  return check_launch();
}

extern "C" int so_field_second_grad_backward(const so_volume_desc* vol_host, const float* points, int64_t n, const float* g_second_grad,
                                             float* g_vol_sdf, void* stream) {
  if (!points || !g_second_grad || !g_vol_sdf || n < 0) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(vol_host);
  if (rc) return rc;
  if (n == 0) return SO_OK;
  VolumeDev V = make_volume(*vol_host, nullptr, nullptr);
  field_hess_bwd_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(V, points, n, g_second_grad, g_vol_sdf);
  note_launch(1);
  return check_launch();
}
