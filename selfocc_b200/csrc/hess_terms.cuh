// `second_grad` of one sample (declared assumption, see field_hess.cu): the row sums of the Hessian of the trilinear
// interpolant in metres, from the sample's tap set.  Shared by so_field_second_grad (field_hess.cu) and the training render
// with the objective fused in (render_objective.cuh), so both evaluate a sample with the same arithmetic.
#pragma once
#include "common.cuh"

namespace so {

__device__ __forceinline__ size_t corner_index(const VolumeDev& v, const Taps& t, int i, int j, int k) {
  int h = min(max(t.h0 + i, 0), v.H - 1), w = min(max(t.w0 + j, 0), v.W - 1), z = min(max(t.z0 + k, 0), v.Z - 1);
  return ((size_t)h * v.W + w) * v.zpitch + z;
}

// the mixed second derivatives (grid units) d2s/dh dw, d2s/dh dz, d2s/dw dz of the cell; zero padding through the masks
__device__ __forceinline__ void hess_grid(const VolumeDev& V, const Taps& t, float& s_hw, float& s_hz, float& s_wz) {
  s_hw = 0.f; s_hz = 0.f; s_wz = 0.f;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        float m = (i ? t.mh1 : t.mh0) * (j ? t.mw1 : t.mw0) * (k ? t.mz1 : t.mz0);
        float a = m * __ldg(V.sdf + corner_index(V, t, i, j, k));
        float si = i ? 1.f : -1.f, sj = j ? 1.f : -1.f, sk = k ? 1.f : -1.f;
        s_hw = fmaf(si * sj * (k ? t.fz : 1.f - t.fz), a, s_hw);
        s_hz = fmaf(si * sk * (j ? t.fw : 1.f - t.fw), a, s_hz);
        s_wz = fmaf(sj * sk * (i ? t.fh : 1.f - t.fh), a, s_wz);
      }
}

// second_grad = (Hxy + Hxz, Hxy + Hyz, Hxz + Hyz) in metres (x <-> w, y <-> h, z <-> d)
__device__ __forceinline__ void second_grad_at(const VolumeDev& V, const Taps& t, float kh, float kw, float kd, float out[3]) {
  float s_hw, s_hz, s_wz;
  hess_grid(V, t, s_hw, s_hz, s_wz);
  float Hxy = kw * kh * s_hw, Hxz = kw * kd * s_wz, Hyz = kh * kd * s_hz;
  out[0] = Hxy + Hxz;
  out[1] = Hxy + Hyz;
  out[2] = Hxz + Hyz;
}

__device__ __forceinline__ void hess_weights(const Taps& t, float kh, float kw, float kd, float ghw, float ghz, float gwz,
                                             float c[2][2][2]) {
  // contribution of corner (i, j, k) to  ghw * s_hw + ghz * s_hz + gwz * s_wz  (signs: +1 for index 1, -1 for index 0)
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        float si = i ? 1.f : -1.f, sj = j ? 1.f : -1.f, sk = k ? 1.f : -1.f;
        float wh = i ? t.fh : 1.f - t.fh, ww = j ? t.fw : 1.f - t.fw, wz = k ? t.fz : 1.f - t.fz;
        float m = (i ? t.mh1 : t.mh0) * (j ? t.mw1 : t.mw0) * (k ? t.mz1 : t.mz0);
        c[i][j][k] = m * (ghw * si * sj * wz + ghz * si * sk * ww + gwz * sj * sk * wh);
      }
}

// corner coefficients of the gradient of  g . second_grad  (g = d loss / d second_grad of the sample)
__device__ __forceinline__ void second_grad_weights(const Taps& t, float kh, float kw, float kd, float g0, float g1, float g2,
                                                    float c[2][2][2]) {
  hess_weights(t, kh, kw, kd, (g0 + g1) * kw * kh, (g1 + g2) * kh * kd, (g0 + g2) * kw * kd, c);
}

}  // namespace so
