// EikonalLoss (loss/eikonal_loss.py:19-21) per sample: f = (|g|_2 - 1)^2 of the metre gradient g of the sdf, and the
// gradient of s * f.  Shared by the sample-mean kernels (loss_terms.cu) and the training render with the objective fused
// in (render_train.cu), so both evaluate every sample with the same arithmetic.
#pragma once
#include "common.cuh"

namespace so {

__device__ __forceinline__ float eik_norm(float x, float y, float z) { return sqrtf(fmaf(x, x, fmaf(y, y, z * z))); }

__device__ __forceinline__ double eik_row(float x, float y, float z) {
  const double d = (double)eik_norm(x, y, z) - 1.0;
  return d * d;
}

// 2 (|g| - 1) g / |g| * s, 0 where |g| = 0 (vector_norm's backward masks zero norms)
__device__ __forceinline__ float eik_coef(float x, float y, float z, float s) {
  const float n = eik_norm(x, y, z);
  return n > 0.f ? 2.f * (n - 1.f) * s / n : 0.f;
}

}  // namespace so
