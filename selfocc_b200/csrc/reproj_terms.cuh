// Per-sample terms of the photometric reprojection loss (SURVEY.md 8f-2): the projection of a ray sample into the
// previous / next frame, its validity mask, the bilinear colours there and the L1 difference to the current image.
// Shared by the per-ray statistics kernels (reproj.cu) and the training render with the objective fused in
// (render_train.cu / render_objective.cu), so both evaluate every sample with the same arithmetic.
#pragma once
#include "common.cuh"

namespace so {

constexpr float kReprojEps = 1.1920928955078125e-07f;   // torch.finfo(float32).eps: the weight-sum clamp and the deltas test

// ATen grid_sampler_2d, bilinear, align_corners=True: the reference normalises x by size_w and samples at
// ((2 x / size_w - 1 + 1) / 2) (W - 1).  BORDER clips the coordinate; corners outside the image read zero either way.
template <bool BORDER>
__device__ __forceinline__ void sample3(const float* __restrict__ img, int H, int W, float size_w, float size_h, float px,
                                        float py, float out[3]) {
  float gx = 2.f * (px / size_w) - 1.f, gy = 2.f * (py / size_h) - 1.f;
  float ix = ((gx + 1.f) * 0.5f) * (float)(W - 1), iy = ((gy + 1.f) * 0.5f) * (float)(H - 1);
  if (BORDER) {
    ix = fminf((float)(W - 1), fmaxf(ix, 0.f));
    iy = fminf((float)(H - 1), fmaxf(iy, 0.f));
  }
  out[0] = out[1] = out[2] = 0.f;
  if (!(ix > -1.f && ix < (float)W && iy > -1.f && iy < (float)H)) return;   // every corner outside (zeros padding; NaN)
  const float x0f = floorf(ix), y0f = floorf(iy);
  const int x0 = (int)x0f, y0 = (int)y0f;
  const float tx = ix - x0f, ty = iy - y0f, ux = (x0f + 1.f) - ix, uy = (y0f + 1.f) - iy;
  const bool vx0 = x0 >= 0, vx1 = x0 + 1 < W, vy0 = y0 >= 0, vy1 = y0 + 1 < H;
  const float wnw = ux * uy, wne = tx * uy, wsw = ux * ty, wse = tx * ty;
  const int64_t plane = (int64_t)H * W;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* p = img + c * plane;
    float v = 0.f;
    if (vy0 && vx0) v += __ldg(p + y0 * W + x0) * wnw;
    if (vy0 && vx1) v += __ldg(p + y0 * W + x0 + 1) * wne;
    if (vy1 && vx0) v += __ldg(p + (y0 + 1) * W + x0) * wsw;
    if (vy1 && vx1) v += __ldg(p + (y0 + 1) * W + x0 + 1) * wse;
    out[c] = v;
  }
}

// Rows 0-2 of one 4x4 matrix.
struct Mat34 { float m[12]; };

__device__ __forceinline__ Mat34 load_mat(const float* __restrict__ M) {
  Mat34 r;
#pragma unroll
  for (int i = 0; i < 12; ++i) r.m[i] = __ldg(M + i);
  return r;
}

// cal_pixel: (u t, v t, t, 1) through the matrix, z > 0, division by max(z, 1e-5), strict in-image test.
__device__ __forceinline__ bool project(const Mat34& M, float ut, float vt, float t, float size_w, float size_h, float& px,
                                        float& py) {
  const float x = M.m[0] * ut + M.m[1] * vt + M.m[2] * t + M.m[3];
  const float y = M.m[4] * ut + M.m[5] * vt + M.m[6] * t + M.m[7];
  const float z = M.m[8] * ut + M.m[9] * vt + M.m[10] * t + M.m[11];
  const float d = fmaxf(z, 1e-5f);
  px = x / d;
  py = y / d;
  return z > 0.f && px > 0.f && px < size_w && py > 0.f && py < size_h;
}

__device__ __forceinline__ float l1_mean3(const float a[3], const float b[3]) {
  return (fabsf(a[0] - b[0]) + fabsf(a[1] - b[1]) + fabsf(a[2] - b[2])) / 3.f;
}

// Per-sample terms of one sample at depth t of the ray through loss pixel (u, v).  COMBINE: one direction set (prev | next
// merged, diff and colour averaged over the valid directions); MultiNew: prev and next kept apart.  Returns the masks;
// diff / rgb of each set in d[], c[][3].  H, W: image shape; size_h, size_w: the loss's img_size.
template <bool COMBINE>
__device__ __forceinline__ void sample_terms(int H, int W, float size_w, float size_h, const Mat34& Mp, const Mat34& Mn,
                                             const float* __restrict__ prev, const float* __restrict__ next, float u, float v,
                                             float t, const float cur[3], bool m[2], float d[2], float c[2][3]) {
  const float ut = u * t, vt = v * t;
  float ppx, ppy, npx, npy;
  m[0] = project(Mp, ut, vt, t, size_w, size_h, ppx, ppy);
  m[1] = project(Mn, ut, vt, t, size_w, size_h, npx, npy);
  float p[3] = {0.f, 0.f, 0.f}, n[3] = {0.f, 0.f, 0.f};
  if (m[0]) sample3<COMBINE>(prev, H, W, size_w, size_h, ppx, ppy, p);
  if (m[1]) sample3<COMBINE>(next, H, W, size_w, size_h, npx, npy, n);
  if (COMBINE) {
    const float fp = m[0] ? 1.f : 0.f, fn = m[1] ? 1.f : 0.f;
    const float cnt = fmaxf(fp + fn, 1.f);
    const float dp = m[0] ? l1_mean3(cur, p) : 0.f, dn = m[1] ? l1_mean3(cur, n) : 0.f;
    d[0] = (dp + dn) / cnt;
#pragma unroll
    for (int k = 0; k < 3; ++k) c[0][k] = (p[k] * fp + n[k] * fn) / cnt;
    m[0] = m[0] || m[1];
  } else {
    d[0] = m[0] ? l1_mean3(cur, p) : 0.f;
    d[1] = m[1] ? l1_mean3(cur, n) : 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) { c[0][k] = p[k]; c[1][k] = n[k]; }
  }
}

}  // namespace so
