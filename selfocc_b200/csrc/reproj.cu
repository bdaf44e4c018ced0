// Photometric reprojection loss, per-ray statistics and their backward (SURVEY.md 8f-2).
//
// Both reference variants (loss/reproj_loss_mono_multi_new_combine.py:70-248, loss/reproj_loss_mono_multi_new.py:72-288)
// use the rendering weights only through masked, weighted sums over each ray's samples that are then divided by the
// ray's masked weight sum.  So the loss is a function of a few per-ray statistics built from sums LINEAR in the weights:
//   W = sum w_s m_s,  l1 = (sum w_s m_s diff_s) / max(W, eps),  rgb = (sum w_s m_s rgb_s) / max(W, eps)  (+ any = OR m_s)
// and d loss / d w_s = f_s m_s (gW + (g_l1 (diff_s - l1) + g_rgb . (rgb_s - rgb)) / W)  for W >= eps
//                    = f_s m_s (gW + (g_l1 diff_s + g_rgb . rgb_s) / eps)                 otherwise (the clamp is flat),
// with diff_s / rgb_s recomputed from ts, the matrices and the images: nothing per sample is stored for the backward.
// The backward subtracts the ray means before it multiplies (rather than adding -g L / W^2 to g diff_s / W): the two
// terms nearly cancel wherever a sample is close to its ray's mean, and fp32 keeps the difference exact only this way.  The per-ray tail (SSIM over the ray grid, the automask
// min, the 1e3 filters, the means) is torch on [N_cam, R] grids (selfocc_b200/loss.py).
#include "reproj_terms.cuh"
#include <math.h>

namespace so {

namespace {

constexpr int kWarpsPerBlock = 8;

struct ReprojArgs {
  const float* weights;   // [N, R, S]
  const float* ts;        // [N, R, S]
  const float* deltas;    // [N, R, S] or nullptr
  const float* pix;       // [R, 2] (x, y) in loss pixels
  const float* m_prev;    // [N, 4, 4] img2prevImg
  const float* m_next;    // [N, 4, 4] img2nextImg
  const float* curr;      // [N, 3, H, W]
  const float* prev;
  const float* next;
  int N, R, S, H, W;
  float size_h, size_w;   // the loss's img_size (normalisation of the pixel coordinates)
};

// weight factor of the optional `deltas` input: w / max(delta, eps), zero where delta < eps (fp32 eps)
__device__ __forceinline__ float delta_scale(const float* __restrict__ deltas, int64_t i, float w) {
  if (!deltas) return w;
  const float dl = __ldg(deltas + i);
  return dl < kReprojEps ? 0.f : w / fmaxf(dl, kReprojEps);
}

// One warp per ray (ray = cam * R + r), lanes stride over the S samples, fixed xor-shuffle reduction (deterministic).
// stats [N, R, 6 * NSET] = per set (W, l1, rgb0, rgb1, rgb2, any); colours [N, R, 9] = (curr, prev, next) at the ray pixel.
template <bool COMBINE>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) reproj_stats_kernel(ReprojArgs a, float* __restrict__ stats,
                                                                           float* __restrict__ colours) {
  constexpr int NSET = COMBINE ? 1 : 2;
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (ray >= (int64_t)a.N * a.R) return;
  const int cam = (int)(ray / a.R), r = (int)(ray - (int64_t)cam * a.R);
  const int64_t img_off = (int64_t)cam * 3 * a.H * a.W;
  const float u = __ldg(a.pix + 2 * r), v = __ldg(a.pix + 2 * r + 1);
  float cur[3];
  sample3<COMBINE>(a.curr + img_off, a.H, a.W, a.size_w, a.size_h, u, v, cur);
  if (colours && lane < 3) {
    float o[3];
    const float* img = lane == 0 ? a.curr : (lane == 1 ? a.prev : a.next);
    sample3<COMBINE>(img + img_off, a.H, a.W, a.size_w, a.size_h, u, v, o);
#pragma unroll
    for (int k = 0; k < 3; ++k) colours[ray * 9 + lane * 3 + k] = o[k];
  }
  const Mat34 Mp = load_mat(a.m_prev + cam * 16), Mn = load_mat(a.m_next + cam * 16);
  float acc[NSET][5];
  bool any[NSET];
#pragma unroll
  for (int j = 0; j < NSET; ++j) {
    any[j] = false;
#pragma unroll
    for (int k = 0; k < 5; ++k) acc[j][k] = 0.f;
  }
  const int64_t base = ray * a.S;
  const float* prev = a.prev + img_off;
  const float* next = a.next + img_off;
  for (int s = lane; s < a.S; s += 32) {
    const float t = __ldg(a.ts + base + s);
    const float w = delta_scale(a.deltas, base + s, __ldg(a.weights + base + s));
    bool m[2];
    float d[2], c[2][3];
    sample_terms<COMBINE>(a.H, a.W, a.size_w, a.size_h, Mp, Mn, prev, next, u, v, t, cur, m, d, c);
#pragma unroll
    for (int j = 0; j < NSET; ++j) {
      if (!m[j]) continue;
      any[j] = true;
      acc[j][0] += w;
      acc[j][1] += w * d[j];
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[j][2 + k] += w * c[j][k];
    }
  }
#pragma unroll
  for (int j = 0; j < NSET; ++j) {
#pragma unroll
    for (int k = 0; k < 5; ++k)
      for (int o = 16; o > 0; o >>= 1) acc[j][k] += __shfl_xor_sync(0xffffffffu, acc[j][k], o);
    any[j] = __any_sync(0xffffffffu, any[j]);
  }
  if (lane == 0) {
    float* st = stats + ray * (6 * NSET);
#pragma unroll
    for (int j = 0; j < NSET; ++j) {
      const float wc = fmaxf(acc[j][0], kReprojEps);
      st[6 * j] = acc[j][0];
#pragma unroll
      for (int k = 1; k < 5; ++k) st[6 * j + k] = acc[j][k] / wc;
      st[6 * j + 5] = any[j] ? 1.f : 0.f;
    }
  }
}

// grad_weights [N, R, S] from the forward's stats and grad_stats [N, R, 6 * NSET] (the `any` slots are ignored), same
// recomputation.
template <bool COMBINE>
__global__ void __launch_bounds__(kWarpsPerBlock * 32) reproj_stats_backward_kernel(ReprojArgs a, const float* __restrict__ stats,
                                                                                    const float* __restrict__ gstats,
                                                                                    float* __restrict__ gw) {
  constexpr int NSET = COMBINE ? 1 : 2;
  const int lane = threadIdx.x & 31;
  const int64_t ray = (int64_t)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (ray >= (int64_t)a.N * a.R) return;
  const int cam = (int)(ray / a.R), r = (int)(ray - (int64_t)cam * a.R);
  const int64_t img_off = (int64_t)cam * 3 * a.H * a.W;
  const float u = __ldg(a.pix + 2 * r), v = __ldg(a.pix + 2 * r + 1);
  float cur[3];
  sample3<COMBINE>(a.curr + img_off, a.H, a.W, a.size_w, a.size_h, u, v, cur);
  // per set: gW, the scaled gradients of l1 / rgb, and the ray means they are taken against (0 on the flat clamp)
  float gW[NSET], gs[NSET][4], mean[NSET][4];
#pragma unroll
  for (int j = 0; j < NSET; ++j) {
    const float* st = stats + ray * (6 * NSET) + 6 * j;
    const float* g = gstats + ray * (6 * NSET) + 6 * j;
    const float W = __ldg(st);
    const bool flat = !(W >= kReprojEps);
    gW[j] = __ldg(g);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      gs[j][k] = __ldg(g + 1 + k) / (flat ? kReprojEps : W);
      mean[j][k] = flat ? 0.f : __ldg(st + 1 + k);
    }
  }
  const Mat34 Mp = load_mat(a.m_prev + cam * 16), Mn = load_mat(a.m_next + cam * 16);
  const int64_t base = ray * a.S;
  const float* prev = a.prev + img_off;
  const float* next = a.next + img_off;
  for (int s = lane; s < a.S; s += 32) {
    const float t = __ldg(a.ts + base + s);
    bool m[2];
    float d[2], c[2][3];
    sample_terms<COMBINE>(a.H, a.W, a.size_w, a.size_h, Mp, Mn, prev, next, u, v, t, cur, m, d, c);
    float G = 0.f;
#pragma unroll
    for (int j = 0; j < NSET; ++j)
      if (m[j])
        G += gW[j] + gs[j][0] * (d[j] - mean[j][0]) + gs[j][1] * (c[j][0] - mean[j][1]) + gs[j][2] * (c[j][1] - mean[j][2]) +
             gs[j][3] * (c[j][2] - mean[j][3]);
    gw[base + s] = delta_scale(a.deltas, base + s, G);
  }
}

int validate(const float* ts, const float* pix, const float* m_prev, const float* m_next, const float* curr,
             const float* prev, const float* next, int32_t n_cam, int32_t rays_per_cam, int32_t S, int32_t img_h, int32_t img_w,
             float size_h, float size_w, int32_t mode) {
  if (!ts || !pix || !m_prev || !m_next || !curr || !prev || !next) return SO_ERR_INVALID_ARG;
  if (n_cam < 1 || rays_per_cam < 1 || S < 1 || img_h < 1 || img_w < 1) return SO_ERR_INVALID_ARG;
  if (!(size_h > 0.f) || !(size_w > 0.f) || !isfinite(size_h) || !isfinite(size_w)) return SO_ERR_INVALID_ARG;
  if (mode != SO_REPROJ_COMBINE && mode != SO_REPROJ_MULTI_NEW) return SO_ERR_INVALID_ARG;
  // 32-bit pixel offsets inside one image plane; the grid covers N * R rays with 8 per block
  if ((int64_t)img_h * img_w >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;
  if (ceil_div64((int64_t)n_cam * rays_per_cam, kWarpsPerBlock) >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;
  return SO_OK;
}

ReprojArgs make_args(const float* weights, const float* ts, const float* deltas, const float* pix, const float* m_prev,
                     const float* m_next, const float* curr, const float* prev, const float* next, int32_t n_cam,
                     int32_t rays_per_cam, int32_t S, int32_t img_h, int32_t img_w, float size_h, float size_w) {
  ReprojArgs a;
  a.weights = weights; a.ts = ts; a.deltas = deltas; a.pix = pix; a.m_prev = m_prev; a.m_next = m_next;
  a.curr = curr; a.prev = prev; a.next = next;
  a.N = n_cam; a.R = rays_per_cam; a.S = S; a.H = img_h; a.W = img_w; a.size_h = size_h; a.size_w = size_w;
  return a;
}

}  // namespace
}  // namespace so

using namespace so;

extern "C" int so_reproj_stats_forward(const float* weights, const float* ts, const float* deltas, const float* pix,
                                       const float* img2prev, const float* img2next, const float* curr_imgs,
                                       const float* prev_imgs, const float* next_imgs, int32_t n_cam, int32_t rays_per_cam,
                                       int32_t S, int32_t img_h, int32_t img_w, float size_h, float size_w, int32_t mode,
                                       float* stats, float* colours, void* stream) {
  if (!weights || !stats) return SO_ERR_INVALID_ARG;
  int rc = validate(ts, pix, img2prev, img2next, curr_imgs, prev_imgs, next_imgs, n_cam, rays_per_cam, S, img_h, img_w,
                    size_h, size_w, mode);
  if (rc) return rc;
  const ReprojArgs a = make_args(weights, ts, deltas, pix, img2prev, img2next, curr_imgs, prev_imgs, next_imgs, n_cam,
                                 rays_per_cam, S, img_h, img_w, size_h, size_w);
  const unsigned grid = (unsigned)ceil_div64((int64_t)n_cam * rays_per_cam, kWarpsPerBlock);
  if (mode == SO_REPROJ_COMBINE)
    reproj_stats_kernel<true><<<grid, kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(a, stats, colours);
  else
    reproj_stats_kernel<false><<<grid, kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(a, stats, colours);
  note_launch(1);
  return check_launch();
}

extern "C" int so_reproj_stats_backward(const float* ts, const float* deltas, const float* pix,
                                        const float* img2prev, const float* img2next, const float* curr_imgs,
                                        const float* prev_imgs, const float* next_imgs, int32_t n_cam, int32_t rays_per_cam,
                                        int32_t S, int32_t img_h, int32_t img_w, float size_h, float size_w, int32_t mode,
                                        const float* stats, const float* grad_stats, float* grad_weights, void* stream) {
  if (!stats || !grad_stats || !grad_weights) return SO_ERR_INVALID_ARG;
  int rc = validate(ts, pix, img2prev, img2next, curr_imgs, prev_imgs, next_imgs, n_cam, rays_per_cam, S, img_h, img_w,
                    size_h, size_w, mode);
  if (rc) return rc;
  const ReprojArgs a = make_args(nullptr, ts, deltas, pix, img2prev, img2next, curr_imgs, prev_imgs, next_imgs, n_cam,
                                 rays_per_cam, S, img_h, img_w, size_h, size_w);
  const unsigned grid = (unsigned)ceil_div64((int64_t)n_cam * rays_per_cam, kWarpsPerBlock);
  if (mode == SO_REPROJ_COMBINE)
    reproj_stats_backward_kernel<true><<<grid, kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(a, stats, grad_stats, grad_weights);
  else
    reproj_stats_backward_kernel<false><<<grid, kWarpsPerBlock * 32, 0, (cudaStream_t)stream>>>(a, stats, grad_stats, grad_weights);
  note_launch(1);
  return check_launch();
}
