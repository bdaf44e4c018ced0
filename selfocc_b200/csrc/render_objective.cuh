// The training objective's per-sample terms folded into the training render (SURVEY.md 8f-2, DESIGN.md section 7): the
// reprojection statistics of so_reproj_stats_forward (deltas == NULL), the eikonal sum of so_sample_mean_forward (EIKONAL)
// and the second-grad sum of so_field_second_grad + so_sample_mean_forward (ABS), accumulated per ray while the render walks
// the ray's samples, and their adjoints formed per sample in the backward.  Nothing per sample reaches memory.
//
// The training kernels (render_train.cu) take an OBJ template parameter: kObjOff is the plain training render; the other
// values add the objective.  ObjFwd / ObjBwd hold one ray's state in the lanes of the warp that renders it (lane = sample),
// so they follow the one-ray-per-warp structure of reproj_stats_kernel: per-lane sums over the lane's samples in sample
// order, then a fixed xor-shuffle reduction.
#pragma once
#include "reproj_terms.cuh"
#include "eikonal_terms.cuh"
#include "hess_terms.cuh"

namespace so {

constexpr int kObjOff = 0;         // no objective: so_render_train_forward / _backward
constexpr int kObjNoReproj = 1;    // objective without a reprojection term (eikonal only, or nothing)
constexpr int kObjCombine = 2;     // SO_REPROJ_COMBINE
constexpr int kObjMultiNew = 3;    // SO_REPROJ_MULTI_NEW

struct ObjectiveDev {
  // reprojection operands (OBJ >= kObjCombine), as so_reproj_stats_forward takes them
  const float *pix, *m_prev, *m_next, *curr, *prev, *next;
  int H, W;
  float size_h, size_w;
  int eikonal;                      // the eikonal term is on
  // forward outputs
  float* stats;                     // [rays, 6 * sets]
  float* colours;                   // [rays, 9] or nullptr
  double* eik_part;                 // [rays] per-ray fp64 sums of (|grad sdf| - 1)^2
  int second_grad;                  // the second-grad term is on
  double* sg_part;                  // [rays] per-ray fp64 sums of |second_grad| over the 3 components
  // backward inputs
  const float *stats_in, *g_stats;  // [rays, 6 * sets]
  const float* g_eik_mean;          // device scalar or nullptr (= 0)
  long long eik_count;              // samples the eikonal mean is taken over
  double* inv_part;                 // [rays] per-ray d loss / d inv_s, or nullptr (no inv_s gradient)
  const float* g_sg_mean;           // device scalar or nullptr (= 0)
  long long sg_count;               // elements the second-grad mean is taken over (3 per sample)
};

template <int OBJ>
struct ObjTraits {
  static constexpr bool kReproj = OBJ >= kObjCombine;
  static constexpr bool kCombine = OBJ == kObjCombine;
  static constexpr int kSets = OBJ == kObjMultiNew ? 2 : 1;
};

// the reprojection operands of one ray: loss pixel, current colour there, matrices and neighbouring frames of its camera
template <int OBJ>
struct ObjRay {
  float u, v, cur[3];
  Mat34 Mp, Mn;
  const float *prev, *next;

  __device__ __forceinline__ void load(const ObjectiveDev& D, int cam, int r) {
    const int64_t img_off = (int64_t)cam * 3 * D.H * D.W;
    u = __ldg(D.pix + 2 * r);
    v = __ldg(D.pix + 2 * r + 1);
    sample3<ObjTraits<OBJ>::kCombine>(D.curr + img_off, D.H, D.W, D.size_w, D.size_h, u, v, cur);
    Mp = load_mat(D.m_prev + cam * 16);
    Mn = load_mat(D.m_next + cam * 16);
    prev = D.prev + img_off;
    next = D.next + img_off;
  }
  __device__ __forceinline__ void terms(const ObjectiveDev& D, float ts, bool m[2], float d[2], float c[2][3]) const {
    sample_terms<ObjTraits<OBJ>::kCombine>(D.H, D.W, D.size_w, D.size_h, Mp, Mn, prev, next, u, v, ts, cur, m, d, c);
  }
};

// forward: begin() at the ray's start, sample() for every live sample (w = weight, ts = mid / |dir|, g = metre gradient of
// the sdf), sample_hess() for every live sample when D.second_grad (t = the sample's taps, k = metre->grid slopes), end()
// once per ray with every lane of the warp
template <int OBJ>
struct ObjFwd {
  using T = ObjTraits<OBJ>;
  ObjRay<OBJ> ray;
  float acc[T::kSets][5];
  bool any[T::kSets];
  double eik, sg;

  __device__ __forceinline__ void begin(const ObjectiveDev& D, int cam, int r, long long out, int lane) {
    eik = 0.0;
    sg = 0.0;
    if (!T::kReproj) return;
    ray.load(D, cam, r);
    if (D.colours && lane < 3) {
      const int64_t img_off = (int64_t)cam * 3 * D.H * D.W;
      const float* img = lane == 0 ? D.curr : (lane == 1 ? D.prev : D.next);
      float o[3];
      sample3<T::kCombine>(img + img_off, D.H, D.W, D.size_w, D.size_h, ray.u, ray.v, o);
#pragma unroll
      for (int k = 0; k < 3; ++k) D.colours[out * 9 + lane * 3 + k] = o[k];
    }
#pragma unroll
    for (int j = 0; j < T::kSets; ++j) {
      any[j] = false;
#pragma unroll
      for (int k = 0; k < 5; ++k) acc[j][k] = 0.f;
    }
  }

  __device__ __forceinline__ void sample(const ObjectiveDev& D, float w, float ts, float gx, float gy, float gz) {
    if (D.eikonal) eik += eik_row(gx, gy, gz);
    if (!T::kReproj) return;
    bool m[2];
    float d[2], c[2][3];
    ray.terms(D, ts, m, d, c);
#pragma unroll
    for (int j = 0; j < T::kSets; ++j) {
      if (!m[j]) continue;
      any[j] = true;
      acc[j][0] += w;
      acc[j][1] += w * d[j];
#pragma unroll
      for (int k = 0; k < 3; ++k) acc[j][2 + k] += w * c[j][k];
    }
  }

  // |second_grad| of the sample, summed as so_sample_mean_forward(ABS) sums each element: fp64 of the fp32 magnitude
  __device__ __forceinline__ void sample_hess(const ObjectiveDev& D, const VolumeDev& V, const Taps& t, float kh, float kw,
                                              float kd) {
    float h[3];
    second_grad_at(V, t, kh, kw, kd, h);
    sg += (double)fabsf(h[0]);
    sg += (double)fabsf(h[1]);
    sg += (double)fabsf(h[2]);
  }

  __device__ __forceinline__ void end(const ObjectiveDev& D, long long out, int lane) {
    if (D.second_grad) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sg += __shfl_xor_sync(0xffffffffu, sg, o);
      if (lane == 0) D.sg_part[out] = sg;
    }
    if (D.eikonal) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) eik += __shfl_xor_sync(0xffffffffu, eik, o);
      if (lane == 0) D.eik_part[out] = eik;
    }
    if (!T::kReproj) return;
#pragma unroll
    for (int j = 0; j < T::kSets; ++j) {
#pragma unroll
      for (int k = 0; k < 5; ++k)
        for (int o = 16; o > 0; o >>= 1) acc[j][k] += __shfl_xor_sync(0xffffffffu, acc[j][k], o);
      any[j] = __any_sync(0xffffffffu, any[j]);
    }
    if (lane == 0) {
      float* st = D.stats + out * (6 * T::kSets);
#pragma unroll
      for (int j = 0; j < T::kSets; ++j) {
        const float wc = fmaxf(acc[j][0], kReprojEps);
        st[6 * j] = acc[j][0];
#pragma unroll
        for (int k = 1; k < 5; ++k) st[6 * j + k] = acc[j][k] / wc;
        st[6 * j + 5] = any[j] ? 1.f : 0.f;
      }
    }
  }
};

// backward: begin() at the ray's start; g_w(ts) = d loss / d w of a sample (reproj_stats_backward_kernel's G),
// add_g_eik adds d loss / d g of the eikonal mean (sample_mean_backward_kernel's x * eik_coef), hess_corners gives the
// sdf-corner gradient of the second-grad mean (sample_mean_backward_kernel's sign(x) * s, then field_hess_bwd_kernel's
// corner coefficients)
template <int OBJ>
struct ObjBwd {
  using T = ObjTraits<OBJ>;
  ObjRay<OBJ> ray;
  float gW[T::kSets], gs[T::kSets][4], mean[T::kSets][4];
  float eik_s, sg_s;

  __device__ __forceinline__ void begin(const ObjectiveDev& D, int cam, int r, long long out) {
    eik_s = (D.eikonal && D.g_eik_mean) ? (float)((double)__ldg(D.g_eik_mean) / (double)D.eik_count) : 0.f;
    sg_s = (D.second_grad && D.g_sg_mean) ? (float)((double)__ldg(D.g_sg_mean) / (double)D.sg_count) : 0.f;
    if (!T::kReproj) return;
    ray.load(D, cam, r);
#pragma unroll
    for (int j = 0; j < T::kSets; ++j) {
      const float* st = D.stats_in + out * (6 * T::kSets) + 6 * j;
      const float* g = D.g_stats + out * (6 * T::kSets) + 6 * j;
      const float W = __ldg(st);
      const bool flat = !(W >= kReprojEps);
      gW[j] = __ldg(g);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        gs[j][k] = __ldg(g + 1 + k) / (flat ? kReprojEps : W);
        mean[j][k] = flat ? 0.f : __ldg(st + 1 + k);
      }
    }
  }

  __device__ __forceinline__ float g_w(const ObjectiveDev& D, float ts) const {
    if (!T::kReproj) return 0.f;
    bool m[2];
    float d[2], c[2][3];
    ray.terms(D, ts, m, d, c);
    float G = 0.f;
#pragma unroll
    for (int j = 0; j < T::kSets; ++j)
      if (m[j])
        G += gW[j] + gs[j][0] * (d[j] - mean[j][0]) + gs[j][1] * (c[j][0] - mean[j][1]) + gs[j][2] * (c[j][1] - mean[j][2]) +
             gs[j][3] * (c[j][2] - mean[j][3]);
    return G;
  }

  __device__ __forceinline__ void add_g_eik(const ObjectiveDev& D, float gx, float gy, float gz, float& ggx, float& ggy,
                                            float& ggz) const {
    if (!D.eikonal) return;
    const float k = eik_coef(gx, gy, gz, eik_s);
    ggx += gx * k; ggy += gy * k; ggz += gz * k;
  }

  __device__ __forceinline__ void hess_corners(const VolumeDev& V, const Taps& t, float kh, float kw, float kd,
                                               float c[2][2][2]) const {
    float h[3], g[3];
    second_grad_at(V, t, kh, kw, kd, h);
#pragma unroll
    for (int i = 0; i < 3; ++i) g[i] = h[i] > 0.f ? sg_s : (h[i] < 0.f ? -sg_s : 0.f);    // sign(x) * s, 0 at 0
    second_grad_weights(t, kh, kw, kd, g[0], g[1], g[2], c);
  }
};

// host side: one launch of the training forward / backward with the objective `obj` (kObj*) -- render_train.cu
int render_train_forward_obj(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* cam_mats,
                             const float* pix, const so_ray_desc* rd, const so_render_params* pr, const float* jitter,
                             const float* bkgd_rand, float* depth, float* acc, float* fars, float* rgb, float* sem,
                             float* max_depth, float* weights, float* ts, float* deltas, float* eik_grad, float* sample_sdf,
                             float* workspace, float* pair_workspace, int obj, const ObjectiveDev& D, void* stream);
int render_train_backward_obj(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* cam_mats,
                              const float* pix, const so_ray_desc* rd, const so_render_params* pr, const float* jitter,
                              const float* bkgd_rand, const float* g_depth, const float* g_acc, const float* g_rgb,
                              const float* g_sem, const float* g_weights, const float* g_eik, const float* g_sdf, float* g_vol_sdf,
                              float* g_vol_feat, float* g_inv_s, float* workspace, int obj, const ObjectiveDev& D, void* stream);

}  // namespace so
