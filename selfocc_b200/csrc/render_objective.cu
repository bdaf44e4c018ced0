// The training render with the objective's per-sample terms fused in (SURVEY.md 8f-2, DESIGN.md section 7): the C entry
// points, their argument checks and the index-ordered pass that reduces per-ray sums (the eikonal and second-grad means in
// the forward, the inv_s gradient in the backward).  The kernels are the training render's (render_train.cu) with the objective hooks of
// render_objective.cuh switched on.
#include "render_objective.cuh"
#include <math.h>

namespace so {
namespace {

constexpr int kEikThreads = 1024;

// sum of the per-ray fp64 values: thread t sums the rays t, t + 1024, ... in order, then a fixed tree over the threads.
// One CTA, no atomics: the value depends on the ray count only, never on the device or the render's grid.
// ADD: out[0] += sum (an accumulated gradient); otherwise out[0] = sum / count (a mean).
template <bool ADD>
__global__ void __launch_bounds__(kEikThreads) ordered_sum_kernel(const double* __restrict__ part, long long n_rays,
                                                                  long long count, float* __restrict__ out) {
  __shared__ double sh[kEikThreads / 32];
  double v = 0.0;
  for (long long i = threadIdx.x; i < n_rays; i += kEikThreads) v += part[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = sh[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) out[0] = ADD ? out[0] + (float)v : (float)(v / (double)count);
  }
}

bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

// the objective's operands; `stats` is the forward's output or the backward's input (both [rays, 6 * sets])
int check_objective(const so_objective_desc* ob, const so_ray_desc* rd, const float* stats) {
  if (!ob || !rd) return SO_ERR_INVALID_ARG;
  if (ob->eikonal != 0 && ob->eikonal != 1) return SO_ERR_INVALID_ARG;
  if (ob->second_grad != 0 && ob->second_grad != 1) return SO_ERR_INVALID_ARG;
  if (ob->reproj_mode == SO_OBJECTIVE_NO_REPROJ) return SO_OK;
  if (ob->reproj_mode != SO_REPROJ_COMBINE && ob->reproj_mode != SO_REPROJ_MULTI_NEW) return SO_ERR_INVALID_ARG;
  const float* ops[] = {ob->pix, ob->img2prev, ob->img2next, ob->curr_imgs, ob->prev_imgs, ob->next_imgs, stats};
  for (const float* p : ops)
    if (!p || misaligned(p, 4)) return SO_ERR_INVALID_ARG;
  if (ob->img_h < 1 || ob->img_w < 1) return SO_ERR_INVALID_ARG;
  if (!(ob->size_h > 0.f) || !(ob->size_w > 0.f) || !isfinite(ob->size_h) || !isfinite(ob->size_w)) return SO_ERR_INVALID_ARG;
  if ((int64_t)ob->img_h * ob->img_w >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;   // 32-bit offsets in one image plane
  return SO_OK;
}

int obj_kind(const so_objective_desc* ob) {
  if (ob->reproj_mode == SO_REPROJ_COMBINE) return kObjCombine;
  if (ob->reproj_mode == SO_REPROJ_MULTI_NEW) return kObjMultiNew;
  return kObjNoReproj;
}

ObjectiveDev make_objective(const so_objective_desc* ob) {
  ObjectiveDev D{};
  D.pix = ob->pix; D.m_prev = ob->img2prev; D.m_next = ob->img2next;
  D.curr = ob->curr_imgs; D.prev = ob->prev_imgs; D.next = ob->next_imgs;
  D.H = ob->img_h; D.W = ob->img_w; D.size_h = ob->size_h; D.size_w = ob->size_w;
  D.eikonal = ob->eikonal;
  D.second_grad = ob->second_grad;
  return D;
}

}  // namespace
}  // namespace so

using namespace so;

extern "C" int so_render_train_objective_forward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                                                 const float* cam_mats, const float* pix, const so_ray_desc* rd,
                                                 const so_render_params* pr, const float* jitter, const float* bkgd_rand,
                                                 const so_objective_desc* objective, float* depth, float* acc, float* fars,
                                                 float* rgb, float* sem, float* max_depth, float* weights, float* ts,
                                                 float* deltas, float* eik_grad, float* sample_sdf, float* reproj_stats,
                                                 float* reproj_colours, float* eikonal_mean, float* workspace,
                                                 float* pair_workspace, void* stream) {
  int rc = check_objective(objective, rd, reproj_stats);
  if (rc) return rc;
  if (reproj_colours && misaligned(reproj_colours, 4)) return SO_ERR_INVALID_ARG;
  if (objective->eikonal && (!eikonal_mean || misaligned(eikonal_mean, 4))) return SO_ERR_INVALID_ARG;
  if (objective->second_grad && (!objective->second_grad_mean || misaligned(objective->second_grad_mean, 4)))
    return SO_ERR_INVALID_ARG;
  const int sums = objective->eikonal + objective->second_grad;     // per-ray fp64 sums in the workspace: eikonal first
  if (sums) {
    if (!objective->workspace || misaligned(objective->workspace, 8)) return SO_ERR_INVALID_ARG;
    if (rd->ray_count < 0 || objective->workspace_bytes < 8 * sums * rd->ray_count) return SO_ERR_INVALID_ARG;
  }
  ObjectiveDev D = make_objective(objective);
  D.stats = reproj_stats;
  D.colours = reproj_colours;
  D.eik_part = static_cast<double*>(objective->workspace);
  D.sg_part = static_cast<double*>(objective->workspace) + (objective->eikonal ? rd->ray_count : 0);
  rc = render_train_forward_obj(vol_sdf, vol_feat, vol_host, cam_mats, pix, rd, pr, jitter, bkgd_rand, depth, acc, fars, rgb, sem,
                                max_depth, weights, ts, deltas, eik_grad, sample_sdf, workspace, pair_workspace, obj_kind(objective),
                                D, stream);
  if (rc || rd->ray_count == 0) return rc;
  const long long samples = rd->ray_count * (long long)pr->num_samples;
  if (objective->eikonal) {
    ordered_sum_kernel<false><<<1, kEikThreads, 0, (cudaStream_t)stream>>>(D.eik_part, rd->ray_count, samples, eikonal_mean);
    note_launch(1);
  }
  if (objective->second_grad) {
    ordered_sum_kernel<false><<<1, kEikThreads, 0, (cudaStream_t)stream>>>(D.sg_part, rd->ray_count, 3 * samples,
                                                                           objective->second_grad_mean);
    note_launch(1);
  }
  return sums ? check_launch() : SO_OK;
}

extern "C" int so_render_train_objective_backward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                                                  const float* cam_mats, const float* pix, const so_ray_desc* rd,
                                                  const so_render_params* pr, const float* jitter, const float* bkgd_rand,
                                                  const so_objective_desc* objective, const float* g_depth, const float* g_acc,
                                                  const float* g_rgb, const float* g_sem, const float* reproj_stats,
                                                  const float* grad_reproj_stats, const float* grad_eikonal_mean,
                                                  float* g_vol_sdf, float* g_vol_feat, float* g_inv_s, float* workspace,
                                                  void* stream) {
  int rc = check_objective(objective, rd, reproj_stats);
  if (rc) return rc;
  if (objective->reproj_mode != SO_OBJECTIVE_NO_REPROJ && (!grad_reproj_stats || misaligned(grad_reproj_stats, 4)))
    return SO_ERR_INVALID_ARG;
  if (grad_eikonal_mean && misaligned(grad_eikonal_mean, 4)) return SO_ERR_INVALID_ARG;
  if (objective->grad_second_grad_mean && misaligned(objective->grad_second_grad_mean, 4)) return SO_ERR_INVALID_ARG;
  if (!pr) return SO_ERR_INVALID_ARG;
  if (g_inv_s) {
    if (misaligned(g_inv_s, 4) || !objective->workspace || misaligned(objective->workspace, 8)) return SO_ERR_INVALID_ARG;
    if (rd->ray_count < 0 || objective->workspace_bytes < 8 * rd->ray_count) return SO_ERR_INVALID_ARG;
  }
  ObjectiveDev D = make_objective(objective);
  D.stats_in = reproj_stats;
  D.g_stats = grad_reproj_stats;
  D.g_eik_mean = grad_eikonal_mean;
  D.eik_count = rd->ray_count * (long long)pr->num_samples;
  D.g_sg_mean = objective->grad_second_grad_mean;
  D.sg_count = 3 * D.eik_count;
  D.inv_part = g_inv_s ? static_cast<double*>(objective->workspace) : nullptr;
  rc = render_train_backward_obj(vol_sdf, vol_feat, vol_host, cam_mats, pix, rd, pr, jitter, bkgd_rand, g_depth, g_acc, g_rgb,
                                 g_sem, nullptr, nullptr, nullptr, g_vol_sdf, g_vol_feat, g_inv_s, workspace, obj_kind(objective),
                                 D, stream);
  if (rc || !g_inv_s || rd->ray_count == 0) return rc;
  ordered_sum_kernel<true><<<1, kEikThreads, 0, (cudaStream_t)stream>>>(D.inv_part, rd->ray_count, 1, g_inv_s);
  note_launch(1);
  return check_launch();
}
