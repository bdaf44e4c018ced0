/*
 * selfocc_b200 -- C ABI of the sm_90a hot-path library (libselfocc_b200.so).
 *
 * The reference (huang-yh/SelfOcc) has no FFI of its own: its boundary for this path is the
 * mmengine registry + nn.Module contracts (SURVEY.md section 8b).  This C ABI sits UNDER
 * those Python modules; each entry point names the reference call site it replaces.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host;
 *   - tensors are dense, row-major, fp32 unless stated; index tensors are int64/int32 as stated;
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *   - no internal allocation, no implicit synchronisation: work is enqueued on `stream`;
 *   - return value: SO_OK (0) or a negative SO_ERR_* code; never throws, never prints;
 *   - thread-safe for concurrent callers that use distinct streams and distinct outputs.
 */
#ifndef SELFOCC_B200_H
#define SELFOCC_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SO_OK 0
#define SO_ERR_INVALID_ARG (-1)   /* null pointer / non-positive size / unsupported shape */
#define SO_ERR_UNSUPPORTED (-2)   /* valid request outside what the kernels implement */
#define SO_ERR_CUDA (-3)          /* a CUDA runtime call or launch failed; see so_last_cuda_error */
#define SO_ERR_NO_DEVICE (-4)

#define SO_ABI_VERSION 10  /* 2: so_render_train_forward gained pair_workspace; 3: packed render volume entry points;
                              4: backward of the fused attention cores; 5: the colour pack holds the SH-0 colour;
                              6: reprojection-loss statistics; 7: training-render sample probe;
                              8: occupancy labels and confusion matrix; 9: per-sample loss-term means;
                              10: test hooks so_linear_force_ss / so_tpv_decode_force_simt removed.
                              Entry points added since (so_mesh_*, so_voxel_*) change no existing signature: same version */

/* ABI version of the loaded library (compare with SO_ABI_VERSION). */
int so_abi_version(void);
/* cudaError_t (as int) of the most recent failing CUDA call on this host thread, 0 if none. */
int so_last_cuda_error(void);
/* Static string for an SO_* code. */
const char* so_error_string(int code);
/* Number of kernel launches enqueued by this library since process start (bench.py's
 * gpu_launches claim is read from here). */
int64_t so_launch_count(void);

/* Optional per-kernel device timing (used by bench.py for the roofline line).  When enabled, the entry
 * points bracket their dominant kernel with cudaEventRecord on the launch stream.  Tags:
 * 0 render_infer, 1 tpv_decode, 2 tpv_cross_attn, 3 tpv_self_attn, 4 msda_forward, 5 msda_backward,
 * 6 render_train_fwd, 7 render_train_bwd, 8 linear_3xtf32.  so_profile_elapsed_ms returns the SUM over the calls since
 * the last so_profile_reset (the caller must have synchronised the stream) and the call count. */
#define SO_PROF_NUM_TAGS 10
int so_profile_enable(int on);
int so_profile_reset(void);
int so_profile_elapsed_ms(int tag, float* total_ms_host, int32_t* calls_host);

/* ---------------------------------------------------------------------------------------
 * Grid <-> metre mapping, one axis.  Restates LinearMapping.meter2grid
 * (reference model/encoder/bevformer/mappings.py:97-150):
 *     c = m - start;  a = |c|
 *     g = sign(c) * (a <= range0 || size1 == 0 ? a / range0 * size0
 *                                             : size0 + (a - range0) / range1 * size1) + offset
 * offset = size0 + size1 for a mirrored (non-half) h/w axis, else 0; start = d_range[0] for d.
 * Axis order everywhere: [0] = h (from metre y), [1] = w (from metre x), [2] = d (from metre z).
 */
typedef struct so_axis_map {
  float start, range0, range1, size0, size1, offset;
} so_axis_map;

typedef struct so_volume_desc {
  int32_t H, W, Z;      /* grid sizes (size_h, size_w, size_d) */
  int32_t zpitch;       /* floats between consecutive (h, w) columns of the sdf plane, >= Z */
  int32_t n_feat;       /* decoded channels besides sdf (colour + semantics), 0 if none */
  int32_t feat_pitch;   /* floats per voxel in the channel-last feature volume (>= n_feat, %4==0) */
  so_axis_map axis[3];
} so_volume_desc;

/* ---------------------------------------------------------------------------------------
 * B5  TPV planes -> decoded volume.  Replaces field.pre_compute_density_color(representation)
 * (call sites model/head/neus_head/neus_head.py:249,302,483; semantics from the in-repo analogue
 * model/head/nerfacc_head/bev_nerf.py:62-95, tpv=True, density_layers=2):
 *     f[h,w,z,:] = hw[h,w,:] + zh[z,h,:] + wz[w,z,:]
 *     out        = W2 * softplus(W1 * softplus(f) + b1) + b2          (C -> C -> 1 + n_feat)
 * tpv_hw [H*W, C], tpv_zh [Z*H, C], tpv_wz [W*Z, C]; w1 [C, C], b1 [C], w2 [1+n_feat, C], b2.
 * Outputs: vol_sdf [H, W, zpitch] (channel 0; pad entries z in [Z, zpitch) written as 0), vol_feat [H, W, Z, feat_pitch]
 * (channels 1.., may be NULL when n_feat == 0; the pad channels [n_feat, feat_pitch) are never written: a caller that reads
 * them clears the buffer first).  C is 32, 64, 96 or 128 and 1 + n_feat <= 32, else SO_ERR_UNSUPPORTED before any launch.
 */
int so_tpv_decode(const float* tpv_hw, const float* tpv_zh, const float* tpv_wz, int32_t C,
                  const float* w1, const float* b1, const float* w2, const float* b2,
                  const so_volume_desc* vol_host, float* vol_sdf, float* vol_feat, void* stream);
/* Same, for the row range [h_begin, h_begin + h_count) of the volume only (voxel-sharded decode: every rank decodes its
 * slab of h rows into the full-size buffers and one all_gather assembles the volume; SURVEY 8e).  Other rows untouched. */
int so_tpv_decode_rows(const float* tpv_hw, const float* tpv_zh, const float* tpv_wz, int32_t C, const float* w1,
                       const float* b1, const float* w2, const float* b2, const so_volume_desc* vol_host, int32_t h_begin,
                       int32_t h_count, float* vol_sdf, float* vol_feat, void* stream);

/* Backward of the decode MLP over one slab of h rows (training).  The two [rows x C x C] products of the slab run through
 * so_linear_3xtf32; these are the element-wise pieces around them (reference: autograd through the decoder MLP,
 * model/head/neus_head/bev_nerf.py:150-190).  rows = h_count * W * Z, voxel order (h, w, z) inside the slab.
 *   features: a0[rows][C] = softplus(hw + zh + wz)
 *   hidden:   z1_a1[rows][C] holds z1 = a0 W1^T + b1 on entry and a1 = softplus(z1) on return;
 *             g1 = (W2^T g_out) * sigmoid(z1); g_out[rows][1 + n_feat] = the slab's output gradient gathered from
 *             g_vol_sdf [H][W][zpitch] (may be NULL = zero) and g_vol_feat [H][W][Z][feat_pitch] (may be NULL = zero)
 *   input:    g0[n] *= 1 - exp(-a0[n])   (= sigmoid of the pre-activation), n % 4 == 0
 * The sdf pads and feature pad channels of g_vol_sdf / g_vol_feat are never read.  softplus and both sigmoid factors are
 * accurate relative to their own value (1e-5 or better down to a pre-activation of -16 and below), not only absolutely:
 * a channel whose activations are all small still gets a gradient that is right relative to itself.                      */
int so_tpv_decode_bwd_features(const float* tpv_hw, const float* tpv_zh, const float* tpv_wz, int32_t C,
                               const so_volume_desc* vol_host, int32_t h_begin, int32_t h_count, float* a0, void* stream);
int so_tpv_decode_bwd_hidden(float* z1_a1, const float* g_vol_sdf, const float* g_vol_feat, const float* w2, int32_t C,
                             const so_volume_desc* vol_host, int32_t h_begin, int32_t h_count, float* g1, float* g_out,
                             void* stream);
int so_tpv_decode_bwd_input(float* g0, const float* a0, int64_t n, void* stream);

/* B5 for tpv=False heads (the BEV-only model; bev_nerf.py:62-81, density_layers=2):
 *     out[r][z * Cf + c] = W2 * softplus(W1 * softplus(bev[r]) + b1) + b2          (C -> C -> Z * Cf), Cf = 1 + n_feat
 * bev [H*W, C] (row r = h * W + w); w1 [C, C], b1 [C], w2 [Z * Cf, C], b2 [Z * Cf].  Column z * Cf + c of row r is voxel
 * (h, w, z), channel c: c = 0 -> vol_sdf [H, W, zpitch] (pads z in [Z, zpitch) written as 0), c >= 1 -> vol_feat
 * [H, W, Z, feat_pitch] channel c - 1 (may be NULL when n_feat == 0; pad channels never written, as so_tpv_decode).
 * One persistent wgmma kernel with the 3xTF32 split; the hidden and output matrices never reach global memory, and every
 * voxel is computed the same way whatever the SM count.  C == 96 and Z * Cf <= 2048, else SO_ERR_UNSUPPORTED before any
 * launch; bev, w1 and w2 16-byte aligned. */
int so_bev_decode(const float* bev, int32_t C, const float* w1, const float* b1, const float* w2, const float* b2,
                  const so_volume_desc* vol_host, float* vol_sdf, float* vol_feat, void* stream);
/* Same, for the row range [h_begin, h_begin + h_count) of the volume only (the decode-sharded training step: every rank
 * decodes its slab of h rows, BEV rows h_begin * W .. (h_begin + h_count) * W - 1, into the full-size buffers).  Other rows
 * untouched, including their sdf pads.  A negative or overflowing range is SO_ERR_INVALID_ARG; h_count == 0 does nothing.
 * so_bev_decode is the range [0, H). */
int so_bev_decode_rows(const float* bev, int32_t C, const float* w1, const float* b1, const float* w2, const float* b2,
                       const so_volume_desc* vol_host, int32_t h_begin, int32_t h_count, float* vol_sdf, float* vol_feat,
                       void* stream);
/* Element-wise pieces of its backward (training), around the products on so_linear_3xtf32 / cuBLAS:
 *   gather:   g_out[row_count][Z * Cf] of rows [row_begin, row_begin + row_count) from g_vol_sdf / g_vol_feat (NULL = zero;
 *             sdf pads and feature pad channels never read)
 *   features: a0[n] = softplus(bev[n])
 *   hidden:   z1_a1[n] holds z1 on entry and a1 = softplus(z1) on return; g1[n] *= sigmoid(z1)
 * with the relative-accuracy softplus / sigmoid forms of so_tpv_decode_bwd_*; the input side is so_tpv_decode_bwd_input. */
int so_bev_decode_bwd_gather(const float* g_vol_sdf, const float* g_vol_feat, const so_volume_desc* vol_host, int64_t row_begin,
                             int64_t row_count, float* g_out, void* stream);
int so_bev_decode_bwd_features(const float* bev, int64_t n, float* a0, void* stream);
int so_bev_decode_bwd_hidden(float* z1_a1, float* g1, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------
 * Ray set of one frame: n_cam cameras x rays_per_cam pixel rays, flattened (cam, ray)-major
 * exactly like neus_head.py:324-325.  Pixel coordinates come either from `pix` ([rays_per_cam, 2]
 * (x, y), RaySampler.forward(), ray_sampler.py:48-68) or, when pix == NULL, from the strided grid
 *     x = j * sx + ox,  y = i * sy + oy,  ray = i * nx + j          (ray_sampler.py:23-31,58-68)
 * cam_mats [n_cam, 4, 4] = metas[trans_kw] (img2lidar.py:25-70): origin = M[:3,3],
 * direction = M[:3,:3] * (x, y, 1), un-normalised; its norm converts ray length <-> camera depth.
 */
typedef struct so_ray_desc {
  int32_t n_cam, rays_per_cam;
  int32_t nx, ny;            /* grid shape, used when pix == NULL (nx * ny == rays_per_cam) */
  float sx, ox, sy, oy;
  int64_t ray_begin;         /* first flat ray index this call renders (ray sharding across GPUs) */
  int64_t ray_count;         /* number of flat rays this call renders */
  int64_t chunk_len;         /* rays per reference chunk (neus_head.py:341-345 `--batch`); the
                                expected-depth clip is taken per chunk.  <= 0: one chunk */
} so_ray_desc;

typedef struct so_render_params {
  float aabb[6];             /* roi_aabb x0 y0 z0 x1 y1 z1 (neus_head.py:189-195) */
  float near_plane;          /* near clamp, applied when `training` (collider) */
  int32_t training;          /* 0: eval (near clamp 0, rgb clamped), 1: train */
  int32_t num_samples;       /* S, uniform bins per ray (neus_head.py:136) */
  float inv_s;               /* exp(10 * variance) of the deviation network, clipped 1e-6..1e6 */
  float cos_anneal;          /* NeuS cos anneal ratio, 1.0 after warm-up */
  int32_t anchor_mid;        /* 1: field queried at bin midpoints, 0: at bin starts */
  int32_t sh_act;            /* 0: relu(C0*f + 0.5), 1: sigmoid(C0*f)  (sh_render.py:84-94, deg 0) */
  int32_t bkgd_mode;         /* 0 black, 1 white, 2 per-ray colours given in bkgd_rand */
} so_render_params;

/* Workspace floats needed by so_render_infer for `n_chunks` depth-clip chunks. */
int64_t so_render_workspace_floats(int64_t n_chunks);

/* B1-B4, B6-B11  fused inference render: ray generation -> AABB -> S samples -> trilinear gather
 * (+ analytic sdf gradient) -> NeuS alpha -> compositing -> depth / max-depth / acc / normal / rgb.
 * Replaces the chunk loop `self.model(ray_bundle)` + post-processing of NeuSHead.render
 * (model/head/neus_head/neus_head.py:319-438).  Outputs are indexed by (flat ray - ray_begin);
 * any output pointer may be NULL.  depth/max_depth are camera-z depths (divided by |direction|).
 *   depth [n], max_depth [n], max_idx int64 [n] (first-max argmax of w/delta, :430-438),
 *   acc [n], normal_vis [n,3], rgb [n,3] (needs n_feat >= 3), sem [n, n_feat-3] (needs n_feat > 3).
 * workspace: so_render_workspace_floats(n_chunks) floats, n_chunks = ceil(total rays / chunk_len).
 */
int so_render_infer(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                    const float* cam_mats, const float* pix, const so_ray_desc* rays_host,
                    const so_render_params* params_host, const float* bkgd_rand,
                    float* depth, float* max_depth, int64_t* max_idx, float* acc,
                    float* normal_vis, float* rgb, float* sem, float* workspace, void* stream);

/* Packed render volume: a once-per-frame repack of the decoded volume into the layout the gather of the inference
 * render wants (built by NeuSHead.prepare, reused by every render of the frame -- eval_novel_depth.py:143-172 renders
 * several poses per prepare):
 *   n_feat == 0 : float2 [H][W][zpitch] {sdf[z], sdf[z+1]}  -- the 8 trilinear taps become 4 aligned 64-bit loads
 *   n_feat == 3 : float4 [H][W][Z]      {C0 r + 0.5, C0 g + 0.5, C0 b + 0.5, sdf}, C0 = 0.28209479177387814 (SH degree 0)
 *                 -- 8 aligned 128-bit loads fetch sdf and colour together.  The colour lanes hold the SH-0 colour before
 *                 its relu (one fmaf per channel), not the decoded features: trilinear weights sum to one, so the map
 *                 commutes with the interpolation and the render applies only the relu.  The sdf lane is the decoded sdf.
 * so_render_pack_floats: floats needed (0: this channel count has no packed form).  pack must be 16-byte aligned. */
int64_t so_render_pack_floats(const so_volume_desc* vol_host);
int so_render_pack(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, float* pack, void* stream);

/* so_render_infer on the packed volume (same outputs, same semantics; `pack` from so_render_pack, NULL = plain
 * so_render_infer).  Used when the metre->grid map is affine, num_samples is a power of two, the cos-anneal is finished,
 * samples are taken at bin midpoints and no semantics are rendered; any other configuration is routed to so_render_infer.
 * Rays that leave the volume take the zero-padding loop inside the same launch.  A warp stops marching when every
 * ray's transmittance is below 1e-9 (changes the outputs by < 1e-9 relative, never the max-depth index).
 * dbg_grid: optional probe [n, S, 3]: the fp32 (h, w, d) grid coordinates of every sample exactly as the kernel computed
 * them (test hook: lets a fp64 oracle be evaluated in the kernel's own cells, the analytic sdf gradient being
 * discontinuous across cell faces); NULL in production. */
int so_render_infer_packed(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* pack,
                           const float* cam_mats, const float* pix, const so_ray_desc* rays_host,
                           const so_render_params* params_host, const float* bkgd_rand,
                           float* depth, float* max_depth, int64_t* max_idx, float* acc,
                           float* normal_vis, float* rgb, float* sem, float* workspace, float* dbg_grid, void* stream);

/* B6-B10, B13  training-form render (NeuSHead.forward, neus_head.py:513-587): same sampling / field / alpha /
 * compositing as so_render_infer but it EMITS the per-sample tensors the losses consume (:667-682) and has a
 * backward.  `jitter` [total rays, S+1] uniforms in [0,1) for the stratified sampler (`perturb=True`), NULL =
 * no jitter.  Per-ray outputs [n]: depth, acc, fars (far / |dir|), max_depth, rgb [n,3], sem [n,n_feat-3];
 * per-sample outputs [n,S]: weights, ts = mid / |dir|, deltas = (end-start) / |dir|, sample_sdf; eik_grad [n,S,3]
 * = d sdf / d metre at the samples.  Any output may be NULL.  S <= 256.
 * pair_workspace: optional scratch of so_render_train_pair_floats(vol) floats (8-byte aligned), NULL = none.  When
 * given, the sdf volume is first repacked as {v[z], v[z+1]} pairs so that the 8 trilinear taps become 4 aligned
 * 64-bit loads (half the L1 requests of the gather-bound forward); results are bit-identical either way. */
int64_t so_render_train_pair_floats(const so_volume_desc* vol_host);
int so_render_train_forward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                            const float* cam_mats, const float* pix, const so_ray_desc* rays_host,
                            const so_render_params* params_host, const float* jitter, const float* bkgd_rand,
                            float* depth, float* acc, float* fars, float* rgb, float* sem, float* max_depth,
                            float* weights, float* ts, float* deltas, float* eik_grad, float* sample_sdf,
                            float* workspace, float* pair_workspace, void* stream);

/* Test hook: force the one-ray-per-warp forward kernel (default: the batched-ray kernel whenever the mapping is affine,
 * num_samples is a power of two >= 64, the cos-anneal is finished and no semantics are rendered). */
int so_render_train_force_fwd32(int on);
/* Test hook: render 24-channel feature volumes through the generic (any channel count) semantic path instead of the
 * vectorised 3 rgb + 21 class specialisation (config/nuscenes/nuscenes_occ.py:350). */
int so_render_train_force_sem_generic(int on);

/* Backward of so_render_train_forward w.r.t. the decoded volume and inv_s.  Incoming gradients (NULL = zero):
 * g_depth, g_acc [n], g_rgb [n,3], g_sem [n,n_feat-3], g_weights, g_sdf [n,S], g_eik [n,S,3].  Results are
 * ACCUMULATED (atomically) into g_vol_sdf [H,W,zpitch], g_vol_feat [H,W,Z,feat_pitch] (needed iff g_rgb/g_sem)
 * and the scalar g_inv_s; the caller zero-fills them.  Recomputes the forward (nothing is saved). */
int so_render_train_backward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                             const float* cam_mats, const float* pix, const so_ray_desc* rays_host,
                             const so_render_params* params_host, const float* jitter, const float* bkgd_rand,
                             const float* g_depth, const float* g_acc, const float* g_rgb, const float* g_sem,
                             const float* g_weights, const float* g_eik, const float* g_sdf,
                             float* g_vol_sdf, float* g_vol_feat, float* g_inv_s, float* workspace, void* stream);

/* Test probe of the training render's sample geometry (the training analogue of so_render_infer_packed's dbg_grid):
 * same ray / param / jitter / volume operands as so_render_train_forward.  grid [n, S, 3] receives the fp32 (h, w, d) grid
 * coordinates of every sample, computed with the device function that so_render_train_forward's one-ray-per-warp kernel
 * and so_render_train_backward use for this configuration (the backward recomputes the samples with the arithmetic of
 * the forward it is paired with).  The batched forward kernel builds the same values with its own edge arithmetic; its
 * `ts` / `deltas` outputs are bit-identical to the one-ray-per-warp kernel's. */
int so_render_train_probe(const so_volume_desc* vol_host, const float* cam_mats, const float* pix, const so_ray_desc* rays_host,
                          const so_render_params* params_host, const float* jitter, float* grid, void* stream);

/* Backward of so_field_query: g_sdf [n], g_grad [n,3], g_feat [n,n_feat] (NULL = zero) accumulated into
 * g_vol_sdf / g_vol_feat (caller zero-fills). */
int so_field_query_backward(const so_volume_desc* vol_host, const float* points, int64_t n, const float* g_sdf,
                            const float* g_grad, const float* g_feat, float* g_vol_sdf, float* g_vol_feat, void* stream);

/* B8  `second_grad` (neus_head.py:177,703-706 -> loss/second_grad_loss.py:19-20), DECLARED ASSUMPTION: the quantity lives in
 * the un-vendored fork; restated as the double-backward idiom d(sum_j d sdf/d x_j)/d x of the trilinear field = the row
 * sums of its Hessian in metres (pure second derivatives vanish inside a cell, the mixed ones do not).  points [n,3]
 * metres -> second_grad [n,3].  Backward: g_second_grad [n,3] accumulated atomically into g_vol_sdf (caller zero-fills). */
int so_field_second_grad(const float* vol_sdf, const so_volume_desc* vol_host, const float* points, int64_t n,
                         float* second_grad, void* stream);
int so_field_second_grad_backward(const so_volume_desc* vol_host, const float* points, int64_t n, const float* g_second_grad,
                                  float* g_vol_sdf, void* stream);

/* 8f-3  device-side DepthMetric step (utils/metric_util.py:247-279,311-349; eval_novel_depth.py:174-200).
 * so_depth_metric_sample: depth_pred [N,h,w], loc [N,n,2] in [0,1] (x,y) -> sampled [N,n] with the arithmetic of
 *   F.grid_sample(pred, loc*2-1, bilinear, padding_mode='border', align_corners=True).
 * so_depth_metric_sums: per camera, over points with mask != 0 and pred' = clamp(scale[cam] * sampled, 1e-3, 80)
 *   (scale NULL = 1): sums [N,8] = (sum |gt-pred'|/gt, sum (gt-pred')^2/gt, sum (gt-pred')^2, sum (log gt - log pred')^2,
 *   #(thresh < 1.25), #(< 1.25^2), #(< 1.25^3), #points); the metrics are sums / #points (rmse: sqrt).  One CTA per
 *   camera, deterministic. */
int so_depth_metric_sample(const float* depth_pred, const float* loc, int32_t N, int32_t n, int32_t h, int32_t w,
                           float* sampled, void* stream);
int so_depth_metric_sums(const float* sampled, const float* depth_gt, const uint8_t* mask, const float* scale, int32_t N,
                         int32_t n, float* sums, void* stream);
/* 8f-3  novel-view depth evaluation (eval_novel_depth.py:159-208, eval_novel_depth_kitti.py): the depth maps of K poses x
 * N cameras, depth_maps [n_seg = K*N, h, w], against a ragged LiDAR set in CSR form with one segment per (pose, camera):
 * segment s is points [offsets[s], offsets[s+1]) of loc [T,2] in [0,1] (x,y), depth_gt [T], mask [T] (uint8).  Each point
 * with mask != 0 samples map s with the arithmetic of so_depth_metric_sample; errors [n_seg, 7] = the segment's
 * compute_depth_errors_torch (utils/metric_util.py:424-445) metrics (abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3) at
 * pred' = clamp(sampled, 1e-3, 80): means over the masked points, rmse / rmse_log the square roots of means.  A segment
 * without a masked point gives NaN in all seven.  One CTA per segment, fp64 sums in a fixed order: bit-identical run to
 * run.  offsets lives on the device; offsets_host is the same array in host memory, checked before the launch: refused
 * (SO_ERR_INVALID_ARG) are null pointers, n_seg < 1, h or w < 1, offsets_host[0] != 0, offsets_host[n_seg] != T and
 * decreasing offsets; h * w >= 2^31 is SO_ERR_UNSUPPORTED. */
int so_novel_depth_errors(const float* depth_maps, int32_t n_seg, int32_t h, int32_t w, const int64_t* offsets,
                          const int64_t* offsets_host, int64_t T, const float* loc, const float* depth_gt, const uint8_t* mask,
                          float* errors, void* stream);

/* B12  field query at arbitrary points.  Replaces field.forward_sdfnetwork / forward_geonetwork
 * as used by NeuSHead.get_uniform_sdf (neus_head.py:265-293).  points [n,3] metres ->
 * sdf [n], grad [n,3] (NULL ok), feat [n, n_feat] raw decoded channels 1.. (NULL ok). */
int so_field_query(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                   const float* points, int64_t n, float* sdf, float* grad, float* feat, void* stream);

/* ---------------------------------------------------------------------------------------
 * Occupancy evaluation (eval_iou.py:196-270, eval_iou_kitti.py:160-190) from the decoded volume.
 * The uniform lattice of NeuSHead.get_uniform_sdf (neus_head.py:265-293) is given by its axes xs [nx], ys [ny], zs [nz]
 * (metres; lattice point (iy, ix, iz) = (xs[ix], ys[iy], zs[iz]), layout [ny, nx, nz]).  A lattice value is the field
 * query of so_field_query at that point, evaluated on the fly: nothing but the byte labels is written.
 * Semantics: the argmax (first maximum, like torch.argmax) over the n_sem vol_feat channels [sem_begin, sem_begin + n_sem)
 * (the head's logits h[..., 4:] are vol_feat channels 3..), mapped through lut (uint8 [n_sem], NULL = the raw argmax).
 *   so_occ_lattice_labels: occ [ny, nx, nz] = sdf <= thresh;  sem [ny, nx, nz] = occ ? lut[argmax] : 0 (sem NULL: not
 *     computed).  Equals thresholding / arg-maxing forward_occ's sdf / logits.
 *   so_occ_sample_labels: points [m, 3] normalised to the lattice's unit cube (u = (p - aabb_min) / expansion); each label
 *     uses the values of F.grid_sample(lattice[None, None], u[..., [2, 0, 1]] * 2 - 1, bilinear, padding_mode='zeros',
 *     align_corners=True) for the sdf and every logit channel: occ [m] = sdf' <= thresh, sem [m] = occ ? lut[argmax'] : 0.
 * Logits are only gathered where occ is set.  Refused: null pointers, sizes < 1, a channel range outside n_feat when sem
 * is requested. */
int so_occ_lattice_labels(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* xs,
                          int32_t nx, const float* ys, int32_t ny, const float* zs, int32_t nz, float thresh, int32_t sem_begin,
                          int32_t n_sem, const uint8_t* lut, uint8_t* occ, uint8_t* sem, void* stream);
int so_occ_sample_labels(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* xs,
                         int32_t nx, const float* ys, int32_t ny, const float* zs, int32_t nz, const float* points, int64_t m,
                         float thresh, int32_t sem_begin, int32_t n_sem, const uint8_t* lut, uint8_t* occ, uint8_t* sem,
                         void* stream);
/* Confusion matrix of two label arrays pred, gt (uint8 [n]) over the elements with mask != 0 (mask NULL = all) and
 * gt != ignore (-1 = none): counts[(n_cls + 1) * g + p] += 1, labels >= n_cls counted in bin n_cls.  counts int64
 * [(n_cls + 1)^2] is ACCUMULATED (the caller zero-fills it).  1 <= n_cls <= 255.  Integer atomics: deterministic. */
int so_occ_confusion(const uint8_t* pred, const uint8_t* gt, const uint8_t* mask, int64_t n, int32_t n_cls, int32_t ignore,
                     int64_t* counts, void* stream);

/* ---------------------------------------------------------------------------------------
 * Surface extraction (the mesh that vis_3d.py / vis_3d_scene.py draw as voxels from forward_occ(..., occ_only=True)):
 * marching cubes over the lattice of so_occ_lattice_labels (axes xs [nx], ys [ny], zs [nz], layout [ny, nx, nz], values the
 * so_field_query sdf, evaluated on the fly).  Point p = (iy, ix, iz), index (iy * nx + ix) * nz + iz, is inside when
 * sdf <= thresh, so the surface bounds exactly the points so_occ_lattice_labels marks occupied; it is open where it leaves
 * the lattice.  Point p owns its +x, +y and +z edges; an edge crosses when its ends lie on different sides, and its vertex
 * is p_a + t (p_b - p_a), t = (thresh - s_a) / (s_b - s_a).  Cell p is the cube whose lowest corner is p; its triangles
 * come from the case table of selfocc_b200/mc_table.py (csrc/mc_table.cuh), counter-clockwise seen from the outside
 * (sdf > thresh).
 *   so_mesh_count: counts int32 [2, N] (N = nx * ny * nz): counts[0][p] = crossing edges owned by p, counts[1][p] =
 *     triangles of cell p (0 on the upper border); edge_mask uint8 [N], bit a = p's +a edge crosses (a = x, y, z).
 *   so_mesh_emit: given scans = the INCLUSIVE scans of both rows of counts (int32 [2, N]), the same edge_mask and their
 *     totals n_vertices = sum(counts[0]), n_faces = sum(counts[1]): vertices [n_vertices, 3] fp32 metres in ascending
 *     owner index then axis, faces [n_faces, 3] int32 vertex ids in ascending cell index then table order.  One thread
 *     writes each output: bit-identical run to run.
 * Refused (SO_ERR_INVALID_ARG): null pointers, an axis shorter than 2, negative totals.  N >= 2^31 and totals >= 2^31
 * (int32 ids) are SO_ERR_UNSUPPORTED.  Both checks come before any CUDA call. */
int so_mesh_count(const float* vol_sdf, const so_volume_desc* vol_host, const float* xs, int32_t nx, const float* ys, int32_t ny,
                  const float* zs, int32_t nz, float thresh, int32_t* counts, uint8_t* edge_mask, void* stream);
int so_mesh_emit(const float* vol_sdf, const so_volume_desc* vol_host, const float* xs, int32_t nx, const float* ys, int32_t ny,
                 const float* zs, int32_t nz, float thresh, const int32_t* scans, const uint8_t* edge_mask, int64_t n_vertices,
                 int64_t n_faces, float* vertices, int32_t* faces, void* stream);

/* ---------------------------------------------------------------------------------------
 * Voxel-cube drawing of a label volume (what vis_3d.py / vis_3d_scene.py draw with mayavi's cube glyphs).
 * Grid: labels uint8 [H, W, D] contiguous on the device, the layout NeuSHead.occupancy returns; voxel (h, w, d), index
 * (h * W + w) * D + d, is the cube of side voxel_size whose lowest corner is origin_host + (w, h, d) * voxel_size (x, y, z
 * metres; origin_host is 3 floats in host memory).  Face code 2a + s: axis a (0 x, 1 y, 2 z), s = 0 the cube's lower
 * face on that axis, s = 1 its upper face.  A label l is drawn when palette_host[4 l + 3] (its alpha) is non-zero
 * (so_voxel_render) or drawn_host[l] is non-zero (the face kernels).
 *
 * so_voxel_render: K cameras, each 16 floats of cams (device, 16-byte aligned): origin (3), a row-major 3x3 matrix M (9),
 *   near, far, 2 unused.  Pixel (u, v) of an img_h x img_w image (v down) is the ray o + t M (u + 1/2, v + 1/2, 1), t the
 *   ray parameter (for look-at and Img2LiDAR cameras: the depth along the optical axis, the quantity a VTK clipping
 *   range bounds).  The ray is clipped to the grid's box and walks its cells with an Amanatides-Woo DDA in fp64
 *   (integer cell steps; a zero direction component never steps).  The hit is the first drawn voxel the ray enters
 *   within [near, far]; a voxel that holds the ray's point at near was entered before near and is skipped.  Its colour is
 *   round-half-even(palette[label].rgb * shade_host[face]) in fp32, face the face entered; a pixel with no hit gets
 *   background_host (3 bytes).  Outputs (device, any may be null, not all): rgb uint8 [K, img_h, img_w, 3], voxel int32
 *   [K, img_h, img_w] hit index or -1, face int8 [K, img_h, img_w] or -1, dist fp32 [K, img_h, img_w] hit t or +inf.
 *   palette_host [256 * 4] RGBA bytes and shade_host [6] floats in [0, 1] are host memory, copied into the launch.
 * so_voxel_faces_count: counts int32 [H W D], the number of exposed faces of each voxel: a face of a drawn voxel whose
 *   6-neighbour is not drawn or lies outside the grid.
 * so_voxel_faces_emit: given scans = the INCLUSIVE scan of counts and its total n_faces: each exposed face as 4 vertices
 *   fp32 [4 n_faces, 3] and 2 triangles int32 [2 n_faces, 3], counter-clockwise seen from outside, in ascending voxel
 *   index then face code; per vertex the outward unit normal fp32 [4 n_faces, 3] and the voxel's label (sem uint8
 *   [4 n_faces], may be null).  Quad corners: with (b, c) = (a + 1, a + 2) mod 3, (b, c) offsets (0,0) (1,0) (1,1) (0,1)
 *   on an upper face, (0,0) (0,1) (1,1) (1,0) on a lower one; triangles (0, 1, 2) and (0, 2, 3).
 * One thread writes each output: bit-identical run to run, no host synchronisation.
 * Refused (SO_ERR_INVALID_ARG) before any CUDA call: null pointers, non-positive sizes, K = 0, voxel_size not positive and
 * finite, n_faces < 1, a shade outside [0, 1], misaligned cams (16 bytes) or 4-byte outputs.  H W D >= 2^31, K > 65535
 * and 4 n_faces >= 2^31 are SO_ERR_UNSUPPORTED. */
int so_voxel_render(const uint8_t* labels, int32_t H, int32_t W, int32_t D, const float* origin_host, float voxel_size,
                    const float* cams, int32_t K, int32_t img_h, int32_t img_w, const uint8_t* palette_host,
                    const float* shade_host, const uint8_t* background_host, uint8_t* rgb, int32_t* voxel, int8_t* face,
                    float* dist, void* stream);
int so_voxel_faces_count(const uint8_t* labels, int32_t H, int32_t W, int32_t D, const uint8_t* drawn_host, int32_t* counts,
                         void* stream);
int so_voxel_faces_emit(const uint8_t* labels, int32_t H, int32_t W, int32_t D, const float* origin_host, float voxel_size,
                        const uint8_t* drawn_host, const int32_t* scans, int64_t n_faces, float* vertices, int32_t* faces,
                        float* normals, uint8_t* sem, void* stream);

/* ---------------------------------------------------------------------------------------
 * A7/A8  multi-scale deformable attention forward.  Drop-in for
 * MultiScaleDeformableAttnFunction.apply(value, spatial_shapes, level_start_index,
 * sampling_locations, attention_weights, im2col_step) of mmcv==2.0.1 (reference call sites
 * model/encoder/bevformer/attention/image_cross_attention.py:340-342 and
 * model/encoder/tpvformer/attention/cross_view_hybrid_attention.py:111-113).
 *   value [B, Nv, Hd, Dh]   spatial_shapes int64 [L,2] (h,w)   level_start_index int64 [L]
 *   loc [B, Nq, Hd, L, P, 2] normalised (x,y)   weights [B, Nq, Hd, L, P]   out [B, Nq, Hd*Dh]
 * Dh must be 16 or 32.
 */
int so_msda_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                    const float* loc, const float* weights, float* out,
                    int32_t B, int32_t Nv, int32_t Hd, int32_t Dh, int32_t Nq, int32_t L, int32_t P,
                    void* stream);

/* Backward of so_msda_forward (the mmcv op's autograd contract): grad_out [B,Nq,Hd*Dh] ->
 * grad_value [B,Nv,Hd,Dh] (must be zero-filled by the caller; accumulated atomically),
 * grad_loc [B,Nq,Hd,L,P,2], grad_weights [B,Nq,Hd,L,P]. */
int so_msda_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                     const float* loc, const float* weights, const float* grad_out,
                     float* grad_value, float* grad_loc, float* grad_weights,
                     int32_t B, int32_t Nv, int32_t Hd, int32_t Dh, int32_t Nq, int32_t L, int32_t P,
                     void* stream);

/* A6/A9  dense projection on the Hopper tensor cores (wgmma) with fp32-level accuracy ("3xTF32" operand splitting):
 *     y[M,N] = act(x[M,K] * w[N,K]^T + bias[N]) (+ residual[M,N])
 * Replaces the nn.Linear calls of the attention modules and the FFN (image_cross_attention.py:36,218-223,309-317,
 * cross_view_hybrid_attention.py:79-86,118, tpvformer_encoder_layer.py:198-206).  w_hi / w_lo = so_split_tf32(w)
 * (w_hi = w with the low 13 mantissa bits cleared, w_lo = w - w_hi), computed once per weight.  K % 96 == 0, N even;
 * x, w_hi, w_lo 16-byte aligned (TMA), y and residual 8-byte aligned; relu: 0/1; bias / residual may be NULL. */
int so_split_tf32(const float* w, float* w_hi, float* w_lo, int64_t n, void* stream);
int so_linear_3xtf32(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                     float* y, int64_t M, int32_t N, int32_t K, int32_t relu, void* stream);

/* A9  projection + LayerNorm in ONE launch: y = LayerNorm(act(x w^T + bias) + residual) * gamma + beta over the N output
 * columns, computed in the GEMM epilogue (an epilogue thread owns a whole output row, so the statistics are register-local).
 * Replaces `output_proj -> (+ identity) -> norm` and `ffn.layers[1] -> (+ identity) -> norm` of TPVFormerLayer
 * (tpvformer_encoder_layer.py:185-218).  N % 32 == 0, N <= 128; otherwise as so_linear_3xtf32. */
int so_linear_3xtf32_ln(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                        const float* gamma, const float* beta, float eps, float* y, int64_t M, int32_t N, int32_t K,
                        int32_t relu, void* stream);

/* A9  y = LayerNorm(x [+ add]) over the last dimension C (nn.LayerNorm(C), biased variance, eps inside the sqrt),
 * replaces the norm steps of TPVFormerLayer (tpvformer_encoder_layer.py:185-196).  x, add, y [rows, C]; C <= 256. */
int so_layer_norm(const float* x, const float* add, const float* gamma, const float* beta, float* y, int64_t rows,
                  int32_t C, float eps, void* stream);

/* A3  one FPN level into the flattened token tensor (tpvformer_encoder.py:261-277): feat [N, C, hw] ->
 * out[n, level_start + p, :] = (feat[n, :, p] + cams_embeds[n, :]) + level_embed[:], out being [N, total, C].  Replaces
 * flatten(3).permute(...) + the two embedding adds + torch.cat over levels + .contiguous() (five passes over 59 MB). */
int so_flatten_level(const float* feat, const float* cams_embeds, const float* level_embed, float* out, int32_t N, int32_t C,
                     int32_t hw, int64_t level_start, int64_t total, void* stream);

/* A4  projection of pillar reference points into the cameras.  Replaces point_sampling
 * (model/encoder/bevformer/utils.py:116-206, including the focal_ratios branch through
 * so_point_sampling_scaled; the post_rots branch, which no shipped pipeline produces, is not covered).
 *   ref_3d [D, Q, 3] metres, lidar2img [N, 4, 4], img_h/img_w = metas[0]['img_shape']
 *   -> uv [N, Q, D, 2] normalised (x, y), mask uint8 [N, Q, D] (1 = in frustum),
 *      vis uint8 [N, Q] = any_d mask (the per-camera query visibility of
 *      image_cross_attention.py:92; NULL ok).
 * Arithmetic order is fixed (plain fp32 mul/add, no FMA contraction) so that `mask`, an index-
 * generating quantity, is reproducible bit for bit.  Same as so_point_sampling_scaled with scale_xy = NULL. */
int so_point_sampling(const float* ref_3d, const float* lidar2img, int32_t D, int32_t Q, int32_t N,
                      float img_h, float img_w, float* uv, uint8_t* mask, uint8_t* vis, void* stream);

/* A4 with the focal-ratio rescale of bevformer/utils.py:198-204 (metas[0]['focal_ratios_x' / '_y'],
 * written by RandomScaleImageMultiViewImage).  scale_xy [N, 2] fp32 device memory holds
 * (ratio_x, ratio_y) per camera, or NULL for none (bit-identical to so_point_sampling).  After the
 * frustum test, uv[cam, ..., 0] *= ratio_x[cam] and uv[cam, ..., 1] *= ratio_y[cam], each one fp32
 * multiply; mask and vis are those of the unscaled coordinates, as in the reference, so a visible
 * sample may lie outside [0, 1] when a ratio exceeds 1.  The ratios are read on the device when the
 * kernel runs (a captured graph picks up new values written into scale_xy).  Same error returns as
 * so_point_sampling. */
int so_point_sampling_scaled(const float* ref_3d, const float* lidar2img, const float* scale_xy, int32_t D,
                             int32_t Q, int32_t N, float img_h, float img_w, float* uv, uint8_t* mask,
                             uint8_t* vis, void* stream);

/* A5+A6+A7  rebatch-free image cross-attention core for one TPV plane.  Replaces the
 * nonzero()/rebatch/scatter-add/count machinery of BEVCrossAttention.forward together with the
 * location arithmetic, softmax and op call of BEVDeformableAttention.forward
 * (model/encoder/bevformer/attention/image_cross_attention.py:84-136, 313-345):
 *   for every query q:  slots[q] = (1 / max(1, #visible cams)) *
 *        sum_{cam visible(q)} MSDA(value[cam], uv[cam,q,:] + offsets[q] / (w_l, h_l), softmax(logits[q]))
 * where visible(q, cam) = vis[cam, q] = any_d mask[cam, q, d] (from so_point_sampling).  offsets/logits depend on the query only, so they
 * are computed once per query instead of once per (camera, padded slot).
 *   value [N, Nv, Hd, Dh] (after value_proj), offsets [Q, Hd, L, D, 2], logits [Q, Hd, L, D],
 *   uv [N, Q, D, 2], vis uint8 [N, Q], spatial_shapes int64 [L,2], level_start_index int64 [L]
 *   -> slots [Q, Hd*Dh] (input of output_proj), count int32 [Q] (NULL ok). */
int so_tpv_cross_attn_forward(const float* value, const int64_t* spatial_shapes,
                              const int64_t* level_start_index, const float* offsets, const float* logits,
                              const float* uv, const uint8_t* vis, float* slots, int32_t* count,
                              int32_t N, int32_t Nv, int32_t Hd, int32_t Dh, int32_t Q, int32_t L, int32_t D,
                              void* stream);

/* Strided variants: the value / offsets / logits operands may be column slices of wider row-major matrices (row strides
 * value_ld / offsets_ld / logits_ld in floats), so ONE projection GEMM can produce the offsets and logits of a query (and
 * the value tensors of all three planes) side by side without a repacking copy. */
int so_tpv_cross_attn_forward_strided(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                      const float* offsets, const float* logits, const float* uv, const uint8_t* vis,
                                      float* slots, int32_t* count, int32_t N, int32_t Nv, int32_t Hd, int32_t Dh, int32_t Q,
                                      int32_t L, int32_t D, int32_t value_ld, int32_t offsets_ld, int32_t logits_ld, void* stream);

/* Test hook: 1 = run so_tpv_cross_attn_forward* / so_tpv_self_attn_forward* on the first-generation kernels (every lane of
 * a (query, head) redoes the sample set-up) instead of the shared-set-up kernels.  Both are parity-tested. */
int so_attn_force_v1(int on);

/* A5  visible-query index lists, as the reference builds them with nonzero()
 * (image_cross_attention.py:90-94), without a host sync: for each camera, ascending int64 query
 * indices with any in-frustum point.  index_lists [N, Q] (first lens[cam] entries valid),
 * lens int32 [N].  Single-CTA-per-camera ordered compaction. */
int so_visible_index_lists(const uint8_t* mask, int32_t N, int32_t Q, int32_t D,
                           int64_t* index_lists, int32_t* lens, void* stream);

/* A8 fused  cross-view hybrid (self) attention core: softmax + location arithmetic + sampling.
 * Replaces cross_view_hybrid_attention.py:83-116.
 *   value [Nv, Hd, Dh] (after value_proj; levels = the three planes), offsets [Q, Hd, L, P, 2],
 *   logits [Q, Hd, L, P], ref [Q, L, P, 2] -> out [Q, Hd*Dh] (input of output_proj). */
int so_tpv_self_attn_forward(const float* value, const int64_t* spatial_shapes,
                             const int64_t* level_start_index, const float* offsets, const float* logits,
                             const float* ref, float* out,
                             int32_t Nv, int32_t Hd, int32_t Dh, int32_t Q, int32_t L, int32_t P,
                             void* stream);

int so_tpv_self_attn_forward_strided(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                     const float* offsets, const float* logits, const float* ref, float* out, int32_t Nv,
                                     int32_t Hd, int32_t Dh, int32_t Q, int32_t L, int32_t P, int32_t value_ld,
                                     int32_t offsets_ld, int32_t logits_ld, void* stream);

/* Backward of so_tpv_cross_attn_forward (training).  Takes the forward's operands (contiguous, no strided form) plus
 *   count int32 [Q]       the forward's per-query visible-camera count (so_tpv_cross_attn_forward's `count` output)
 *   grad_slots [Q, Hd*Dh] the gradient of `slots`
 * and writes
 *   grad_value [N, Nv, Hd, Dh]      ACCUMULATED with atomics: the caller zero-fills it
 *   grad_offsets [Q, Hd, L, D, 2]   summed over the visible cameras; overwritten
 *   grad_logits [Q, Hd, L, D]       softmax backward over the (L, D) samples of each (query, head); overwritten
 * Each sample's softmax weight and location are recomputed with the forward's arithmetic (nothing else is saved), so
 * this is the adjoint of the function the forward evaluated.  A query visible in no camera gets zero gradients.
 * grad_offsets and grad_logits are deterministic (fixed loop and shuffle order, no atomics); grad_value is not.
 * value, grad_value and grad_slots 16-byte aligned, offsets and grad_offsets 8-byte aligned.  Dh must be 16 or 32. */
int so_tpv_cross_attn_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                               const float* offsets, const float* logits, const float* uv, const uint8_t* vis,
                               const int32_t* count, const float* grad_slots, float* grad_value, float* grad_offsets,
                               float* grad_logits, int32_t N, int32_t Nv, int32_t Hd, int32_t Dh, int32_t Q, int32_t L,
                               int32_t D, void* stream);

/* Backward of so_tpv_self_attn_forward (training): grad_out [Q, Hd*Dh] ->
 *   grad_value [Nv, Hd, Dh] (ACCUMULATED with atomics: the caller zero-fills it), grad_offsets [Q, Hd, L, P, 2],
 *   grad_logits [Q, Hd, L, P] (both overwritten, deterministic).
 * Same recomputation, alignment and Dh rules as so_tpv_cross_attn_backward; ref is a constant (no gradient). */
int so_tpv_self_attn_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                              const float* offsets, const float* logits, const float* ref, const float* grad_out,
                              float* grad_value, float* grad_offsets, float* grad_logits, int32_t Nv, int32_t Hd, int32_t Dh,
                              int32_t Q, int32_t L, int32_t P, void* stream);

/* ---------------------------------------------------------------------------------------
 * 8f-2  photometric reprojection loss: per-ray statistics of the rendering weights.  Replaces the per-sample part of
 * ReprojLossMonoMultiNewCombine (mode SO_REPROJ_COMBINE, loss/reproj_loss_mono_multi_new_combine.py:108-198, grid_sample
 * padding 'border') and ReprojLossMonoMultiNew (mode SO_REPROJ_MULTI_NEW, loss/reproj_loss_mono_multi_new.py:117-192,
 * padding 'zeros').  Both use the weights only through masked sums over each ray's samples, normalised by the masked
 * weight sum:
 *   per set: W = sum w m,  l1 = (sum w m diff) / max(W, eps),  rgb[3] = (sum w m rgb) / max(W, eps),  any = OR m
 * where, for the sample point (u t, v t, t, 1) of ray pixel (u, v) at depth t projected through img2prevImg / img2nextImg,
 * divided by max(z, 1e-5) and valid when z > 0, 0 < x < size_w and 0 < y < size_h:
 *   COMBINE (one set):  m = prev valid | next valid, cnt = max(#valid, 1),
 *                       diff = (sum over valid d of mean_c |cur - rgb_d|) / cnt, rgb = (sum over valid d of rgb_d) / cnt
 *   MULTI_NEW (two sets, prev then next): m, diff = mean_c |cur - rgb_d|, rgb = rgb_d of that direction.
 * cur / rgb_d are bilinear samples (align_corners=True) of the current / prev / next image at pixel (x / size_w * (W - 1),
 * y / size_h * (H - 1)); w = weights, or with `deltas` w / max(delta, eps) and 0 where delta < eps; eps = 2^-23 (fp32).
 *   weights, ts, deltas (NULL = none) [n_cam, rays_per_cam, S] ray-major; pix [rays_per_cam, 2] (x, y) pixel of each ray;
 *   img2prev, img2next [n_cam, 4, 4]; curr/prev/next images [n_cam, 3, img_h, img_w] fp32;
 *   size_h, size_w: the loss's img_size (may differ from img_h, img_w)
 *   -> stats [n_cam, rays_per_cam, 6 * sets] = per set (W, l1, rgb0, rgb1, rgb2, any as 0/1),
 *      colours [n_cam, rays_per_cam, 9] = current, prev, next image at the ray pixel (NULL ok; no gradient).
 * One warp per ray, fixed reduction order: deterministic, no atomics.
 * so_reproj_stats_backward: the forward's `stats` and grad_stats [n_cam, rays_per_cam, 6 * sets] (the `any` slots are
 *   ignored) -> grad_weights [n_cam, rays_per_cam, S], overwritten: the exact adjoint of the stats above (the clamp of W
 *   passes no gradient below eps).  The per-sample terms are recomputed with the forward's arithmetic. */
#define SO_REPROJ_COMBINE 0
#define SO_REPROJ_MULTI_NEW 1
int so_reproj_stats_forward(const float* weights, const float* ts, const float* deltas, const float* pix,
                            const float* img2prev, const float* img2next, const float* curr_imgs, const float* prev_imgs,
                            const float* next_imgs, int32_t n_cam, int32_t rays_per_cam, int32_t S, int32_t img_h,
                            int32_t img_w, float size_h, float size_w, int32_t mode, float* stats, float* colours,
                            void* stream);
int so_reproj_stats_backward(const float* ts, const float* deltas, const float* pix, const float* img2prev,
                             const float* img2next, const float* curr_imgs, const float* prev_imgs, const float* next_imgs,
                             int32_t n_cam, int32_t rays_per_cam, int32_t S, int32_t img_h, int32_t img_w, float size_h,
                             float size_w, int32_t mode, const float* stats, const float* grad_stats, float* grad_weights,
                             void* stream);

/* ---------------------------------------------------------------------------------------
 * 8f-2  per-sample regularisers of the training objective: mean of an elementwise function over a fp32 tensor, and the
 * gradient of that mean.
 *   SO_SAMPLE_MEAN_EIKONAL  EikonalLoss (loss/eikonal_loss.py:19-21): x is rows of 3, f = (|g|_2 - 1)^2 per row,
 *                           df/dg = 2 (|g| - 1) g / |g| and 0 where |g| = 0 (torch's vector_norm backward); n % 3 == 0
 *   SO_SAMPLE_MEAN_ABS      SecondGradLoss (loss/second_grad_loss.py:19-20): f = |x|, df/dx = sign(x), 0 at 0
 *   SO_SAMPLE_MEAN_NEG_RELU SoftSparsityLoss (loss/sparsity_loss.py:80-81): f = relu(-x), df/dx = -1 where x < 0, else 0
 * count = n / 3 rows (EIKONAL) or n elements.  x [n] fp32 (4-byte aligned; 128-bit words are used from the first aligned
 * one on, the unaligned head and the tail element by element).
 * so_sample_mean_forward -> out[0] = sum f / count (fp32, device scalar).  Each CTA of a fixed grid (a function of n only)
 *   accumulates in fp64 into workspace, SO_SAMPLE_MEAN_WORKSPACE_BYTES of 8-byte aligned device memory (contents on entry
 *   ignored), and a second one-CTA launch sums those partials in index order: deterministic, no atomics.
 * so_sample_mean_backward: grad_out [1] on the device -> grad_x [n] = grad_out[0] / count * df/dx, overwritten.  One
 *   read of x, one write of grad_x; the scale never reaches the host. */
#define SO_SAMPLE_MEAN_EIKONAL 0
#define SO_SAMPLE_MEAN_ABS 1
#define SO_SAMPLE_MEAN_NEG_RELU 2
#define SO_SAMPLE_MEAN_WORKSPACE_BYTES 8192
int so_sample_mean_forward(const float* x, int64_t n, int32_t op, void* workspace, float* out, void* stream);
int so_sample_mean_backward(const float* x, int64_t n, int32_t op, const float* grad_out, float* grad_x, void* stream);

/* ---------------------------------------------------------------------------------------
 * 8f-2  the sparsity terms of loss/sparsity_loss.py, on the launches and conventions of so_sample_mean_* (fixed grid, fp64
 * partials in SO_SAMPLE_MEAN_WORKSPACE_BYTES of workspace summed in index order, grad_out read on the device).
 * so_sparsity_forward: SparsityLoss (:24-27), out[0] = mean over x [n] of sech^2(x / (2 scale)), evaluated as
 *   4e / (1 + e)^2 with e = exp(-|x| / scale): 0, not NaN, where cosh overflows.  scale finite and != 0.
 * so_sparsity_backward: grad_x = grad_out[0] / n * (-tanh(u) sech^2(u) / scale), u = x / (2 scale); overwritten.
 * so_hard_sparsity_forward: HardSparsityLoss (:46-63) on the lattice x [H, W, D] (H * W * D < 2^31):
 *   out[0] = relu(mean sigmoid(-scale x') - thresh), the mean in fp32 as the reference's, where x' is x with the crop
 *   borders read as 100: crop (host, NULL = none) = {h0, h1, w0, w1, d0, d1}, the first h0 and last h1 cells along h (and
 *   so on) are cropped, 0 = none, negative values are SO_ERR_INVALID_ARG.  x is never written.
 * so_hard_sparsity_backward: grad_x = grad_out[0] / n * (-scale) sigmoid (1 - sigmoid), 0 in the cropped cells and
 *   everywhere unless loss[0] (the forward's out, on the device) is > 0: relu's gradient, read without the host.
 * AdaptiveSparsityLoss (:102-114) per ray: sdf, ts [n_rays, S] ray-major, depth [n_rays] fp32; a sample counts where
 *   ts > depth + slack (fp32, as the reference's mask).
 * so_adaptive_sparsity_rays -> ray_stats [n_rays] of (sum of relu(-sdf) over the counted samples, their count) in fp64
 *   (16-byte aligned).  One warp per ray, fixed reduction order.  n_rays == 0 does nothing.
 * so_adaptive_sparsity_reduce: ray_stats [n_rays >= 1] -> out[0] = (float)(sum / count) over all rays, NaN when no sample
 *   counts (torch's mean of an empty tensor); total (NULL ok) [2] = the fp64 (sum, count).  A fixed grid sums the pairs
 *   into workspace (SO_SAMPLE_MEAN_WORKSPACE_BYTES, 16-byte aligned) and one CTA sums those in index order: the result
 *   is a function of ray_stats alone, so per-ray pairs gathered from ray-sharded ranks reduce to the unsharded value.
 * so_adaptive_sparsity_backward: grad_stats [n_rays] (d loss / d sum, d loss / d count; the count slot is ignored, the
 *   mask has no gradient) -> grad_sdf [n_rays, S] = -grad_stats[ray].sum where the sample counts and sdf < 0, else 0. */
int so_sparsity_forward(const float* x, int64_t n, float scale, void* workspace, float* out, void* stream);
int so_sparsity_backward(const float* x, int64_t n, float scale, const float* grad_out, float* grad_x, void* stream);
int so_hard_sparsity_forward(const float* x, int32_t H, int32_t W, int32_t D, const int32_t* crop, float scale,
                             float thresh, void* workspace, float* out, void* stream);
int so_hard_sparsity_backward(const float* x, int32_t H, int32_t W, int32_t D, const int32_t* crop, float scale,
                              const float* loss, const float* grad_out, float* grad_x, void* stream);
int so_adaptive_sparsity_rays(const float* sdf, const float* ts, const float* depth, int64_t n_rays, int32_t S,
                              float slack, double* ray_stats, void* stream);
int so_adaptive_sparsity_reduce(const double* ray_stats, int64_t n_rays, void* workspace, float* out, double* total,
                                void* stream);
int so_adaptive_sparsity_backward(const float* sdf, const float* ts, const float* depth, int64_t n_rays, int32_t S,
                                  float slack, const double* grad_stats, float* grad_sdf, void* stream);

/* ---------------------------------------------------------------------------------------
 * 8f-2  training render with the objective's per-sample terms fused in.  Renders exactly as so_render_train_forward
 * (same sampling, field, alpha, compositing and kernel choice: the per-ray outputs are bit-identical) and, instead of
 * storing the per-sample tensors the losses read, reduces them per ray while it renders:
 *   reprojection (reproj_mode SO_REPROJ_COMBINE / SO_REPROJ_MULTI_NEW): reproj_stats [rays, 6 * sets] and reproj_colours
 *     [rays, 9] (NULL ok) with the contract and the arithmetic of so_reproj_stats_forward with deltas == NULL, from the
 *     weights and ts of the render.  Row i is flat ray ray_begin + i, of camera (ray_begin + i) / rays_per_cam and loss pixel
 *     pix[(ray_begin + i) % rays_per_cam]; images and matrices are indexed by that camera.
 *   eikonal (eikonal = 1): eikonal_mean [1] = mean over the call's rays x S samples of (|eik_grad| - 1)^2, as
 *     so_sample_mean_forward(EIKONAL): per-ray fp64 sums in `workspace` (8-byte aligned, >= 8 * ray_count bytes), then one
 *     index-ordered pass.  Deterministic, no float atomics, the same value on every device.
 *   second grad (second_grad = 1): second_grad_mean [1] = mean over the call's rays x S samples x 3 of |second_grad|, as
 *     so_field_second_grad followed by so_sample_mean_forward(ABS), with second_grad taken at the render's own sample point
 *     (the point eik_grad is taken at: the bin mid-point, or its start with anchor_mid = 0).  Per-ray fp64 sums in
 *     `workspace` after the eikonal sums (>= 16 * ray_count bytes with both terms, >= 8 * ray_count with this one alone),
 *     then one index-ordered pass.  Deterministic, no float atomics.
 * The per-sample outputs of so_render_train_forward stay available and NULL = not written (a head that also needs the
 * sample positions asks for ts / deltas).
 * so_render_train_objective_backward recomputes the forward as so_render_train_backward does and forms every sample's
 * d loss / d w (the adjoint of so_reproj_stats_backward: reproj_stats = the forward's, grad_reproj_stats [rays, 6 * sets])
 * and d loss / d eik_grad (the adjoint of so_sample_mean_backward: grad_eikonal_mean [1] on the device, NULL = 0, never
 * read on the host) in registers; with second_grad = 1 it adds the second-grad mean's sdf-corner gradients
 * (grad_second_grad_mean [1] / (3 rays S) * sign(second_grad), sign(0) = 0, through so_field_second_grad_backward's
 * corner coefficients; NULL = 0, never read on the host) to each sample's sdf scatter; with the per-ray g_depth / g_acc / g_rgb / g_sem it ACCUMULATES into g_vol_sdf,
 * g_vol_feat and g_inv_s as so_render_train_backward does (the caller zero-fills them).  g_inv_s is formed from per-ray
 * fp64 values in `workspace` (as the forward's eikonal sums: >= 8 * ray_count bytes when g_inv_s != NULL) summed in ray
 * order, so it is the same on every run; g_vol_sdf / g_vol_feat are accumulated with atomics.
 * Argument errors return SO_ERR_INVALID_ARG / SO_ERR_UNSUPPORTED before any launch: the checks of so_render_train_forward /
 * _backward (S <= 256) and, for the objective, those of so_reproj_stats_forward (operands, image sizes) plus 4-byte
 * alignment of every float operand, eikonal and second_grad in {0, 1}, and the workspace's size and alignment.
 * A zero-initialised descriptor tail (second_grad = 0, NULL pointers) leaves the second-grad term off. */
#define SO_OBJECTIVE_NO_REPROJ (-1)
typedef struct so_objective_desc {
  int32_t reproj_mode;       /* SO_REPROJ_COMBINE, SO_REPROJ_MULTI_NEW or SO_OBJECTIVE_NO_REPROJ */
  int32_t eikonal;           /* 1: the eikonal mean is computed, 0: not */
  const float* pix;          /* [rays_per_cam, 2] (x, y) loss pixel of each ray */
  const float* img2prev;     /* [n_cam, 4, 4] img2prevImg */
  const float* img2next;     /* [n_cam, 4, 4] img2nextImg */
  const float* curr_imgs;    /* [n_cam, 3, img_h, img_w] fp32 */
  const float* prev_imgs;
  const float* next_imgs;
  int32_t img_h, img_w;
  float size_h, size_w;      /* the loss's img_size */
  void* workspace;           /* forward: >= 8 * ray_count bytes per mean computed (eikonal, second grad), backward with
                                g_inv_s: >= 8 * ray_count bytes; 8-byte aligned */
  int64_t workspace_bytes;
  int32_t second_grad;       /* 1: the second-grad mean is computed (forward) and differentiated (backward), 0: not */
  float* second_grad_mean;   /* forward output [1] when second_grad = 1 */
  const float* grad_second_grad_mean;  /* backward input [1] on the device, NULL = 0 */
} so_objective_desc;
int so_render_train_objective_forward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                                      const float* cam_mats, const float* pix, const so_ray_desc* rays_host,
                                      const so_render_params* params_host, const float* jitter, const float* bkgd_rand,
                                      const so_objective_desc* objective, float* depth, float* acc, float* fars, float* rgb,
                                      float* sem, float* max_depth, float* weights, float* ts, float* deltas, float* eik_grad,
                                      float* sample_sdf, float* reproj_stats, float* reproj_colours, float* eikonal_mean,
                                      float* workspace, float* pair_workspace, void* stream);
int so_render_train_objective_backward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                                       const float* cam_mats, const float* pix, const so_ray_desc* rays_host,
                                       const so_render_params* params_host, const float* jitter, const float* bkgd_rand,
                                       const so_objective_desc* objective, const float* g_depth, const float* g_acc,
                                       const float* g_rgb, const float* g_sem, const float* reproj_stats,
                                       const float* grad_reproj_stats, const float* grad_eikonal_mean, float* g_vol_sdf,
                                       float* g_vol_feat, float* g_inv_s, float* workspace, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SELFOCC_B200_H */
