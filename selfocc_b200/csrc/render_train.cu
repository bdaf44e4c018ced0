// Training-form render (SURVEY.md section 8a rows B6-B10, B13): NeuSHead.forward must emit per-sample tensors
// (weights / ts / deltas / eik_grad [/ sample_sdf], neus_head.py:667-682) and be differentiable w.r.t. the
// decoded volume and the NeuS deviation parameter.
//
// Mapping: one WARP per ray, lane = sample (s = 32*k + lane, k = 0..S/32-1), so every per-sample tensor is written
// fully coalesced (32 consecutive floats per store) -- this form is HBM-write bound (~6 KB/ray).  The
// transmittance is an exclusive product scan along the sample dimension done with warp shuffles (5 steps per
// 32-sample chunk + a carried prefix); the backward needs the matching suffix sums and runs the chunks in reverse.
#include "render_common.cuh"
#ifndef SO_TRAIN_FWD_MIN_CTAS
#define SO_TRAIN_FWD_MIN_CTAS 8   // H100 SXM (700 W), cfg-5 sizes, Cf = 25: 0.664-0.668 ms, 4 CTAs/SM the same; latency-bound
#endif

#ifndef SO_TRAIN_FWD24_MIN_CTAS
#define SO_TRAIN_FWD24_MIN_CTAS 3    // 24-channel semantic forward: 168 registers, no spills
#endif
#ifndef SO_TRAIN_BWD24_MIN_CTAS
#define SO_TRAIN_BWD24_MIN_CTAS 3    // 24-channel semantic backward: 168 registers + 328 B of L1-resident spills (2: 255 registers, 44 B)
#endif

namespace so {

constexpr int kTrainMaxChunks = 8;  // S <= 256

struct TrainOut {
  float *depth, *acc, *fars, *rgb, *sem, *max_depth;      // per ray
  float *weights, *ts, *deltas, *eik, *sdf;               // per sample
};

struct TrainGrad {
  const float *g_depth, *g_acc, *g_rgb, *g_sem, *g_weights, *g_eik, *g_sdf;
  float *g_vol_sdf, *g_vol_feat, *g_inv_s;
};

// one sample of one ray: geometry + field + alpha.  `s` must be < S.
struct Sample {
  float mid, delta, sdf, gx, gy, gz, alpha;
  // pieces the backward needs
  float half, pa, pb, tc;
  Taps t;
  float kh, kw, kd;
};

// Per-ray constants of the training kernels (hoisted out of the per-sample work)
struct RayCtx {
  float o[3], d[3], nrm, inv_nrm, tn, tf;
  float gh0, gdh, gw0, gdw, gd0, gdd;   // affine grid-space ray (valid when the mapping has no outer ring)
  bool affine;
  const float* u;                       // this ray's jitter row or nullptr
};

__device__ __forceinline__ void make_ctx(const VolumeDev& V, const RayDev& R, const RenderDev& P, long long gid, RayCtx& c) {
  make_ray(R, gid, c.o, c.d, c.nrm);
  slab(P, c.o, c.d, c.tn, c.tf);
  c.inv_nrm = 1.0f / c.nrm;
  c.affine = V.ax[0].k1 == 0.f && V.ax[1].k1 == 0.f && V.ax[2].k1 == 0.f;
  affine_grid_ray(V, c.o, c.d, c.gh0, c.gdh, c.gw0, c.gdw, c.gd0, c.gdd);
  c.u = P.jitter ? P.jitter + gid * (long long)(P.S + 1) : nullptr;
}

// FAST = affine metre->grid map, S a power of two (multiple of 32), cos-anneal finished, mid-point anchor (see
// train_fast).  Every training kernel of a FAST launch -- both forwards, the backward and the probe -- takes its sample
// positions from these two helpers, so the backward differentiates exactly the cells the forward rendered.
// Edge i is re-drawn inside [max(i - 1/2, 0), min(i + 1/2, S)] / S (exact arithmetic for power-of-two S).
__device__ __forceinline__ float fast_edge(int i, float u, bool jit, int S, float step, float span, float tn) {
  float fi = (float)i;
  float lo_b = fmaxf(fi - 0.5f, 0.f) * step, up_b = fminf(fi + 0.5f, (float)S) * step;
  float b = jit ? fmaf(up_b - lo_b, u, lo_b) : fi * step;
  return fmaf(b, span, tn);
}
// mid-point, width and affine grid coordinates of the bin [e0, e1]
__device__ __forceinline__ void fast_mid_grid(float e0, float e1, float gh0, float gdh, float gw0, float gdw, float gd0, float gdd,
                                              float& mid, float& delta, float& gh, float& gw, float& gd) {
  mid = 0.5f * (e0 + e1);
  delta = e1 - e0;
  gh = fmaf(gdh, mid, gh0); gw = fmaf(gdw, mid, gw0); gd = fmaf(gdd, mid, gd0);
}

// geometry of one sample of one ray (lane = sample): bin mid-point, width, grid coordinates and metre->grid slopes.
// `s` must be < S.  Edges are shared between neighbouring lanes with one shuffle (lane 31 computes its own right edge).
// FAST: the shipped forwards' arithmetic; otherwise the reference form b * tf + (1 - b) * tn of the edges.
template <bool FAST>
__device__ __forceinline__ void sample_geom(const VolumeDev& V, const RenderDev& P, const RayCtx& c, int s, int lane, float& mid,
                                            float& delta, float& gh, float& gw, float& gd, float& kh, float& kw, float& kd) {
  const int S = P.S;
  const float step = 1.0f / (float)S;
  if (FAST) {
    const float span = c.tf - c.tn;
    float e0 = fast_edge(s, c.u ? __ldg(c.u + s) : 0.f, c.u != nullptr, S, step, span, c.tn);
    float e1 = __shfl_down_sync(0xffffffffu, e0, 1);
    const int s1 = min(s + 1, S);
    if (lane == 31 || s + 1 >= S) e1 = fast_edge(s1, c.u ? __ldg(c.u + s1) : 0.f, c.u != nullptr, S, step, span, c.tn);
    fast_mid_grid(e0, e1, c.gh0, c.gdh, c.gw0, c.gdw, c.gd0, c.gdd, mid, delta, gh, gw, gd);
    kh = V.ax[0].k0; kw = V.ax[1].k0; kd = V.ax[2].k0;
    return;
  }
  float e0 = edge_t(bin_edge01_jit(s, S, step, c.u), c.tn, c.tf);
  float e1 = __shfl_down_sync(0xffffffffu, e0, 1);
  if (lane == 31 || s + 1 >= S) e1 = edge_t(bin_edge01_jit(min(s + 1, S), S, step, c.u), c.tn, c.tf);
  mid = __fmul_rn(__fadd_rn(e0, e1), 0.5f);
  delta = __fsub_rn(e1, e0);
  float tq = P.anchor_mid ? mid : e0;
  if (c.affine) {
    gh = fmaf(c.gdh, tq, c.gh0); gw = fmaf(c.gdw, tq, c.gw0); gd = fmaf(c.gdd, tq, c.gd0);
    kh = V.ax[0].k0; kw = V.ax[1].k0; kd = V.ax[2].k0;
  } else {
    float x = fmaf(c.d[0], tq, c.o[0]), y = fmaf(c.d[1], tq, c.o[1]), z = fmaf(c.d[2], tq, c.o[2]);
    gh = axis_m2g(V.ax[0], y, kh); gw = axis_m2g(V.ax[1], x, kw); gd = axis_m2g(V.ax[2], z, kd);
  }
}

// one sample of one ray (lane = sample): geometry + field + alpha.  `s` must be < S.  FAST: the alpha value is the
// shipped forwards' neus_alpha_log2 as well (pa / pb, which the backward differentiates, are the same logistics).
template <bool FAST>
__device__ __forceinline__ void eval_sample(const VolumeDev& V, const RenderDev& P, const RayCtx& c, int s, int lane, Sample& q) {
  float gh, gw, gd;
  sample_geom<FAST>(V, P, c, s, lane, q.mid, q.delta, gh, gw, gd, q.kh, q.kw, q.kd);
  q.t = make_taps(V, gh, gw, gd);
  float dgh, dgw, dgd;
  const bool interior = (unsigned)q.t.h0 < (unsigned)(V.H - 1) && (unsigned)q.t.w0 < (unsigned)(V.W - 1) &&
                        (unsigned)q.t.z0 < (unsigned)(V.Z - 1);
  if (__all_sync(0xffffffffu, interior)) gather_sdf_interior(V, q.t.h0, q.t.w0, q.t.z0, q.t.fh, q.t.fw, q.t.fz, q.sdf, dgh, dgw, dgd);
  else gather_sdf(V, q.t, q.sdf, dgh, dgw, dgd);
  q.gx = dgw * q.kw; q.gy = dgh * q.kh; q.gz = dgd * q.kd;
  q.tc = c.d[0] * q.gx + c.d[1] * q.gy + c.d[2] * q.gz;
  float ic = -(fmaxf(fmaf(-q.tc, 0.5f, 0.5f), 0.f) * (1.0f - P.cos_anneal) + fmaxf(-q.tc, 0.f) * P.cos_anneal);
  q.half = ic * q.delta * 0.5f;
  float a = (q.sdf - q.half) * P.inv_s, b = (q.sdf + q.half) * P.inv_s;
  q.pa = sigmoid_fast(a);
  q.pb = sigmoid_fast(b);
  if (FAST) {
    const float k_log2 = P.inv_s * 1.4426950408889634f;
    q.alpha = neus_alpha_log2(q.sdf * k_log2, fminf(q.tc, 0.f) * (q.delta * (0.5f * k_log2)));
  } else {
    float diff = q.pa * sigmoid_fast(-b) * one_minus_exp_neg(-2.0f * q.half * P.inv_s);
    q.alpha = __saturatef(__fdividef(diff + 1e-5f, q.pa + 1e-5f));
  }
}

__device__ __forceinline__ float warp_incl_prod(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float n = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v *= n;
  }
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// transmittance of this lane's sample from the factors f = 1 - alpha + 1e-7 of one 32-sample chunk: the exclusive product
// along the lanes times `carry`, the product over the earlier chunks, which then takes on this chunk's product
__device__ __forceinline__ float warp_transmittance(float f, int lane, float& carry) {
  float incl = warp_incl_prod(f, lane);
  float excl = __shfl_up_sync(0xffffffffu, incl, 1);
  float T = carry * (lane == 0 ? 1.0f : excl);
  carry *= __shfl_sync(0xffffffffu, incl, 31);
  return T;
}
// reverse inclusive sum: out[lane] = sum_{i >= lane} v[i]
__device__ __forceinline__ float warp_rev_incl_sum(float v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    float n = __shfl_down_sync(0xffffffffu, v, o);
    if (lane + o < 32) v += n;
  }
  return v;
}

__device__ __forceinline__ void sample_colour(const VolumeDev& V, const RenderDev& P, const Taps& t, float col[3], float raw[3]) {
  float f[3];
  gather_feat<3>(V, t, 0, f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    raw[c] = f[c] * kC0;
    col[c] = P.sh_act == 0 ? fmaxf(raw[c] + 0.5f, 0.f) : sigmoidf_acc(raw[c]);
  }
}

// ---- the shipped semantic configuration (config/nuscenes/nuscenes_occ.py:350: color_dims = 24 = 3 rgb + 21 classes) --------
// SEM template parameter of the one-ray-per-warp kernels: 0 = no semantics, 1 = any channel count (runtime loops over
// scalar gathers), 24 = exactly 24 feature channels with feat_pitch 24: a voxel's 96 bytes are read / accumulated as six
// float4 (48 LDG.128 instead of 192 LDG.32 per sample; 48 128-bit reductions instead of 192 atomics in the backward) and every
// per-class array has a compile-time size, so nothing lives in local memory (runtime-count arrays spill to local memory).
constexpr int kSem24 = 21;

__device__ __forceinline__ void gather_feat24(const VolumeDev& v, const Taps& t, float out[24]) {
#pragma unroll
  for (int i = 0; i < 24; ++i) out[i] = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int dh = k >> 2, dw = (k >> 1) & 1, dz = k & 1;
    float wgt = (dh ? t.fh * t.mh1 : (1.f - t.fh) * t.mh0) * (dw ? t.fw * t.mw1 : (1.f - t.fw) * t.mw0) *
                (dz ? t.fz * t.mz1 : (1.f - t.fz) * t.mz0);
    int h = min(max(t.h0 + dh, 0), v.H - 1), w = min(max(t.w0 + dw, 0), v.W - 1), z = min(max(t.z0 + dz, 0), v.Z - 1);
    const float4* p = reinterpret_cast<const float4*>(v.feat + (((size_t)h * v.W + w) * v.Z + z) * 24);
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      float4 f = __ldg(p + j);
      out[4 * j] = fmaf(wgt, f.x, out[4 * j]); out[4 * j + 1] = fmaf(wgt, f.y, out[4 * j + 1]);
      out[4 * j + 2] = fmaf(wgt, f.z, out[4 * j + 2]); out[4 * j + 3] = fmaf(wgt, f.w, out[4 * j + 3]);
    }
  }
}

__device__ __forceinline__ void scatter_feat24(const VolumeDev& V, float* __restrict__ gfeat, const Taps& t, const float g[24]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int dh = k >> 2, dw = (k >> 1) & 1, dz = k & 1;
    float m = (dh ? t.mh1 : t.mh0) * (dw ? t.mw1 : t.mw0) * (dz ? t.mz1 : t.mz0);
    if (m == 0.f) continue;
    float wgt = (dh ? t.fh : 1.f - t.fh) * (dw ? t.fw : 1.f - t.fw) * (dz ? t.fz : 1.f - t.fz);
    float4* p = reinterpret_cast<float4*>(gfeat + (((size_t)(t.h0 + dh) * V.W + (t.w0 + dw)) * V.Z + (t.z0 + dz)) * 24);
#pragma unroll
    for (int j = 0; j < 6; ++j)
      atomicAdd(p + j, make_float4(wgt * g[4 * j], wgt * g[4 * j + 1], wgt * g[4 * j + 2], wgt * g[4 * j + 3]));   // red.global.add.v4.f32
  }
}

// the training kernels' form of colour_act(sh_act, ...) (render_common.cuh): the same values; the two forms are kept because
// each compiles to the machine code its kernels were tuned with
__device__ __forceinline__ void colour_act(const RenderDev& P, const float f[3], float col[3], float raw[3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    raw[c] = f[c] * kC0;
    col[c] = P.sh_act == 0 ? fmaxf(raw[c] + 0.5f, 0.f) : sigmoidf_acc(raw[c]);
  }
}

// FAST = affine metre->grid map, S a power of two (multiple of 32), cos-anneal finished, mid-point anchor: lean per-sample
// path (closed-form jittered edges, interior gather chosen by a warp vote, base-2 alpha), ~2.4x fewer instructions.
template <bool HAS_RGB, int SEM, bool FAST>
__global__ void __launch_bounds__(128, SEM == 24 ? SO_TRAIN_FWD24_MIN_CTAS : SO_TRAIN_FWD_MIN_CTAS) render_train_fwd_kernel(VolumeDev V, RayDev R, RenderDev P, const float* __restrict__ ws,
                                                               const float* __restrict__ bkgd_rand, TrainOut O) {
  constexpr bool HAS_SEM = SEM != 0;
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const int S = P.S;
  const int K = (S + 31) >> 5;
  const int n_sem = HAS_SEM ? V.n_feat - 3 : 0;
  const float eps = 1.1920928955078125e-07f;
  for (long long ray = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); ray < R.ray_count; ray += warps) {
    long long gid = R.ray_begin + ray;
    RayCtx c;
    make_ctx(V, R, P, gid, c);
    const float nrm = c.nrm, tf = c.tf;
    float carry = 1.0f, acc = 0.f, dsum = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
    float best = -INFINITY, best_ts = 0.f;
    int best_i = 0x7fffffff;
    float sem_acc[SEM == 24 ? kSem24 : (HAS_SEM ? kMaxSem : 1)];
    if (SEM == 24) {
#pragma unroll
      for (int c = 0; c < kSem24; ++c) sem_acc[c] = 0.f;
    } else if (HAS_SEM) {
      for (int c = 0; c < kMaxSem; ++c) sem_acc[c] = 0.f;
    }
    const float step = 1.0f / (float)S, span = c.tf - c.tn, k_log2 = P.inv_s * 1.4426950408889634f;
    // the jitter value of the NEXT chunk is requested one iteration ahead, so its DRAM latency is off the critical path
    float u_cur = (FAST && c.u) ? __ldg(c.u + lane) : 0.f;
    for (int k = 0; k < K; ++k) {
      int s = k * 32 + lane;
      bool live = s < S;
      Sample q;
      if (FAST) {
        const int s_nxt = s + 32;
        const float u_nxt = (c.u && s_nxt <= S) ? __ldg(c.u + s_nxt) : 0.f;
        auto edge = [&](int i, float u) { return fast_edge(i, u, c.u != nullptr, S, step, span, c.tn); };
        float e0 = edge(s, u_cur);
        float e_next = edge(k * 32 + 32, __shfl_sync(0xffffffffu, u_nxt, 0));   // right edge of lane 31 = first edge of the next chunk
        float e1 = __shfl_down_sync(0xffffffffu, e0, 1);
        if (lane == 31) e1 = e_next;
        u_cur = u_nxt;
        float gh, gw, gd;
        fast_mid_grid(e0, e1, c.gh0, c.gdh, c.gw0, c.gdw, c.gd0, c.gdd, q.mid, q.delta, gh, gw, gd);
        q.kh = V.ax[0].k0; q.kw = V.ax[1].k0; q.kd = V.ax[2].k0;
        float flh = floorf(gh), flw = floorf(gw), flz = floorf(gd);
        int h0 = (int)flh, w0 = (int)flw, z0 = (int)flz;
        bool interior = (unsigned)h0 < (unsigned)(V.H - 1) && (unsigned)w0 < (unsigned)(V.W - 1) && (unsigned)z0 < (unsigned)(V.Z - 1);
        float dgh, dgw, dgd;
        if (__all_sync(0xffffffffu, interior)) {
          gather_sdf_interior(V, h0, w0, z0, gh - flh, gw - flw, gd - flz, q.sdf, dgh, dgw, dgd);
          if (HAS_RGB) q.t = make_taps(V, gh, gw, gd);
        } else {
          q.t = make_taps(V, gh, gw, gd);
          gather_sdf(V, q.t, q.sdf, dgh, dgw, dgd);
        }
        q.gx = dgw * q.kw; q.gy = dgh * q.kh; q.gz = dgd * q.kd;
        float tc = c.d[0] * q.gx + c.d[1] * q.gy + c.d[2] * q.gz;
        q.alpha = neus_alpha_log2(q.sdf * k_log2, fminf(tc, 0.f) * (q.delta * (0.5f * k_log2)));
      } else {
        eval_sample<false>(V, P, c, live ? s : S - 1, lane, q);
      }
      float alpha = live ? q.alpha : 0.f;
      float f = live ? (1.0f - alpha + 1e-7f) : 1.0f;
      float T = warp_transmittance(f, lane, carry);
      float w = alpha * T;
      if (live) {
        long long oidx = ray * S + s;
        float ts = q.mid * c.inv_nrm, dl = q.delta * c.inv_nrm;     // neus_head.py:571-577 (reciprocal multiply, <= 1 ulp)
        if (O.weights) O.weights[oidx] = w;
        if (O.ts) O.ts[oidx] = ts;
        if (O.deltas) O.deltas[oidx] = dl;
        if (O.sdf) O.sdf[oidx] = q.sdf;
        if (O.eik) { O.eik[3 * oidx] = q.gx; O.eik[3 * oidx + 1] = q.gy; O.eik[3 * oidx + 2] = q.gz; }
        acc += w;
        dsum = fmaf(w, q.mid, dsum);
        float cand = (dl < eps ? 0.f : w) * __fdividef(1.0f, fmaxf(dl, eps));  // neus_head.py:579-587
        if (cand > best) { best = cand; best_i = s; best_ts = ts; }
        if (SEM == 24) {
          float F[24], col[3], raw[3];
          gather_feat24(V, q.t, F);
          colour_act(P, F, col, raw);
          cr = fmaf(w, col[0], cr); cg = fmaf(w, col[1], cg); cb = fmaf(w, col[2], cb);
          float mx = F[3];
#pragma unroll
          for (int c = 1; c < kSem24; ++c) mx = fmaxf(mx, F[3 + c]);
          float den = 0.f;
#pragma unroll
          for (int c = 0; c < kSem24; ++c) { F[3 + c] = expf(F[3 + c] - mx); den += F[3 + c]; }
          float sc = w / den;
#pragma unroll
          for (int c = 0; c < kSem24; ++c) sem_acc[c] = fmaf(sc, F[3 + c], sem_acc[c]);
        } else if (HAS_RGB) {
          float col[3], raw[3];
          sample_colour(V, P, q.t, col, raw);
          cr = fmaf(w, col[0], cr); cg = fmaf(w, col[1], cg); cb = fmaf(w, col[2], cb);
        }
        if (SEM == 1) {
          float lg[kMaxSem];
          float mx = -INFINITY;
          for (int c = 0; c < n_sem; ++c) { float f1[1]; gather_feat<1>(V, q.t, 3 + c, f1); lg[c] = f1[0]; mx = fmaxf(mx, f1[0]); }
          float den = 0.f;
          for (int c = 0; c < n_sem; ++c) { lg[c] = expf(lg[c] - mx); den += lg[c]; }
          float sc = w / den;
          for (int c = 0; c < n_sem; ++c) sem_acc[c] = fmaf(sc, lg[c], sem_acc[c]);
        }
      }
    }
    acc = warp_sum(acc);
    dsum = warp_sum(dsum);
    // first-max argmax across lanes: larger score wins, ties go to the smaller sample index
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      float ob = __shfl_xor_sync(0xffffffffu, best, off);
      int oi = __shfl_xor_sync(0xffffffffu, best_i, off);
      float ot = __shfl_xor_sync(0xffffffffu, best_ts, off);
      if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; best_ts = ot; }
    }
    if (HAS_RGB) { cr = warp_sum(cr); cg = warp_sum(cg); cb = warp_sum(cb); }
    if (SEM == 24) {
#pragma unroll
      for (int c = 0; c < kSem24; ++c) sem_acc[c] = warp_sum(sem_acc[c]);
    } else if (HAS_SEM) {
      for (int c = 0; c < n_sem; ++c) sem_acc[c] = warp_sum(sem_acc[c]);
    }
    if (lane == 0) {
      long long chunk = R.chunk_len > 0 ? gid / R.chunk_len : 0;
      float lo = ws[2 * chunk], hi = ws[2 * chunk + 1];
      float dd = fminf(fmaxf(dsum / (acc + 1e-10f), lo), hi);
      if (O.depth) O.depth[ray] = dd / nrm;
      if (O.acc) O.acc[ray] = acc;
      if (O.fars) O.fars[ray] = tf / nrm;
      if (O.max_depth) O.max_depth[ray] = best_ts;
      if (HAS_RGB && O.rgb) {
        float b0, b1, b2;
        if (P.bkgd_mode == 2) { b0 = bkgd_rand[3 * ray]; b1 = bkgd_rand[3 * ray + 1]; b2 = bkgd_rand[3 * ray + 2]; }
        else { b0 = b1 = b2 = (P.bkgd_mode == 1) ? 1.f : 0.f; }
        float rem = 1.0f - acc;
        float r = fmaf(b0, rem, cr), g = fmaf(b1, rem, cg), b = fmaf(b2, rem, cb);
        if (P.eval_clamp) { r = __saturatef(r); g = __saturatef(g); b = __saturatef(b); }
        O.rgb[3 * ray] = r; O.rgb[3 * ray + 1] = g; O.rgb[3 * ray + 2] = b;
      }
      if (SEM == 24 && O.sem) {
#pragma unroll
        for (int c = 0; c < kSem24; ++c) O.sem[ray * kSem24 + c] = sem_acc[c];
      } else if (HAS_SEM && O.sem) {
        for (int c = 0; c < n_sem; ++c) O.sem[ray * n_sem + c] = sem_acc[c];
      }
    }
  }
}

// ---- forward, batched rays + U chunks in flight + z-pair volume ---------------------------------------------------
// Same contract and the same per-sample arithmetic as render_train_fwd_kernel<., false, true> (lane = sample, so the 32
// lanes of a load touch neighbouring voxels: the gathers are bound by distinct 128-byte lines per L1 request), with the
// three things that kernel lacks:
//  (a) a warp takes a BATCH of consecutive rays: lane b computes ray b's set-up (camera ray, slab test, affine
//      grid-space ray: ~300 instructions the one-ray-per-warp kernel repeats in all 32 lanes) and, after the batch, its
//      tail (depth clip, divisions, per-ray stores); the 12 per-ray constants are broadcast with shuffles;
//  (b) U chunks (32 U samples) are evaluated per loop iteration, so 8 U (4 U with the pair volume) independent gathers
//      are in flight per thread instead of 8;
//  (c) PAIR: the sdf volume is first repacked as float2 {v[z], v[z + 1]} (zpair_pack_kernel, 2 x 8 MB, L2 resident),
//      which turns the 8 taps into 4 aligned 64-bit loads: half the L1 requests and half the tag look-ups.
// The jittered edge b_i = lo_i + (up_i - lo_i) u_i of the upstream sampler is evaluated as
// fma(w_i, u_i, max(i - 1/2, 0)) * step with w_i = 1 (1/2 at the two ends); for power-of-two S this is the same
// fp32 value as the one-ray-per-warp kernel's.
#ifndef SO_TRAIN_FWD5_U
#define SO_TRAIN_FWD5_U 4            // H100 SXM (700 W), cfg-5 sizes, Cf = 1, ms: U=2 0.129, U=4 0.125, U=8 0.160 (latency-bound)
#endif
#ifndef SO_TRAIN_FWD5_PREFETCH
#define SO_TRAIN_FWD5_PREFETCH 1     // 1 / 2: prefetch.global.L2 / .L1 of the batch's jitter rows before the ray set-up (109 -> 101 us)
#endif
#ifndef SO_TRAIN_FWD5_AHEAD
#define SO_TRAIN_FWD5_AHEAD 1        // 1: the jitter of group k + 1 is requested while group k is evaluated (101 -> 98 us)
#endif
#ifndef SO_TRAIN_FWD5_WARPS
#define SO_TRAIN_FWD5_WARPS 4
#endif
#ifndef SO_TRAIN_FWD5_MIN_CTAS
#define SO_TRAIN_FWD5_MIN_CTAS 4
#endif
#ifndef SO_TRAIN_FWD5_BATCH
#define SO_TRAIN_FWD5_BATCH 4
#endif
#ifndef SO_TRAIN_FWD5_CONST_PITCH
#define SO_TRAIN_FWD5_CONST_PITCH 1  // specialise for zpitch 32, W 257 (every nuScenes config): the taps = 1 address + immediates
#endif

__device__ __forceinline__ void prefetch_global(const void* p) {
#if SO_TRAIN_FWD5_PREFETCH == 2
  asm volatile("prefetch.global.L1 [%0];" ::"l"(__cvta_generic_to_global(p)));
#else
  asm volatile("prefetch.global.L2 [%0];" ::"l"(__cvta_generic_to_global(p)));
#endif
}

// ZP / WZP: compile-time zpitch and W * zpitch (0 = take them from the descriptor)
template <bool HAS_RGB, bool PAIR, int ZP, int WZP>
__global__ void __launch_bounds__(32 * SO_TRAIN_FWD5_WARPS, SO_TRAIN_FWD5_MIN_CTAS)
render_train_fwd5_kernel(VolumeDev V, RayDev R, RenderDev P, const float* __restrict__ ws, const float2* __restrict__ vpair,
                         const float* __restrict__ bkgd_rand, TrainOut O) {
  constexpr int B = SO_TRAIN_FWD5_BATCH, U = SO_TRAIN_FWD5_U;
  constexpr unsigned kFull = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const int S = P.S;
  const int K = S >> 5;                    // the launcher guarantees S % (32 U) == 0
  const float eps = 1.1920928955078125e-07f;
  const float k_log2 = P.inv_s * 1.4426950408889634f;
  const float kh = V.ax[0].k0, kw = V.ax[1].k0, kd = V.ax[2].k0;
  const int zp = ZP ? ZP : V.zpitch, wzp = WZP ? WZP : V.W * V.zpitch;
  const bool want_max = O.max_depth != nullptr;
  const long long n_batches = (R.ray_count + B - 1) / B;
  for (long long batch = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); batch < n_batches; batch += warps) {
    const long long ray0 = batch * B;
    const int nb = (int)min((long long)B, R.ray_count - ray0);
    if (SO_TRAIN_FWD5_PREFETCH && P.jitter) {     // the batch's jitter rows are contiguous: one line per lane, before the set-up
      const char* jb = reinterpret_cast<const char*>(P.jitter + (R.ray_begin + ray0) * (long long)(S + 1));
      const long long span = (long long)nb * (S + 1) * 4;
      for (long long off = lane * 128LL; off < span; off += 32 * 128) prefetch_global(jb + off);
      if (lane == 0) prefetch_global(jb + span - 4);
    }
    // ---- set-up of ray (ray0 + lane) in lane `lane` (lanes >= nb repeat the batch's first ray: no divergence, unused)
    const bool own = lane < nb;
    const long long my_ray = own ? ray0 + lane : ray0;
    const long long my_gid = R.ray_begin + my_ray;
    RayCtx c;
    make_ctx(V, R, P, my_gid, c);
    const float my_span_s = (c.tf - c.tn) * (1.0f / (float)S);      // exact: 1/S is a power of two
    float r_acc = 0.f, r_dsum = 0.f, r_best = 0.f, r_cr = 0.f, r_cg = 0.f, r_cb = 0.f;
    for (int b = 0; b < nb; ++b) {
      const long long ray = ray0 + b;
      const float d0 = __shfl_sync(kFull, c.d[0], b), d1 = __shfl_sync(kFull, c.d[1], b), d2 = __shfl_sync(kFull, c.d[2], b);
      const float inv_nrm = __shfl_sync(kFull, c.inv_nrm, b), tn = __shfl_sync(kFull, c.tn, b), span_s = __shfl_sync(kFull, my_span_s, b);
      const float gh0 = __shfl_sync(kFull, c.gh0, b), gdh = __shfl_sync(kFull, c.gdh, b);
      const float gw0 = __shfl_sync(kFull, c.gw0, b), gdw = __shfl_sync(kFull, c.gdw, b);
      const float gd0 = __shfl_sync(kFull, c.gd0, b), gdd = __shfl_sync(kFull, c.gdd, b);
      const float* __restrict__ u = P.jitter ? P.jitter + (R.ray_begin + ray) * (long long)(S + 1) : nullptr;
      float carry = 1.0f, acc = 0.f, dsum = 0.f, cr = 0.f, cg = 0.f, cb = 0.f;
      float best = -INFINITY, best_ts = 0.f;
      int best_i = 0x7fffffff;
#if SO_TRAIN_FWD5_AHEAD
      float ucur[U], unx = 0.f;           // jitter of the current group's samples / of the first edge of the next group
#pragma unroll
      for (int j = 0; j < U; ++j) ucur[j] = u ? __ldcs(u + (j << 5) + lane) : 0.f;
      if (u) unx = __ldcs(u + (U << 5));
#endif
      for (int k = 0; k < K; k += U) {
        // ---- left bin edges (ray length) of this lane's U samples, and the first edge of the next group
        float e0[U];
        const int inx = (k + U) << 5;               // <= S; the jitter row has S + 1 entries
        float bnx = (float)inx;
#if SO_TRAIN_FWD5_AHEAD
        float unext[U], unx2 = 0.f;
#pragma unroll
        for (int j = 0; j < U; ++j) unext[j] = 0.f;
        if (u && k + U < K) {                       // then (k + 2 U) * 32 <= S
#pragma unroll
          for (int j = 0; j < U; ++j) unext[j] = __ldcs(u + ((k + U + j) << 5) + lane);
          unx2 = __ldcs(u + ((k + 2 * U) << 5));
        }
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int s = ((k + j) << 5) + lane;
          const float fs = (float)s;
          float bb = fs;
          if (u) bb = s == 0 ? 0.5f * ucur[j] : ucur[j] + (fs - 0.5f);
          e0[j] = fmaf(bb, span_s, tn);
          ucur[j] = unext[j];
        }
        if (u) bnx = inx == S ? fmaf(0.5f, unx, bnx - 0.5f) : unx + (bnx - 0.5f);
        unx = unx2;
#else
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int s = ((k + j) << 5) + lane;
          const float fs = (float)s;
          float bb = fs;
          if (u) { float uu = __ldcs(u + s); bb = s == 0 ? 0.5f * uu : uu + (fs - 0.5f); }
          e0[j] = fmaf(bb, span_s, tn);
        }
        if (u) { float un = __ldcs(u + inx); bnx = inx == S ? fmaf(0.5f, un, bnx - 0.5f) : un + (bnx - 0.5f); }
#endif
        const float e_next = fmaf(bnx, span_s, tn);
        // ---- positions in grid space
        float mid[U], delta[U], fh[U], fw[U], fz[U], gh[U], gw[U], gd[U];
        int h0[U], w0[U], z0[U];
        bool interior = true;
#pragma unroll
        for (int j = 0; j < U; ++j) {
          // right edge = left edge of the next sample: lane l + 1, or lane 0 of the next chunk for lane 31
          const float src = lane == 0 ? (j + 1 < U ? e0[j + 1 < U ? j + 1 : j] : e_next) : e0[j];
          const float e1 = __shfl_sync(kFull, src, (lane + 1) & 31);
          fast_mid_grid(e0[j], e1, gh0, gdh, gw0, gdw, gd0, gdd, mid[j], delta[j], gh[j], gw[j], gd[j]);
          float flh = floorf(gh[j]), flw = floorf(gw[j]), flz = floorf(gd[j]);
          h0[j] = (int)flh; w0[j] = (int)flw; z0[j] = (int)flz;
          fh[j] = gh[j] - flh; fw[j] = gw[j] - flw; fz[j] = gd[j] - flz;
          interior = interior && (unsigned)h0[j] < (unsigned)(V.H - 1) && (unsigned)w0[j] < (unsigned)(V.W - 1) &&
                     (unsigned)z0[j] < (unsigned)(V.Z - 1);
        }
        // ---- field: trilinear sdf + analytic gradient
        float sdf[U], gx[U], gy[U], gz[U], alpha[U];
        if (__all_sync(kFull, interior)) {
          float a[U][8];
#pragma unroll
          for (int j = 0; j < U; ++j) {               // every load of the group is issued before the first use
            const int idx = h0[j] * wzp + w0[j] * zp + z0[j];
            if (PAIR) {
              const float2* q00 = vpair + idx;
              float2 v00 = __ldg(q00), v01 = __ldg(q00 + zp), v10 = __ldg(q00 + wzp), v11 = __ldg(q00 + wzp + zp);
              a[j][0] = v00.x; a[j][1] = v00.y; a[j][2] = v01.x; a[j][3] = v01.y;
              a[j][4] = v10.x; a[j][5] = v10.y; a[j][6] = v11.x; a[j][7] = v11.y;
            } else {
              const float* p00 = V.sdf + idx;
              a[j][0] = __ldg(p00); a[j][1] = __ldg(p00 + 1);
              a[j][2] = __ldg(p00 + zp); a[j][3] = __ldg(p00 + zp + 1);
              a[j][4] = __ldg(p00 + wzp); a[j][5] = __ldg(p00 + wzp + 1);
              a[j][6] = __ldg(p00 + wzp + zp); a[j][7] = __ldg(p00 + wzp + zp + 1);
            }
          }
#pragma unroll
          for (int j = 0; j < U; ++j) {
            float dz00 = a[j][1] - a[j][0], dz01 = a[j][3] - a[j][2], dz10 = a[j][5] - a[j][4], dz11 = a[j][7] - a[j][6];
            float c00 = fmaf(fz[j], dz00, a[j][0]), c01 = fmaf(fz[j], dz01, a[j][2]);
            float c10 = fmaf(fz[j], dz10, a[j][4]), c11 = fmaf(fz[j], dz11, a[j][6]);
            float dw0 = c01 - c00, dw1 = c11 - c10;
            float c0 = fmaf(fw[j], dw0, c00), c1 = fmaf(fw[j], dw1, c10);
            float dz0 = fmaf(fw[j], dz01 - dz00, dz00), dz1 = fmaf(fw[j], dz11 - dz10, dz10);
            float dgh = c1 - c0;
            sdf[j] = fmaf(fh[j], dgh, c0);
            gy[j] = dgh * kh;
            gx[j] = fmaf(fh[j], dw1 - dw0, dw0) * kw;
            gz[j] = fmaf(fh[j], dz1 - dz0, dz0) * kd;
          }
        } else {
#pragma unroll
          for (int j = 0; j < U; ++j) {
            Taps t = make_taps(V, gh[j], gw[j], gd[j]);
            float dgh, dgw, dgd;
            gather_sdf(V, t, sdf[j], dgh, dgw, dgd);
            gx[j] = dgw * kw; gy[j] = dgh * kh; gz[j] = dgd * kd;
          }
        }
        // ---- NeuS alpha
#pragma unroll
        for (int j = 0; j < U; ++j) {
          float tc = d0 * gx[j] + d1 * gy[j] + d2 * gz[j];
          alpha[j] = neus_alpha_log2(sdf[j] * k_log2, fminf(tc, 0.f) * (delta[j] * (0.5f * k_log2)));
        }
        // ---- transmittance (one warp product scan per chunk), per-sample outputs (streaming stores), ray sums
#pragma unroll
        for (int j = 0; j < U; ++j) {
          const int s = ((k + j) << 5) + lane;
          float f = 1.0f - alpha[j] + 1e-7f;
          // warp_transmittance written out: calling it changes this kernel's machine code
          float incl = warp_incl_prod(f, lane);
          float excl = __shfl_up_sync(kFull, incl, 1);
          float T = carry * (lane == 0 ? 1.0f : excl);
          carry *= __shfl_sync(kFull, incl, 31);
          float w = alpha[j] * T;
          const long long oidx = ray * S + s;
          float ts = mid[j] * inv_nrm, dl = delta[j] * inv_nrm;      // neus_head.py:571-577 (reciprocal multiply, <= 1 ulp)
          if (O.weights) __stcs(O.weights + oidx, w);
          if (O.ts) __stcs(O.ts + oidx, ts);
          if (O.deltas) __stcs(O.deltas + oidx, dl);
          if (O.sdf) __stcs(O.sdf + oidx, sdf[j]);
          if (O.eik) { __stcs(O.eik + 3 * oidx, gx[j]); __stcs(O.eik + 3 * oidx + 1, gy[j]); __stcs(O.eik + 3 * oidx + 2, gz[j]); }
          acc += w;
          dsum = fmaf(w, mid[j], dsum);
          if (want_max) {
            float cand = (dl < eps ? 0.f : w) * __fdividef(1.0f, fmaxf(dl, eps));  // neus_head.py:579-587
            if (cand > best) { best = cand; best_i = s; best_ts = ts; }
          }
          if (HAS_RGB) {
            float col[3], raw[3];
            Taps t = make_taps(V, gh[j], gw[j], gd[j]);
            sample_colour(V, P, t, col, raw);
            cr = fmaf(w, col[0], cr); cg = fmaf(w, col[1], cg); cb = fmaf(w, col[2], cb);
          }
        }
      }
      acc = warp_sum(acc);
      dsum = warp_sum(dsum);
      if (want_max) {
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {   // first-max argmax: larger score wins, ties go to the smaller sample index
          float ob = __shfl_xor_sync(kFull, best, off);
          int oi = __shfl_xor_sync(kFull, best_i, off);
          float ot = __shfl_xor_sync(kFull, best_ts, off);
          if (ob > best || (ob == best && oi < best_i)) { best = ob; best_i = oi; best_ts = ot; }
        }
      }
      if (HAS_RGB) { cr = warp_sum(cr); cg = warp_sum(cg); cb = warp_sum(cb); }
      if (lane == b) { r_acc = acc; r_dsum = dsum; r_best = best_ts; if (HAS_RGB) { r_cr = cr; r_cg = cg; r_cb = cb; } }
    }
    // ---- per-ray tail of ray (ray0 + lane)
    if (own) {
      const long long ray = my_ray;
      long long chunk = R.chunk_len > 0 ? my_gid / R.chunk_len : 0;
      float lo = ws[2 * chunk], hi = ws[2 * chunk + 1];
      float dd = fminf(fmaxf(r_dsum / (r_acc + 1e-10f), lo), hi);
      if (O.depth) O.depth[ray] = dd / c.nrm;
      if (O.acc) O.acc[ray] = r_acc;
      if (O.fars) O.fars[ray] = c.tf / c.nrm;
      if (O.max_depth) O.max_depth[ray] = r_best;
      if (HAS_RGB && O.rgb) {
        float b0, b1, b2;
        if (P.bkgd_mode == 2) { b0 = bkgd_rand[3 * ray]; b1 = bkgd_rand[3 * ray + 1]; b2 = bkgd_rand[3 * ray + 2]; }
        else { b0 = b1 = b2 = (P.bkgd_mode == 1) ? 1.f : 0.f; }
        float rem = 1.0f - r_acc;
        float r = fmaf(b0, rem, r_cr), g = fmaf(b1, rem, r_cg), bb = fmaf(b2, rem, r_cb);
        if (P.eval_clamp) { r = __saturatef(r); g = __saturatef(g); bb = __saturatef(bb); }
        O.rgb[3 * ray] = r; O.rgb[3 * ray + 1] = g; O.rgb[3 * ray + 2] = bb;
      }
    }
  }
}

// scatter d(loss)/d(sdf value), d/d(metre-gradient) of one sample into the 8 corners of the sdf volume
__device__ __forceinline__ void scatter_sdf(const VolumeDev& V, float* __restrict__ gvol, const Taps& t, float g_s, float g_gh,
                                            float g_gw, float g_gd) {
  // interpolant:  s = sum_c Wh(c) Ww(c) Wz(c) v_c ;  d s / d gh = sum_c Wh'(c) Ww Wz v_c  etc. (masks = zero padding)
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int dh = k >> 2, dw = (k >> 1) & 1, dz = k & 1;
    float mh = dh ? t.mh1 : t.mh0, mw = dw ? t.mw1 : t.mw0, mz = dz ? t.mz1 : t.mz0;
    float m = mh * mw * mz;
    if (m == 0.f) continue;
    float wh = dh ? t.fh : 1.f - t.fh, ww = dw ? t.fw : 1.f - t.fw, wz = dz ? t.fz : 1.f - t.fz;
    float sh = dh ? 1.f : -1.f, sw = dw ? 1.f : -1.f, sz = dz ? 1.f : -1.f;
    float g = g_s * wh * ww * wz + g_gh * sh * ww * wz + g_gw * wh * sw * wz + g_gd * wh * ww * sz;
    atomicAdd(gvol + ((size_t)(t.h0 + dh) * V.W + (t.w0 + dw)) * V.zpitch + (t.z0 + dz), g);
  }
}

template <int N>
__device__ __forceinline__ void scatter_feat(const VolumeDev& V, float* __restrict__ gfeat, const Taps& t, int c0, const float g[N]) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int dh = k >> 2, dw = (k >> 1) & 1, dz = k & 1;
    float m = (dh ? t.mh1 : t.mh0) * (dw ? t.mw1 : t.mw0) * (dz ? t.mz1 : t.mz0);
    if (m == 0.f) continue;
    float wgt = (dh ? t.fh : 1.f - t.fh) * (dw ? t.fw : 1.f - t.fw) * (dz ? t.fz : 1.f - t.fz);
    float* p = gfeat + (((size_t)(t.h0 + dh) * V.W + (t.w0 + dw)) * V.Z + (t.z0 + dz)) * V.feat_pitch + c0;
#pragma unroll
    for (int i = 0; i < N; ++i) atomicAdd(p + i, wgt * g[i]);
  }
}

// FAST: recompute the samples with the arithmetic of the FAST forwards (sample_geom<true>, neus_alpha_log2)
template <bool HAS_RGB, int SEM, bool FAST>
__global__ void __launch_bounds__(128, SEM == 24 ? SO_TRAIN_BWD24_MIN_CTAS : 1) render_train_bwd_kernel(VolumeDev V, RayDev R, RenderDev P, const float* __restrict__ ws,
                                                               const float* __restrict__ bkgd_rand, TrainGrad G) {
  constexpr bool HAS_SEM = SEM != 0;
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const int S = P.S;
  const int K = (S + 31) >> 5;
  const int n_sem = HAS_SEM ? V.n_feat - 3 : 0;
  float g_invs_local = 0.f;
  for (long long ray = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); ray < R.ray_count; ray += warps) {
    long long gid = R.ray_begin + ray;
    RayCtx c;
    make_ctx(V, R, P, gid, c);
    const float nrm = c.nrm;
    const float* d = c.d;
    // ---- pass 1: transmittance per sample, ray sums
    float Tk[kTrainMaxChunks], Ak[kTrainMaxChunks];
    float carry = 1.0f, acc = 0.f, dsum = 0.f;
#pragma unroll
    for (int k = 0; k < kTrainMaxChunks; ++k) {
      if (k >= K) break;
      int s = k * 32 + lane;
      bool live = s < S;
      Sample q;
      eval_sample<FAST>(V, P, c, live ? s : S - 1, lane, q);
      float alpha = live ? q.alpha : 0.f;
      float f = live ? (1.0f - alpha + 1e-7f) : 1.0f;
      float T = warp_transmittance(f, lane, carry);
      Tk[k] = T; Ak[k] = alpha;
      acc += alpha * T;
      dsum = fmaf(alpha * T, q.mid, dsum);
    }
    acc = warp_sum(acc);
    dsum = warp_sum(dsum);
    long long chunk = R.chunk_len > 0 ? gid / R.chunk_len : 0;
    float lo = ws[2 * chunk], hi = ws[2 * chunk + 1];
    float draw = dsum / (acc + 1e-10f);
    bool clipped = draw < lo || draw > hi;
    float gd = (G.g_depth && !clipped) ? G.g_depth[ray] / nrm : 0.f;   // d depth / d depth_raw (depth = clip(raw)/|dir|)
    float ga = G.g_acc ? G.g_acc[ray] : 0.f;
    float gr[3] = {0.f, 0.f, 0.f}, bg[3] = {0.f, 0.f, 0.f};
    if (HAS_RGB && G.g_rgb) {
      gr[0] = G.g_rgb[3 * ray]; gr[1] = G.g_rgb[3 * ray + 1]; gr[2] = G.g_rgb[3 * ray + 2];
      if (P.bkgd_mode == 2) { bg[0] = bkgd_rand[3 * ray]; bg[1] = bkgd_rand[3 * ray + 1]; bg[2] = bkgd_rand[3 * ray + 2]; }
      else bg[0] = bg[1] = bg[2] = (P.bkgd_mode == 1) ? 1.f : 0.f;
    }
    // ---- pass 2: reverse over chunks
    float tail = 0.f;   // sum_{j in later chunks} G_j w_j
#pragma unroll
    for (int kk = kTrainMaxChunks - 1; kk >= 0; --kk) {
      if (kk >= K) continue;
      int s = kk * 32 + lane;
      bool live = s < S;
      Sample q;
      eval_sample<FAST>(V, P, c, live ? s : S - 1, lane, q);
      float T = Tk[kk], alpha = Ak[kk];
      float w = alpha * T;
      long long oidx = ray * S + (live ? s : S - 1);
      // dL/dw_s
      float Gw = (G.g_weights ? G.g_weights[oidx] : 0.f) + ga + gd * (q.mid - draw) / (acc + 1e-10f);
      float col[3] = {0.f, 0.f, 0.f}, raw[3] = {0.f, 0.f, 0.f};
      float lg[SEM == 24 ? 24 : (HAS_SEM ? kMaxSem : 1)];      // SEM == 24: the 24 gathered channels, then [3..23] = softmax
      float gdot = 0.f;
      if (SEM == 24) {
        gather_feat24(V, q.t, lg);
        colour_act(P, lg, col, raw);
        if (G.g_rgb) Gw += gr[0] * (col[0] - bg[0]) + gr[1] * (col[1] - bg[1]) + gr[2] * (col[2] - bg[2]);
        if (G.g_sem) {
          float mx = lg[3];
#pragma unroll
          for (int c = 1; c < kSem24; ++c) mx = fmaxf(mx, lg[3 + c]);
          float den = 0.f;
#pragma unroll
          for (int c = 0; c < kSem24; ++c) { lg[3 + c] = expf(lg[3 + c] - mx); den += lg[3 + c]; }
          const float* gs = G.g_sem + ray * kSem24;
#pragma unroll
          for (int c = 0; c < kSem24; ++c) { lg[3 + c] /= den; gdot += __ldg(gs + c) * lg[3 + c]; }
          Gw += gdot;
        }
      } else if (HAS_RGB && G.g_rgb) {
        sample_colour(V, P, q.t, col, raw);
        Gw += gr[0] * (col[0] - bg[0]) + gr[1] * (col[1] - bg[1]) + gr[2] * (col[2] - bg[2]);
      }
      if (SEM == 1 && G.g_sem) {
        float mx = -INFINITY;
        for (int c = 0; c < n_sem; ++c) { float f1[1]; gather_feat<1>(V, q.t, 3 + c, f1); lg[c] = f1[0]; mx = fmaxf(mx, f1[0]); }
        float den = 0.f;
        for (int c = 0; c < n_sem; ++c) { lg[c] = expf(lg[c] - mx); den += lg[c]; }
        for (int c = 0; c < n_sem; ++c) { lg[c] /= den; gdot += G.g_sem[ray * n_sem + c] * lg[c]; }
        Gw += gdot;
      }
      if (!live) Gw = 0.f;
      float gw_w = live ? Gw * w : 0.f;
      float rinc = warp_rev_incl_sum(gw_w, lane);
      float B = tail + rinc - gw_w;                         // sum_{j > s} G_j w_j
      tail += __shfl_sync(0xffffffffu, rinc, 0);
      float dalpha = Gw * T - B / (1.0f - alpha + 1e-7f);
      if (!live) dalpha = 0.f;   // (the raw alpha lies in (0, 1] by construction, so the clip never cuts a gradient)
      // alpha = (Pa - Pb + e) / (Pa + e):  d/da = Pa' Pb / (Pa+e)^2,  d/db = -Pb' / (Pa+e)
      float den = q.pa + 1e-5f;
      float da = q.pa * (1.0f - q.pa) * q.pb / (den * den);
      float db = -q.pb * (1.0f - q.pb) / den;
      float g_sdf = dalpha * (da + db) * P.inv_s;
      float g_half = dalpha * (db - da) * P.inv_s;
      g_invs_local += dalpha * (da * (q.sdf - q.half) + db * (q.sdf + q.half));
      // half = ic * delta / 2,  ic = -(relu(-tc/2 + 1/2)(1-r) + relu(-tc) r)
      float dic = 0.f;
      if (fmaf(-q.tc, 0.5f, 0.5f) > 0.f) dic += 0.5f * (1.0f - P.cos_anneal);
      if (-q.tc > 0.f) dic += P.cos_anneal;
      float g_tc = g_half * 0.5f * q.delta * dic;
      float ggx = g_tc * d[0], ggy = g_tc * d[1], ggz = g_tc * d[2];
      if (live) {
        if (G.g_sdf) g_sdf += G.g_sdf[oidx];
        if (G.g_eik) { ggx += G.g_eik[3 * oidx]; ggy += G.g_eik[3 * oidx + 1]; ggz += G.g_eik[3 * oidx + 2]; }
        // metre gradient (gx, gy, gz) = (dgw kw, dgh kh, dgd kd)
        scatter_sdf(V, G.g_vol_sdf, q.t, g_sdf, ggy * q.kh, ggx * q.kw, ggz * q.kd);
        if (SEM == 24 && G.g_vol_feat && (G.g_rgb || G.g_sem)) {
          // the gradient w.r.t. the 24 interpolated channels, built in place of the gathered values
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            float dact = P.sh_act == 0 ? (raw[c] + 0.5f > 0.f ? 1.f : 0.f) : col[c] * (1.f - col[c]);
            lg[c] = G.g_rgb ? w * gr[c] * dact * kC0 : 0.f;
          }
          const float* gs = G.g_sem + ray * kSem24;
#pragma unroll
          for (int c = 0; c < kSem24; ++c) lg[3 + c] = G.g_sem ? w * lg[3 + c] * (__ldg(gs + c) - gdot) : 0.f;
          if (w != 0.f) scatter_feat24(V, G.g_vol_feat, q.t, lg);            // w == 0 (transmittance underflowed): every entry is 0
        } else if (HAS_RGB && G.g_rgb && G.g_vol_feat) {
          float gf[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            float dact = P.sh_act == 0 ? (raw[c] + 0.5f > 0.f ? 1.f : 0.f) : col[c] * (1.f - col[c]);
            gf[c] = w * gr[c] * dact * kC0;
          }
          scatter_feat<3>(V, G.g_vol_feat, q.t, 0, gf);
        }
        if (SEM == 1 && G.g_sem && G.g_vol_feat) {
          for (int c = 0; c < n_sem; ++c) {
            float gl[1] = {w * lg[c] * (G.g_sem[ray * n_sem + c] - gdot)};
            scatter_feat<1>(V, G.g_vol_feat, q.t, 3 + c, gl);
          }
        }
      }
    }
  }
  if (G.g_inv_s) {
    g_invs_local = warp_sum(g_invs_local);
    if (lane == 0 && g_invs_local != 0.f) atomicAdd(G.g_inv_s, g_invs_local);
  }
}

__global__ void __launch_bounds__(256) field_query_bwd_kernel(VolumeDev V, const float* __restrict__ pts, long long n,
                                                              const float* __restrict__ g_sdf, const float* __restrict__ g_grad,
                                                              const float* __restrict__ g_feat, float* __restrict__ gvs,
                                                              float* __restrict__ gvf) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
  float kh, kw, kd;
  float gh = axis_m2g(V.ax[0], y, kh), gw = axis_m2g(V.ax[1], x, kw), gd = axis_m2g(V.ax[2], z, kd);
  Taps t = make_taps(V, gh, gw, gd);
  float gs = g_sdf ? g_sdf[i] : 0.f;
  float gx = g_grad ? g_grad[3 * i] : 0.f, gy = g_grad ? g_grad[3 * i + 1] : 0.f, gz = g_grad ? g_grad[3 * i + 2] : 0.f;
  scatter_sdf(V, gvs, t, gs, gy * kh, gx * kw, gz * kd);
  if (g_feat && gvf)
    for (int c = 0; c < V.n_feat; ++c) { float g1[1] = {g_feat[i * V.n_feat + c]}; scatter_feat<1>(V, gvf, t, c, g1); }
}

// test probe: the fp32 grid coordinates of every sample as the forwards and the backward of this launch compute them
template <bool FAST>
__global__ void __launch_bounds__(128) render_train_probe_kernel(VolumeDev V, RayDev R, RenderDev P, float* __restrict__ grid) {
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (blockDim.x >> 5);
  const int S = P.S;
  const int K = (S + 31) >> 5;
  for (long long ray = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5); ray < R.ray_count; ray += warps) {
    RayCtx c;
    make_ctx(V, R, P, R.ray_begin + ray, c);
    for (int k = 0; k < K; ++k) {
      const int s = k * 32 + lane;
      const bool live = s < S;
      float mid, delta, gh, gw, gd, kh, kw, kd;
      sample_geom<FAST>(V, P, c, live ? s : S - 1, lane, mid, delta, gh, gw, gd, kh, kw, kd);
      if (live) {
        float* o = grid + 3 * (ray * S + s);
        o[0] = gh; o[1] = gw; o[2] = gd;
      }
    }
  }
}

// the lean per-sample path of the forwards applies (see fast_edge)
static bool train_fast(const VolumeDev& V, const RenderDev& P) { return uniform_affine_march(V, P) && P.S >= 32; }

static int train_num_samples_check(const so_render_params* pr) {
  if (pr->num_samples < 1) return SO_ERR_INVALID_ARG;
  if (pr->num_samples > 32 * kTrainMaxChunks) return SO_ERR_UNSUPPORTED;
  return SO_OK;
}

static int train_common_checks(const float* vol_sdf, const float* vol_feat, const so_volume_desc* d, const float* cam_mats,
                               const so_ray_desc* rd, const so_render_params* pr, const float* workspace, bool want_rgb,
                               bool want_sem, const float* bkgd_rand) {
  int rc = check_render_operands(vol_sdf, workspace, cam_mats, rd, pr, d);
  if (rc || (rc = train_num_samples_check(pr))) return rc;
  return check_shading(d, vol_feat, pr, want_rgb, want_sem, bkgd_rand);
}

// persistent-style grid of the one-ray-per-warp kernels: warps stride over rays; 4 warps per CTA, enough CTAs to fill
// every SM several times over
static unsigned train_grid(long long ray_count) {
  const long long ctas = ceil_div64(ray_count, 4), cap = (long long)num_sms() * 16;
  return (unsigned)(ctas < cap ? ctas : cap);
}

}  // namespace so

using namespace so;

static bool g_force_sem_generic = false;
// test hook: route 24-channel volumes through the generic (runtime channel count) semantic path
extern "C" int so_render_train_force_sem_generic(int on) { g_force_sem_generic = on != 0; return SO_OK; }
static bool g_force_fwd32 = false;
// test hook: route so_render_train_forward through the one-ray-per-warp kernel even when the batched one applies
extern "C" int so_render_train_force_fwd32(int on) { g_force_fwd32 = on != 0; return SO_OK; }

extern "C" int64_t so_render_train_pair_floats(const so_volume_desc* vol_host) {
  if (!vol_host || validate_volume(vol_host)) return 0;
  return zpair_floats(*vol_host);
}

extern "C" int so_render_train_forward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                                       const float* cam_mats, const float* pix, const so_ray_desc* rd,
                                       const so_render_params* pr, const float* jitter, const float* bkgd_rand,
                                       float* depth, float* acc, float* fars, float* rgb, float* sem, float* max_depth,
                                       float* weights, float* ts, float* deltas, float* eik_grad, float* sample_sdf,
                                       float* workspace, float* pair_workspace, void* stream) {
  bool want_rgb = rgb != nullptr, want_sem = sem != nullptr;
  if (pair_workspace && (reinterpret_cast<uintptr_t>(pair_workspace) & 7)) return SO_ERR_INVALID_ARG;
  int rc = train_common_checks(vol_sdf, vol_feat, vol_host, cam_mats, rd, pr, workspace, want_rgb, want_sem, bkgd_rand);
  if (rc) return rc;
  RayDev R;
  if ((rc = make_ray_dev(rd, cam_mats, pix, &R))) return rc;
  if (R.ray_count == 0) return SO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  VolumeDev V = make_volume(*vol_host, vol_sdf, vol_feat);
  RenderDev P = make_render_dev(*pr, jitter);
  if ((rc = launch_depth_bounds(R, P, workspace, st))) return rc;
  TrainOut O{depth, acc, fars, rgb, sem, max_depth, weights, ts, deltas, eik_grad, sample_sdf};
  const unsigned grid = train_grid(R.ray_count);
  ProfScope prof(6, st);
  const bool fast = train_fast(V, P);
  // batched-ray kernel (U chunks in flight, optional z-pair volume); the one-ray-per-warp kernel covers semantics,
  // non-affine mappings, S not a multiple of 32 U and the cos-anneal phase
  const bool sem24 = want_sem && V.n_feat == 24 && V.feat_pitch == 24 && (reinterpret_cast<uintptr_t>(vol_feat) & 15) == 0 && !g_force_sem_generic;
  const bool v5 = fast && !want_sem && ((P.S >> 5) % SO_TRAIN_FWD5_U) == 0 && !g_force_fwd32;
#define SO_TRAIN_FWD(RGB, SEM, F) render_train_fwd_kernel<RGB, SEM, F><<<grid, 128, 0, st>>>(V, R, P, workspace, bkgd_rand, O)
  if (v5) {
    const float2* vp = nullptr;
    if (pair_workspace) {
      launch_zpair_pack(vol_sdf, *vol_host, pair_workspace, st);
      note_launch(1);
      vp = reinterpret_cast<const float2*>(pair_workspace);
    }
    const long long n_batches = ceil_div64(R.ray_count, SO_TRAIN_FWD5_BATCH);
    const unsigned grid5 = (unsigned)ceil_div64(n_batches, SO_TRAIN_FWD5_WARPS);   // one batch per warp
    const bool cp = SO_TRAIN_FWD5_CONST_PITCH && V.zpitch == 32 && V.W == 257;
#define SO_TRAIN_FWD5(RGB, PAIR, ZP, WZP) \
  render_train_fwd5_kernel<RGB, PAIR, ZP, WZP><<<grid5, 32 * SO_TRAIN_FWD5_WARPS, 0, st>>>(V, R, P, workspace, vp, bkgd_rand, O)
#define SO_TRAIN_FWD5_P(RGB, PAIR) do { if (cp) SO_TRAIN_FWD5(RGB, PAIR, 32, 257 * 32); else SO_TRAIN_FWD5(RGB, PAIR, 0, 0); } while (0)
    if (want_rgb) { if (vp) SO_TRAIN_FWD5_P(true, true); else SO_TRAIN_FWD5_P(true, false); }
    else { if (vp) SO_TRAIN_FWD5_P(false, true); else SO_TRAIN_FWD5_P(false, false); }
#undef SO_TRAIN_FWD5_P
#undef SO_TRAIN_FWD5
  } else if (want_sem && sem24) { if (fast) SO_TRAIN_FWD(true, 24, true); else SO_TRAIN_FWD(true, 24, false); }
  else if (want_sem) { if (fast) SO_TRAIN_FWD(true, 1, true); else SO_TRAIN_FWD(true, 1, false); }
  else if (want_rgb) { if (fast) SO_TRAIN_FWD(true, 0, true); else SO_TRAIN_FWD(true, 0, false); }
  else { if (fast) SO_TRAIN_FWD(false, 0, true); else SO_TRAIN_FWD(false, 0, false); }
#undef SO_TRAIN_FWD
  note_launch(1);
  return check_launch();
}

extern "C" int so_render_train_backward(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host,
                                        const float* cam_mats, const float* pix, const so_ray_desc* rd,
                                        const so_render_params* pr, const float* jitter, const float* bkgd_rand,
                                        const float* g_depth, const float* g_acc, const float* g_rgb, const float* g_sem,
                                        const float* g_weights, const float* g_eik, const float* g_sdf, float* g_vol_sdf,
                                        float* g_vol_feat, float* g_inv_s, float* workspace, void* stream) {
  bool want_rgb = g_rgb != nullptr, want_sem = g_sem != nullptr;
  if (!g_vol_sdf) return SO_ERR_INVALID_ARG;
  int rc = train_common_checks(vol_sdf, vol_feat, vol_host, cam_mats, rd, pr, workspace, want_rgb, want_sem, bkgd_rand);
  if (rc) return rc;
  if ((want_rgb || want_sem) && !g_vol_feat) return SO_ERR_INVALID_ARG;
  RayDev R;
  if ((rc = make_ray_dev(rd, cam_mats, pix, &R))) return rc;
  if (R.ray_count == 0) return SO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  VolumeDev V = make_volume(*vol_host, vol_sdf, vol_feat);
  RenderDev P = make_render_dev(*pr, jitter);
  if ((rc = launch_depth_bounds(R, P, workspace, st))) return rc;
  TrainGrad G{g_depth, g_acc, g_rgb, g_sem, g_weights, g_eik, g_sdf, g_vol_sdf, g_vol_feat, g_inv_s};
  const unsigned grid = train_grid(R.ray_count);
  ProfScope prof(7, st);
  const bool sem24 = V.n_feat == 24 && V.feat_pitch == 24 && (want_rgb || want_sem) && !g_force_sem_generic &&
                     ((reinterpret_cast<uintptr_t>(vol_feat) | reinterpret_cast<uintptr_t>(g_vol_feat)) & 15) == 0;
  const bool fast = train_fast(V, P);      // recompute the samples with the arithmetic of the paired forward
#define SO_TRAIN_BWD(RGB, SEM) do { \
    if (fast) render_train_bwd_kernel<RGB, SEM, true><<<grid, 128, 0, st>>>(V, R, P, workspace, bkgd_rand, G); \
    else render_train_bwd_kernel<RGB, SEM, false><<<grid, 128, 0, st>>>(V, R, P, workspace, bkgd_rand, G); } while (0)
  if (sem24) SO_TRAIN_BWD(true, 24);
  else if (want_sem) SO_TRAIN_BWD(true, 1);
  else if (want_rgb) SO_TRAIN_BWD(true, 0);
  else SO_TRAIN_BWD(false, 0);
#undef SO_TRAIN_BWD
  note_launch(1);
  return check_launch();
}

extern "C" int so_render_train_probe(const so_volume_desc* vol_host, const float* cam_mats, const float* pix, const so_ray_desc* rd,
                                     const so_render_params* pr, const float* jitter, float* grid, void* stream) {
  int rc = check_render_operands(vol_host, grid, cam_mats, rd, pr, vol_host);
  if (rc || (rc = train_num_samples_check(pr))) return rc;
  RayDev R;
  if ((rc = make_ray_dev(rd, cam_mats, pix, &R))) return rc;
  if (R.ray_count == 0) return SO_OK;
  VolumeDev V = make_volume(*vol_host, nullptr, nullptr);
  RenderDev P = make_render_dev(*pr, jitter);
  const unsigned g = train_grid(R.ray_count);
  cudaStream_t st = (cudaStream_t)stream;
  if (train_fast(V, P)) render_train_probe_kernel<true><<<g, 128, 0, st>>>(V, R, P, grid);
  else render_train_probe_kernel<false><<<g, 128, 0, st>>>(V, R, P, grid);
  note_launch(1);
  return check_launch();
}

extern "C" int so_field_query_backward(const so_volume_desc* vol_host, const float* points, int64_t n, const float* g_sdf,
                                       const float* g_grad, const float* g_feat, float* g_vol_sdf, float* g_vol_feat,
                                       void* stream) {
  if (!points || n < 0 || !g_vol_sdf) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(vol_host);
  if (rc) return rc;
  if (g_feat && !g_vol_feat) return SO_ERR_INVALID_ARG;
  if (n == 0) return SO_OK;
  VolumeDev V = make_volume(*vol_host, nullptr, nullptr);
  field_query_bwd_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(V, points, n, g_sdf, g_grad, g_feat,
                                                                                         g_vol_sdf, g_vol_feat);
  note_launch(1);
  return check_launch();
}
