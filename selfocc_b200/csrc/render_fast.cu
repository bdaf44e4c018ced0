// Packed-volume inference render (SURVEY.md section 8a rows B1-B4, B6-B11): the second-generation kernels behind
// so_render_infer_packed.  Same contract and the same per-ray recurrence as render_infer_kernel (render.cu); what changes
// is how a sample is fetched and how many instructions it costs:
//
//  * the decoded volume is first repacked once per frame (so_render_pack) into the layout the gather wants:
//      n_feat == 0 : float2 [H][W][zpitch]  {sdf[z], sdf[z+1]}     -> the 8 trilinear taps are 4 aligned 64-bit loads
//      n_feat == 3 : float4 [H][W][Z]       {C0 r + 1/2, C0 g + 1/2, C0 b + 1/2, sdf}
//                                                                   -> 8 aligned 128-bit loads fetch sdf AND colour
//    (the reference gathers 8 + 24 scalars per sample for colour, bev_nerf.py:99-117; the SH-0 colour map is affine, so
//    it is applied once per voxel in the pack and the loop keeps only the relu);
//  * the interior loop is scalar FP32 (sm_90 has no packed fp32x2 pipe): only the sdf is lerped with its gradient terms
//    (the gradient falls out of the lerp differences); r, g, b take one shared set of 8 trilinear weights;
//  * "all 8 corners inside the volume" is decided ONCE per ray: for the affine metre->grid map g(t) = g0 + gd * t is
//    monotone along the ray (so is its fp32 evaluation fma(gd, t, g0)), so if the first and the last sample are interior,
//    every sample is; warps with a non-interior ray take the general zero-padding loop;
//  * NeuS alpha with ONE reciprocal:  alpha = (omen + c (1 + B)) / ((1 + B) (1 + c)),  A = e^-(s-h), B = e^(s+h),
//    c = 1e-5 (1 + A)  (algebraically equal to (Phi(prev) - Phi(next) + 1e-5) / (Phi(prev) + 1e-5), no cancellation),
//    and in the interior loop two exponentials: omen = 1 - e^-x = 1 - A B;
//  * with colour, a lane keeps its last cell's corners in registers and reloads only when its cell changes;
//  * cell indices come from the float floor through the 2^23 magic add (integer pipe) instead of F2I (XU pipe);
//  * a warp stops marching once every ray's transmittance is below 1e-9: the dropped tail changes acc / depth / rgb by
//    < 1e-9 relative and cannot hold the max-depth argmax (a later w is <= T < 1e-9 <= max_s w_s since sum_s w_s >= 1 - T).
#include "render_common.cuh"

// Tuning knobs, timed on an H100 80GB HBM3 (400 W) with scripts/bench_render.py, analytic scene, 8.64 M rays, depth-only /
// colour ms, before the scalar rewrite: defaults (unroll 4; 6 / 4 CTAs per SM) 6.93-7.18 / 12.06-12.12 over two runs;
// unroll 1 7.27 / 12.08, unroll 2 7.04 / 12.18; 4 / 3 CTAs 6.98 / 12.14; 8 / 5 CTAs 6.92 / 12.12.  After it (same card and
// limit, one session): previous kernel 6.94 / 12.10; cell cache in both kernels 6.74 / 10.81; in neither 6.54 / 11.51.
// bench.py render per step agrees: with the cache depth-only 9.84 / 9.70 vs 9.40 / 9.28 without, colour 15.35 / 15.33 vs
// 16.04 / 15.95 (previous kernel 10.13 / 10.16 and 16.60 / 16.53).  So the cache is on for the colour kernel, whose 8
// 128-bit corner loads it saves, and off for the depth-only one, whose 4 64-bit loads cost less than the vote and the
// register-held corners.  Unroll, CTAs per SM and the exit period were not re-timed after the rewrite.
#ifndef SO_RF_BLOCK
#define SO_RF_BLOCK 128
#endif
#ifndef SO_RF_MIN_CTAS
#define SO_RF_MIN_CTAS 6
#endif
#ifndef SO_RF_MIN_CTAS_RGB
#define SO_RF_MIN_CTAS_RGB 4
#endif
#ifndef SO_RF_UNROLL
#define SO_RF_UNROLL 4
#endif
#ifndef SO_RF_CELL_CACHE
#define SO_RF_CELL_CACHE 0      // depth-only: keep the last cell's corners in registers (0: load them every sample)
#endif
#ifndef SO_RF_CELL_CACHE_RGB
#define SO_RF_CELL_CACHE_RGB 1  // the same for the colour kernel
#endif
#ifndef SO_RF_EXIT_T
#define SO_RF_EXIT_T 1e-9f
#endif
#ifndef SO_RF_EXIT_EVERY
#define SO_RF_EXIT_EVERY 4      // the exit vote is taken every 4th sample (power of two)
#endif

namespace so {

struct RayAcc {
  float T, acc, dsum, n0, n1, n2, best, best_mid, c_r, c_g, c_b;
  int best_i;
};

struct RayGeo {        // per-ray constants of the affine march (grid units)
  float tn, span, step;
  float gh0, gw0, gd0, gdh, gdw, gdd;   // g(t) = g0 + gd * t
  float kh, kw, kd;                     // d grid / d metre
  float dx, dy, dz;                     // unit direction (metres)
  float h_const;                        // delta * inv_s * log2(e) / 2
  float k_log2;
};

// NeuS alpha, one-reciprocal form (see the file header).  s2 = sdf * inv_s * log2(e), h2 = half * inv_s * log2(e) <= 0.
// The exponents are clamped at 64: beyond that alpha is 1 (A huge) or the 1e-5 floor (B huge) to within 2^-40.
// kTwoExp (interior loop): e^-x = 2^(2 h2) = A B whenever neither exponent is clamped, so omen needs no third
// exponential.  A clamped A or B makes A B smaller than e^-x, but then alpha is 1 (resp. the 1e-5 floor) to within 2^-40
// whatever omen is; A B <= 1 always (the exponents sum to 2 h2 <= 0 and cannot both exceed 64), so omen stays in [0, 1].
// A flushed A or B means e^-x < 2^-62, where 1 - e^-x rounds to 1 anyway.
template <bool kTwoExp>
__device__ __forceinline__ float neus_alpha_rcp1(float s2, float h2) {
  float A = exp2f(fminf(h2 - s2, 64.f));
  float B = exp2f(fminf(s2 + h2, 64.f));
  float pB = 1.0f + B;
  float c = fmaf(A, 1e-5f, 1e-5f);                               // 1e-5 (1 + A)
  float x = h2 * (-2.0f * 0.6931471805599453f);                  // (s - h) - (s + h) in natural units, >= 0
  float ser = x * fmaf(x, fmaf(x, fmaf(x, fmaf(x, 1.0f / 120.0f, -1.0f / 24.0f), 1.0f / 6.0f), -0.5f), 1.0f);
  float omen = x < 0.125f ? ser : (kTwoExp ? fmaf(-A, B, 1.0f) : 1.0f - exp2f(h2 + h2));   // 1 - e^-x
  float num = fmaf(c, pB, omen);
  float den = fmaf(pB, c, pB);
  return __saturatef(__fdividef(num, den));
}

__device__ __forceinline__ void composite(RayAcc& a, float alpha, float mid, float gx, float gy, float gz, int s, float& w_out) {
  float w = alpha * a.T;
  a.T *= (1.0f - alpha + 1e-7f);
  a.acc += w;
  a.dsum = fmaf(w, mid, a.dsum);
  float wn = w * rsqrtf(fmaxf(fmaf(gx, gx, fmaf(gy, gy, gz * gz)), 1e-24f));   // F.normalize(eps=1e-12)
  a.n0 = fmaf(wn, gx, a.n0); a.n1 = fmaf(wn, gy, a.n1); a.n2 = fmaf(wn, gz, a.n2);
  // max-depth candidate (neus_head.py:430-438): delta is a positive per-ray constant here, so argmax(w / delta) = argmax(w)
  if (w > a.best) { a.best = w; a.best_i = s; }     // best_mid is recomputed from best_i after the loop (same fp32 formula)
  w_out = w;
}

// General (zero-padding) march for warps that hold a ray leaving the volume: the arithmetic of render_infer_kernel<.., FAST>.
template <bool RGB>
__device__ __noinline__ void march_padded(const VolumeDev& V, const RayGeo& G, int S, int sh_act, float* __restrict__ dbg, RayAcc& a) {
  float bm = 0.5f * G.step;
  for (int s = 0; s < S; ++s) {
    float mid = fmaf(bm, G.span, G.tn);
    bm += G.step;
    float gh = fmaf(G.gdh, mid, G.gh0), gw = fmaf(G.gdw, mid, G.gw0), gd = fmaf(G.gdd, mid, G.gd0);
    if (dbg) { dbg[3 * s] = gh; dbg[3 * s + 1] = gw; dbg[3 * s + 2] = gd; }
    Taps t = make_taps(V, gh, gw, gd);
    float sdf, dgh, dgw, dgd;
    gather_sdf(V, t, sdf, dgh, dgw, dgd);
    float tc = fmaf(G.gdh, dgh, fmaf(G.gdw, dgw, G.gdd * dgd));
    float alpha = neus_alpha_rcp1<false>(sdf * G.k_log2, fminf(tc, 0.f) * G.h_const);
    float w;
    composite(a, alpha, mid, dgw * G.kw, dgh * G.kh, dgd * G.kd, s, w);
    if (RGB) {
      float f[3], col[3], raw[3];
      gather_feat<3>(V, t, 0, f);
      colour_act(sh_act, f, col, raw);
      a.c_r = fmaf(w, col[0], a.c_r); a.c_g = fmaf(w, col[1], a.c_g); a.c_b = fmaf(w, col[2], a.c_b);
    }
  }
}

constexpr float kMagic = 8388608.0f;          // 2^23: float(n) + 2^23 has the bit pattern 0x4B000000 + n for 0 <= n < 2^23
constexpr unsigned kMagicBits = 0x4B000000u;

// ZP / WZ: compile-time pitches (0 = take them from the descriptor).
//   pair volume: ZP = zpitch, WZ = W * zpitch (float2 elements);  rgbs volume: ZP = Z, WZ = W * Z (float4 elements)
template <bool RGB, bool DBG, int ZP, int WZ>
__global__ void __launch_bounds__(SO_RF_BLOCK, RGB ? SO_RF_MIN_CTAS_RGB : SO_RF_MIN_CTAS)
render_packed_kernel(VolumeDev V, const void* __restrict__ pack, RayDev R, RenderDev P, const float* __restrict__ ws,
                     const float* __restrict__ bkgd_rand, float* __restrict__ depth, float* __restrict__ max_depth,
                     long long* __restrict__ max_idx, float* __restrict__ acc_out, float* __restrict__ normal_vis,
                     float* __restrict__ rgb_out, float* __restrict__ dbg_grid) {
  constexpr unsigned kFull = 0xffffffffu;
  long long lid = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const bool valid = lid < R.ray_count;            // lanes past the end stay alive for the warp votes below
  if (!valid) lid = R.ray_count - 1;
  const long long gid = R.ray_begin + lid;
  float o[3], d[3], nrm, tn, tf;
  make_ray(R, gid, o, d, nrm);
  slab(P, o, d, tn, tf);

  const int S = P.S;
  RayGeo G;
  G.tn = tn; G.span = tf - tn; G.step = 1.0f / (float)S;
  G.kh = V.ax[0].k0; G.kw = V.ax[1].k0; G.kd = V.ax[2].k0;
  affine_grid_ray(V, o, d, G.gh0, G.gdh, G.gw0, G.gdw, G.gd0, G.gdd);
  G.dx = d[0]; G.dy = d[1]; G.dz = d[2];
  G.k_log2 = P.inv_s * 1.4426950408889634f;
  const float delta_c = G.span * G.step;
  G.h_const = delta_c * (0.5f * G.k_log2);

  RayAcc a;
  a.T = 1.0f; a.acc = a.dsum = a.n0 = a.n1 = a.n2 = 0.f;
  a.best = -INFINITY; a.best_mid = 0.f; a.best_i = 0;
  a.c_r = a.c_g = a.c_b = 0.f;

  // ---- interior for the whole ray?  first / last sample coordinates, computed exactly like the loop computes them
  const float bm_first = 0.5f * G.step, bm_last = 1.0f - 0.5f * G.step;     // (s + 1/2) / S is exact for power-of-two S
  const float m_first = fmaf(bm_first, G.span, tn), m_last = fmaf(bm_last, G.span, tn);
  bool inside = true;
  {
    const float g0[3] = {G.gh0, G.gw0, G.gd0}, gd[3] = {G.gdh, G.gdw, G.gdd};
    const int top[3] = {V.H - 2, V.W - 2, V.Z - 2};
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      float fa = floorf(fmaf(gd[k], m_first, g0[k])), fb = floorf(fmaf(gd[k], m_last, g0[k]));
      inside = inside && fminf(fa, fb) >= 0.f && fmaxf(fa, fb) <= (float)top[k];
    }
  }
  float* dbg_ray = DBG ? dbg_grid + lid * (long long)S * 3 : nullptr;

  if (!__all_sync(kFull, inside)) {
    march_padded<RGB>(V, G, S, P.sh_act, valid ? dbg_ray : nullptr, a);
  } else {
    const unsigned zp = ZP ? ZP : (RGB ? V.Z : V.zpitch), wz = WZ ? WZ : V.W * zp;
    // Address of the cell's (h0, w0, z0) corner.  With compile-time pitches the element index goes through fp32: every
    // partial sum is an integer below 2^24 (the launcher checks H * W * Z <= 2^23), so both FFMAs are exact and the float's
    // bits are 0x4B000000 + index.  Otherwise the index is formed on the integer
    // pipe from the magic-added floors (kcorr removes their 0x4B000000s, modulo 2^32).
    const unsigned kIdx0 = ZP ? kMagicBits : 0u;
    const unsigned kcorr = 0u - kMagicBits * (wz + zp + 1u);
    // The last cell's corners (and the differences that depend on the cell only) stay in registers: a lane reloads
    // when its cell changes, the warp branches over the reload when no lane's cell did.  `cell` starts at a key no
    // cell has (0x4B000000 + index < 0x4C000000 on the fp32 path; the pack holds fewer than 2^32 - 1 elements).
    constexpr bool kCache = (RGB ? SO_RF_CELL_CACHE_RGB : SO_RF_CELL_CACHE) != 0;
    unsigned cell = 0xffffffffu;
    float4 k[8];                         // RGB: corners {r, g, b, sdf}, order (h, w, z) = 000 001 010 011 100 101 110 111
    float dz[4] = {}, ddz0 = 0.f, ddz1 = 0.f;   // RGB: sdf differences along z per (h, w) column, and their w-differences
    float2 a00, a10, e0, e1, ee;         // depth-only: z-pairs at (h0, w0) / (h1, w0), their w-differences, e1 - e0
#pragma unroll
    for (int i = 0; i < 8; ++i) k[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    a00 = a10 = e0 = e1 = ee = make_float2(0.f, 0.f);
    float bm = bm_first;
    constexpr int kUnroll = SO_RF_UNROLL;
#pragma unroll kUnroll
    for (int s = 0; s < S; ++s) {
      const float mid = fmaf(bm, G.span, tn);
      bm += G.step;
      const float gh = fmaf(G.gdh, mid, G.gh0), gw = fmaf(G.gdw, mid, G.gw0), gd = fmaf(G.gdd, mid, G.gd0);
      if (DBG) { dbg_ray[3 * s] = gh; dbg_ray[3 * s + 1] = gw; dbg_ray[3 * s + 2] = gd; }
      const float flh = floorf(gh), flw = floorf(gw), flz = floorf(gd);
      const float fh = gh - flh, fw = gw - flw, fz = gd - flz;
      const float rz = flz + kMagic;
      unsigned idx;
      if (ZP) idx = __float_as_uint(fmaf(flh, (float)WZ, fmaf(flw, (float)ZP, rz)));
      else idx = __float_as_uint(flh + kMagic) * wz + (__float_as_uint(flw + kMagic) * zp + (__float_as_uint(rz) + kcorr));
      if (!kCache || __any_sync(kFull, idx != cell)) {
        if (!kCache || idx != cell) {
          cell = idx;
          if (!RGB) {
            const float2* p = reinterpret_cast<const float2*>(pack) + (idx - kIdx0);
            a00 = __ldg(p); a10 = __ldg(p + wz);
            const float2 a01 = __ldg(p + zp), a11 = __ldg(p + wz + zp);
            e0 = make_float2(a01.x - a00.x, a01.y - a00.y);
            e1 = make_float2(a11.x - a10.x, a11.y - a10.y);
            ee = make_float2(e1.x - e0.x, e1.y - e0.y);
          } else {
            const float4* p = reinterpret_cast<const float4*>(pack) + (idx - kIdx0);
            k[0] = __ldg(p); k[1] = __ldg(p + 1); k[2] = __ldg(p + zp); k[3] = __ldg(p + zp + 1);
            k[4] = __ldg(p + wz); k[5] = __ldg(p + wz + 1); k[6] = __ldg(p + wz + zp); k[7] = __ldg(p + wz + zp + 1);
#pragma unroll
            for (int j = 0; j < 4; ++j) dz[j] = k[2 * j + 1].w - k[2 * j].w;
            ddz0 = dz[1] - dz[0]; ddz1 = dz[3] - dz[2];
          }
        }
      }
      float sdf, dgh, dgw, dgd;
      if (!RGB) {
        // lanes = (z0, z1): lerp along w, then h, both lanes; z last
        const float2 c0 = make_float2(fmaf(fw, e0.x, a00.x), fmaf(fw, e0.y, a00.y));
        const float2 c1 = make_float2(fmaf(fw, e1.x, a10.x), fmaf(fw, e1.y, a10.y));
        const float2 dh = make_float2(c1.x - c0.x, c1.y - c0.y);
        const float c_x = fmaf(fh, dh.x, c0.x), c_y = fmaf(fh, dh.y, c0.y);
        const float e_x = fmaf(fh, ee.x, e0.x), e_y = fmaf(fh, ee.y, e0.y);
        dgd = c_y - c_x;
        sdf = fmaf(fz, dgd, c_x);
        dgh = fmaf(fz, dh.y - dh.x, dh.x);
        dgw = fmaf(fz, e_y - e_x, e_x);
      } else {
        // sdf: lerp along z, w, h; the gradient from the lerp differences
        const float c00 = fmaf(fz, dz[0], k[0].w), c01 = fmaf(fz, dz[1], k[2].w);
        const float c10 = fmaf(fz, dz[2], k[4].w), c11 = fmaf(fz, dz[3], k[6].w);
        const float dw0 = c01 - c00, dw1 = c11 - c10;
        const float u0 = fmaf(fw, dw0, c00), u1 = fmaf(fw, dw1, c10);
        dgh = u1 - u0;
        sdf = fmaf(fh, dgh, u0);
        dgw = fmaf(fh, dw1 - dw0, dw0);
        const float dzw0 = fmaf(fw, ddz0, dz[0]), dzw1 = fmaf(fw, ddz1, dz[2]);
        dgd = fmaf(fh, dzw1 - dzw0, dzw0);
      }
      const float tc = fmaf(G.gdh, dgh, fmaf(G.gdw, dgw, G.gdd * dgd));     // direction . d sdf / d metre
      const float alpha = neus_alpha_rcp1<true>(sdf * G.k_log2, fminf(tc, 0.f) * G.h_const);
      float w;
      composite(a, alpha, mid, dgw * G.kw, dgh * G.kh, dgd * G.kd, s, w);
      if (RGB) {
        // colour: one set of 8 trilinear weights for r, g, b (value only).  SH degree 0 with relu (sh_render.py:84-94):
        // the pack holds C0 f + 0.5 and the weights sum to one, so only the relu is left; the launcher routes
        // sh_act != 0 to the general kernel
        const float oh = 1.0f - fh, ow = 1.0f - fw, oz = 1.0f - fz;
        const float m00 = oh * ow, m01 = oh * fw, m10 = fh * ow, m11 = fh * fw;
        const float wt[8] = {m00 * oz, m00 * fz, m01 * oz, m01 * fz, m10 * oz, m10 * fz, m11 * oz, m11 * fz};
        float r0 = wt[0] * k[0].x, r1 = wt[0] * k[0].y, r2 = wt[0] * k[0].z;
#pragma unroll
        for (int j = 1; j < 8; ++j) { r0 = fmaf(wt[j], k[j].x, r0); r1 = fmaf(wt[j], k[j].y, r1); r2 = fmaf(wt[j], k[j].z, r2); }
        a.c_r = fmaf(w, fmaxf(r0, 0.f), a.c_r); a.c_g = fmaf(w, fmaxf(r1, 0.f), a.c_g); a.c_b = fmaf(w, fmaxf(r2, 0.f), a.c_b);
      }
      if (!DBG && (s & (SO_RF_EXIT_EVERY - 1)) == SO_RF_EXIT_EVERY - 1 && __all_sync(kFull, a.T < SO_RF_EXIT_T)) break;
    }
  }
  if (!valid) return;
  const float eps_len = 1.1920928955078125e-07f * nrm;   // torch.finfo(float32).eps * |dir| (neus_head.py:431)
  if (delta_c < eps_len) a.best_i = 0;                   // every candidate is 0: first index
  a.best_mid = fmaf(((float)a.best_i + 0.5f) * G.step, G.span, tn);   // (i + 1/2) / S is exact: the loop's mid_i bit for bit

  float lo, hi;
  depth_clip_range(ws, R, gid, lo, hi);
  if (depth) depth[lid] = clipped_depth(a.dsum, a.acc, lo, hi, nrm);
  if (max_depth) max_depth[lid] = a.best_mid / nrm;
  if (max_idx) max_idx[lid] = a.best_i;
  if (acc_out) acc_out[lid] = a.acc;
  if (normal_vis) {
    normal_vis[3 * lid + 0] = (a.n0 + 1.0f) * 0.5f;
    normal_vis[3 * lid + 1] = (a.n1 + 1.0f) * 0.5f;
    normal_vis[3 * lid + 2] = (a.n2 + 1.0f) * 0.5f;
  }
  if (RGB && rgb_out) store_rgb(P, bkgd_rand, lid, a.acc, a.c_r, a.c_g, a.c_b, rgb_out);
}

// ---- repack of the decoded volume: once per frame for inference (so_render_pack), per launch for the training forward
__global__ void __launch_bounds__(256) zpair_pack_kernel(const float* __restrict__ v, float2* __restrict__ out, long long n, int zp) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int z = (int)(i % zp);
  out[i] = make_float2(v[i], z + 1 < zp ? v[i + 1] : 0.f);       // the volume's z pad is already zero (so_tpv_decode)
}

void launch_zpair_pack(const float* vol_sdf, const so_volume_desc& d, float* pack, cudaStream_t st) {
  const long long n = (long long)d.H * d.W * d.zpitch;
  zpair_pack_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(vol_sdf, reinterpret_cast<float2*>(pack), n, d.zpitch);
}

__global__ void __launch_bounds__(256) pack_rgbs_kernel(const float* __restrict__ sdf, const float* __restrict__ feat,
                                                        float4* __restrict__ out, long long n, int Z, int zp, int fp) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long col = i / Z;
  int z = (int)(i - col * Z);
  const float* f = feat + i * fp;
  // the SH-0 colour map C0 f + 0.5 is affine and trilinear weights sum to one, so it is applied here once per voxel
  // instead of once per sample; render_packed_kernel only applies the relu
  out[i] = make_float4(fmaf(f[0], kC0, 0.5f), fmaf(f[1], kC0, 0.5f), fmaf(f[2], kC0, 0.5f), sdf[col * zp + z]);
}

}  // namespace so

using namespace so;

extern "C" int64_t so_render_pack_floats(const so_volume_desc* d) {
  if (!d || validate_volume(d)) return 0;
  if (d->n_feat == 0) return zpair_floats(*d);
  if (d->n_feat == 3) return 4 * (int64_t)d->H * d->W * d->Z;
  return 0;
}

extern "C" int so_render_pack(const float* vol_sdf, const float* vol_feat, const so_volume_desc* d, float* pack, void* stream) {
  if (!vol_sdf || !pack) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(d);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->n_feat == 0) {
    launch_zpair_pack(vol_sdf, *d, pack, st);
  } else if (d->n_feat == 3) {
    if (!vol_feat) return SO_ERR_INVALID_ARG;
    long long n = (long long)d->H * d->W * d->Z;
    if (n * 4 >= ((long long)1 << 32)) return SO_ERR_UNSUPPORTED;      // 32-bit element offsets in the gather
    pack_rgbs_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(vol_sdf, vol_feat, reinterpret_cast<float4*>(pack), n, d->Z,
                                                                     d->zpitch, d->feat_pitch);
  } else {
    return SO_ERR_UNSUPPORTED;
  }
  note_launch(1);
  return check_launch();
}

extern "C" int so_render_infer_packed(const float* vol_sdf, const float* vol_feat, const so_volume_desc* vol_host, const float* pack,
                                      const float* cam_mats, const float* pix, const so_ray_desc* rd,
                                      const so_render_params* pr, const float* bkgd_rand, float* depth, float* max_depth,
                                      int64_t* max_idx, float* acc, float* normal_vis, float* rgb, float* sem,
                                      float* workspace, float* dbg_grid, void* stream) {
  int rc = check_render_operands(vol_sdf, workspace, cam_mats, rd, pr, vol_host);
  if (rc) return rc;
  VolumeDev V = make_volume(*vol_host, vol_sdf, vol_feat);
  RenderDev P = make_render_dev(*pr, nullptr);
  const bool want_rgb = rgb != nullptr;
  const bool shape_ok = (vol_host->n_feat == 0 && !want_rgb) || (vol_host->n_feat == 3 && (!want_rgb || pr->sh_act == 0));
  if (!pack || !uniform_affine_march(V, P) || P.S < 2 || !shape_ok || sem) {
    if (dbg_grid) return SO_ERR_UNSUPPORTED;         // the sample-coordinate probe exists on the packed kernels only
    return so_render_infer(vol_sdf, vol_feat, vol_host, cam_mats, pix, rd, pr, bkgd_rand, depth, max_depth, max_idx, acc,
                           normal_vis, rgb, sem, workspace, stream);
  }
  if ((rc = check_background(pr, want_rgb, bkgd_rand))) return rc;
  RayDev R;
  if ((rc = make_ray_dev(rd, cam_mats, pix, &R))) return rc;
  if (rd->ray_count == 0) return SO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if ((rc = launch_depth_bounds(R, P, workspace, st))) return rc;

  const unsigned grid = (unsigned)ceil_div64(rd->ray_count, SO_RF_BLOCK);
  ProfScope prof(0, st);
  long long* midx = reinterpret_cast<long long*>(max_idx);
  const bool rgbs = vol_host->n_feat == 3;
  // the nuScenes depth volume: constant pitches; its element index fits the exact fp32 index path (<= 2^23 elements)
  const bool nus = V.W == 257 && (rgbs ? V.Z == 31 : V.zpitch == 32) && (long long)V.H * V.W * (rgbs ? V.Z : V.zpitch) <= (1 << 23);
#define SO_RP(RGB, DBG, ZP, WZ) render_packed_kernel<RGB, DBG, ZP, WZ><<<grid, SO_RF_BLOCK, 0, st>>>( \
    V, pack, R, P, workspace, bkgd_rand, depth, max_depth, midx, acc, normal_vis, rgb, dbg_grid)
  if (dbg_grid) { if (rgbs) SO_RP(true, true, 0, 0); else SO_RP(false, true, 0, 0); }
  else if (rgbs) { if (nus) SO_RP(true, false, 31, 257 * 31); else SO_RP(true, false, 0, 0); }
  else { if (nus) SO_RP(false, false, 32, 257 * 32); else SO_RP(false, false, 0, 0); }
#undef SO_RP
  note_launch(1);
  return check_launch();
}
