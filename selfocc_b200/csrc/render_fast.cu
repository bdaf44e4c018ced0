// Packed-volume inference render (SURVEY.md section 8a rows B1-B4, B6-B11): the second-generation kernels behind
// so_render_infer_packed.  Same contract and the same per-ray recurrence as render_infer_kernel (render.cu); what changes
// is how a sample is fetched and how many instructions it costs:
//
//  * the decoded volume is first repacked once per frame (so_render_pack) into the layout the gather wants:
//      n_feat == 0 : float2 [H][W][zpitch]  {sdf[z], sdf[z+1]}     -> the 8 trilinear taps are 4 aligned 64-bit loads
//      n_feat == 3 : float4 [H][W][Z]       {r, g, b, sdf}          -> 8 aligned 128-bit loads fetch sdf AND colour
//    (the reference gathers 8 + 24 scalars per sample for colour, bev_nerf.py:99-117);
//  * the trilinear interpolation works on register pairs: the two lanes of a loaded pair are lerped together, the sdf
//    gradient falls out of the lerp differences;
//  * "all 8 corners inside the volume" is decided ONCE per ray: for the affine metre->grid map g(t) = g0 + gd * t is
//    monotone along the ray (so is its fp32 evaluation fma(gd, t, g0)), so if the first and the last sample are interior,
//    every sample is; warps with a non-interior ray take the general zero-padding loop;
//  * NeuS alpha with ONE reciprocal:  alpha = (omen + c (1 + B)) / ((1 + B) (1 + c)),  A = e^-(s-h), B = e^(s+h),
//    c = 1e-5 (1 + A)  (algebraically equal to (Phi(prev) - Phi(next) + 1e-5) / (Phi(prev) + 1e-5), no cancellation);
//  * cell indices come from the float floor through the 2^23 magic add (integer pipe) instead of F2I (XU pipe);
//  * a warp stops marching once every ray's transmittance is below 1e-9: the dropped tail changes acc / depth / rgb by
//    < 1e-9 relative and cannot hold the max-depth argmax (a later w is <= T < 1e-9 <= max_s w_s since sum_s w_s >= 1 - T).
#include "render_common.cuh"

// Tuning knobs, timed on an H100 SXM (400 W) with scripts/bench_render.py, analytic scene, 8.64 M rays, depth-only / colour
// ms: defaults (unroll 4; 6 / 4 CTAs per SM) 6.93-7.18 / 12.06-12.12 over two runs; unroll 1 7.27 / 12.08, unroll 2
// 7.04 / 12.18; 4 / 3 CTAs 6.98 / 12.14; 8 / 5 CTAs 6.92 / 12.12.  No alternative beats the run-to-run spread.
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

__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 bc2(float a) { return make_float2(a, a); }
// two-lane helpers: one rounded fmaf / add per lane (sm_90 has no packed fp32x2 pipe; the results are the same)
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 sub2(float2 a, float2 b) { return fma2(b, make_float2(-1.f, -1.f), a); }   // a - b, exact
__device__ __forceinline__ float2 lerp2(float2 t, float2 d, float2 a) { return fma2(t, d, a); }               // a + t * d

// NeuS alpha, one-reciprocal form (see the file header).  s2 = sdf * inv_s * log2(e), h2 = half * inv_s * log2(e) <= 0.
// The exponents are clamped at 64: beyond that alpha is 1 (A huge) or the 1e-5 floor (B huge) to within 2^-40.
__device__ __forceinline__ float neus_alpha_rcp1(float s2, float h2) {
  float A = exp2f(fminf(h2 - s2, 64.f));
  float B = exp2f(fminf(s2 + h2, 64.f));
  float pB = 1.0f + B;
  float c = fmaf(A, 1e-5f, 1e-5f);                               // 1e-5 (1 + A)
  float x = h2 * (-2.0f * 0.6931471805599453f);                  // (s - h) - (s + h) in natural units, >= 0
  float ser = x * fmaf(x, fmaf(x, fmaf(x, fmaf(x, 1.0f / 120.0f, -1.0f / 24.0f), 1.0f / 6.0f), -0.5f), 1.0f);
  float omen = x < 0.125f ? ser : 1.0f - exp2f(h2 + h2);         // 1 - e^-x
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
    float alpha = neus_alpha_rcp1(sdf * G.k_log2, fminf(tc, 0.f) * G.h_const);
    float w;
    composite(a, alpha, mid, dgw * G.kw, dgh * G.kh, dgd * G.kd, s, w);
    if (RGB) {
      float f[3];
      gather_feat<3>(V, t, 0, f);
      float r0 = f[0] * kC0, r1 = f[1] * kC0, r2 = f[2] * kC0;
      if (sh_act == 0) { r0 = fmaxf(r0 + 0.5f, 0.f); r1 = fmaxf(r1 + 0.5f, 0.f); r2 = fmaxf(r2 + 0.5f, 0.f); }
      else { r0 = sigmoidf_acc(r0); r1 = sigmoidf_acc(r1); r2 = sigmoidf_acc(r2); }
      a.c_r = fmaf(w, r0, a.c_r); a.c_g = fmaf(w, r1, a.c_g); a.c_b = fmaf(w, r2, a.c_b);
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
  G.gh0 = fmaf(o[1] - V.ax[0].start, G.kh, V.ax[0].offset); G.gdh = d[1] * G.kh;
  G.gw0 = fmaf(o[0] - V.ax[1].start, G.kw, V.ax[1].offset); G.gdw = d[0] * G.kw;
  G.gd0 = fmaf(o[2] - V.ax[2].start, G.kd, V.ax[2].offset); G.gdd = d[2] * G.kd;
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
    const float2 span2 = bc2(G.span), tn2 = bc2(tn), step2 = bc2(G.step);
    const float2 gdhw = f2(G.gdh, G.gdw), ghw0 = f2(G.gh0, G.gw0), magic2 = bc2(kMagic);
    float2 bm2 = bc2(bm_first);
    const unsigned zp = ZP ? ZP : (RGB ? V.Z : V.zpitch), wz = WZ ? WZ : V.W * zp;
    const unsigned kcorr = 0u - kMagicBits * (wz + zp + 1u);
    constexpr int kUnroll = SO_RF_UNROLL;
#pragma unroll kUnroll
    for (int s = 0; s < S; ++s) {
      const float2 mid2 = fma2(bm2, span2, tn2);
      bm2 = add2(bm2, step2);
      const float mid = mid2.x;
      const float2 ghw = fma2(gdhw, mid2, ghw0);
      const float gd = fmaf(G.gdd, mid, G.gd0);
      if (DBG) { dbg_ray[3 * s] = ghw.x; dbg_ray[3 * s + 1] = ghw.y; dbg_ray[3 * s + 2] = gd; }
      const float flh = floorf(ghw.x), flw = floorf(ghw.y), flz = floorf(gd);
      const float2 fhw = sub2(ghw, f2(flh, flw));
      const float fz = gd - flz;
      const float2 rhw = add2(f2(flh, flw), magic2);
      const float rz = flz + kMagic;
      const unsigned idx = __float_as_uint(rhw.x) * wz + (__float_as_uint(rhw.y) * zp + (__float_as_uint(rz) + kcorr));
      const float2 fh2 = bc2(fhw.x), fw2 = bc2(fhw.y);
      float sdf, dgh, dgw, dgd;
      float2 rg;
      float bl;
      if (!RGB) {
        const float2* p = reinterpret_cast<const float2*>(pack) + idx;
        const float2 a00 = __ldg(p), a01 = __ldg(p + zp), a10 = __ldg(p + wz), a11 = __ldg(p + wz + zp);
        // lanes = (z0, z1): lerp along w, then h, with both lanes at once; z last
        const float2 e0 = sub2(a01, a00), e1 = sub2(a11, a10);
        const float2 c0 = lerp2(fw2, e0, a00), c1 = lerp2(fw2, e1, a10);
        const float2 dh = sub2(c1, c0);
        const float2 c = lerp2(fh2, dh, c0);
        const float2 e = lerp2(fh2, sub2(e1, e0), e0);
        dgd = c.y - c.x;
        sdf = fmaf(fz, dgd, c.x);
        dgh = fmaf(fz, dh.y - dh.x, dh.x);
        dgw = fmaf(fz, e.y - e.x, e.x);
      } else {
        const float4* p = reinterpret_cast<const float4*>(pack) + idx;
        const float4 q000 = __ldg(p), q001 = __ldg(p + 1), q010 = __ldg(p + zp), q011 = __ldg(p + zp + 1);
        const float4 q100 = __ldg(p + wz), q101 = __ldg(p + wz + 1), q110 = __ldg(p + wz + zp), q111 = __ldg(p + wz + zp + 1);
        const float2 fz2 = bc2(fz);
        // lanes lo = (r, g), hi = (b, sdf): lerp along z, w, h
#define SO_LO(q) f2((q).x, (q).y)
#define SO_HI(q) f2((q).z, (q).w)
        const float2 dz00l = sub2(SO_LO(q001), SO_LO(q000)), dz00h = sub2(SO_HI(q001), SO_HI(q000));
        const float2 dz01l = sub2(SO_LO(q011), SO_LO(q010)), dz01h = sub2(SO_HI(q011), SO_HI(q010));
        const float2 dz10l = sub2(SO_LO(q101), SO_LO(q100)), dz10h = sub2(SO_HI(q101), SO_HI(q100));
        const float2 dz11l = sub2(SO_LO(q111), SO_LO(q110)), dz11h = sub2(SO_HI(q111), SO_HI(q110));
        const float2 t00l = lerp2(fz2, dz00l, SO_LO(q000)), t00h = lerp2(fz2, dz00h, SO_HI(q000));
        const float2 t01l = lerp2(fz2, dz01l, SO_LO(q010)), t01h = lerp2(fz2, dz01h, SO_HI(q010));
        const float2 t10l = lerp2(fz2, dz10l, SO_LO(q100)), t10h = lerp2(fz2, dz10h, SO_HI(q100));
        const float2 t11l = lerp2(fz2, dz11l, SO_LO(q110)), t11h = lerp2(fz2, dz11h, SO_HI(q110));
#undef SO_LO
#undef SO_HI
        const float2 dw0l = sub2(t01l, t00l), dw0h = sub2(t01h, t00h), dw1l = sub2(t11l, t10l), dw1h = sub2(t11h, t10h);
        const float2 u0l = lerp2(fw2, dw0l, t00l), u0h = lerp2(fw2, dw0h, t00h);
        const float2 u1l = lerp2(fw2, dw1l, t10l), u1h = lerp2(fw2, dw1h, t10h);
        const float2 dhl = sub2(u1l, u0l), dhh = sub2(u1h, u0h);
        const float2 vl = lerp2(fh2, dhl, u0l), vh = lerp2(fh2, dhh, u0h);
        rg = vl; bl = vh.x; sdf = vh.y;
        dgh = dhh.y;
        dgw = fmaf(fhw.x, dw1h.y - dw0h.y, dw0h.y);
        const float dzw0 = fmaf(fhw.y, dz01h.y - dz00h.y, dz00h.y), dzw1 = fmaf(fhw.y, dz11h.y - dz10h.y, dz10h.y);
        dgd = fmaf(fhw.x, dzw1 - dzw0, dzw0);
      }
      const float tc = fmaf(G.gdh, dgh, fmaf(G.gdw, dgw, G.gdd * dgd));     // direction . d sdf / d metre
      const float alpha = neus_alpha_rcp1(sdf * G.k_log2, fminf(tc, 0.f) * G.h_const);
      float w;
      composite(a, alpha, mid, dgw * G.kw, dgh * G.kh, dgd * G.kd, s, w);
      if (RGB) {
        // SH degree 0, relu activation (sh_render.py:84-94); the launcher routes sh_act != 0 to the general kernel
        const float2 c2 = fma2(rg, bc2(kC0), bc2(0.5f));
        const float r0 = fmaxf(c2.x, 0.f), r1 = fmaxf(c2.y, 0.f), r2 = fmaxf(fmaf(bl, kC0, 0.5f), 0.f);
        a.c_r = fmaf(w, r0, a.c_r); a.c_g = fmaf(w, r1, a.c_g); a.c_b = fmaf(w, r2, a.c_b);
      }
      if (!DBG && (s & (SO_RF_EXIT_EVERY - 1)) == SO_RF_EXIT_EVERY - 1 && __all_sync(kFull, a.T < SO_RF_EXIT_T)) break;
    }
  }
  if (!valid) return;
  const float eps_len = 1.1920928955078125e-07f * nrm;   // torch.finfo(float32).eps * |dir| (neus_head.py:431)
  if (delta_c < eps_len) a.best_i = 0;                   // every candidate is 0: first index
  a.best_mid = fmaf(((float)a.best_i + 0.5f) * G.step, G.span, tn);   // (i + 1/2) / S is exact: the loop's mid_i bit for bit

  const long long chunk = R.chunk_len > 0 ? gid / R.chunk_len : 0;
  const float lo = __ldg(ws + 2 * chunk), hi = __ldg(ws + 2 * chunk + 1);
  if (depth) {
    float dd = a.dsum / (a.acc + 1e-10f);
    dd = fminf(fmaxf(dd, lo), hi);
    depth[lid] = dd / nrm;
  }
  if (max_depth) max_depth[lid] = a.best_mid / nrm;
  if (max_idx) max_idx[lid] = a.best_i;
  if (acc_out) acc_out[lid] = a.acc;
  if (normal_vis) {
    normal_vis[3 * lid + 0] = (a.n0 + 1.0f) * 0.5f;
    normal_vis[3 * lid + 1] = (a.n1 + 1.0f) * 0.5f;
    normal_vis[3 * lid + 2] = (a.n2 + 1.0f) * 0.5f;
  }
  if (RGB && rgb_out) {
    float b0, b1, b2;
    if (P.bkgd_mode == 2) { b0 = bkgd_rand[3 * lid]; b1 = bkgd_rand[3 * lid + 1]; b2 = bkgd_rand[3 * lid + 2]; }
    else { b0 = b1 = b2 = (P.bkgd_mode == 1) ? 1.f : 0.f; }
    const float rem = 1.0f - a.acc;
    float r = fmaf(b0, rem, a.c_r), g = fmaf(b1, rem, a.c_g), b = fmaf(b2, rem, a.c_b);
    if (P.eval_clamp) { r = fminf(fmaxf(r, 0.f), 1.f); g = fminf(fmaxf(g, 0.f), 1.f); b = fminf(fmaxf(b, 0.f), 1.f); }
    rgb_out[3 * lid] = r; rgb_out[3 * lid + 1] = g; rgb_out[3 * lid + 2] = b;
  }
}

// ---- once-per-frame repack of the decoded volume -------------------------------------------------------
__global__ void __launch_bounds__(256) pack_pair_kernel(const float* __restrict__ v, float2* __restrict__ out, long long n, int zp) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int z = (int)(i % zp);
  out[i] = make_float2(v[i], z + 1 < zp ? v[i + 1] : 0.f);       // the volume's z pad is already zero (so_tpv_decode)
}

__global__ void __launch_bounds__(256) pack_rgbs_kernel(const float* __restrict__ sdf, const float* __restrict__ feat,
                                                        float4* __restrict__ out, long long n, int Z, int zp, int fp) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long col = i / Z;
  int z = (int)(i - col * Z);
  const float* f = feat + i * fp;
  out[i] = make_float4(f[0], f[1], f[2], sdf[col * zp + z]);
}

}  // namespace so

using namespace so;

extern "C" int64_t so_render_pack_floats(const so_volume_desc* d) {
  if (!d || validate_volume(d)) return 0;
  if (d->n_feat == 0) return 2 * (int64_t)d->H * d->W * d->zpitch;
  if (d->n_feat == 3) return 4 * (int64_t)d->H * d->W * d->Z;
  return 0;
}

extern "C" int so_render_pack(const float* vol_sdf, const float* vol_feat, const so_volume_desc* d, float* pack, void* stream) {
  if (!vol_sdf || !pack) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(d);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->n_feat == 0) {
    long long n = (long long)d->H * d->W * d->zpitch;
    pack_pair_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(vol_sdf, reinterpret_cast<float2*>(pack), n, d->zpitch);
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
  if (!vol_sdf || !cam_mats || !rd || !pr || !workspace) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(vol_host);
  if (rc) return rc;
  VolumeDev V = make_volume(*vol_host, vol_sdf, vol_feat);
  const bool fast = V.ax[0].k1 == 0.f && V.ax[1].k1 == 0.f && V.ax[2].k1 == 0.f && pr->num_samples >= 2 &&
                    (pr->num_samples & (pr->num_samples - 1)) == 0 && pr->cos_anneal == 1.0f && pr->anchor_mid;
  const bool want_rgb = rgb != nullptr;
  const bool shape_ok = (vol_host->n_feat == 0 && !want_rgb) || (vol_host->n_feat == 3 && (!want_rgb || pr->sh_act == 0));
  if (!pack || !fast || !shape_ok || sem) {
    if (dbg_grid) return SO_ERR_UNSUPPORTED;         // the sample-coordinate probe exists on the packed kernels only
    return so_render_infer(vol_sdf, vol_feat, vol_host, cam_mats, pix, rd, pr, bkgd_rand, depth, max_depth, max_idx, acc,
                           normal_vis, rgb, sem, workspace, stream);
  }
  if (rd->n_cam < 1 || rd->rays_per_cam < 1) return SO_ERR_INVALID_ARG;
  if (pr->bkgd_mode == 2 && want_rgb && !bkgd_rand) return SO_ERR_INVALID_ARG;
  if (pr->bkgd_mode < 0 || pr->bkgd_mode > 2 || pr->sh_act < 0 || pr->sh_act > 1) return SO_ERR_INVALID_ARG;
  RayDev R;
  if ((rc = make_ray_dev(rd, cam_mats, pix, &R))) return rc;
  if (rd->ray_count == 0) return SO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  RenderDev P = make_render_dev(*pr, nullptr);
  if ((rc = launch_depth_bounds(R, P, workspace, st))) return rc;

  const unsigned grid = (unsigned)ceil_div64(rd->ray_count, SO_RF_BLOCK);
  ProfScope prof(0, st);
  long long* midx = reinterpret_cast<long long*>(max_idx);
  const bool rgbs = vol_host->n_feat == 3;
  const bool nus = V.W == 257 && (rgbs ? V.Z == 31 : V.zpitch == 32);     // the nuScenes depth volume: constant pitches
#define SO_RP(RGB, DBG, ZP, WZ) render_packed_kernel<RGB, DBG, ZP, WZ><<<grid, SO_RF_BLOCK, 0, st>>>( \
    V, pack, R, P, workspace, bkgd_rand, depth, max_depth, midx, acc, normal_vis, rgb, dbg_grid)
  if (dbg_grid) { if (rgbs) SO_RP(true, true, 0, 0); else SO_RP(false, true, 0, 0); }
  else if (rgbs) { if (nus) SO_RP(true, false, 31, 257 * 31); else SO_RP(true, false, 0, 0); }
  else { if (nus) SO_RP(false, false, 32, 257 * 32); else SO_RP(false, false, 0, 0); }
#undef SO_RP
  note_launch(1);
  return check_launch();
}
