// Image -> tri-plane lifting kernels (SURVEY.md section 8a rows A4-A8).
//
// Thread mapping of every sampling kernel: one "item" = one (query, head); DH/4 lanes own an item and
// each lane owns 4 consecutive channels (one float4) of the head, so a bilinear corner is one coalesced
// 64-byte (DH=16) read per item and the (query, head*DH) output row is written as float4, 512 B per warp.
// Value tensors are 30-65 MB fp32, i.e. largely L2-resident on H100 (50 MB): these kernels are L2/L1-gather
// bound, not HBM bound.
#include "common.cuh"
#include <math.h>
// Tuning knobs, timed on an H100 SXM (700 W) over the bench frame with `bench.py`'s per-kernel breakdown, ms per step.
// Cross-attention: 4.63-4.66 at the defaults (two runs); unroll 2 / 8: 4.65 / 4.63; 4 / 6 CTAs per SM: 4.66 / 4.63.
// Self-attention: 1.66-1.67 at the defaults; unroll 4: 1.66; 3 / 5 CTAs per SM: 1.67 / 1.67.  Every alternative is
// within the run-to-run spread, so the defaults stay.
#ifndef SO_ATTN_UNROLL
#define SO_ATTN_UNROLL 4
#endif
#ifndef SO_SELF_ATTN_MIN_CTAS
#define SO_SELF_ATTN_MIN_CTAS 4
#endif
#ifndef SO_SELF_ATTN_UNROLL
#define SO_SELF_ATTN_UNROLL 8
#endif
#ifndef SO_ATTN_MIN_CTAS
#define SO_ATTN_MIN_CTAS 5
#endif

namespace so {

constexpr int kMaxLevels = 8;

struct Levels {
  int n;
  int h[kMaxLevels], w[kMaxLevels];
  long long start[kMaxLevels];
};

__device__ __forceinline__ void load_levels(Levels& lv, const long long* __restrict__ shapes,
                                            const long long* __restrict__ lsi, int L) {
  // spatial_shapes / level_start_index are device int64 tensors (the mmcv op contract); every CTA
  // copies the <= 8 entries into shared memory once.
  if (threadIdx.x < L) {
    lv.h[threadIdx.x] = (int)shapes[2 * threadIdx.x];
    lv.w[threadIdx.x] = (int)shapes[2 * threadIdx.x + 1];
    lv.start[threadIdx.x] = lsi[threadIdx.x];
  }
  if (threadIdx.x == 0) lv.n = L;
  __syncthreads();
}

// bilinear read of 4 channels at normalised location (lx, ly) of level (Hl, Wl); align_corners=False,
// zero padding (mmcv ms_deform_attn / F.grid_sample semantics).  vbase points at channel 0 of this lane
// in pixel 0 of the level; pstride = floats between consecutive pixels.
__device__ __forceinline__ float4 bilinear4(const float* __restrict__ vbase, int pstride, int Hl, int Wl, float lx, float ly) {
  float x = lx * (float)Wl - 0.5f, y = ly * (float)Hl - 0.5f;
  float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
  if (!(y > -1.f && x > -1.f && y < (float)Hl && x < (float)Wl)) return r;
  float xf = floorf(x), yf = floorf(y);
  int x0 = (int)xf, y0 = (int)yf;
  float fx = x - xf, fy = y - yf;
  float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
  bool xa = x0 >= 0, xb = x0 + 1 < Wl, ya = y0 >= 0, yb = y0 + 1 < Hl;
  const float* p = vbase + ((long long)y0 * Wl + x0) * pstride;
  float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 v00 = (ya && xa) ? __ldg(reinterpret_cast<const float4*>(p)) : z;
  float4 v01 = (ya && xb) ? __ldg(reinterpret_cast<const float4*>(p + pstride)) : z;
  float4 v10 = (yb && xa) ? __ldg(reinterpret_cast<const float4*>(p + (long long)Wl * pstride)) : z;
  float4 v11 = (yb && xb) ? __ldg(reinterpret_cast<const float4*>(p + (long long)(Wl + 1) * pstride)) : z;
  r.x = w00 * v00.x + w01 * v01.x + w10 * v10.x + w11 * v11.x;
  r.y = w00 * v00.y + w01 * v01.y + w10 * v10.y + w11 * v11.y;
  r.z = w00 * v00.z + w01 * v01.z + w10 * v10.z + w11 * v11.z;
  r.w = w00 * v00.w + w01 * v01.w + w10 * v10.w + w11 * v11.w;
  return r;
}

// ---- A7/A8 generic op (the mmcv contract) -------------------------------------------------------------
template <int DH>
__global__ void __launch_bounds__(256) msda_forward_kernel(const float* __restrict__ value, const long long* __restrict__ shapes, const long long* __restrict__ lsi,
                                                           const float* __restrict__ loc, const float* __restrict__ wts,
                                                           float* __restrict__ out, int B, int Nv, int Hd, int Nq, int L, int P) {
  constexpr int LPI = DH / 4;
  __shared__ Levels lv;
  load_levels(lv, shapes, lsi, L);
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long item = t / LPI;
  int lc = (int)(t % LPI);
  long long n_items = (long long)B * Nq * Hd;
  if (item >= n_items) return;
  int h = (int)(item % Hd);
  long long bq = item / Hd;
  int b = (int)(bq / Nq);
  const int pstride = Hd * DH;
  const float* lp = loc + item * (long long)L * P * 2;
  const float* wp = wts + item * (long long)L * P;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int l = 0; l < L; ++l) {
    const int Hl = lv.h[l], Wl = lv.w[l];
    const float* vbase = value + (((long long)b * Nv + lv.start[l]) * Hd + h) * DH + lc * 4;
#pragma unroll 4
    for (int p = 0; p < P; ++p) {
      float2 xy = __ldg(reinterpret_cast<const float2*>(lp) + l * P + p);
      float aw = __ldg(wp + l * P + p);
      float4 s = bilinear4(vbase, pstride, Hl, Wl, xy.x, xy.y);
      acc.x = fmaf(aw, s.x, acc.x); acc.y = fmaf(aw, s.y, acc.y);
      acc.z = fmaf(aw, s.z, acc.z); acc.w = fmaf(aw, s.w, acc.w);
    }
  }
  *reinterpret_cast<float4*>(out + item * DH + lc * 4) = acc;
}

// Backward of the generic op.  Same mapping; channel reductions for grad_loc / grad_weights run over the
// LPI lanes of an item with xor-shuffles; grad_value is accumulated with 128-bit vector atomics.
template <int DH>
__global__ void __launch_bounds__(256) msda_backward_kernel(const float* __restrict__ value, const long long* __restrict__ shapes, const long long* __restrict__ lsi,
                                                            const float* __restrict__ loc, const float* __restrict__ wts,
                                                            const float* __restrict__ gout, float* __restrict__ gvalue,
                                                            float* __restrict__ gloc, float* __restrict__ gw, int B, int Nv,
                                                            int Hd, int Nq, int L, int P) {
  constexpr int LPI = DH / 4;
  __shared__ Levels lv;
  load_levels(lv, shapes, lsi, L);
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long item = t / LPI;
  int lc = (int)(t % LPI);
  long long n_items = (long long)B * Nq * Hd;
  bool live = item < n_items;
  if (!live) item = n_items - 1;  // keep the warp converged for the shuffles
  int h = (int)(item % Hd);
  long long bq = item / Hd;
  int b = (int)(bq / Nq);
  const int pstride = Hd * DH;
  const float* lp = loc + item * (long long)L * P * 2;
  const float* wp = wts + item * (long long)L * P;
  float4 go = __ldg(reinterpret_cast<const float4*>(gout + item * DH + lc * 4));
  for (int l = 0; l < L; ++l) {
    const int Hl = lv.h[l], Wl = lv.w[l];
    const long long voff = (((long long)b * Nv + lv.start[l]) * Hd + h) * DH + lc * 4;
    for (int p = 0; p < P; ++p) {
      float2 xy = __ldg(reinterpret_cast<const float2*>(lp) + l * P + p);
      float aw = __ldg(wp + l * P + p);
      float x = xy.x * (float)Wl - 0.5f, y = xy.y * (float)Hl - 0.5f;
      float g_w = 0.f, g_x = 0.f, g_y = 0.f;
      if (y > -1.f && x > -1.f && y < (float)Hl && x < (float)Wl) {
        float xf = floorf(x), yf = floorf(y);
        int x0 = (int)xf, y0 = (int)yf;
        float fx = x - xf, fy = y - yf;
        bool xa = x0 >= 0, xb = x0 + 1 < Wl, ya = y0 >= 0, yb = y0 + 1 < Hl;
        long long o00 = voff + ((long long)y0 * Wl + x0) * pstride;
        long long o01 = o00 + pstride, o10 = o00 + (long long)Wl * pstride, o11 = o10 + pstride;
        float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        float4 v00 = (ya && xa) ? __ldg(reinterpret_cast<const float4*>(value + o00)) : z;
        float4 v01 = (ya && xb) ? __ldg(reinterpret_cast<const float4*>(value + o01)) : z;
        float4 v10 = (yb && xa) ? __ldg(reinterpret_cast<const float4*>(value + o10)) : z;
        float4 v11 = (yb && xb) ? __ldg(reinterpret_cast<const float4*>(value + o11)) : z;
        float w00 = (1.f - fy) * (1.f - fx), w01 = (1.f - fy) * fx, w10 = fy * (1.f - fx), w11 = fy * fx;
        // dot products with grad_out over this lane's 4 channels
        float d00 = go.x * v00.x + go.y * v00.y + go.z * v00.z + go.w * v00.w;
        float d01 = go.x * v01.x + go.y * v01.y + go.z * v01.z + go.w * v01.w;
        float d10 = go.x * v10.x + go.y * v10.y + go.z * v10.z + go.w * v10.w;
        float d11 = go.x * v11.x + go.y * v11.y + go.z * v11.z + go.w * v11.w;
        g_w = w00 * d00 + w01 * d01 + w10 * d10 + w11 * d11;
        g_x = aw * (float)Wl * ((1.f - fy) * (d01 - d00) + fy * (d11 - d10));
        g_y = aw * (float)Hl * ((1.f - fx) * (d10 - d00) + fx * (d11 - d01));
        if (live) {
          float4 g;
          if (ya && xa) { float s = aw * w00; g = make_float4(s * go.x, s * go.y, s * go.z, s * go.w); atomicAdd(reinterpret_cast<float4*>(gvalue + o00), g); }
          if (ya && xb) { float s = aw * w01; g = make_float4(s * go.x, s * go.y, s * go.z, s * go.w); atomicAdd(reinterpret_cast<float4*>(gvalue + o01), g); }
          if (yb && xa) { float s = aw * w10; g = make_float4(s * go.x, s * go.y, s * go.z, s * go.w); atomicAdd(reinterpret_cast<float4*>(gvalue + o10), g); }
          if (yb && xb) { float s = aw * w11; g = make_float4(s * go.x, s * go.y, s * go.z, s * go.w); atomicAdd(reinterpret_cast<float4*>(gvalue + o11), g); }
        }
      }
#pragma unroll
      for (int s = LPI / 2; s > 0; s >>= 1) {
        g_w += __shfl_xor_sync(0xffffffffu, g_w, s);
        g_x += __shfl_xor_sync(0xffffffffu, g_x, s);
        g_y += __shfl_xor_sync(0xffffffffu, g_y, s);
      }
      if (live && lc == 0) {
        long long o = item * (long long)L * P + l * P + p;
        gw[o] = g_w;
        gloc[2 * o] = g_x;
        gloc[2 * o + 1] = g_y;
      }
    }
  }
}

// ---- softmax statistics of one item's logits, computed cooperatively by its LPI lanes -------------------
template <int LPI>
__device__ __forceinline__ void softmax_stats(const float* __restrict__ lg, int n, int lc, float& mx, float& inv_sum) {
  float m = -INFINITY;
  for (int i = lc; i < n; i += LPI) m = fmaxf(m, __ldg(lg + i));
#pragma unroll
  for (int s = LPI / 2; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
  float sum = 0.f;
  for (int i = lc; i < n; i += LPI) sum += __expf(__ldg(lg + i) - m);
#pragma unroll
  for (int s = LPI / 2; s > 0; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
  mx = m;
  inv_sum = 1.0f / sum;
}

// ---- A5+A6+A7 fused, rebatch-free image cross-attention core --------------------------------------------
// SPLIT sample-groups share one (query, head): group g takes pillar points d = g, g + SPLIT, ...  Planes with long
// pillars (D = 48: only ~48 k items but 192 x cams samples each) would otherwise run as ~1 wave of long threads.
template <int DH, int SPLIT>
__global__ void __launch_bounds__(256, SO_ATTN_MIN_CTAS) tpv_cross_attn_kernel(const float* __restrict__ value, const long long* __restrict__ shapes,
                                                             const long long* __restrict__ lsi, const float* __restrict__ offsets,
                                                             const float* __restrict__ logits, const float* __restrict__ uv,
                                                             const unsigned char* __restrict__ vis, float* __restrict__ slots,
                                                             int* __restrict__ count, int N, int Nv, int Hd, int Q, int L, int D,
                                                             int value_ld, int off_ld, int lg_ld) {
  constexpr int LPI = DH / 4;
  constexpr int LANES = LPI * SPLIT;
  __shared__ Levels lv;
  load_levels(lv, shapes, lsi, L);
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long item = t / LANES;
  const int li = (int)(t % LANES);
  const int lc = li % LPI, sg = li / LPI;
  long long n_items = (long long)Q * Hd;
  bool live = item < n_items;
  if (!live) item = n_items - 1;
  int h = (int)(item % Hd);
  int q = (int)(item / Hd);
  const int pstride = value_ld;                       // floats between consecutive pixels of the value tensor
  const int LD = L * D;
  const float* op = offsets + (long long)q * off_ld + (long long)h * LD * 2;
  const float* lg = logits + (long long)q * lg_ld + (long long)h * LD;
  float mx, inv_sum;
  softmax_stats<LANES>(lg, LD, li, mx, inv_sum);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int cnt = 0;
  for (int cam = 0; cam < N; ++cam) {
    if (!__ldg(vis + (long long)cam * Q + q)) continue;  // image_cross_attention.py:92 (query visible in cam)
    ++cnt;
    const float* uvp = uv + ((long long)cam * Q + q) * D * 2;
    float4 part = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int l = 0; l < L; ++l) {
      const int Hl = lv.h[l], Wl = lv.w[l];
      const float rw = 1.0f / (float)Wl, rh = 1.0f / (float)Hl;
      const float* vbase = value + ((long long)cam * Nv + lv.start[l]) * value_ld + h * DH + lc * 4;
      constexpr int kUnroll = SO_ATTN_UNROLL;
#pragma unroll kUnroll
      for (int d = sg; d < D; d += SPLIT) {
        float2 r = __ldg(reinterpret_cast<const float2*>(uvp) + d);
        float2 o = __ldg(reinterpret_cast<const float2*>(op) + l * D + d);
        float aw = __expf(__ldg(lg + l * D + d) - mx) * inv_sum;
        // image_cross_attention.py:326-328: ref + offset / (w_l, h_l)   (reciprocal multiply: <= 1 ulp from the division)
        float4 s = bilinear4(vbase, pstride, Hl, Wl, fmaf(o.x, rw, r.x), fmaf(o.y, rh, r.y));
        part.x = fmaf(aw, s.x, part.x); part.y = fmaf(aw, s.y, part.y);
        part.z = fmaf(aw, s.z, part.z); part.w = fmaf(aw, s.w, part.w);
      }
    }
    acc.x += part.x; acc.y += part.y; acc.z += part.z; acc.w += part.w;  // :129-131, camera order
  }
#pragma unroll
  for (int s = LPI; s < LANES; s <<= 1) {   // fold the sample groups
    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, s); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, s);
    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, s); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, s);
  }
  if (!live || sg != 0) return;
  float c = (float)max(cnt, 1);  // :133-136
  acc.x /= c; acc.y /= c; acc.z /= c; acc.w /= c;
  *reinterpret_cast<float4*>(slots + item * DH + lc * 4) = acc;
  if (count && h == 0 && lc == 0) count[q] = cnt;
}

// ---- A8 fused cross-view hybrid attention core -----------------------------------------------------------
template <int DH>
__global__ void __launch_bounds__(256, SO_SELF_ATTN_MIN_CTAS) tpv_self_attn_kernel(const float* __restrict__ value, const long long* __restrict__ shapes, const long long* __restrict__ lsi,
                                                            const float* __restrict__ offsets, const float* __restrict__ logits,
                                                            const float* __restrict__ ref, float* __restrict__ out, int Nv, int Hd,
                                                            int Q, int L, int P, int value_ld, int off_ld, int lg_ld) {
  constexpr int LPI = DH / 4;
  __shared__ Levels lv;
  load_levels(lv, shapes, lsi, L);
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long item = t / LPI;
  int lc = (int)(t % LPI);
  long long n_items = (long long)Q * Hd;
  bool live = item < n_items;
  if (!live) item = n_items - 1;
  int h = (int)(item % Hd);
  int q = (int)(item / Hd);
  const int pstride = value_ld;
  const int LP = L * P;
  const float* op = offsets + (long long)q * off_ld + (long long)h * LP * 2;
  const float* lg = logits + (long long)q * lg_ld + (long long)h * LP;
  const float* rp = ref + (long long)q * LP * 2;
  float mx, inv_sum;
  softmax_stats<LPI>(lg, LP, lc, mx, inv_sum);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int l = 0; l < L; ++l) {
    const int Hl = lv.h[l], Wl = lv.w[l];
    const float rw = 1.0f / (float)Wl, rh = 1.0f / (float)Hl;
    const float* vbase = value + (long long)lv.start[l] * value_ld + h * DH + lc * 4;
    constexpr int kUnroll = SO_SELF_ATTN_UNROLL;
#pragma unroll kUnroll
    for (int p = 0; p < P; ++p) {
      float2 r = __ldg(reinterpret_cast<const float2*>(rp) + l * P + p);
      float2 o = __ldg(reinterpret_cast<const float2*>(op) + l * P + p);
      float aw = __expf(__ldg(lg + l * P + p) - mx) * inv_sum;
      float4 s = bilinear4(vbase, pstride, Hl, Wl, fmaf(o.x, rw, r.x), fmaf(o.y, rh, r.y));  // cross_view_hybrid_attention.py:97-99
      acc.x = fmaf(aw, s.x, acc.x); acc.y = fmaf(aw, s.y, acc.y);
      acc.z = fmaf(aw, s.z, acc.z); acc.w = fmaf(aw, s.w, acc.w);
    }
  }
  if (live) *reinterpret_cast<float4*>(out + item * DH + lc * 4) = acc;
}

// ======================================================================================================================
// v2 of the two fused attention cores: the per-sample set-up is computed ONCE per (query, head, sample) instead of once
// per lane.  In the kernels above the DH/4 lanes of an item each redo the whole set-up of every sample (location
// arithmetic, floor, bounds, 4 bilinear weights, softmax weight: ~70 of the ~116 instructions per sample, plus three
// parameter loads and spill traffic under the register cap).  Here the LANES lanes of an
// item set up LANES DIFFERENT samples of a round (lane j: point d0 + j), park the result -- 4 corner weights already
// multiplied by the attention weight and by the zero-padding mask, and the 4 (clamped, always in-bounds) absolute pixel
// indices -- in 32 bytes of shared memory, and then each 4-lane sub-group walks over its 4 samples of the round reading
// the parked set-up with two broadcast LDS.128 and issuing the 4 coalesced 64-byte corner reads + 16 FMAs.  Same
// arithmetic per sample as bilinear4 (weights are the same products; the attention weight is folded in before the
// corner sum instead of after), so results agree to rounding with the v1 kernels (tests: both vs the fp64 oracle).
struct SamplePark { float w[4]; int p[4]; };     // 32 B: parked as one float4 + one int4 in two shared arrays
// Slot layout inside a warp's 32 entries (conflict-free on both sides): the lane L = 4 g + j that sets sample j of sub-group
// g up writes slot j * 8 + g; at step j the 8 sub-groups read slots j * 8 + 0..7 = 128 contiguous bytes (one wavefront; the
// first version parked array-of-structs at a 128-byte stride between sub-groups: 8-way bank conflicts).
__device__ __forceinline__ int park_write_slot(int lane) { return (lane & 3) * 8 + (lane >> 2); }
__device__ __forceinline__ int park_read_slot(int lane, int j) { return j * 8 + (lane >> 2); }

// set-up of one bilinear sample at normalised (lx, ly) of a level [Hl, Wl] whose first pixel has absolute index `base`
__device__ __forceinline__ SamplePark park_sample(float lx, float ly, int Hl, int Wl, int base, float aw) {
  SamplePark s;
  float x = lx * (float)Wl - 0.5f, y = ly * (float)Hl - 0.5f;
  const bool inside = y > -1.f && x > -1.f && y < (float)Hl && x < (float)Wl;
  float xf = floorf(x), yf = floorf(y);
  int x0 = (int)xf, y0 = (int)yf;
  float fx = x - xf, fy = y - yf;
  const bool xa = x0 >= 0, xb = x0 + 1 < Wl, ya = y0 >= 0, yb = y0 + 1 < Hl;
  const float a = inside ? aw : 0.f;
  s.w[0] = (ya && xa) ? a * ((1.f - fy) * (1.f - fx)) : 0.f;
  s.w[1] = (ya && xb) ? a * ((1.f - fy) * fx) : 0.f;
  s.w[2] = (yb && xa) ? a * (fy * (1.f - fx)) : 0.f;
  s.w[3] = (yb && xb) ? a * (fy * fx) : 0.f;
  // clamped indices: a masked corner re-reads a valid pixel with weight 0 (no predicated loads, no out-of-bounds address)
  int xc0 = min(max(x0, 0), Wl - 1), xc1 = min(max(x0 + 1, 0), Wl - 1);
  int yc0 = min(max(y0, 0), Hl - 1), yc1 = min(max(y0 + 1, 0), Hl - 1);
  if (!inside) { xc0 = xc1 = yc0 = yc1 = 0; }
  s.p[0] = base + yc0 * Wl + xc0; s.p[1] = base + yc0 * Wl + xc1;
  s.p[2] = base + yc1 * Wl + xc0; s.p[3] = base + yc1 * Wl + xc1;
  return s;
}

__device__ __forceinline__ void consume_sample(const float4 w, const int4 p, const float* __restrict__ vlane, int value_ld, float4& acc) {
  if (w.x == 0.f && w.y == 0.f && w.z == 0.f && w.w == 0.f) return;       // uniform over the 4 lanes of the sub-group
  const float4 v0 = __ldg(reinterpret_cast<const float4*>(vlane + (long long)p.x * value_ld));
  const float4 v1 = __ldg(reinterpret_cast<const float4*>(vlane + (long long)p.y * value_ld));
  const float4 v2 = __ldg(reinterpret_cast<const float4*>(vlane + (long long)p.z * value_ld));
  const float4 v3 = __ldg(reinterpret_cast<const float4*>(vlane + (long long)p.w * value_ld));
  acc.x = fmaf(w.x, v0.x, acc.x); acc.y = fmaf(w.x, v0.y, acc.y); acc.z = fmaf(w.x, v0.z, acc.z); acc.w = fmaf(w.x, v0.w, acc.w);
  acc.x = fmaf(w.y, v1.x, acc.x); acc.y = fmaf(w.y, v1.y, acc.y); acc.z = fmaf(w.y, v1.z, acc.z); acc.w = fmaf(w.y, v1.w, acc.w);
  acc.x = fmaf(w.z, v2.x, acc.x); acc.y = fmaf(w.z, v2.y, acc.y); acc.z = fmaf(w.z, v2.z, acc.z); acc.w = fmaf(w.z, v2.w, acc.w);
  acc.x = fmaf(w.w, v3.x, acc.x); acc.y = fmaf(w.w, v3.y, acc.y); acc.z = fmaf(w.w, v3.z, acc.z); acc.w = fmaf(w.w, v3.w, acc.w);
}

#ifndef SO_ATTN2_MIN_CTAS
#define SO_ATTN2_MIN_CTAS 4
#endif

// DH = 16 only (4 lanes x float4).  Requires D % (4 * SPLIT) == 0 (every round lies inside one level of one camera).
template <int SPLIT>
__global__ void __launch_bounds__(256, SO_ATTN2_MIN_CTAS) tpv_cross_attn2_kernel(
    const float* __restrict__ value, const long long* __restrict__ shapes, const long long* __restrict__ lsi,
    const float* __restrict__ offsets, const float* __restrict__ logits, const float* __restrict__ uv,
    const unsigned char* __restrict__ vis, float* __restrict__ slots, int* __restrict__ count, int N, int Nv, int Hd, int Q, int L,
    int D, int value_ld, int off_ld, int lg_ld) {
  constexpr int DH = 16, LPI = 4, LANES = LPI * SPLIT;
  __shared__ Levels lv;
  __shared__ float4 park_w[256];
  __shared__ int4 park_p[256];
  load_levels(lv, shapes, lsi, L);
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long item = t / LANES;
  const int li = (int)(t % LANES);
  const int lc = li % LPI, sg = li / LPI;
  const long long n_items = (long long)Q * Hd;
  const bool live = item < n_items;
  if (!live) item = n_items - 1;
  const int h = (int)(item % Hd);
  const int q = (int)(item / Hd);
  const int LD = L * D;
  const float* op = offsets + (long long)q * off_ld + (long long)h * LD * 2;
  const float* lg = logits + (long long)q * lg_ld + (long long)h * LD;
  float mx, inv_sum;
  softmax_stats<LANES>(lg, LD, li, mx, inv_sum);
  const float* vlane = value + h * DH + lc * 4;
  const int wbase = threadIdx.x & ~31, wl = threadIdx.x & 31;
  const int slot_w = wbase + park_write_slot(wl);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  int cnt = 0;
  for (int cam = 0; cam < N; ++cam) {
    const bool visible = __ldg(vis + (long long)cam * Q + q) != 0;       // image_cross_attention.py:92 (query visible in cam)
    if (!__any_sync(0xffffffffu, visible)) continue;
    cnt += visible ? 1 : 0;
    const float* uvp = uv + ((long long)cam * Q + q) * D * 2;
    float4 part = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int l = 0; l < L; ++l) {
      const int Hl = lv.h[l], Wl = lv.w[l];
      const float rw = 1.0f / (float)Wl, rh = 1.0f / (float)Hl;
      const int base = cam * Nv + (int)lv.start[l];
      for (int d0 = 0; d0 < D; d0 += LANES) {
        const int d = d0 + li;
        const float2 r = __ldg(reinterpret_cast<const float2*>(uvp) + d);
        const float2 o = __ldg(reinterpret_cast<const float2*>(op) + l * D + d);
        const float aw = visible ? __expf(__ldg(lg + l * D + d) - mx) * inv_sum : 0.f;
        // image_cross_attention.py:326-328: ref + offset / (w_l, h_l)   (reciprocal multiply: <= 1 ulp from the division)
        const SamplePark sp = park_sample(fmaf(o.x, rw, r.x), fmaf(o.y, rh, r.y), Hl, Wl, base, aw);
        park_w[slot_w] = make_float4(sp.w[0], sp.w[1], sp.w[2], sp.w[3]);
        park_p[slot_w] = make_int4(sp.p[0], sp.p[1], sp.p[2], sp.p[3]);
        __syncwarp();
#pragma unroll
        for (int j = 0; j < LPI; ++j) {
          const int rs = wbase + park_read_slot(wl, j);
          consume_sample(park_w[rs], park_p[rs], vlane, value_ld, part);
        }
        __syncwarp();
      }
    }
    acc.x += part.x; acc.y += part.y; acc.z += part.z; acc.w += part.w;  // :129-131, camera order
  }
#pragma unroll
  for (int s2 = LPI; s2 < LANES; s2 <<= 1) {   // fold the sample groups
    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, s2); acc.y += __shfl_xor_sync(0xffffffffu, acc.y, s2);
    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, s2); acc.w += __shfl_xor_sync(0xffffffffu, acc.w, s2);
  }
  if (!live || sg != 0) return;
  float c = (float)max(cnt, 1);  // :133-136
  acc.x /= c; acc.y /= c; acc.z /= c; acc.w /= c;
  *reinterpret_cast<float4*>(slots + item * DH + lc * 4) = acc;
  if (count && h == 0 && lc == 0) count[q] = cnt;
}

// self-attention (cross-view hybrid), DH = 16, P % 4 == 0
__global__ void __launch_bounds__(256, SO_ATTN2_MIN_CTAS) tpv_self_attn2_kernel(
    const float* __restrict__ value, const long long* __restrict__ shapes, const long long* __restrict__ lsi,
    const float* __restrict__ offsets, const float* __restrict__ logits, const float* __restrict__ ref, float* __restrict__ out, int Nv,
    int Hd, int Q, int L, int P, int value_ld, int off_ld, int lg_ld) {
  constexpr int DH = 16, LPI = 4;
  __shared__ Levels lv;
  __shared__ float4 park_w[256];
  __shared__ int4 park_p[256];
  load_levels(lv, shapes, lsi, L);
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  long long item = t / LPI;
  const int lc = (int)(t % LPI);
  const long long n_items = (long long)Q * Hd;
  const bool live = item < n_items;
  if (!live) item = n_items - 1;
  const int h = (int)(item % Hd);
  const int q = (int)(item / Hd);
  const int LP = L * P;
  const float* op = offsets + (long long)q * off_ld + (long long)h * LP * 2;
  const float* lg = logits + (long long)q * lg_ld + (long long)h * LP;
  const float* rp = ref + (long long)q * LP * 2;
  float mx, inv_sum;
  softmax_stats<LPI>(lg, LP, lc, mx, inv_sum);
  const float* vlane = value + h * DH + lc * 4;
  const int wbase = threadIdx.x & ~31, wl = threadIdx.x & 31;
  const int slot_w = wbase + park_write_slot(wl);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int l = 0; l < L; ++l) {
    const int Hl = lv.h[l], Wl = lv.w[l];
    const float rw = 1.0f / (float)Wl, rh = 1.0f / (float)Hl;
    const int base = (int)lv.start[l];
    for (int p0 = 0; p0 < P; p0 += LPI) {
      const int p = p0 + lc;
      const float2 r = __ldg(reinterpret_cast<const float2*>(rp) + l * P + p);
      const float2 o = __ldg(reinterpret_cast<const float2*>(op) + l * P + p);
      const float aw = __expf(__ldg(lg + l * P + p) - mx) * inv_sum;
      const SamplePark sp = park_sample(fmaf(o.x, rw, r.x), fmaf(o.y, rh, r.y), Hl, Wl, base, aw);    // cross_view_hybrid_attention.py:97-99
      park_w[slot_w] = make_float4(sp.w[0], sp.w[1], sp.w[2], sp.w[3]);
      park_p[slot_w] = make_int4(sp.p[0], sp.p[1], sp.p[2], sp.p[3]);
      __syncwarp();
#pragma unroll
      for (int j = 0; j < LPI; ++j) {
        const int rs = wbase + park_read_slot(wl, j);
        consume_sample(park_w[rs], park_p[rs], vlane, value_ld, acc);
      }
      __syncwarp();
    }
  }
  if (live) *reinterpret_cast<float4*>(out + item * DH + lc * 4) = acc;
}

// ---- A4 point_sampling (bevformer/utils.py:116-206) ---------------------------------------------------------
// One thread per (camera, query, pillar point): fully coalesced uv / mask stores.  The projection uses plain fp32
// mul/add in a fixed left-to-right order (no FMA contraction): `mask` generates index lists.  `vis` (any over the
// pillar) is zero-filled first and set with idempotent byte stores.
__global__ void __launch_bounds__(256) point_sampling_kernel(const float* __restrict__ ref3d, const float* __restrict__ l2i,
                                                             int D, int Q, int N, float img_h, float img_w,
                                                             float* __restrict__ uv, unsigned char* __restrict__ mask,
                                                             unsigned char* __restrict__ vis) {
  long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (t >= (long long)N * Q * D) return;
  int d = (int)(t % D);
  long long cq = t / D;
  int cam = (int)(cq / Q), q = (int)(cq % Q);
  const float* m = l2i + cam * 16;
  const float eps = 1e-5f;
  const float* p = ref3d + ((long long)d * Q + q) * 3;
  float x = __ldg(p), y = __ldg(p + 1), z = __ldg(p + 2);
  float cx = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 0), x), __fmul_rn(__ldg(m + 1), y)), __fmul_rn(__ldg(m + 2), z)), __ldg(m + 3));
  float cy = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 4), x), __fmul_rn(__ldg(m + 5), y)), __fmul_rn(__ldg(m + 6), z)), __ldg(m + 7));
  float cz = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 8), x), __fmul_rn(__ldg(m + 9), y)), __fmul_rn(__ldg(m + 10), z)), __ldg(m + 11));
  bool ok = cz > eps;
  float den = fmaxf(cz, eps);
  float u = __fdiv_rn(__fdiv_rn(cx, den), img_w);
  float v = __fdiv_rn(__fdiv_rn(cy, den), img_h);
  ok = ok && (v > 0.f) && (v < 1.f) && (u < 1.f) && (u > 0.f);
  reinterpret_cast<float2*>(uv)[t] = make_float2(u, v);
  if (mask) mask[t] = ok ? 1 : 0;
  if (vis && ok) vis[cq] = 1;
}

__global__ void zero_bytes_kernel(unsigned char* p, long long n) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) p[i] = 0;
}

// ---- A5 ordered index lists (nonzero) ---------------------------------------------------------------------
// One CTA per camera; chunks of 1024 queries are compacted in order with a block-wide ballot scan.
__global__ void __launch_bounds__(1024) visible_index_kernel(const unsigned char* __restrict__ mask, int Q, int D,
                                                             long long* __restrict__ lists, int* __restrict__ lens) {
  __shared__ int warp_cnt[32];
  __shared__ int base;
  int cam = blockIdx.x;
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int q0 = 0; q0 < Q; q0 += 1024) {
    int q = q0 + threadIdx.x;
    bool v = false;
    if (q < Q) {
      const unsigned char* m = mask + ((long long)cam * Q + q) * D;
      for (int d = 0; d < D; ++d) v = v || m[d];
    }
    unsigned bal = __ballot_sync(0xffffffffu, v);
    if (lane == 0) warp_cnt[wid] = __popc(bal);
    __syncthreads();
    int off = base;
    for (int w = 0; w < wid; ++w) off += warp_cnt[w];
    if (v) lists[(long long)cam * Q + off + __popc(bal & ((1u << lane) - 1u))] = q;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < 32; ++w) tot += warp_cnt[w];
      base += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) lens[cam] = base;
}

}  // namespace so

using namespace so;

#define SO_DISPATCH_DH(Dh, EXPR16, EXPR32) \
  do {                                     \
    if ((Dh) == 16) { EXPR16; }            \
    else if ((Dh) == 32) { EXPR32; }       \
    else return SO_ERR_UNSUPPORTED;        \
  } while (0)

static bool g_attn_force_v1 = false;
// Test hook: 1 = route the fused attention cores through the first-generation kernels (one set-up per lane).
extern "C" int so_attn_force_v1(int on) { g_attn_force_v1 = on != 0; return SO_OK; }

extern "C" int so_msda_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                               const float* loc, const float* weights, float* out, int32_t B, int32_t Nv, int32_t Hd,
                               int32_t Dh, int32_t Nq, int32_t L, int32_t P, void* stream) {
  if (!value || !spatial_shapes || !level_start_index || !loc || !weights || !out) return SO_ERR_INVALID_ARG;
  if (B < 1 || Nv < 1 || Hd < 1 || Nq < 0 || L < 1 || P < 1) return SO_ERR_INVALID_ARG;
  if (Nq == 0) return SO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (L > kMaxLevels) return SO_ERR_UNSUPPORTED;
  const long long* shp = reinterpret_cast<const long long*>(spatial_shapes);
  const long long* lsi = reinterpret_cast<const long long*>(level_start_index);
  long long threads = (long long)B * Nq * Hd * (Dh / 4);
  unsigned grid = (unsigned)ceil_div64(threads, 256);
  ProfScope prof(4, st);
  SO_DISPATCH_DH(Dh, (msda_forward_kernel<16><<<grid, 256, 0, st>>>(value, shp, lsi, loc, weights, out, B, Nv, Hd, Nq, L, P)),
                 (msda_forward_kernel<32><<<grid, 256, 0, st>>>(value, shp, lsi, loc, weights, out, B, Nv, Hd, Nq, L, P)));
  note_launch(1);
  return check_launch();
}

extern "C" int so_msda_backward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                const float* loc, const float* weights, const float* grad_out, float* grad_value,
                                float* grad_loc, float* grad_weights, int32_t B, int32_t Nv, int32_t Hd, int32_t Dh,
                                int32_t Nq, int32_t L, int32_t P, void* stream) {
  if (!value || !spatial_shapes || !level_start_index || !loc || !weights || !grad_out || !grad_value || !grad_loc ||
      !grad_weights)
    return SO_ERR_INVALID_ARG;
  if (B < 1 || Nv < 1 || Hd < 1 || Nq < 0 || L < 1 || P < 1) return SO_ERR_INVALID_ARG;
  if (Nq == 0) return SO_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (L > kMaxLevels) return SO_ERR_UNSUPPORTED;
  const long long* shp = reinterpret_cast<const long long*>(spatial_shapes);
  const long long* lsi = reinterpret_cast<const long long*>(level_start_index);
  long long threads = (long long)B * Nq * Hd * (Dh / 4);
  unsigned grid = (unsigned)ceil_div64(threads, 256);
  ProfScope prof(5, st);
  SO_DISPATCH_DH(Dh,
                 (msda_backward_kernel<16><<<grid, 256, 0, st>>>(value, shp, lsi, loc, weights, grad_out, grad_value, grad_loc, grad_weights, B, Nv, Hd, Nq, L, P)),
                 (msda_backward_kernel<32><<<grid, 256, 0, st>>>(value, shp, lsi, loc, weights, grad_out, grad_value, grad_loc, grad_weights, B, Nv, Hd, Nq, L, P)));
  note_launch(1);
  return check_launch();
}

extern "C" int so_point_sampling(const float* ref_3d, const float* lidar2img, int32_t D, int32_t Q, int32_t N, float img_h,
                                 float img_w, float* uv, uint8_t* mask, uint8_t* vis, void* stream) {
  if (!ref_3d || !lidar2img || !uv) return SO_ERR_INVALID_ARG;
  if (D < 1 || Q < 1 || N < 1 || !(img_h > 0.f) || !(img_w > 0.f)) return SO_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (vis) {
    zero_bytes_kernel<<<(unsigned)ceil_div64((long long)N * Q, 256), 256, 0, st>>>(vis, (long long)N * Q);
    note_launch(1);
  }
  long long n = (long long)N * Q * D;
  point_sampling_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(ref_3d, lidar2img, D, Q, N, img_h, img_w, uv, mask, vis);
  note_launch(1);
  return check_launch();
}

extern "C" int so_tpv_cross_attn_forward_strided(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                                 const float* offsets, const float* logits, const float* uv, const uint8_t* vis,
                                                 float* slots, int32_t* count, int32_t N, int32_t Nv, int32_t Hd, int32_t Dh,
                                                 int32_t Q, int32_t L, int32_t D, int32_t value_ld, int32_t offsets_ld,
                                                 int32_t logits_ld, void* stream) {
  if (!value || !spatial_shapes || !level_start_index || !offsets || !logits || !uv || !vis || !slots) return SO_ERR_INVALID_ARG;
  if (N < 1 || Nv < 1 || Hd < 1 || Q < 1 || L < 1 || D < 1) return SO_ERR_INVALID_ARG;
  if (value_ld < Hd * Dh || offsets_ld < Hd * L * D * 2 || logits_ld < Hd * L * D || (value_ld & 3)) return SO_ERR_INVALID_ARG;
  // the kernels read value rows as float4 and (x, y) offsets as float2
  if ((offsets_ld & 1) || (reinterpret_cast<uintptr_t>(offsets) & 7) || (reinterpret_cast<uintptr_t>(value) & 15)) return SO_ERR_INVALID_ARG;
  if (L > kMaxLevels) return SO_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const long long* shp = reinterpret_cast<const long long*>(spatial_shapes);
  const long long* lsi = reinterpret_cast<const long long*>(level_start_index);
  const int split = D >= 32 ? 4 : (D >= 16 ? 2 : 1);
  long long threads = (long long)Q * Hd * (Dh / 4) * split;
  unsigned grid = (unsigned)ceil_div64(threads, 256);
  ProfScope prof(2, st);
#define SO_CROSS2(SP) tpv_cross_attn2_kernel<SP><<<grid, 256, 0, st>>>(value, shp, lsi, offsets, logits, uv, vis, slots, count, N, Nv, Hd, Q, L, D, value_ld, offsets_ld, logits_ld)
  if (Dh == 16 && D % (4 * split) == 0 && !g_attn_force_v1 && (long long)N * Nv < (1LL << 31)) {
    if (split == 4) SO_CROSS2(4); else if (split == 2) SO_CROSS2(2); else SO_CROSS2(1);
    note_launch(1);
    return check_launch();
  }
#undef SO_CROSS2
#define SO_CROSS(DHV, SP) tpv_cross_attn_kernel<DHV, SP><<<grid, 256, 0, st>>>(value, shp, lsi, offsets, logits, uv, vis, slots, count, N, Nv, Hd, Q, L, D, value_ld, offsets_ld, logits_ld)
  if (Dh == 16) { if (split == 4) SO_CROSS(16, 4); else if (split == 2) SO_CROSS(16, 2); else SO_CROSS(16, 1); }
  else if (Dh == 32) { if (split == 4) SO_CROSS(32, 4); else if (split == 2) SO_CROSS(32, 2); else SO_CROSS(32, 1); }
  else return SO_ERR_UNSUPPORTED;
#undef SO_CROSS
  note_launch(1);
  return check_launch();
}

extern "C" int so_tpv_cross_attn_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                         const float* offsets, const float* logits, const float* uv, const uint8_t* vis,
                                         float* slots, int32_t* count, int32_t N, int32_t Nv, int32_t Hd, int32_t Dh, int32_t Q,
                                         int32_t L, int32_t D, void* stream) {
  return so_tpv_cross_attn_forward_strided(value, spatial_shapes, level_start_index, offsets, logits, uv, vis, slots, count, N, Nv,
                                           Hd, Dh, Q, L, D, Hd * Dh, Hd * L * D * 2, Hd * L * D, stream);
}

extern "C" int so_tpv_self_attn_forward_strided(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                                const float* offsets, const float* logits, const float* ref, float* out, int32_t Nv,
                                                int32_t Hd, int32_t Dh, int32_t Q, int32_t L, int32_t P, int32_t value_ld,
                                                int32_t offsets_ld, int32_t logits_ld, void* stream) {
  if (!value || !spatial_shapes || !level_start_index || !offsets || !logits || !ref || !out) return SO_ERR_INVALID_ARG;
  if (Nv < 1 || Hd < 1 || Q < 1 || L < 1 || P < 1) return SO_ERR_INVALID_ARG;
  if (value_ld < Hd * Dh || offsets_ld < Hd * L * P * 2 || logits_ld < Hd * L * P || (value_ld & 3)) return SO_ERR_INVALID_ARG;
  if ((offsets_ld & 1) || (reinterpret_cast<uintptr_t>(offsets) & 7) || (reinterpret_cast<uintptr_t>(value) & 15)) return SO_ERR_INVALID_ARG;
  if (L > kMaxLevels) return SO_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const long long* shp = reinterpret_cast<const long long*>(spatial_shapes);
  const long long* lsi = reinterpret_cast<const long long*>(level_start_index);
  long long threads = (long long)Q * Hd * (Dh / 4);
  unsigned grid = (unsigned)ceil_div64(threads, 256);
  ProfScope prof(3, st);
  if (Dh == 16 && P % 4 == 0 && !g_attn_force_v1) {
    tpv_self_attn2_kernel<<<grid, 256, 0, st>>>(value, shp, lsi, offsets, logits, ref, out, Nv, Hd, Q, L, P, value_ld, offsets_ld, logits_ld);
    note_launch(1);
    return check_launch();
  }
  SO_DISPATCH_DH(Dh, (tpv_self_attn_kernel<16><<<grid, 256, 0, st>>>(value, shp, lsi, offsets, logits, ref, out, Nv, Hd, Q, L, P, value_ld, offsets_ld, logits_ld)),
                 (tpv_self_attn_kernel<32><<<grid, 256, 0, st>>>(value, shp, lsi, offsets, logits, ref, out, Nv, Hd, Q, L, P, value_ld, offsets_ld, logits_ld)));
  note_launch(1);
  return check_launch();
}

extern "C" int so_tpv_self_attn_forward(const float* value, const int64_t* spatial_shapes, const int64_t* level_start_index,
                                        const float* offsets, const float* logits, const float* ref, float* out, int32_t Nv,
                                        int32_t Hd, int32_t Dh, int32_t Q, int32_t L, int32_t P, void* stream) {
  return so_tpv_self_attn_forward_strided(value, spatial_shapes, level_start_index, offsets, logits, ref, out, Nv, Hd, Dh, Q, L, P,
                                          Hd * Dh, Hd * L * P * 2, Hd * L * P, stream);
}

extern "C" int so_visible_index_lists(const uint8_t* mask, int32_t N, int32_t Q, int32_t D, int64_t* index_lists, int32_t* lens,
                                      void* stream) {
  if (!mask || !index_lists || !lens || N < 1 || Q < 1 || D < 1) return SO_ERR_INVALID_ARG;
  visible_index_kernel<<<N, 1024, 0, (cudaStream_t)stream>>>(mask, Q, D, reinterpret_cast<long long*>(index_lists), lens);
  note_launch(1);
  return check_launch();
}
