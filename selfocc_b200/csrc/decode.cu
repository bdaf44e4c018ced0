// B5: TPV planes -> decoded volume (SURVEY.md section 8a row B5; semantics bev_nerf.py:62-95).
//
// One CTA decodes 128 consecutive (w, z) voxels of one h row:
//   A[r][:]  = softplus(hw[h,w] + zh[z,h] + wz[w,z])           built in shared memory, never in HBM
//   H1       = softplus(A * W1^T + b1)                           fp32 register-tiled 128x96x96 GEMM
//   out[r,:] = H1 * W2^T + b2                                    (1 + n_feat outputs)
// The reference materialises the [H,W,Z,C] broadcast sum (750 MB at cfg 2); here the only HBM traffic
// is the 30 MB of planes (L2-resident across CTAs) and the decoded volume itself.
// fp32 SIMT on purpose: the decoded sdf feeds a 1e-4-relative depth parity bar (fp32 reference,
// autocast disabled at bev_nerf.py:73).
#include "tc_common.cuh"

namespace so {

constexpr int kRows = 128;      // voxels per CTA
constexpr int kThreads = 256;
constexpr int kMaxOut = 32;

__device__ __forceinline__ float softplus_fast(float x) {
  // F.softplus(beta=1, threshold=20): max(x,0) + log1p(exp(-|x|)); identical to x beyond the threshold in fp32.
  // Forward kernels only.  1 + e is rounded to fp32 and __logf is accurate to 2^-21.4 absolute, so the ABSOLUTE error stays
  // below 1e-6 everywhere, which is what the decoded volume needs (every consumer of an activation multiplies it by a
  // weight and adds it to an O(1) sum), but the error RELATIVE to the value grows as the value shrinks (1e-2 at x = -10).
  // The backward needs the relative kind (softplus_rel below) and does not share this function.
  return fmaxf(x, 0.f) + __logf(1.0f + __expf(-fabsf(x)));
}

// log1p(e) for e = exp(-|x|) in [0, 1], accurate relative to its value: 2 atanh(s) with s = e / (2 + e) <= 1/3 by the odd
// series up to s^11 (next term 1.5e-7 relative at e = 1).  No 1 + e is formed and no logarithm taken, so a small e keeps all
// its digits; one MUFU.RCP instead of softplus_fast's MUFU.LG2, plus five FMAs.
__device__ __forceinline__ float log1p_small(float e) {
  const float s = __fdividef(e, 2.0f + e), t = s * s;
  float p = fmaf(t, 1.0f / 11.0f, 1.0f / 9.0f);
  p = fmaf(t, p, 1.0f / 7.0f);
  p = fmaf(t, p, 1.0f / 5.0f);
  p = fmaf(t, p, 1.0f / 3.0f);
  p = fmaf(t, p, 1.0f);
  return 2.0f * s * p;
}

// Backward kernels: softplus and the sigmoid factors accurate RELATIVE to their values on the negative side too (a few
// 1e-7 down to the underflow of exp at x = -87).  A plane channel or hidden unit whose pre-activation sits below about
// -6 has activations and sigmoid factors of 1e-3 and less; its gradient is a sum of products with exactly those, and
// Adam divides every gradient by its own running magnitude, so an error relative to the small value is an error of the
// same size in the update.
__device__ __forceinline__ float softplus_rel(float x) { return fmaxf(x, 0.f) + log1p_small(__expf(-fabsf(x))); }

// softplus(z) and sigmoid(z) from one exponential: sigmoid = 1 / (1 + e) for z >= 0, e / (1 + e) below
__device__ __forceinline__ float softplus_sigmoid(float z, float* sig) {
  const float e = __expf(-fabsf(z)), r = __fdividef(1.0f, 1.0f + e);
  *sig = z >= 0.f ? r : e * r;
  return fmaxf(z, 0.f) + log1p_small(e);
}

// sigmoid(x) from a = softplus(x) alone: 1 - exp(-a).  Below 1/8 the subtraction would cancel (sigmoid ~ a), so -expm1(-a)
// is taken by its series up to a^5 (next term 4e-8 relative at 1/8); above, the difference keeps 2e-6 relative or better.
__device__ __forceinline__ float sigmoid_of_softplus(float a) {
  float p = fmaf(a, 1.0f / 120.0f, -1.0f / 24.0f);
  p = fmaf(a, p, 1.0f / 6.0f);
  p = fmaf(a, p, -0.5f);
  p = fmaf(a, p, 1.0f);
  return a < 0.125f ? a * p : 1.0f - __expf(-a);
}

// Split v into TF32 hi / lo (hi + lo == v exactly) and store both at byte offset off of the hi and lo operand atoms.
__device__ __forceinline__ void store_split_tf32(uint8_t* hi, uint8_t* lo, uint32_t off, float4 v) {
  float4 h, l;
  h.x = tf32_rn(v.x); l.x = v.x - h.x; h.y = tf32_rn(v.y); l.y = v.y - h.y;
  h.z = tf32_rn(v.z); l.z = v.z - h.z; h.w = tf32_rn(v.w); l.w = v.w - h.w;
  *reinterpret_cast<float4*>(hi + off) = h;
  *reinterpret_cast<float4*>(lo + off) = l;
}

// Builder step of the tensor-core decodes (TPV and BEV): softplus of one 16-byte chunk x of a row's pre-activations, split
// into TF32 hi / lo and stored at (row, chunk c4) of the 128B-swizzled K-major A atoms.  Rows past the end (ok false) are 0.
__device__ __forceinline__ void build_a_chunk(uint8_t* hi, uint8_t* lo, int row, int c4, float4 x, bool ok) {
  float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
  if (ok) {
    f.x = softplus_fast(x.x); f.y = softplus_fast(x.y);
    f.z = softplus_fast(x.z); f.w = softplus_fast(x.w);
  }
  store_split_tf32(hi, lo, swz_off(row, c4), f);
}

// C = channels (multiple of 32), LD = padded leading dimension (C + 4) in floats
template <int C>
__global__ void __launch_bounds__(kThreads) tpv_decode_kernel(
    const float* __restrict__ hw, const float* __restrict__ zh, const float* __restrict__ wz,
    const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
    const float* __restrict__ b2, int H, int W, int Z, int zpitch, int n_out, int feat_pitch,
    float* __restrict__ vol_sdf, float* __restrict__ vol_feat, int h_begin) {
  constexpr int LD = C + 4;
  constexpr int TN = C / 16;  // output columns per thread (strided by 16)
  extern __shared__ __align__(16) float smem[];
  float* As = smem;                 // [kRows][LD]
  float* Ws = As + kRows * LD;      // [C][LD]   (W1 as given: [out][in])
  float* W2s = Ws + C * LD;         // [n_out][C]
  float* b1s = W2s + kMaxOut * C;   // [C]
  float* b2s = b1s + C;             // [kMaxOut]

  const int tid = threadIdx.x;
  const int h = h_begin + blockIdx.y;     // row range [h_begin, h_begin + gridDim.y): so_tpv_decode_rows
  const int v0 = blockIdx.x * kRows;
  const int WZ = W * Z;

  // stage weights
  for (int i = tid; i < C * C / 4; i += kThreads) {
    int j = (i * 4) / C, k = (i * 4) % C;
    *reinterpret_cast<float4*>(Ws + j * LD + k) = __ldg(reinterpret_cast<const float4*>(w1) + i);
  }
  for (int i = tid; i < n_out * C; i += kThreads) W2s[i] = __ldg(w2 + i);
  for (int i = tid; i < C; i += kThreads) b1s[i] = __ldg(b1 + i);
  for (int i = tid; i < n_out; i += kThreads) b2s[i] = __ldg(b2 + i);

  // build A = softplus(broadcast sum); a warp walks one voxel row's C channels with float4 (coalesced)
  constexpr int kVecPerRow = C / 4;
  for (int i = tid; i < kRows * kVecPerRow; i += kThreads) {
    int r = i / kVecPerRow, c4 = i % kVecPerRow;
    int v = v0 + r;
    float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
    if (v < WZ) {
      int w = v / Z, z = v - w * Z;
      float4 a = __ldg(reinterpret_cast<const float4*>(hw + ((size_t)h * W + w) * C) + c4);
      float4 b = __ldg(reinterpret_cast<const float4*>(zh + ((size_t)z * H + h) * C) + c4);
      float4 c = __ldg(reinterpret_cast<const float4*>(wz + (size_t)v * C) + c4);
      f.x = softplus_fast(a.x + b.x + c.x);
      f.y = softplus_fast(a.y + b.y + c.y);
      f.z = softplus_fast(a.z + b.z + c.z);
      f.w = softplus_fast(a.w + b.w + c.w);
    }
    *reinterpret_cast<float4*>(As + r * LD + c4 * 4) = f;
  }
  __syncthreads();

  // GEMM1: thread (ty, tx) owns rows ty*8..+7 and columns tx + 16*j
  const int tx = tid & 15, ty = tid >> 4;
  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;
#pragma unroll 2
  for (int k = 0; k < C; k += 4) {
    float4 a[8], b[TN];
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = *reinterpret_cast<const float4*>(As + (ty * 8 + i) * LD + k);
#pragma unroll
    for (int j = 0; j < TN; ++j) b[j] = *reinterpret_cast<const float4*>(Ws + (tx + 16 * j) * LD + k);
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        acc[i][j] = fmaf(a[i].x, b[j].x, acc[i][j]);
        acc[i][j] = fmaf(a[i].y, b[j].y, acc[i][j]);
        acc[i][j] = fmaf(a[i].z, b[j].z, acc[i][j]);
        acc[i][j] = fmaf(a[i].w, b[j].w, acc[i][j]);
      }
  }
  __syncthreads();  // everyone done reading As
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) As[(ty * 8 + i) * LD + tx + 16 * j] = softplus_fast(acc[i][j] + b1s[tx + 16 * j]);
  __syncthreads();

  // GEMM2: (row, out-channel) pairs, K = C
  for (int idx = tid; idx < kRows * n_out; idx += kThreads) {
    int r = idx % kRows, c = idx / kRows;
    int v = v0 + r;
    if (v >= WZ) continue;
    float s = b2s[c];
    const float4* hp = reinterpret_cast<const float4*>(As + r * LD);
    const float4* wp = reinterpret_cast<const float4*>(W2s + c * C);
#pragma unroll 4
    for (int k = 0; k < C / 4; ++k) {
      float4 x = hp[k], y = wp[k];
      s = fmaf(x.x, y.x, s); s = fmaf(x.y, y.y, s); s = fmaf(x.z, y.z, s); s = fmaf(x.w, y.w, s);
    }
    int w = v / Z, z = v - w * Z;
    if (c == 0) vol_sdf[((size_t)h * W + w) * zpitch + z] = s;
    else vol_feat[(((size_t)h * W + w) * Z + z) * feat_pitch + (c - 1)] = s;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Tensor-core variant (wgmma, same 3xTF32 operand splitting as gemm.cu so the decoded sdf keeps fp32-level accuracy).
// Persistent CTA per SM, 16 warps:
//   warps 0-7   builders   A tile = softplus(hw + zh + wz) for 128 voxels x 32 channels at a time, split into TF32 hi / lo and
//                          written straight into the 128B-swizzled K-major operand layout (no TMA: the operand is computed)
//   warps 8-15  two consumer warpgroups, 64 voxels each: 12 x wgmma.m64nCk8.tf32 per atom (hi*hi, lo*hi, hi*lo) into a
//                          register accumulator; epilogue +b1 -> softplus -> second Linear (1 + n_feat outputs, dot products
//                          over the 4 threads that share a row) -> volume
// W1 (hi and lo, swizzled) stays resident in shared memory for the whole kernel.
constexpr int kDecBuilders = 256;
constexpr int kDecThreads = kDecBuilders + 256;
constexpr int kDecStagesMax = 4;

struct DecSmem {
  int atoms, stages, w_bytes, ring, w2, b1, b2, bars, total;
};
__host__ __device__ inline DecSmem dec_smem(int C, int n_out) {
  DecSmem m;
  m.atoms = C / kAtomK;
  m.w_bytes = 2 * m.atoms * C * 128;                          // W1 hi + lo: atoms x [C rows x 128 B]
  const int fixed = m.w_bytes + n_out * C * 4 + C * 4 + 128 + 256;
  int st = (227 * 1024 - 1024 - fixed) / (2 * kAtomBytesA);
  m.stages = st > kDecStagesMax ? kDecStagesMax : st;
  m.ring = m.w_bytes;
  m.w2 = m.ring + m.stages * 2 * kAtomBytesA;
  m.b1 = m.w2 + n_out * C * 4;
  m.b2 = m.b1 + C * 4;
  m.bars = m.b2 + 128;
  m.total = m.bars + 256 + 1024;
  return m;
}

// C = channels (wgmma N); NOUT = compile-time upper bound of the second layer's width (1 + n_feat): the per-row outputs
// stay in registers
template <int C, int NOUT>
__global__ void __launch_bounds__(kDecThreads, 1)
tpv_decode_tc_kernel(const float* __restrict__ hw, const float* __restrict__ zh, const float* __restrict__ wz,
                     const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ w2,
                     const float* __restrict__ b2, int H, int W, int Z, int zpitch, int n_out, int feat_pitch,
                     float* __restrict__ vol_sdf, float* __restrict__ vol_feat, int tiles_per_row, int n_tiles, int h_begin) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const DecSmem L = dec_smem(C, n_out);
  constexpr int KA = C / kAtomK;
  const int stages = L.stages;
  uint8_t* w_hi = sm;
  uint8_t* w_lo = sm + KA * C * 128;
  uint8_t* ring = sm + L.ring;
  float* W2s = reinterpret_cast<float*>(sm + L.w2);
  float* b1s = reinterpret_cast<float*>(sm + L.b1);
  float* b2s = reinterpret_cast<float*>(sm + L.b2);
  uint64_t* conv = reinterpret_cast<uint64_t*>(sm + L.bars);
  uint64_t* empty = conv + kDecStagesMax;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int WZ = W * Z;

  if (tid == 0) {
    for (int s = 0; s < kDecStagesMax; ++s) { mbar_init(conv + s, kDecBuilders); mbar_init(empty + s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // W1 [out j][in k] is K-major already: split it and lay it out as KA swizzled atoms of [C rows x 32 k]
  for (int i = tid; i < C * C / 4; i += kDecThreads) {
    int j = (i * 4) / C, k = (i * 4) % C;
    store_split_tf32(w_hi, w_lo, (uint32_t)((k / kAtomK) * C * 128) + swz_off(j, (k % kAtomK) / 4),
                     __ldg(reinterpret_cast<const float4*>(w1) + i));
  }
  for (int i = tid; i < n_out * C; i += kDecThreads) W2s[i] = __ldg(w2 + i);
  for (int i = tid; i < C; i += kDecThreads) b1s[i] = __ldg(b1 + i);
  for (int i = tid; i < n_out; i += kDecThreads) b2s[i] = __ldg(b2 + i);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  if (warp < 8) {
    // ===== builders: thread owns 16-byte chunk c4 of rows r = tid/8 + 32 j =====
    const int c4 = tid & 7, r0 = tid >> 3;
    const float inv_z = 1.0f / (float)Z;
    int s = 0; uint32_t ph = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      const int hr = t / tiles_per_row, h = h_begin + hr, v0 = (t - hr * tiles_per_row) * kBM;
      // (w, z) of this thread's four voxel rows; (v + 1/2) / Z is at least 1/(2Z) away from an integer, so the float
      // floor is exact
      int vv[4], ww[4], zz[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        vv[j] = v0 + r0 + 32 * j;
        ww[j] = __float2int_rd(((float)vv[j] + 0.5f) * inv_z);
        zz[j] = vv[j] - ww[j] * Z;
      }
      for (int a = 0; a < KA; ++a) {
        mbar_wait(empty + s, ph ^ 1);
        uint8_t* hi = ring + s * 2 * kAtomBytesA;
        uint8_t* lo = hi + kAtomBytesA;
        const int kc = a * kAtomK + c4 * 4;
        float4 x[4], y[4], u[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {       // all 12 loads of the atom in flight before any use
          const bool ok = vv[j] < WZ;
          x[j] = ok ? __ldg(reinterpret_cast<const float4*>(hw + ((size_t)h * W + ww[j]) * C + kc)) : make_float4(0.f, 0.f, 0.f, 0.f);
          y[j] = ok ? __ldg(reinterpret_cast<const float4*>(zh + ((size_t)zz[j] * H + h) * C + kc)) : make_float4(0.f, 0.f, 0.f, 0.f);
          u[j] = ok ? __ldg(reinterpret_cast<const float4*>(wz + (size_t)vv[j] * C + kc)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < 4; ++j)
          build_a_chunk(hi, lo, r0 + 32 * j, c4,
                        make_float4(x[j].x + y[j].x + u[j].x, x[j].y + y[j].y + u[j].y, x[j].z + y[j].z + u[j].z,
                                    x[j].w + y[j].w + u[j].w), vv[j] < WZ);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(conv + s);
        if (++s == stages) { s = 0; ph ^= 1; }
      }
    }
  } else {
    // ===== consumers: warpgroup wg owns voxels 64 wg .. 64 wg + 63 of every tile =====
    const int wg = (warp - 8) >> 2, wl = warp & 3, g = lane >> 2, t4 = lane & 3;
    const int frag_row = wg * kWgRows + wl * 16 + g;          // this thread's voxel rows: frag_row and frag_row + 8
    const uint32_t whi = smem_u32(w_hi), wlo = smem_u32(w_lo);
    float acc[C / 2];
#pragma unroll
    for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
    int s = 0; uint32_t ph = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      const int hr = t / tiles_per_row, h = h_begin + hr, v0 = (t - hr * tiles_per_row) * kBM;
      uint32_t accum = 0;
      for (int a = 0; a < KA; ++a) {
        mbar_wait(conv + s, ph);
        const uint32_t ahi = smem_u32(ring + s * 2 * kAtomBytesA) + wg * kWgRows * 128, alo = ahi + kAtomBytesA;
        const uint32_t bhi = whi + a * C * 128, blo = wlo + a * C * 128;
#pragma unroll
        for (int i = 0; i < C / 2; ++i) asm volatile("" : "+f"(acc[i])::"memory");
        wg_fence();
#pragma unroll
        for (int prod = 0; prod < 3; ++prod) {
          const uint32_t ab = prod == 1 ? alo : ahi;
          const uint32_t bb = prod == 2 ? blo : bhi;
#pragma unroll
          for (int k = 0; k < kAtomK / 8; ++k) {
            Wgmma<C>::ss(acc, make_desc(ab + k * 32), make_desc(bb + k * 32), accum);
            accum = 1u;
          }
        }
        wg_commit();
        wg_wait0();
#pragma unroll
        for (int i = 0; i < C / 2; ++i) asm volatile("" : "+f"(acc[i])::"memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(empty + s);
        if (++s == stages) { s = 0; ph ^= 1; }
      }
      // ===== epilogue: hidden = softplus(acc + b1); out = W2 hidden + b2 =====
      // RP voxel rows per pass over the 8-column blocks.  With a narrow second layer both rows go in one pass, so each
      // block's accumulator registers die as it is consumed; with NOUT = 32 one row at a time keeps 32 sums live, not 64.
      // Either way a row's sums are accumulated in the same order.
      constexpr int RP = NOUT <= 4 ? 2 : 1;
#pragma unroll
      for (int p = 0; p < 2 / RP; ++p) {
        float out[RP][NOUT];
#pragma unroll
        for (int r = 0; r < RP; ++r)
#pragma unroll
          for (int c = 0; c < NOUT; ++c) out[r][c] = 0.f;
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const int col = 8 * j + 2 * t4;
#pragma unroll
          for (int r = 0; r < RP; ++r) {
            const int hh = p * RP + r;
            const float h0 = softplus_fast(acc[4 * j + 2 * hh] + b1s[col]);
            const float h1 = softplus_fast(acc[4 * j + 2 * hh + 1] + b1s[col + 1]);
#pragma unroll
            for (int c = 0; c < NOUT; ++c)
              if (c < n_out) out[r][c] = fmaf(h1, W2s[c * C + col + 1], fmaf(h0, W2s[c * C + col], out[r][c]));
          }
        }
#pragma unroll
        for (int r = 0; r < RP; ++r) {
#pragma unroll
          for (int c = 0; c < NOUT; ++c) {
            out[r][c] += __shfl_xor_sync(0xffffffffu, out[r][c], 1);
            out[r][c] += __shfl_xor_sync(0xffffffffu, out[r][c], 2);
          }
          const int v = v0 + frag_row + 8 * (p * RP + r);
          if (v < WZ) {
            const int w = v / Z, z = v - w * Z;
#pragma unroll
            for (int c = 0; c < NOUT; ++c) {
              if (c >= n_out || (c & 3) != t4) continue;
              const float o = out[r][c] + b2s[c];
              if (c == 0) vol_sdf[((size_t)h * W + w) * zpitch + z] = o;
              else vol_feat[(((size_t)h * W + w) * Z + z) * feat_pitch + (c - 1)] = o;
            }
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// BEV decode (tpv=False heads, bev_nerf.py:62-81): one row per BEV cell, N = Z * Cf outputs per row,
//   a0 = softplus(bev[r])     a1 = softplus(a0 W1^T + b1)     out[r][z * Cf + c] = a1 W2[z * Cf + c]^T + b2   -> voxel (r, z), c
// N is far beyond a register-resident second layer (625 at the shipped geometry), so both layers run on the tensor cores
// with the 3xTF32 split.  Persistent CTA per SM, 12 warps:
//   warps 0-3   builders  per 128-row tile: the A atoms of a0 (build_a_chunk, shared with the TPV decode), then every
//                         n-tile of W2 split into hi / lo, read from L2 (every CTA splits the same 240 KB, so no split copy
//                         of the weights has to live in global memory); the next n-tile's loads are in flight while one
//                         is split and stored
//   warps 4-11  two consumer warpgroups, 64 rows each: GEMM 1 with resident W1 hi / lo, + b1, softplus; the hidden tile
//                         stays in registers as the A operand of GEMM 2 (wgmma with A from registers), one n-tile of W2 at a
//                         time from the ring, + b2, staged in shared memory and written out row by row.  Neither the
//                         [rows, C] hidden nor the [rows, N] output matrix reaches HBM.
// GEMM 2's A fragment holds hidden columns (8j + 2t, 8j + 2t + 1) where wgmma reads k = (t, t + 4) of the k-block: the
// builders store W2's k in the same order (even columns in the first four positions of each 8-column block, odd in the
// last four), so the contraction is unchanged.  Every output takes the same products in the same order whatever the grid.
constexpr int kBevBuilders = 128;
constexpr int kBevThreads = kBevBuilders + 256;
constexpr int kBevBN = 64;            // GEMM 2 n-tile
constexpr int kBevStagesA = 1, kBevStagesW = 2;   // 72 KB W1 + 32 KB A (also the output staging) + 2 x 48 KB W2
constexpr int kBevMaxCols = 2048;     // Z * Cf: every CTA splits all of W2 per tile; beyond this that outweighs the tile's output

struct BevSmem {
  int w1, ring_a, ring_w, b1, bars, total;
};
__host__ __device__ inline BevSmem bev_smem(int C) {
  BevSmem m;
  m.w1 = 0;                                                        // W1 hi + lo: (C / 32) atoms x [C rows x 128 B] each
  m.ring_a = 2 * C * C * 4;
  m.ring_w = m.ring_a + kBevStagesA * 2 * kAtomBytesA;             // A stage: hi + lo atom of 128 rows
  m.b1 = m.ring_w + kBevStagesW * 2 * C * kBevBN * 4;              // W2 stage: hi + lo, (C / 32) atoms x [BN rows x 128 B]
  m.bars = m.b1 + C * 4;
  m.total = m.bars + 256 + 1024;
  return m;
}

template <int C>
__global__ void __launch_bounds__(kBevThreads, 1)
bev_decode_tc_kernel(const float* __restrict__ bev, const float* __restrict__ w1, const float* __restrict__ b1,
                     const float* __restrict__ w2, const float* __restrict__ b2, int rows, int Z, int Cf, int zpitch,
                     int feat_pitch, float* __restrict__ vol_sdf, float* __restrict__ vol_feat, int n_tiles) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int KA = C / kAtomK;
  constexpr int kWAtom = kBevBN * 128;                             // bytes of one W2 atom (BN rows)
  const BevSmem L = bev_smem(C);
  uint8_t* w_hi = sm + L.w1;
  uint8_t* w_lo = w_hi + KA * C * 128;
  uint8_t* ring_a = sm + L.ring_a;
  uint8_t* ring_w = sm + L.ring_w;
  float* b1s = reinterpret_cast<float*>(sm + L.b1);
  uint64_t* full_a = reinterpret_cast<uint64_t*>(sm + L.bars);
  uint64_t* empty_a = full_a + kBevStagesA;
  uint64_t* full_w = empty_a + kBevStagesA;
  uint64_t* empty_w = full_w + kBevStagesW;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int N = Z * Cf, n_tiles_w = (N + kBevBN - 1) / kBevBN;

  if (tid == 0) {
    for (int s = 0; s < kBevStagesA; ++s) { mbar_init(full_a + s, kBevBuilders); mbar_init(empty_a + s, 8); }
    for (int s = 0; s < kBevStagesW; ++s) { mbar_init(full_w + s, kBevBuilders); mbar_init(empty_w + s, 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < C * C / 4; i += kBevThreads) {
    const int j = (i * 4) / C, k = (i * 4) % C;
    store_split_tf32(w_hi, w_lo, (uint32_t)((k / kAtomK) * C * 128) + swz_off(j, (k % kAtomK) / 4),
                     __ldg(reinterpret_cast<const float4*>(w1) + i));
  }
  for (int i = tid; i < C; i += kBevThreads) b1s[i] = __ldg(b1 + i);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();

  if (warp < kBevBuilders / 32) {
    // ===== builders =====
    const int c4 = tid & 7, r0 = tid >> 3;                         // A: 16-byte chunk c4 of rows r0 + 16 j
    const int wr = tid >> 2, wq = tid & 3;       // W2: rows wr + 32 i of the n-tile, 8-column block wq of every atom
    constexpr int WR = kBevBN / 32;
    int sa = 0, sw = 0;
    uint32_t pa = 0, pw = 0;
    float4 w[WR][KA][2];                         // the n-tile being loaded: [row][atom][even / odd half of the block]
    auto load_w2 = [&](int nt) {
#pragma unroll
      for (int i = 0; i < WR; ++i) {
        const int n = nt * kBevBN + wr + 32 * i;
#pragma unroll
        for (int a = 0; a < KA; ++a) {
          const float4* src = reinterpret_cast<const float4*>(w2 + (size_t)n * C + a * kAtomK + wq * 8);
          w[i][a][0] = n < N ? __ldg(src) : make_float4(0.f, 0.f, 0.f, 0.f);
          w[i][a][1] = n < N ? __ldg(src + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
    };
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      const int row0 = t * kBM;
      for (int a = 0; a < KA; ++a) {
        float4 x[kBM / 16];
#pragma unroll
        for (int j = 0; j < kBM / 16; ++j) {
          const int r = row0 + r0 + 16 * j;
          x[j] = r < rows ? __ldg(reinterpret_cast<const float4*>(bev + (size_t)r * C + a * kAtomK + c4 * 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        mbar_wait(empty_a + sa, pa ^ 1);
        uint8_t* hi = ring_a + sa * 2 * kAtomBytesA;
#pragma unroll
        for (int j = 0; j < kBM / 16; ++j) build_a_chunk(hi, hi + kAtomBytesA, r0 + 16 * j, c4, x[j], row0 + r0 + 16 * j < rows);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(full_a + sa);
        if (++sa == kBevStagesA) { sa = 0; pa ^= 1; }
      }
      load_w2(0);
      for (int nt = 0; nt < n_tiles_w; ++nt) {
        float4 cur[WR][KA][2];
#pragma unroll
        for (int i = 0; i < WR; ++i)
#pragma unroll
          for (int a = 0; a < KA; ++a) { cur[i][a][0] = w[i][a][0]; cur[i][a][1] = w[i][a][1]; }
        if (nt + 1 < n_tiles_w) load_w2(nt + 1);
        mbar_wait(empty_w + sw, pw ^ 1);
        uint8_t* hi = ring_w + sw * 2 * KA * kWAtom;
#pragma unroll
        for (int i = 0; i < WR; ++i)
#pragma unroll
          for (int a = 0; a < KA; ++a) {
            const float4 u = cur[i][a][0], v = cur[i][a][1];
            uint8_t* ah = hi + a * kWAtom;
            store_split_tf32(ah, ah + KA * kWAtom, swz_off(wr + 32 * i, 2 * wq), make_float4(u.x, u.z, v.x, v.z));      // even
            store_split_tf32(ah, ah + KA * kWAtom, swz_off(wr + 32 * i, 2 * wq + 1), make_float4(u.y, u.w, v.y, v.w));  // odd
          }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        mbar_arrive(full_w + sw);
        if (++sw == kBevStagesW) { sw = 0; pw ^= 1; }
      }
    }
  } else {
    // ===== consumers: warpgroup wg owns rows 64 wg .. 64 wg + 63 of every tile =====
    const int wg = (warp - kBevBuilders / 32) >> 2, wl = warp & 3, g = lane >> 2, t4 = lane & 3;
    const int frag_row = wg * kWgRows + wl * 16 + g;               // this thread's rows: frag_row and frag_row + 8
    const uint32_t whi = smem_u32(w_hi), wlo = smem_u32(w_lo);
    const float inv_cf = 1.0f / (float)Cf;
    const int wrow0 = wg * kWgRows + wl * 16;                       // the warp's 16 rows of every tile
    // the warp's staging: its rows of the A stage's hi (warps 0, 1 of the warpgroup) or lo (warps 2, 3) atom
    float* stage = reinterpret_cast<float*>(ring_a + (wl >> 1) * kAtomBytesA + wg * kWgRows * 128 + (wl & 1) * 32 * 128);
    int sa = 0, sw = 0;
    uint32_t pa = 0, pw = 0;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
      const int row0 = t * kBM;
      // ---- GEMM 1: z1 = a0 W1^T ----
      float acc[C / 2];
#pragma unroll
      for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
      uint32_t accum = 0;
      for (int a = 0; a < KA; ++a) {
        mbar_wait(full_a + sa, pa);
        const uint32_t ahi = smem_u32(ring_a + sa * 2 * kAtomBytesA) + wg * kWgRows * 128, alo = ahi + kAtomBytesA;
        const uint32_t bhi = whi + a * C * 128, blo = wlo + a * C * 128;
#pragma unroll
        for (int i = 0; i < C / 2; ++i) asm volatile("" : "+f"(acc[i])::"memory");
        wg_fence();
#pragma unroll
        for (int prod = 0; prod < 3; ++prod) {
          const uint32_t ab = prod == 1 ? alo : ahi;
          const uint32_t bb = prod == 2 ? blo : bhi;
#pragma unroll
          for (int k = 0; k < kAtomK / 8; ++k) {
            Wgmma<C>::ss(acc, make_desc(ab + k * 32), make_desc(bb + k * 32), accum);
            accum = 1u;
          }
        }
        wg_commit();
        wg_wait0();
#pragma unroll
        for (int i = 0; i < C / 2; ++i) asm volatile("" : "+f"(acc[i])::"memory");
        __syncwarp();
        if (lane == 0 && a < KA - 1) mbar_arrive(empty_a + sa);      // the last atom's rows stage the output (below)
        if (a < KA - 1 && ++sa == kBevStagesA) { sa = 0; pa ^= 1; }
      }
      // ---- a1 = softplus(z1 + b1) as GEMM 2's A fragments, split into TF32 hi / lo ----
      uint32_t fh[C / 8][4], fl[C / 8][4];
#pragma unroll
      for (int j = 0; j < C / 8; ++j) {
        const int col = 8 * j + 2 * t4;
        const float h[4] = {softplus_fast(acc[4 * j] + b1s[col]), softplus_fast(acc[4 * j + 2] + b1s[col]),
                            softplus_fast(acc[4 * j + 1] + b1s[col + 1]), softplus_fast(acc[4 * j + 3] + b1s[col + 1])};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float hh = tf32_rn(h[q]);
          fh[j][q] = __float_as_uint(hh);
          fl[j][q] = __float_as_uint(h[q] - hh);
        }
      }
      // ---- GEMM 2, one n-tile of W2 at a time.  Epilogue: the warp's 16 rows x BN columns go through its own 4 KB of the A
      // stage (rows this warpgroup read in GEMM 1, free until the next tile's A), then out row by row while the next
      // n-tile's products run: column n = z * Cf + c -> voxel (r, z), channel c, so 32 lanes write 32 consecutive columns,
      // one contiguous run of vol_feat (and the few sdf entries among them).
      auto write_out = [&](int nt) {
        int zq[2], cq[2];
        float bq[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int n = nt * kBevBN + lane + 32 * q;
          // (n + 1/2) / Cf is at least 1/(2 Cf) away from an integer, far beyond the product's rounding: the floor is exact
          zq[q] = __float2int_rd(((float)n + 0.5f) * inv_cf);
          cq[q] = n < N ? n - zq[q] * Cf : -1;
          bq[q] = n < N ? __ldg(b2 + n) : 0.f;
        }
#pragma unroll 4
        for (int lr = 0; lr < 16; ++lr) {
          const int r = row0 + wrow0 + lr;
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const float o = stage[lr * kBevBN + ((lane + 32 * q) ^ ((lr & 7) << 3))] + bq[q];
            if (r >= rows) continue;
            if (cq[q] == 0) vol_sdf[(size_t)r * zpitch + zq[q]] = o;
            else if (cq[q] > 0) vol_feat[((size_t)r * Z + zq[q]) * feat_pitch + (cq[q] - 1)] = o;
          }
        }
      };
      for (int nt = 0; nt < n_tiles_w; ++nt) {
        mbar_wait(full_w + sw, pw);
        const uint32_t bhi = smem_u32(ring_w + sw * 2 * KA * kWAtom), blo = bhi + KA * kWAtom;
        float acc2[kBevBN / 2];
#pragma unroll
        for (int i = 0; i < kBevBN / 2; ++i) acc2[i] = 0.f;
#pragma unroll
        for (int j = 0; j < C / 8; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) asm volatile("" : "+r"(fh[j][q]), "+r"(fl[j][q])::"memory");
        wg_fence();
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const uint32_t off = (j / 4) * kWAtom + (j % 4) * 32;
          Wgmma<kBevBN>::rs(acc2, fh[j], make_desc(bhi + off), j ? 1u : 0u);
          Wgmma<kBevBN>::rs(acc2, fl[j], make_desc(bhi + off), 1u);
          Wgmma<kBevBN>::rs(acc2, fh[j], make_desc(blo + off), 1u);
        }
        wg_commit();
        if (nt > 0) write_out(nt - 1);
        wg_wait0();
#pragma unroll
        for (int i = 0; i < kBevBN / 2; ++i) asm volatile("" : "+f"(acc2[i])::"memory");
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_w + sw);
        if (++sw == kBevStagesW) { sw = 0; pw ^= 1; }
#pragma unroll
        for (int jb = 0; jb < kBevBN / 8; ++jb)
#pragma unroll
          for (int hr = 0; hr < 2; ++hr)
            *reinterpret_cast<float2*>(stage + (g + 8 * hr) * kBevBN + ((8 * jb + 2 * t4) ^ (g << 3))) =
                make_float2(acc2[4 * jb + 2 * hr], acc2[4 * jb + 2 * hr + 1]);
        __syncwarp();
      }
      write_out(n_tiles_w - 1);
      __syncwarp();
      if (lane == 0) mbar_arrive(empty_a + sa);                     // the staging rows are free for the next tile's A
      if (++sa == kBevStagesA) { sa = 0; pa ^= 1; }
    }
  }
}

// ---- BEV decode backward pieces (BEVDecodeFunction: the products run on the 3xTF32 GEMM / cuBLAS between them) ----
// g_out[r][z * Cf + c] of rows [row_begin, row_begin + n / N) gathered from the volume gradients (NULL: zero; pads ignored)
__global__ void __launch_bounds__(256) bev_decode_bwd_gather_kernel(const float* __restrict__ g_vs, const float* __restrict__ g_vf,
                                                                    int Z, int zpitch, int Cf, int feat_pitch, long long row_begin,
                                                                    long long n, float* __restrict__ g_out) {
  const int N = Z * Cf;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = row_begin + i / N;
    const int col = (int)(i % N), z = col / Cf, c = col - z * Cf;
    float g = 0.f;
    if (c == 0) { if (g_vs) g = __ldg(g_vs + r * zpitch + z); }
    else if (g_vf) g = __ldg(g_vf + (r * Z + z) * feat_pitch + c - 1);
    g_out[i] = g;
  }
}

// a0 = softplus(x), accurate relative to its value (softplus_rel)
__global__ void __launch_bounds__(256) bev_decode_bwd_features_kernel(const float* __restrict__ x, long long n, float* __restrict__ a0) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    a0[i] = softplus_rel(__ldg(x + i));
}

// z1 -> a1 = softplus(z1) in place, g1 *= sigmoid(z1) (one exponential: softplus_sigmoid)
__global__ void __launch_bounds__(256) bev_decode_bwd_hidden_kernel(float* __restrict__ z1_a1, float* __restrict__ g1, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float sg;
    z1_a1[i] = softplus_sigmoid(z1_a1[i], &sg);
    g1[i] *= sg;
  }
}

__global__ void zero_pad_kernel(float* vol_sdf, long long columns, int Z, int zpitch) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  int pad = zpitch - Z;
  if (i >= columns * pad) return;
  long long col = i / pad;
  int z = Z + (int)(i - col * pad);
  vol_sdf[col * zpitch + z] = 0.f;
}

template <int C>
int launch_decode(const float* hw, const float* zh, const float* wz, const float* w1, const float* b1, const float* w2,
                  const float* b2, const so_volume_desc* d, float* vol_sdf, float* vol_feat, int h_begin, int h_count, cudaStream_t st) {
  constexpr int LD = C + 4;
  size_t smem = sizeof(float) * ((size_t)kRows * LD + (size_t)C * LD + (size_t)kMaxOut * C + C + kMaxOut);
  static PerDeviceOnce attr_simt;
  int rc_attr = attr_simt.run([smem] {
    return check_cuda(cudaFuncSetAttribute(tpv_decode_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  });
  if (rc_attr) return rc_attr;
  dim3 grid((unsigned)ceil_div64((int64_t)d->W * d->Z, kRows), (unsigned)h_count);
  ProfScope prof(1, st);
  tpv_decode_kernel<C><<<grid, kThreads, smem, st>>>(hw, zh, wz, w1, b1, w2, b2, d->H, d->W, d->Z, d->zpitch,
                                                       1 + d->n_feat, d->feat_pitch, vol_sdf, vol_feat, h_begin);
  note_launch(1);
  return check_launch();
}

}  // namespace so

using namespace so;

static bool g_decode_force_simt = false;
// Test hook: 1 = use the fp32 SIMT decode kernel even where the tensor-core kernel applies (both are parity-tested).
extern "C" int so_tpv_decode_force_simt(int on) { g_decode_force_simt = on != 0; return SO_OK; }

extern "C" int so_tpv_decode(const float* tpv_hw, const float* tpv_zh, const float* tpv_wz, int32_t C, const float* w1,
                             const float* b1, const float* w2, const float* b2, const so_volume_desc* d,
                             float* vol_sdf, float* vol_feat, void* stream) {
  if (!d) return SO_ERR_INVALID_ARG;
  return so_tpv_decode_rows(tpv_hw, tpv_zh, tpv_wz, C, w1, b1, w2, b2, d, 0, d->H, vol_sdf, vol_feat, stream);
}

// Row range [h_begin, h_begin + h_count) of the volume only (voxel-sharded decode across GPUs: every rank decodes its
// slab of h rows into the full-size volume buffer, one all_gather assembles it).  Rows outside the range are untouched.
extern "C" int so_tpv_decode_rows(const float* tpv_hw, const float* tpv_zh, const float* tpv_wz, int32_t C, const float* w1,
                                  const float* b1, const float* w2, const float* b2, const so_volume_desc* d, int32_t h_begin,
                                  int32_t h_count, float* vol_sdf, float* vol_feat, void* stream) {
  if (!tpv_hw || !tpv_zh || !tpv_wz || !w1 || !b1 || !w2 || !b2 || !vol_sdf) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(d);
  if (rc) return rc;
  if (h_begin < 0 || h_count < 0 || h_begin + h_count > d->H) return SO_ERR_INVALID_ARG;
  if (h_count == 0) return SO_OK;
  if (d->n_feat > 0 && !vol_feat) return SO_ERR_INVALID_ARG;
  if (1 + d->n_feat > kMaxOut) return SO_ERR_UNSUPPORTED;
  if (C != 32 && C != 64 && C != 96 && C != 128) return SO_ERR_UNSUPPORTED;   // before the pad kernel below is launched
  if (d->H > 65535) return SO_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  if (d->zpitch > d->Z) {
    long long cols = (long long)h_count * d->W, n = cols * (d->zpitch - d->Z);
    zero_pad_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(vol_sdf + (long long)h_begin * d->W * d->zpitch, cols, d->Z, d->zpitch);
    note_launch(1);
  }
  if (C % 32 == 0 && C >= 32 && C <= 128 && !g_decode_force_simt) {
    const int n_out = 1 + d->n_feat;
    DecSmem Ls = dec_smem(C, n_out);
    if (Ls.stages >= 2) {
      static PerDeviceOnce attr_tc;
      if ((rc = attr_tc.run([] {
             int r = SO_OK;
#define SO_DEC_ATTR(C_, NO) if (!r) r = check_cuda(cudaFuncSetAttribute(tpv_decode_tc_kernel<C_, NO>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024))
#define SO_DEC_ATTR_C(C_) SO_DEC_ATTR(C_, 1); SO_DEC_ATTR(C_, 4); SO_DEC_ATTR(C_, 32)
             SO_DEC_ATTR_C(32); SO_DEC_ATTR_C(64); SO_DEC_ATTR_C(96); SO_DEC_ATTR_C(128);
#undef SO_DEC_ATTR_C
#undef SO_DEC_ATTR
             return r;
           })))
        return rc;
      const int tiles_per_row = (int)ceil_div64((int64_t)d->W * d->Z, kBM);
      const int n_tiles = tiles_per_row * h_count;
      const int sms = num_sms(), grid = n_tiles < sms ? n_tiles : sms;
      ProfScope prof(1, st);
#define SO_DEC_TC(C_, NO) tpv_decode_tc_kernel<C_, NO><<<grid, kDecThreads, Ls.total, st>>>(tpv_hw, tpv_zh, tpv_wz, w1, b1, w2, b2, d->H, d->W, \
                                                                                  d->Z, d->zpitch, n_out, d->feat_pitch, vol_sdf, vol_feat, tiles_per_row, n_tiles, h_begin)
#define SO_DEC_TC_C(C_) if (n_out == 1) SO_DEC_TC(C_, 1); else if (n_out <= 4) SO_DEC_TC(C_, 4); else SO_DEC_TC(C_, 32)
      switch (C) {
        case 32: SO_DEC_TC_C(32); break;
        case 64: SO_DEC_TC_C(64); break;
        case 96: SO_DEC_TC_C(96); break;
        default: SO_DEC_TC_C(128); break;
      }
#undef SO_DEC_TC_C
#undef SO_DEC_TC
      note_launch(1);
      return check_launch();
    }
  }
  switch (C) {
    case 32: return launch_decode<32>(tpv_hw, tpv_zh, tpv_wz, w1, b1, w2, b2, d, vol_sdf, vol_feat, h_begin, h_count, st);
    case 64: return launch_decode<64>(tpv_hw, tpv_zh, tpv_wz, w1, b1, w2, b2, d, vol_sdf, vol_feat, h_begin, h_count, st);
    case 96: return launch_decode<96>(tpv_hw, tpv_zh, tpv_wz, w1, b1, w2, b2, d, vol_sdf, vol_feat, h_begin, h_count, st);
    case 128: return launch_decode<128>(tpv_hw, tpv_zh, tpv_wz, w1, b1, w2, b2, d, vol_sdf, vol_feat, h_begin, h_count, st);
    default: return SO_ERR_UNSUPPORTED;
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward of the decode MLP, one slab of h rows at a time (reference: autograd through TPVDecoder.forward,
// model/head/base_head... the SDF/colour MLP in model/head/neus_head/bev_nerf.py:150-190 at the 1.65 M voxel centres).
// The two M x C x C products of each slab run on the tensor-core 3xTF32 GEMM (so_linear_3xtf32); the kernels here are the
// element-wise pieces fused around them so every slab intermediate is written once and read once:
//   features:  a0 = softplus(hw + zh + wz)                                       (recomputed, never stored by forward)
//   hidden:    z1 -> a1 = softplus(z1);  g1 = (W2^T g_out) * sigmoid(z1);  g_out packed [rows][n_out]
//   input:     g0 *= sigmoid(f) = 1 - exp(-a0)
// sigmoid(x) = 1 - exp(-softplus(x)) lets the input kernel reuse a0 without keeping the pre-activation; the hidden kernel
// has z1 in hand and takes its sigmoid from the same exponential as the softplus.  All three use the relative-accuracy
// forms above (softplus_rel, softplus_sigmoid, sigmoid_of_softplus).
__global__ void __launch_bounds__(256) decode_bwd_features_kernel(const float* __restrict__ hw, const float* __restrict__ zh,
                                                                  const float* __restrict__ wz, int C4, int H, int W, int Z,
                                                                  int h_begin, long long n_vec, float4* __restrict__ a0) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    long long v = i / C4;
    int c4 = (int)(i - v * C4);
    int z = (int)(v % Z);
    long long t = v / Z;
    int w = (int)(t % W), h = h_begin + (int)(t / W);
    float4 a = __ldg(reinterpret_cast<const float4*>(hw + ((size_t)h * W + w) * C4 * 4) + c4);
    float4 b = __ldg(reinterpret_cast<const float4*>(zh + ((size_t)z * H + h) * C4 * 4) + c4);
    float4 c = __ldg(reinterpret_cast<const float4*>(wz + ((size_t)w * Z + z) * C4 * 4) + c4);
    a0[i] = make_float4(softplus_rel(a.x + b.x + c.x), softplus_rel(a.y + b.y + c.y), softplus_rel(a.z + b.z + c.z),
                        softplus_rel(a.w + b.w + c.w));
  }
}

constexpr int kBwdMaxOut = 32;
__global__ void __launch_bounds__(256) decode_bwd_hidden_kernel(float4* __restrict__ z1_a1, const float* __restrict__ g_vs,
                                                                const float* __restrict__ g_vf, const float* __restrict__ w2,
                                                                int C4, int W, int Z, int zpitch, int n_out, int feat_pitch,
                                                                int h_begin, long long n_vec, float4* __restrict__ g1,
                                                                float* __restrict__ g_out) {
  extern __shared__ float4 w2s[];  // [n_out][C4]
  for (int i = threadIdx.x; i < n_out * C4; i += blockDim.x) w2s[i] = __ldg(reinterpret_cast<const float4*>(w2) + i);
  __syncthreads();
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    long long v = i / C4;
    int c4 = (int)(i - v * C4);
    int z = (int)(v % Z);
    long long col = (long long)h_begin * W + v / Z;  // (h, w) column of the full volume
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float go = g_vs ? __ldg(g_vs + col * zpitch + z) : 0.f;
    {
      float4 wv = w2s[c4];
      acc.x = go * wv.x; acc.y = go * wv.y; acc.z = go * wv.z; acc.w = go * wv.w;
    }
    if (c4 == 0) g_out[v * n_out] = go;
    const float* gf = g_vf ? g_vf + (col * Z + z) * feat_pitch : nullptr;
    for (int o = 1; o < n_out; ++o) {
      float g = gf ? __ldg(gf + o - 1) : 0.f;
      float4 wv = w2s[o * C4 + c4];
      acc.x = fmaf(g, wv.x, acc.x); acc.y = fmaf(g, wv.y, acc.y); acc.z = fmaf(g, wv.z, acc.z); acc.w = fmaf(g, wv.w, acc.w);
      if (c4 == 0) g_out[v * n_out + o] = g;
    }
    float4 zv = z1_a1[i];
    float4 a, sg;
    a.x = softplus_sigmoid(zv.x, &sg.x); a.y = softplus_sigmoid(zv.y, &sg.y);
    a.z = softplus_sigmoid(zv.z, &sg.z); a.w = softplus_sigmoid(zv.w, &sg.w);
    z1_a1[i] = a;
    g1[i] = make_float4(acc.x * sg.x, acc.y * sg.y, acc.z * sg.z, acc.w * sg.w);
  }
}

__global__ void __launch_bounds__(256) decode_bwd_input_kernel(float4* __restrict__ g0, const float4* __restrict__ a0, long long n_vec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    float4 g = g0[i], a = __ldg(a0 + i);
    g0[i] = make_float4(g.x * sigmoid_of_softplus(a.x), g.y * sigmoid_of_softplus(a.y), g.z * sigmoid_of_softplus(a.z),
                        g.w * sigmoid_of_softplus(a.w));
  }
}

static inline bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }
static int bwd_slab_check(const so_volume_desc* d, int32_t C, int32_t h_begin, int32_t h_count) {
  int rc = validate_volume(d);
  if (rc) return rc;
  if (C <= 0 || C % 4) return SO_ERR_UNSUPPORTED;
  if (h_begin < 0 || h_count < 0 || h_begin + h_count > d->H) return SO_ERR_INVALID_ARG;
  return SO_OK;
}
static unsigned bwd_grid(long long n_vec) {
  long long g = ceil_div64(n_vec, 256), cap = (long long)num_sms() * 16;
  return (unsigned)(g < cap ? g : cap);
}

extern "C" int so_tpv_decode_bwd_features(const float* tpv_hw, const float* tpv_zh, const float* tpv_wz, int32_t C,
                                          const so_volume_desc* d, int32_t h_begin, int32_t h_count, float* a0, void* stream) {
  if (!tpv_hw || !tpv_zh || !tpv_wz || !a0) return SO_ERR_INVALID_ARG;
  int rc = bwd_slab_check(d, C, h_begin, h_count);
  if (rc) return rc;
  if (misaligned16(tpv_hw) || misaligned16(tpv_zh) || misaligned16(tpv_wz) || misaligned16(a0)) return SO_ERR_INVALID_ARG;
  long long n_vec = (long long)h_count * d->W * d->Z * (C / 4);
  if (n_vec == 0) return SO_OK;
  decode_bwd_features_kernel<<<bwd_grid(n_vec), 256, 0, (cudaStream_t)stream>>>(tpv_hw, tpv_zh, tpv_wz, C / 4, d->H, d->W, d->Z, h_begin,
                                                                              n_vec, reinterpret_cast<float4*>(a0));
  note_launch(1);
  return check_launch();
}

extern "C" int so_tpv_decode_bwd_hidden(float* z1_a1, const float* g_vol_sdf, const float* g_vol_feat, const float* w2, int32_t C,
                                        const so_volume_desc* d, int32_t h_begin, int32_t h_count, float* g1, float* g_out,
                                        void* stream) {
  if (!z1_a1 || !w2 || !g1 || !g_out) return SO_ERR_INVALID_ARG;
  int rc = bwd_slab_check(d, C, h_begin, h_count);
  if (rc) return rc;
  const int n_out = 1 + d->n_feat;
  if (n_out > kBwdMaxOut) return SO_ERR_UNSUPPORTED;
  if (misaligned16(z1_a1) || misaligned16(w2) || misaligned16(g1)) return SO_ERR_INVALID_ARG;
  long long n_vec = (long long)h_count * d->W * d->Z * (C / 4);
  if (n_vec == 0) return SO_OK;
  size_t smem = (size_t)n_out * C * sizeof(float);
  if (smem > 48 * 1024) return SO_ERR_UNSUPPORTED;
  decode_bwd_hidden_kernel<<<bwd_grid(n_vec), 256, smem, (cudaStream_t)stream>>>(
      reinterpret_cast<float4*>(z1_a1), g_vol_sdf, d->n_feat ? g_vol_feat : nullptr, w2, C / 4, d->W, d->Z, d->zpitch, n_out, d->feat_pitch,
      h_begin, n_vec, reinterpret_cast<float4*>(g1), g_out);
  note_launch(1);
  return check_launch();
}

extern "C" int so_tpv_decode_bwd_input(float* g0, const float* a0, int64_t n, void* stream) {
  if (!g0 || !a0 || n < 0 || n % 4) return SO_ERR_INVALID_ARG;
  if (misaligned16(g0) || misaligned16(a0)) return SO_ERR_INVALID_ARG;
  if (n == 0) return SO_OK;
  decode_bwd_input_kernel<<<bwd_grid(n / 4), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<float4*>(g0), reinterpret_cast<const float4*>(a0), n / 4);
  note_launch(1);
  return check_launch();
}

extern "C" int so_bev_decode(const float* bev, int32_t C, const float* w1, const float* b1, const float* w2, const float* b2,
                             const so_volume_desc* d, float* vol_sdf, float* vol_feat, void* stream) {
  if (!bev || !w1 || !b1 || !w2 || !b2 || !vol_sdf) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(d);
  if (rc) return rc;
  if (d->n_feat > 0 && !vol_feat) return SO_ERR_INVALID_ARG;
  if (C != 96) return SO_ERR_UNSUPPORTED;
  if ((int64_t)d->Z * (1 + d->n_feat) > kBevMaxCols) return SO_ERR_UNSUPPORTED;
  if (misaligned16(bev) || misaligned16(w1) || misaligned16(w2)) return SO_ERR_INVALID_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const long long cols = (long long)d->H * d->W;
  if (d->zpitch > d->Z) {
    long long n = cols * (d->zpitch - d->Z);
    zero_pad_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, st>>>(vol_sdf, cols, d->Z, d->zpitch);
    note_launch(1);
  }
  const BevSmem L = bev_smem(96);
  static PerDeviceOnce attr;
  if ((rc = attr.run([&L] {
         return check_cuda(cudaFuncSetAttribute(bev_decode_tc_kernel<96>, cudaFuncAttributeMaxDynamicSharedMemorySize, L.total));
       })))
    return rc;
  const int n_tiles = (int)ceil_div64(cols, kBM), sms = num_sms(), grid = n_tiles < sms ? n_tiles : sms;
  bev_decode_tc_kernel<96><<<grid, kBevThreads, L.total, st>>>(bev, w1, b1, w2, b2, (int)cols, d->Z, 1 + d->n_feat, d->zpitch,
                                                              d->feat_pitch, vol_sdf, vol_feat, n_tiles);
  note_launch(1);
  return check_launch();
}

extern "C" int so_bev_decode_bwd_gather(const float* g_vol_sdf, const float* g_vol_feat, const so_volume_desc* d, int64_t row_begin,
                                        int64_t row_count, float* g_out, void* stream) {
  if (!g_out) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(d);
  if (rc) return rc;
  if (row_begin < 0 || row_count < 0 || row_begin + row_count > (int64_t)d->H * d->W) return SO_ERR_INVALID_ARG;
  const long long n = row_count * (long long)d->Z * (1 + d->n_feat);
  if (n == 0) return SO_OK;
  bev_decode_bwd_gather_kernel<<<bwd_grid(n), 256, 0, (cudaStream_t)stream>>>(g_vol_sdf, d->n_feat ? g_vol_feat : nullptr, d->Z,
                                                                             d->zpitch, 1 + d->n_feat, d->feat_pitch, row_begin, n, g_out);
  note_launch(1);
  return check_launch();
}

extern "C" int so_bev_decode_bwd_features(const float* bev, int64_t n, float* a0, void* stream) {
  if (!bev || !a0 || n < 0) return SO_ERR_INVALID_ARG;
  if (n == 0) return SO_OK;
  bev_decode_bwd_features_kernel<<<bwd_grid(n), 256, 0, (cudaStream_t)stream>>>(bev, n, a0);
  note_launch(1);
  return check_launch();
}

extern "C" int so_bev_decode_bwd_hidden(float* z1_a1, float* g1, int64_t n, void* stream) {
  if (!z1_a1 || !g1 || n < 0) return SO_ERR_INVALID_ARG;
  if (n == 0) return SO_OK;
  bev_decode_bwd_hidden_kernel<<<bwd_grid(n), 256, 0, (cudaStream_t)stream>>>(z1_a1, g1, n);
  note_launch(1);
  return check_launch();
}
