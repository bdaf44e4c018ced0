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
  // F.softplus(beta=1, threshold=20): max(x,0) + log1p(exp(-|x|)); identical to x beyond the threshold in fp32
  return fmaxf(x, 0.f) + __logf(1.0f + __expf(-fabsf(x)));
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
    float4 v = __ldg(reinterpret_cast<const float4*>(w1) + i), h, l;
    h.x = tf32_rn(v.x); l.x = v.x - h.x; h.y = tf32_rn(v.y); l.y = v.y - h.y;
    h.z = tf32_rn(v.z); l.z = v.z - h.z; h.w = tf32_rn(v.w); l.w = v.w - h.w;
    uint32_t off = (uint32_t)((k / kAtomK) * C * 128) + swz_off(j, (k % kAtomK) / 4);
    *reinterpret_cast<float4*>(w_hi + off) = h;
    *reinterpret_cast<float4*>(w_lo + off) = l;
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
        for (int j = 0; j < 4; ++j) {
          float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
          if (vv[j] < WZ) {
            f.x = softplus_fast(x[j].x + y[j].x + u[j].x); f.y = softplus_fast(x[j].y + y[j].y + u[j].y);
            f.z = softplus_fast(x[j].z + y[j].z + u[j].z); f.w = softplus_fast(x[j].w + y[j].w + u[j].w);
          }
          float4 hh, ll;
          hh.x = tf32_rn(f.x); ll.x = f.x - hh.x; hh.y = tf32_rn(f.y); ll.y = f.y - hh.y;
          hh.z = tf32_rn(f.z); ll.z = f.z - hh.z; hh.w = tf32_rn(f.w); ll.w = f.w - hh.w;
          const uint32_t off = swz_off(r0 + 32 * j, c4);
          *reinterpret_cast<float4*>(hi + off) = hh;
          *reinterpret_cast<float4*>(lo + off) = ll;
        }
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
// sigmoid(x) = 1 - exp(-softplus(x)) lets the activations be reused without keeping the pre-activations.
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
    a0[i] = make_float4(softplus_fast(a.x + b.x + c.x), softplus_fast(a.y + b.y + c.y), softplus_fast(a.z + b.z + c.z),
                        softplus_fast(a.w + b.w + c.w));
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
    float4 a = make_float4(softplus_fast(zv.x), softplus_fast(zv.y), softplus_fast(zv.z), softplus_fast(zv.w));
    z1_a1[i] = a;
    g1[i] = make_float4(acc.x * (1.f - __expf(-a.x)), acc.y * (1.f - __expf(-a.y)), acc.z * (1.f - __expf(-a.z)),
                        acc.w * (1.f - __expf(-a.w)));
  }
}

__global__ void __launch_bounds__(256) decode_bwd_input_kernel(float4* __restrict__ g0, const float4* __restrict__ a0, long long n_vec) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_vec; i += (long long)gridDim.x * blockDim.x) {
    float4 g = g0[i], a = __ldg(a0 + i);
    g0[i] = make_float4(g.x * (1.f - __expf(-a.x)), g.y * (1.f - __expf(-a.y)), g.z * (1.f - __expf(-a.z)), g.w * (1.f - __expf(-a.w)));
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
