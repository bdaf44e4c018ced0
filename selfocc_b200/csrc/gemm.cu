// Dense projections of the lifting path on the Hopper tensor cores (SURVEY.md section 8a rows A6, A9: value / offset /
// weight / output Linear, FFN) with fp32-level accuracy:  Y = act(X W^T + b) [+ R]
//
//   X [M, K] fp32, W [N, K] fp32 (torch Linear layout, both K-major)  ->  Y [M, N] fp32
//
// Accuracy: the path feeds a 1e-4-relative depth bar, so plain TF32 (10-bit mantissa) is not acceptable.  Each
// operand is split  v = hi + lo,  hi = v rounded to the nearest TF32 number (low 13 mantissa bits zero), lo = v - hi
// (exact in fp32), and the product is accumulated as  hi*hi + lo*hi + hi*lo  in the fp32 register accumulator
// ("3xTF32", error ~2^-21).  W is split once on the host side (so_split_tf32); X is split by the consumer warps.
// Every output element takes the same products in the same order (32-wide k-atoms ascending; per atom hi*hi, lo*hi,
// hi*lo; per product 4 k-steps of 8), whatever the tile width, M or the CTA: results are bit-reproducible across
// shardings of the rows.
//
// Persistent, warp-specialised ping-pong pipeline (one CTA per SM, 9 warps):
//   warp 8      TMA producer   W tile (hi, lo; all K) once per CTA, then X atoms [64 x 32] (128B swizzle) into a ring of stages
//   warps 0-7   two consumer warpgroups.  The CTA's m-tiles (64 rows each) alternate between them, so one warpgroup's
//               epilogue (+bias, ReLU, +residual, optional LayerNorm over the row; registers -> global) runs while the
//               other issues its MMAs.  Per k-atom: split the X atom into hi / lo, then 3 products x 4 k-steps of
//               wgmma.m64nBNk8.f32.tf32 into a register accumulator.
// A CTA owns ONE n-tile (its W tile stays resident in shared memory) and walks m-tiles, so the streamed traffic per
// output tile is the X tile and the Y tile only.  mbarriers: w_full | full[s] (TMA landed) -> empty[s] (stage consumed).
// Each warpgroup has its own half of the ring, so every stage has one consumer and each warpgroup waits on consecutive
// fills of its own stages (with one shared ring, a warpgroup waiting K/32 atoms ahead of the producer could take an
// older phase of the same parity for its own).
//
// The A operand (X hi / lo) comes from REGISTERS: each thread loads its wgmma fragment from the swizzled stage and
// splits it in registers, so the tensor core reads only W from shared memory and a stage holds the raw X atom only.
// Two fragment sets: atom a + 1 is loaded and split while the MMAs of atom a run (wgmma.wait_group 1).
//
// Tuning, one H100 80GB HBM3 at a 400 W power limit, the 12 launches of one encoder layer (scripts/bench_gemm.py, sum):
//   both warpgroups on one 128-row tile, wait_group 0 per atom, BN = fewest padded columns   1.244 ms
//   ping-pong 64-row tiles, two fragment sets at every BN (before the ring split; spills)    1.027 ms
//   ping-pong, ring halves per warpgroup, two fragment sets at BN <= 80, BN by bn_cost       1.038 ms  (shipped)
//   bn_cost picks BN = 80 for N = 3456: 0.138 -> 0.100 ms per zh / wz launch.  The 64-row tiles are slower for
//   M = 7967 x N = 96 with LayerNorm (0.016 -> 0.031 ms: 125 CTAs with one tile each, one warpgroup busy).
#include "tc_common.cuh"

namespace so {

constexpr int kGemmConsumers = 256;                 // two warpgroups
constexpr int kGemmThreads = kGemmConsumers + 32;   // + the TMA producer warp
constexpr int kGemmTileM = kWgRows;                 // rows per m-tile: one warpgroup, one m64 wgmma
constexpr int kGemmTileBytes = kGemmTileM * 128;    // one X atom of one m-tile
constexpr int kMaxStages = 12;
constexpr int kMaxBN = 128;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 2-D row-major fp32 matrix [rows, cols] (cols contiguous), box = [box_rows x 32 floats], 128-byte swizzle, zero OOB fill
static int make_tmap(CUtensorMap* m, const float* base, int64_t rows, int64_t cols, int box_rows) {  // box = [box_rows x 32]
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return SO_ERR_CUDA;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols * 4};
  cuuint32_t box[2] = {(cuuint32_t)kAtomK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? SO_OK : SO_ERR_CUDA;
}

struct PipeCfg {
  int BN, KA, stages;       // n-tile width, atoms along K (K / 32), ring depth (one raw X atom per stage)
  int w_bytes;              // resident W bytes = 2 * KA * BN * 128
  int smem;                 // dynamic shared memory request (incl. 1 KB alignment slack)
  int n_tiles, m_tiles, groups;  // grid = n_tiles x groups CTAs; group g walks m-tiles g, g + groups, ...
};

// Per-CTA cost of an n-tile width: the m-tiles of the busiest CTA times (BN + a fixed per-tile cost, in columns, for
// loading and splitting the X tile).  Balances padding against filling the SMs: N = 3456 at BN = 128 gives 27 n-tiles,
// 4 CTAs each, 108 of 132 SMs busy; BN = 80 gives 44 n-tiles x 3 = 132.
static long long bn_cost(int bn, int N, int m_tiles, int sms, int* n_tiles_out, int* groups_out) {
  const int n_tiles = (int)ceil_div64(N, bn);
  int groups = sms / n_tiles;
  if (groups < 1) groups = 1;
  if (groups > m_tiles) groups = m_tiles;
  if (n_tiles_out) *n_tiles_out = n_tiles;
  if (groups_out) *groups_out = groups;
  constexpr int kTileCostCols = 32;
  return ceil_div64(m_tiles, groups) * (long long)(bn + kTileCostCols) * ((n_tiles + sms - 1) / sms);
}

// n-tile width: the lowest bn_cost, ties to the wider tile.  The LayerNorm epilogue needs the whole row in one tile.
static int pick_bn(int N, int m_tiles, int sms, bool whole_row) {
  if (whole_row) return N;
  int best = kMaxBN;
  long long best_cost = bn_cost(kMaxBN, N, m_tiles, sms, nullptr, nullptr);
  for (int bn : {96, 80, 64, 32}) {
    const long long c = bn_cost(bn, N, m_tiles, sms, nullptr, nullptr);
    if (c < best_cost) { best = bn; best_cost = c; }
  }
  return best;
}

static PipeCfg make_pipe_cfg(int64_t M, int N, int K, bool whole_row, int sms) {
  PipeCfg c;
  c.m_tiles = (int)ceil_div64(M, kGemmTileM);
  c.BN = pick_bn(N, c.m_tiles, sms, whole_row);
  bn_cost(c.BN, N, c.m_tiles, sms, &c.n_tiles, &c.groups);
  c.KA = K / kAtomK;
  c.w_bytes = 2 * c.KA * c.BN * 128;
  const int fixed = c.w_bytes + 256;                          // + mbarriers
  c.stages = (227 * 1024 - 1024 - fixed) / kGemmTileBytes & ~1;  // even: half of the ring per warpgroup
  if (c.stages > kMaxStages) c.stages = kMaxStages;
  c.smem = fixed + c.stages * kGemmTileBytes + 1024;
  return c;
}

// keeps the compiler from moving accumulator / A-fragment reads and writes across the asynchronous wgmma
template <int NR>
__device__ __forceinline__ void fence_regs(float* r) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+f"(r[i])::"memory");
}
template <int NR>
__device__ __forceinline__ void fence_regs(uint32_t* r) {
#pragma unroll
  for (int i = 0; i < NR; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// next position (stage s, phase ph) in a ring of n stages
__device__ __forceinline__ void ring_advance(int& s, uint32_t& ph, int n) {
  if (++s == n) { s = 0; ph ^= 1; }
}

// register-A fragment of one 64-row X atom: rows frag_row and frag_row + 8, k = 8 kk + t and 8 kk + t + 4, i.e. 16-byte
// chunks 2 kk and 2 kk + 1; both rows have (row & 7) == g, so the swizzle is the same for the pair.  Split into hi / lo.
__device__ __forceinline__ void load_split_frag(const uint8_t* stage, int frag_row, int g, int t, uint32_t* ah, uint32_t* al) {
  const uint8_t* r0 = stage + frag_row * 128 + 4 * t;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const float v[4] = {*reinterpret_cast<const float*>(r0 + (((2 * kk) ^ g) << 4)),
                        *reinterpret_cast<const float*>(r0 + 8 * 128 + (((2 * kk) ^ g) << 4)),
                        *reinterpret_cast<const float*>(r0 + (((2 * kk + 1) ^ g) << 4)),
                        *reinterpret_cast<const float*>(r0 + 8 * 128 + (((2 * kk + 1) ^ g) << 4))};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float h = tf32_rn(v[i]);
      ah[4 * kk + i] = __float_as_uint(h);
      al[4 * kk + i] = __float_as_uint(v[i] - h);
    }
  }
  fence_regs<16>(ah);
  fence_regs<16>(al);
}

// the 12 MMAs of one k-atom, A from registers: hi*hi, lo*hi, hi*lo, 4 k-steps each, as one commit group
template <int BN>
__device__ __forceinline__ void mma_atom_rs(float* acc, uint32_t* ah, uint32_t* al, uint32_t bhi, uint32_t blo, uint32_t& accum) {
  fence_regs<BN / 2>(acc);
  wg_fence();
#pragma unroll
  for (int prod = 0; prod < 3; ++prod) {
    const uint32_t* af = prod == 1 ? al : ah;
    const uint32_t bb = prod == 2 ? blo : bhi;
#pragma unroll
    for (int kk = 0; kk < kAtomK / 8; ++kk) {
      Wgmma<BN>::rs(acc, af + 4 * kk, make_desc(bb + kk * 32), accum);
      accum = 1u;
    }
  }
  wg_commit();
}

template <int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
linear_3xtf32_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_whi,
                     const __grid_constant__ CUtensorMap map_wlo, const float* __restrict__ bias,
                     const float* __restrict__ residual, float* __restrict__ y, long long M, int N, int KA, int stages,
                     int n_tiles, int m_tiles, int relu, const float* __restrict__ ln_gamma, const float* __restrict__ ln_beta,
                     float ln_eps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  const int w_bytes = 2 * KA * BN * 128;
  uint8_t* w_hi = sm;
  uint8_t* w_lo = sm + KA * BN * 128;
  uint8_t* ring = sm + w_bytes;                                   // stages x kGemmTileBytes, 1 KB aligned
  uint64_t* bars = reinterpret_cast<uint64_t*>(ring + stages * kGemmTileBytes);
  uint64_t* w_full = bars;
  uint64_t* full = bars + 1;
  uint64_t* empty = full + kMaxStages;
  const int half = stages / 2;                                    // ring stages per warpgroup

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int n_tile = blockIdx.x % n_tiles;
  const int group = blockIdx.x / n_tiles, n_groups = gridDim.x / n_tiles;
  const int n0 = n_tile * BN;

  if (tid == 0) {
    mbar_init(w_full, 1);
    for (int s = 0; s < kMaxStages; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, kGemmConsumers / 2 / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == kGemmConsumers / 32) {
    // ===== TMA producer: the CTA's m-tiles in order, KA atoms each =====
    if (lane == 0) {
      mbar_expect_tx(w_full, (uint32_t)w_bytes);
      for (int a = 0; a < KA; ++a) {
        tma_load_2d(w_hi + a * BN * 128, &map_whi, a * kAtomK, n0, w_full);
        tma_load_2d(w_lo + a * BN * 128, &map_wlo, a * kAtomK, n0, w_full);
      }
      int s0 = 0, s1 = 0; uint32_t ph0 = 0, ph1 = 0;   // position in each warpgroup's half of the ring
      constexpr int kPrefetchTiles = 8;                 // X tiles requested into L2 ahead of the smem ring
      for (int p = 0; p < kPrefetchTiles; ++p) {
        int mt = group + p * n_groups;
        if (mt < m_tiles)
          for (int a = 0; a < KA; ++a) tma_prefetch_l2_2d(&map_x, a * kAtomK, mt * kGemmTileM);
      }
      int w = 0;                                        // warpgroup of the current tile
      for (int mt = group; mt < m_tiles; mt += n_groups, w ^= 1) {
        const int mt_pf = mt + kPrefetchTiles * n_groups;
        if (mt_pf < m_tiles)
          for (int a = 0; a < KA; ++a) tma_prefetch_l2_2d(&map_x, a * kAtomK, mt_pf * kGemmTileM);
        for (int a = 0; a < KA; ++a) {
          const int slot = w ? half + s1 : s0;
          mbar_wait(empty + slot, (w ? ph1 : ph0) ^ 1);
          mbar_expect_tx(full + slot, (uint32_t)kGemmTileBytes);
          tma_load_2d(ring + slot * kGemmTileBytes, &map_x, a * kAtomK, mt * kGemmTileM, full + slot);
          if (w) ring_advance(s1, ph1, half); else ring_advance(s0, ph0, half);
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg takes the CTA's m-tiles j = wg, wg + 2, ... (64 rows each) =====
  const int wg = warp >> 2, wl = warp & 3, g = lane >> 2, t = lane & 3;
  const int frag_row = wl * 16 + g;                               // this thread's rows: frag_row and frag_row + 8
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  const uint32_t whi = smem_u32(w_hi), wlo = smem_u32(w_lo);
  mbar_wait(w_full, 0);
  uint8_t* my_ring = ring + wg * half * kGemmTileBytes;           // this warpgroup's half of the ring
  uint64_t* my_full = full + wg * half;
  uint64_t* my_empty = empty + wg * half;
  int s = 0; uint32_t ph = 0;
  for (int mt = group + wg * n_groups; mt < m_tiles; mt += 2 * n_groups) {
    uint32_t accum = 0;
    // two fragment sets: atom a + 1 is loaded and split while the MMAs of atom a run.  At BN >= 96 the second set
    // does not fit in the 168 registers a thread gets: one set, and each atom's MMAs complete before the next load.
    constexpr bool kTwoSets = BN <= 80;
    uint32_t ah0[16], al0[16], ah1_[kTwoSets ? 16 : 1], al1_[kTwoSets ? 16 : 1];
    uint32_t* ah1 = kTwoSets ? ah1_ : ah0;
    uint32_t* al1 = kTwoSets ? al1_ : al0;
    // A stage goes back to the producer only once the MMAs that took their A fragments from it have completed.  The
    // fragments are read with generic loads and the next TMA write into the stage is an async-proxy write: releasing
    // the stage right after the loads were issued let that write overtake loads still in flight (wrong rows in a few
    // m-tiles of long runs).  An MMA cannot complete before its register operands have arrived.
    int pending = -1;                                    // two sets: the stage of the MMA group still in flight
    auto release = [&](int slot) {
      if (slot < 0) return;
      __syncwarp();
      if (lane == 0) mbar_arrive(my_empty + slot);
    };
    auto fetch = [&](uint32_t* ah, uint32_t* al) {
      mbar_wait(my_full + s, ph);
      load_split_frag(my_ring + s * kGemmTileBytes, frag_row, g, t, ah, al);
      const int slot = s;
      ring_advance(s, ph, half);
      return slot;
    };
    auto issue = [&](uint32_t* ah, uint32_t* al, int a, int slot) {
      mma_atom_rs<BN>(acc, ah, al, whi + a * BN * 128, wlo + a * BN * 128, accum);
      if constexpr (kTwoSets) {
        wg_wait1();                                      // atom a - 1 is done: its set and its stage are free
        release(pending);
        pending = slot;
      } else {
        wg_wait0();                                      // atom a is done: the one set and its stage are free
        release(slot);
      }
    };
    int cur = fetch(ah0, al0);
    for (int a = 0; a < KA; a += 2) {
      issue(ah0, al0, a, cur);
      if (a + 1 < KA) {
        cur = fetch(ah1, al1);
        issue(ah1, al1, a + 1, cur);
        if (a + 2 < KA) cur = fetch(ah0, al0);
      }
    }
    wg_wait0();
    release(pending);
    fence_regs<BN / 2>(acc);

    // ===== epilogue: accumulator registers -> (+bias, ReLU, +residual [, LayerNorm]) -> global =====
    const long long row[2] = {(long long)mt * kGemmTileM + frag_row, (long long)mt * kGemmTileM + frag_row + 8};
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int gc = n0 + 8 * j + 2 * t;                // N is even: the column pair is in range or out of range together
      const float b0 = (bias && gc < N) ? __ldg(bias + gc) : 0.f, b1 = (bias && gc < N) ? __ldg(bias + gc + 1) : 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
        if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        if (residual && row[h] < M && gc < N) {
          const float2 rr = __ldg(reinterpret_cast<const float2*>(residual + row[h] * N + gc));
          v0 += rr.x; v1 += rr.y;
        }
        acc[4 * j + 2 * h] = v0;
        acc[4 * j + 2 * h + 1] = v1;
      }
    }
    if (ln_gamma) {
      // LayerNorm over the row (the launcher guarantees one n-tile: BN == N).  A row is spread over the 4 threads of a quad.
      float mean[2], rstd[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) sum += acc[4 * j + 2 * h] + acc[4 * j + 2 * h + 1];
        sum += __shfl_xor_sync(0xffffffffu, sum, 1);
        sum += __shfl_xor_sync(0xffffffffu, sum, 2);
        mean[h] = sum / (float)BN;
        float sq = 0.f;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const float d0 = acc[4 * j + 2 * h] - mean[h], d1 = acc[4 * j + 2 * h + 1] - mean[h];
          sq = fmaf(d0, d0, sq);
          sq = fmaf(d1, d1, sq);
        }
        sq += __shfl_xor_sync(0xffffffffu, sq, 1);
        sq += __shfl_xor_sync(0xffffffffu, sq, 2);
        rstd[h] = rsqrtf(sq / (float)BN + ln_eps);
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * t;
        const float g0 = __ldg(ln_gamma + c), g1 = __ldg(ln_gamma + c + 1), e0 = __ldg(ln_beta + c), e1 = __ldg(ln_beta + c + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          acc[4 * j + 2 * h] = (acc[4 * j + 2 * h] - mean[h]) * rstd[h] * g0 + e0;
          acc[4 * j + 2 * h + 1] = (acc[4 * j + 2 * h + 1] - mean[h]) * rstd[h] * g1 + e1;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int gc = n0 + 8 * j + 2 * t;
      if (gc >= N) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (row[h] < M) *reinterpret_cast<float2*>(y + row[h] * N + gc) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    }
  }
}

__global__ void split_tf32_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, long long n) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  float v = w[i];
  float h = tf32_rn(v);
  hi[i] = h;
  lo[i] = v - h;
}

template <int BN>
static int set_smem_attr() {
  return check_cuda(cudaFuncSetAttribute(linear_3xtf32_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
}

}  // namespace so

using namespace so;

extern "C" int so_split_tf32(const float* w, float* hi, float* lo, int64_t n, void* stream) {
  if (!w || !hi || !lo || n < 0) return SO_ERR_INVALID_ARG;
  if (n == 0) return SO_OK;
  split_tf32_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(w, hi, lo, n);
  note_launch(1);
  return check_launch();
}

static int linear_impl(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* residual, float* y,
                       int64_t M, int32_t N, int32_t K, int32_t relu, const float* ln_gamma, const float* ln_beta, float ln_eps,
                       void* stream);

extern "C" int so_linear_3xtf32(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                                float* y, int64_t M, int32_t N, int32_t K, int32_t relu, void* stream) {
  return linear_impl(x, w_hi, w_lo, bias, residual, y, M, N, K, relu, nullptr, nullptr, 0.f, stream);
}

// y = LayerNorm(act(x w^T + bias) + residual) * gamma + beta over the N output columns, in the GEMM epilogue.
// N must be a multiple of 32 and <= 128 (one n-tile holds the whole row).
extern "C" int so_linear_3xtf32_ln(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* residual,
                                   const float* gamma, const float* beta, float eps, float* y, int64_t M, int32_t N, int32_t K,
                                   int32_t relu, void* stream) {
  if (!gamma || !beta) return SO_ERR_INVALID_ARG;
  if (N % 32 != 0 || N > 128) return SO_ERR_UNSUPPORTED;
  return linear_impl(x, w_hi, w_lo, bias, residual, y, M, N, K, relu, gamma, beta, eps, stream);
}

static int linear_impl(const float* x, const float* w_hi, const float* w_lo, const float* bias, const float* residual, float* y,
                       int64_t M, int32_t N, int32_t K, int32_t relu, const float* ln_gamma, const float* ln_beta, float ln_eps,
                       void* stream) {
  if (!x || !w_hi || !w_lo || !y || M < 0 || N < 1 || K < 1) return SO_ERR_INVALID_ARG;
  if (K % 96 != 0 || K > 192) return SO_ERR_UNSUPPORTED;                         // K = 96 or 192
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(w_hi) | reinterpret_cast<uintptr_t>(w_lo)) & 15)
    return SO_ERR_INVALID_ARG;                                                    // TMA needs 16-byte aligned bases
  if (M == 0) return SO_OK;
  if (M > 0x7fffffffLL) return SO_ERR_UNSUPPORTED;
  // the epilogue stores Y and reads the residual as column pairs (float2)
  if ((reinterpret_cast<uintptr_t>(y) & 7) || (reinterpret_cast<uintptr_t>(residual) & 7) || (N % 2)) return SO_ERR_UNSUPPORTED;
  PipeCfg cfg = make_pipe_cfg(M, N, K, ln_gamma != nullptr, num_sms());
  if (cfg.stages < 2) return SO_ERR_UNSUPPORTED;
  CUtensorMap mx, mhi, mlo;
  int rc;
  if ((rc = make_tmap(&mx, x, M, K, kGemmTileM))) return rc;
  if ((rc = make_tmap(&mhi, w_hi, N, K, cfg.BN))) return rc;
  if ((rc = make_tmap(&mlo, w_lo, N, K, cfg.BN))) return rc;
  static PerDeviceOnce smem_attr;
  if ((rc = smem_attr.run([] {
         int r;
         if ((r = set_smem_attr<32>()) || (r = set_smem_attr<64>()) || (r = set_smem_attr<80>()) || (r = set_smem_attr<96>()) ||
             (r = set_smem_attr<128>()))
           return r;
         return SO_OK;
       })))
    return rc;
  cudaStream_t st = (cudaStream_t)stream;
  ProfScope prof(8, st);
#define SO_GEMM(BN_)                                                                                                           \
  linear_3xtf32_kernel<BN_><<<cfg.n_tiles * cfg.groups, kGemmThreads, cfg.smem, st>>>(                                         \
      mx, mhi, mlo, bias, residual, y, (long long)M, N, cfg.KA, cfg.stages, cfg.n_tiles, cfg.m_tiles, relu, ln_gamma, ln_beta, \
      ln_eps)
  switch (cfg.BN) {
    case 32: SO_GEMM(32); break;
    case 64: SO_GEMM(64); break;
    case 80: SO_GEMM(80); break;
    case 96: SO_GEMM(96); break;
    default: SO_GEMM(128); break;
  }
#undef SO_GEMM
  note_launch(1);
  return check_launch();
}
