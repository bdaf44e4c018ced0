// wgmma / mbarrier / TMA PTX wrappers and the shared-memory matrix descriptor shared by the tensor-core kernels
// (gemm.cu: projections, decode.cu: TPV decode MLP).  sm_90a only.
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace so {

constexpr int kBM = 128;            // rows per CTA tile (two consumer warpgroups x 64 rows)
constexpr int kAtomK = 32;          // fp32 elements per 128-byte swizzle atom
constexpr int kAtomBytesA = kBM * 128;
constexpr int kWgRows = 64;         // rows of one wgmma (M = 64)

// ---- PTX wrappers ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0, spins = 0;
  const uint32_t addr = smem_u32(bar);
  while (!done) {
    if (++spins > (1u << 26)) __trap();   // a lost TMA / MMA completion must fail loudly, never hang the GPU
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}\n"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(smem_u32(dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
// TMA prefetch of one box into L2 only: raises the bytes in flight beyond what the shared-memory ring can hold
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(map), "r"(c0), "r"(c1) : "memory");
}

// ---- wgmma (warpgroup = 4 consecutive warps, 128 threads) ----------------------------------------------------------
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// named barrier of the 128 threads of one warpgroup (ids 1.. are free: __syncthreads uses 0)
__device__ __forceinline__ void wg_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

// Shared-memory matrix descriptor: K-major operand, 128-byte swizzle, 8-row groups 1024 B apart.  The atom base must be
// 1024-byte aligned; a K step inside the atom advances the start address by 32 bytes (8 tf32).
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3ffff) >> 4);       // start address
  d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major; canonical value 1)
  d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset: 8 rows x 128 B
  d |= (uint64_t)1 << 62;                        // layout type SWIZZLE_128B
  return d;
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, fp32 accumulator in registers (N / 2 per thread), tf32 operands.
// Accumulator layout: thread (warp w of the warpgroup, lane = 4 g + t) holds for every 8-column block j
//   d[4j] = D[16w + g][8j + 2t], d[4j+1] = D[16w + g][8j + 2t + 1], d[4j+2] / d[4j+3] = the same columns of row 16w + g + 8.
// A from registers (same thread mapping): a[0] = A[16w + g][t], a[1] = A[16w + g + 8][t], a[2] = A[16w + g][t + 4],
// a[3] = A[16w + g + 8][t + 4].
template <int N>
struct Wgmma;

#define SO_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])

template <>
struct Wgmma<32> {
  __device__ __forceinline__ static void ss(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8)
        : "l"(da), "l"(db), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float* d, const uint32_t* a, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
};

template <>
struct Wgmma<64> {
  __device__ __forceinline__ static void ss(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8), SO_ACC8(16), SO_ACC8(24)
        : "l"(da), "l"(db), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float* d, const uint32_t* a, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8), SO_ACC8(16), SO_ACC8(24)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
};

template <>
struct Wgmma<96> {
  __device__ __forceinline__ static void ss(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %50, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8), SO_ACC8(16), SO_ACC8(24), SO_ACC8(32), SO_ACC8(40)
        : "l"(da), "l"(db), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float* d, const uint32_t* a, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %53, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, {%48, %49, %50, %51}, %52, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8), SO_ACC8(16), SO_ACC8(24), SO_ACC8(32), SO_ACC8(40)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
};

template <>
struct Wgmma<128> {
  __device__ __forceinline__ static void ss(float* d, uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8), SO_ACC8(16), SO_ACC8(24), SO_ACC8(32), SO_ACC8(40), SO_ACC8(48), SO_ACC8(56)
        : "l"(da), "l"(db), "r"(acc));
  }
  __device__ __forceinline__ static void rs(float* d, const uint32_t* a, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}\n"
        : SO_ACC8(0), SO_ACC8(8), SO_ACC8(16), SO_ACC8(24), SO_ACC8(32), SO_ACC8(40), SO_ACC8(48), SO_ACC8(56)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
  }
};
#undef SO_ACC8

// nearest TF32 number (low 13 mantissa bits zero), so the tensor core's own operand truncation is exact on it and the
// remainder v - hi (exact in fp32) is at most half a TF32 ulp
__device__ __forceinline__ float tf32_rn(float v) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
  return __uint_as_float(u & 0xffffe000u);
}

// byte offset of 16-byte chunk `chunk` of row `row` in a 128B-swizzled K-major atom
__host__ __device__ inline uint32_t swz_off(int row, int chunk) { return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4)); }

}  // namespace so
