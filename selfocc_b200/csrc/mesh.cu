// Surface extraction: marching cubes over the lattice of NeuSHead.get_uniform_sdf, the lattice values evaluated on the fly
// (the lattice itself is never stored).
//   so_mesh_count  per lattice point: its crossing owned edges; per cell: its triangle count
//   so_mesh_emit   vertices and faces at the offsets of the exclusive scans of those counts
// Lattice point p = (iy, ix, iz), index (iy * nx + ix) * nz + iz, owns its +x, +y and +z edges; cell p is the cube whose
// lowest corner is p.  Vertices go in ascending owner index, then by axis; faces in ascending cell index, then in table
// order.  Every output is written by one thread at a scanned offset: no atomics, bit-identical from run to run.
#include "lattice.cuh"
#include "mc_table.cuh"

namespace so {

// CTA tile: 8 (z) x 8 (x) x 4 (y) lattice points, one per thread; their values plus a +1 halo on each axis (the far
// corners of the tile's cells) are evaluated once per tile and staged in shared memory.
constexpr int kTZ = 8, kTX = 8, kTY = 4;
constexpr int kMeshBlock = kTZ * kTX * kTY;
constexpr int kSZ = kTZ + 1, kSX = kTX + 1, kSY = kTY + 1;

struct MeshPoint {
  int iy, ix, iz;   // lattice indices of this thread's point
  int l;            // its index in the staged tile
  bool valid;       // inside the lattice
};

// Stage the tile's lattice values and locate this thread's point.  Points past the lattice's end are staged as 0 and
// never read: every read below is guarded by the lattice bounds.
__device__ __forceinline__ MeshPoint stage_tile(const VolumeDev& V, const LatticeDev& L, float* s) {
  const int bz = (L.nz + kTZ - 1) / kTZ, bx = (L.nx + kTX - 1) / kTX;
  const int b = blockIdx.x;
  const int z0 = (b % bz) * kTZ, x0 = ((b / bz) % bx) * kTX, y0 = (b / bz / bx) * kTY;
  for (int i = threadIdx.x; i < kSY * kSX * kSZ; i += kMeshBlock) {
    const int lz = i % kSZ, lx = (i / kSZ) % kSX, ly = i / (kSZ * kSX);
    const int iy = y0 + ly, ix = x0 + lx, iz = z0 + lz;
    s[i] = (iy < L.ny && ix < L.nx && iz < L.nz) ? tap_sdf(V, lattice_taps(V, L, iy, ix, iz)) : 0.f;
  }
  __syncthreads();
  const int tz = threadIdx.x % kTZ, tx = (threadIdx.x / kTZ) % kTX, ty = threadIdx.x / (kTZ * kTX);
  MeshPoint p;
  p.iy = y0 + ty; p.ix = x0 + tx; p.iz = z0 + tz;
  p.l = (ty * kSX + tx) * kSZ + tz;
  p.valid = p.iy < L.ny && p.ix < L.nx && p.iz < L.nz;
  return p;
}

// staged-tile stride of each axis (x, y, z), and of cube corner c
__device__ __forceinline__ int tile_step(int a) { return a == 0 ? kSZ : a == 1 ? kSX * kSZ : 1; }
__device__ __forceinline__ int tile_corner(int c) { return (c & 1) * kSZ + ((c >> 1) & 1) * kSX * kSZ + ((c >> 2) & 1); }

// bit a: the point's +a edge exists and crosses thresh
__device__ __forceinline__ unsigned owned_crossings(const LatticeDev& L, const MeshPoint& p, const float* s, float thresh) {
  const bool in0 = s[p.l] <= thresh;
  unsigned m = 0;
  if (p.ix + 1 < L.nx && (s[p.l + tile_step(0)] <= thresh) != in0) m |= 1u;
  if (p.iy + 1 < L.ny && (s[p.l + tile_step(1)] <= thresh) != in0) m |= 2u;
  if (p.iz + 1 < L.nz && (s[p.l + tile_step(2)] <= thresh) != in0) m |= 4u;
  return m;
}

// case index of the cell whose lowest corner is p, or -1 when p is on the lattice's upper border
__device__ __forceinline__ int cell_case(const LatticeDev& L, const MeshPoint& p, const float* s, float thresh) {
  if (p.ix + 1 >= L.nx || p.iy + 1 >= L.ny || p.iz + 1 >= L.nz) return -1;
  int c = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) c |= (s[p.l + tile_corner(k)] <= thresh) << k;
  return c;
}

__global__ void __launch_bounds__(kMeshBlock) mesh_count_kernel(VolumeDev V, LatticeDev L, float thresh, int* __restrict__ counts,
                                                                uint8_t* __restrict__ edge_mask) {
  __shared__ float s[kSY * kSX * kSZ];
  const MeshPoint p = stage_tile(V, L, s);
  if (!p.valid) return;
  const int n = L.ny * L.nx * L.nz;
  const int i = (p.iy * L.nx + p.ix) * L.nz + p.iz;
  const unsigned m = owned_crossings(L, p, s, thresh);
  const int c = cell_case(L, p, s, thresh);
  counts[i] = __popc(m);
  counts[n + i] = c < 0 ? 0 : __ldg(kMcNumTri + c);
  edge_mask[i] = (uint8_t)m;
}

__global__ void __launch_bounds__(kMeshBlock) mesh_emit_kernel(VolumeDev V, LatticeDev L, float thresh, const int* __restrict__ scans,
                                                               const uint8_t* __restrict__ edge_mask, int n_vertices, int n_faces,
                                                               float* __restrict__ vertices, int* __restrict__ faces) {
  __shared__ float s[kSY * kSX * kSZ];
  const MeshPoint p = stage_tile(V, L, s);
  if (!p.valid) return;
  const int n = L.ny * L.nx * L.nz;
  const int i = (p.iy * L.nx + p.ix) * L.nz + p.iz;
  const unsigned m = owned_crossings(L, p, s, thresh);
  if (m) {
    int v = __ldg(scans + i) - __popc(m);        // exclusive scan: the inclusive one minus this point's count
    const float pa[3] = {__ldg(L.xs + p.ix), __ldg(L.ys + p.iy), __ldg(L.zs + p.iz)};
    const float sa = s[p.l];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (!((m >> a) & 1u) || v >= n_vertices) continue;
      const float sb = s[p.l + tile_step(a)];
      const float t = (thresh - sa) / (sb - sa);   // sa and sb lie on different sides of thresh: sb != sa
      const float pb = a == 0 ? __ldg(L.xs + p.ix + 1) : a == 1 ? __ldg(L.ys + p.iy + 1) : __ldg(L.zs + p.iz + 1);
      float* out = vertices + 3 * (int64_t)v;
#pragma unroll
      for (int k = 0; k < 3; ++k) out[k] = k == a ? fmaf(t, pb - pa[a], pa[a]) : pa[k];
      ++v;
    }
  }
  const int c = cell_case(L, p, s, thresh);
  if (c < 0) return;
  const int nt = __ldg(kMcNumTri + c);
  const int f0 = __ldg(scans + n + i) - nt;
  for (int j = 0; j < nt && f0 + j < n_faces; ++j) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int e = __ldg(&kMcTri[c][3 * j + k]);
      const int cq = __ldg(kMcEdgeCorner + e), a = e >> 2;
      const int q = i + (cq & 1) * L.nz + ((cq >> 1) & 1) * L.nx * L.nz + ((cq >> 2) & 1);   // the edge's owner
      const unsigned mq = __ldg(edge_mask + q);
      faces[3 * (int64_t)(f0 + j) + k] = __ldg(scans + q) - __popc(mq) + __popc(mq & ((1u << a) - 1u));
    }
  }
}

int check_mesh(const float* vol_sdf, const so_volume_desc* vol_host, const float* xs, int32_t nx, const float* ys, int32_t ny,
               const float* zs, int32_t nz) {
  if (!vol_sdf || !xs || !ys || !zs || nx < 2 || ny < 2 || nz < 2) return SO_ERR_INVALID_ARG;
  int rc = validate_volume(vol_host);
  if (rc) return rc;
  if ((int64_t)nx * ny * nz >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;   // 32-bit lattice indices and scans
  return SO_OK;
}

unsigned mesh_grid(int32_t nx, int32_t ny, int32_t nz) {
  return (unsigned)(ceil_div64(nz, kTZ) * ceil_div64(nx, kTX) * ceil_div64(ny, kTY));
}

}  // namespace so

using namespace so;

extern "C" int so_mesh_count(const float* vol_sdf, const so_volume_desc* vol_host, const float* xs, int32_t nx, const float* ys,
                             int32_t ny, const float* zs, int32_t nz, float thresh, int32_t* counts, uint8_t* edge_mask,
                             void* stream) {
  if (!counts || !edge_mask) return SO_ERR_INVALID_ARG;
  int rc = check_mesh(vol_sdf, vol_host, xs, nx, ys, ny, zs, nz);
  if (rc) return rc;
  VolumeDev V = make_volume(*vol_host, vol_sdf, nullptr);
  LatticeDev L{xs, ys, zs, nx, ny, nz};
  mesh_count_kernel<<<mesh_grid(nx, ny, nz), kMeshBlock, 0, (cudaStream_t)stream>>>(V, L, thresh, counts, edge_mask);
  note_launch(1);
  return check_launch();
}

extern "C" int so_mesh_emit(const float* vol_sdf, const so_volume_desc* vol_host, const float* xs, int32_t nx, const float* ys,
                            int32_t ny, const float* zs, int32_t nz, float thresh, const int32_t* scans, const uint8_t* edge_mask,
                            int64_t n_vertices, int64_t n_faces, float* vertices, int32_t* faces, void* stream) {
  if (!scans || !edge_mask || !vertices || !faces || n_vertices < 0 || n_faces < 0) return SO_ERR_INVALID_ARG;
  int rc = check_mesh(vol_sdf, vol_host, xs, nx, ys, ny, zs, nz);
  if (rc) return rc;
  if (n_vertices >= (int64_t)1 << 31 || n_faces >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;   // int32 ids and scans
  VolumeDev V = make_volume(*vol_host, vol_sdf, nullptr);
  LatticeDev L{xs, ys, zs, nx, ny, nz};
  mesh_emit_kernel<<<mesh_grid(nx, ny, nz), kMeshBlock, 0, (cudaStream_t)stream>>>(V, L, thresh, scans, edge_mask, (int)n_vertices,
                                                                                     (int)n_faces, vertices, faces);
  note_launch(1);
  return check_launch();
}
