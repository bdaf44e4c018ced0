// The label volume drawn as voxel cubes (the picture vis_3d.py / vis_3d_scene.py make with mayavi's cube glyphs).
//   so_voxel_render       one thread per pixel of K cameras: clip the ray to the grid's box, walk the cells with an
//                         Amanatides-Woo DDA, shade the first drawn voxel entered within [near, far] by the face it entered
//   so_voxel_faces_count  per voxel: its exposed faces (the 6-neighbour is not drawn or lies outside the grid)
//   so_voxel_faces_emit   those faces as quads at the offsets of the inclusive scan of the counts
// Grid: labels uint8 [H, W, D]; voxel (h, w, d), index (h * W + w) * D + d, is the cube [origin + (w, h, d) * voxel_size,
// origin + (w + 1, h + 1, d + 1) * voxel_size] in (x, y, z).  Face code 2a + s: axis a (0 x, 1 y, 2 z), s = 0 the cube's
// lower face on that axis, 1 its upper face.  Every output is written by one thread: no atomics, bit-identical reruns.
#include "common.cuh"

namespace so {

struct VoxelGridDev {
  const uint8_t* labels;
  int n[3];              // cells along x, y, z: W, H, D
  double org[3];         // grid origin, metres
  double vs;             // voxel side, metres
};

struct VoxelStyle {
  uint32_t palette[256];   // RGBA bytes, R lowest
  float shade[6];          // per face code
  uint32_t background;     // RGB bytes, R lowest
};

struct DrawnMask {
  uint32_t bits[8];        // bit l: label l is drawn
};

__device__ __forceinline__ int voxel_index(const VoxelGridDev& G, int ix, int iy, int iz) {
  return (iy * G.n[0] + ix) * G.n[2] + iz;
}

// Pixel tile of a CTA: 16 x 16 pixels, each warp an 8-wide, 4-tall patch so neighbouring rays of a warp walk the same cells.
constexpr int kVisTile = 16;
constexpr int kVisBlock = kVisTile * kVisTile;
constexpr double kVisInf = 1e300;

// The ray arithmetic runs in fp64: a cell boundary ~150 m from the camera is then placed to ~1e-13 m, so the traversal
// picks the nearest entered voxel unless two entries tie to that precision.  The walk is bound by its label loads.
__global__ void __launch_bounds__(kVisBlock) voxel_render_kernel(VoxelGridDev G, const float* __restrict__ cams, int img_h,
                                                                 int img_w, VoxelStyle S, uint8_t* __restrict__ rgb,
                                                                 int32_t* __restrict__ voxel, int8_t* __restrict__ face_out,
                                                                 float* __restrict__ dist) {
  __shared__ uint32_t pal[256];
  __shared__ float shade[6];
  pal[threadIdx.x] = S.palette[threadIdx.x];
  if (threadIdx.x < 6) shade[threadIdx.x] = S.shade[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int u = blockIdx.x * kVisTile + (warp & 1) * 8 + (lane & 7);
  const int v = blockIdx.y * kVisTile + (warp >> 1) * 4 + (lane >> 3);
  if (u >= img_w || v >= img_h) return;
  const float* c = cams + 16 * (int64_t)blockIdx.z;
  const double pu = u + 0.5, pv = v + 0.5;
  double o[3], d[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    o[a] = (double)__ldg(c + a);
    d[a] = (double)__ldg(c + 3 + 3 * a) * pu + (double)__ldg(c + 4 + 3 * a) * pv + (double)__ldg(c + 5 + 3 * a);
  }
  const double near = (double)__ldg(c + 12), far = (double)__ldg(c + 13);

  // clip [near, far] to the grid's box; remember the axis the box is entered through when that happens at or past near
  double t0 = near, t1 = far, inv[3];
  int entry_axis = -1;
  bool miss = !(near <= far);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double lo = G.org[a], hi = fma((double)G.n[a], G.vs, G.org[a]);
    if (d[a] == 0.0) {
      inv[a] = 0.0;
      miss |= o[a] < lo || o[a] > hi;
      continue;
    }
    inv[a] = 1.0 / d[a];
    double ta = (lo - o[a]) * inv[a], tb = (hi - o[a]) * inv[a];
    if (ta > tb) { const double t = ta; ta = tb; tb = t; }
    if (ta > t0) { t0 = ta; entry_axis = a; }
    t1 = fmin(t1, tb);
  }
  miss |= t0 > t1;

  int hit = -1, hit_face = -1;
  double hit_t = 0.0;
  if (!miss) {
    int i[3], step[3];
    double tn[3];
    // a start cell not entered through the box (the ray starts inside the grid at near) is never the hit: its entry lies
    // before near
    int f = -1;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      step[a] = d[a] > 0.0 ? 1 : d[a] < 0.0 ? -1 : 0;
      if (a == entry_axis) {
        i[a] = step[a] > 0 ? 0 : G.n[a] - 1;
        f = 2 * a + (step[a] < 0);
      } else {
        const double p = fma(t0, d[a], o[a]);
        i[a] = (int)fmin(fmax(floor((p - G.org[a]) / G.vs), 0.0), (double)(G.n[a] - 1));
      }
      tn[a] = step[a] == 0 ? kVisInf : (fma((double)(i[a] + (step[a] > 0)), G.vs, G.org[a]) - o[a]) * inv[a];
    }
    double t = t0;
    while (true) {
      if (f >= 0) {
        const int idx = voxel_index(G, i[0], i[1], i[2]);
        const int lab = __ldg(G.labels + idx);
        if (pal[lab] >> 24) { hit = idx; hit_face = f; hit_t = t; break; }
      }
      const int a = (tn[0] <= tn[1] && tn[0] <= tn[2]) ? 0 : (tn[1] <= tn[2] ? 1 : 2);
      bool out = false;
#pragma unroll
      for (int b = 0; b < 3; ++b) {     // the step along axis a, with constant indices so the per-axis state stays in registers
        if (b != a) continue;
        t = tn[b];
        i[b] += step[b];
        out = t > t1 || i[b] < 0 || i[b] >= G.n[b];
        f = 2 * b + (step[b] < 0);
        tn[b] = (fma((double)(i[b] + (step[b] > 0)), G.vs, G.org[b]) - o[b]) * inv[b];
      }
      if (out) break;
    }
  }

  const int64_t px = ((int64_t)blockIdx.z * img_h + v) * img_w + u;
  if (rgb) {
    uint32_t col = S.background;
    if (hit >= 0) {
      const uint32_t p = pal[__ldg(G.labels + hit)];
      const float s = shade[hit_face];
      col = 0;
#pragma unroll
      for (int k = 0; k < 3; ++k)
        col |= (uint32_t)min(max(__float2int_rn((float)((p >> (8 * k)) & 255u) * s), 0), 255) << (8 * k);
    }
    uint8_t* out = rgb + 3 * px;
    out[0] = col & 255u; out[1] = (col >> 8) & 255u; out[2] = (col >> 16) & 255u;
  }
  if (voxel) voxel[px] = hit;
  if (face_out) face_out[px] = (int8_t)hit_face;
  if (dist) dist[px] = hit >= 0 ? (float)hit_t : __int_as_float(0x7f800000);
}

__device__ __forceinline__ bool drawn_at(const VoxelGridDev& G, const DrawnMask& M, int ix, int iy, int iz) {
  if (ix < 0 || iy < 0 || iz < 0 || ix >= G.n[0] || iy >= G.n[1] || iz >= G.n[2]) return false;
  const int lab = __ldg(G.labels + voxel_index(G, ix, iy, iz));
  return (M.bits[lab >> 5] >> (lab & 31)) & 1u;
}

// bit f: the voxel is drawn and its face f is exposed
__device__ __forceinline__ unsigned exposed_faces(const VoxelGridDev& G, const DrawnMask& M, int ix, int iy, int iz) {
  if (!drawn_at(G, M, ix, iy, iz)) return 0;
  unsigned m = 0;
#pragma unroll
  for (int f = 0; f < 6; ++f) {
    const int a = f >> 1, s = (f & 1) ? 1 : -1;
    if (!drawn_at(G, M, ix + (a == 0) * s, iy + (a == 1) * s, iz + (a == 2) * s)) m |= 1u << f;
  }
  return m;
}

constexpr int kFaceBlock = 256;

__device__ __forceinline__ bool locate_voxel(const VoxelGridDev& G, int64_t idx, int& ix, int& iy, int& iz) {
  if (idx >= (int64_t)G.n[0] * G.n[1] * G.n[2]) return false;
  const int i = (int)idx;
  iz = i % G.n[2]; ix = (i / G.n[2]) % G.n[0]; iy = i / (G.n[2] * G.n[0]);
  return true;
}

__global__ void __launch_bounds__(kFaceBlock) voxel_faces_count_kernel(VoxelGridDev G, DrawnMask M, int32_t* __restrict__ counts) {
  const int64_t idx = (int64_t)blockIdx.x * kFaceBlock + threadIdx.x;
  int ix, iy, iz;
  if (!locate_voxel(G, idx, ix, iy, iz)) return;
  counts[idx] = __popc(exposed_faces(G, M, ix, iy, iz));
}

// Face (a, s) as a quad counter-clockwise seen from outside: with (b, c) = (a + 1, a + 2) mod 3, b x c = a, the corners
// (b, c) = (0, 0), (1, 0), (1, 1), (0, 1) on the upper face and the reverse winding (0, 0), (0, 1), (1, 1), (1, 0) on
// the lower face; triangles (0, 1, 2) and (0, 2, 3).
__global__ void __launch_bounds__(kFaceBlock) voxel_faces_emit_kernel(VoxelGridDev G, DrawnMask M, const int32_t* __restrict__ scans,
                                                                      int n_faces, float* __restrict__ vertices,
                                                                      int32_t* __restrict__ faces, float* __restrict__ normals,
                                                                      uint8_t* __restrict__ sem) {
  const int64_t idx = (int64_t)blockIdx.x * kFaceBlock + threadIdx.x;
  int ix, iy, iz;
  if (!locate_voxel(G, idx, ix, iy, iz)) return;
  const unsigned m = exposed_faces(G, M, ix, iy, iz);
  if (!m) return;
  int q = __ldg(scans + idx) - __popc(m);     // exclusive scan: the inclusive one minus this voxel's count
  const uint8_t lab = __ldg(G.labels + idx);
  const int cell[3] = {ix, iy, iz};
#pragma unroll
  for (int f = 0; f < 6; ++f) {
    if (!((m >> f) & 1u) || q >= n_faces) continue;
    const int a = f >> 1, up = f & 1, b = (a + 1) % 3, c = (a + 2) % 3;
    const int cb[4] = {0, up ? 1 : 0, 1, up ? 0 : 1};
    const int cc[4] = {0, up ? 0 : 1, 1, up ? 1 : 0};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      int corner[3];
      corner[a] = cell[a] + up;
      corner[b] = cell[b] + cb[k];
      corner[c] = cell[c] + cc[k];
      const int64_t vtx = 4 * (int64_t)q + k;
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        vertices[3 * vtx + e] = (float)fma((double)corner[e], G.vs, G.org[e]);
        normals[3 * vtx + e] = e == a ? (up ? 1.f : -1.f) : 0.f;
      }
      if (sem) sem[vtx] = lab;
    }
    const int v0 = 4 * q;
    int32_t* tri = faces + 6 * (int64_t)q;
    tri[0] = v0; tri[1] = v0 + 1; tri[2] = v0 + 2;
    tri[3] = v0; tri[4] = v0 + 2; tri[5] = v0 + 3;
    ++q;
  }
}

int make_voxel_grid(const uint8_t* labels, int32_t H, int32_t W, int32_t D, const float* origin, float voxel_size,
                    VoxelGridDev& G) {
  if (!labels || !origin || H < 1 || W < 1 || D < 1 || !(voxel_size > 0.f) || !(voxel_size < 3.4e38f)) return SO_ERR_INVALID_ARG;
  if ((int64_t)H * W * D >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;   // 32-bit voxel indices and scans
  G.labels = labels;
  G.n[0] = W; G.n[1] = H; G.n[2] = D;
  for (int a = 0; a < 3; ++a) G.org[a] = origin[a];
  G.vs = voxel_size;
  return SO_OK;
}

DrawnMask make_drawn(const uint8_t* drawn) {
  DrawnMask M = {};
  for (int l = 0; l < 256; ++l)
    if (drawn[l]) M.bits[l >> 5] |= 1u << (l & 31);
  return M;
}

inline bool aligned(const void* p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

}  // namespace so

using namespace so;

extern "C" int so_voxel_render(const uint8_t* labels, int32_t H, int32_t W, int32_t D, const float* origin, float voxel_size,
                               const float* cams, int32_t K, int32_t img_h, int32_t img_w, const uint8_t* palette,
                               const float* shade, const uint8_t* background, uint8_t* rgb, int32_t* voxel, int8_t* face,
                               float* dist, void* stream) {
  VoxelGridDev G;
  int rc = make_voxel_grid(labels, H, W, D, origin, voxel_size, G);
  if (rc) return rc;
  if (!cams || !palette || !shade || !background || K < 1 || img_h < 1 || img_w < 1) return SO_ERR_INVALID_ARG;
  if (!rgb && !voxel && !face && !dist) return SO_ERR_INVALID_ARG;
  if (!aligned(cams, 16) || !aligned(voxel, 4) || !aligned(dist, 4)) return SO_ERR_INVALID_ARG;
  if (K > 65535 || img_h > 65535 * kVisTile || img_w > 65535 * kVisTile) return SO_ERR_UNSUPPORTED;   // grid dimensions
  VoxelStyle S;
  for (int l = 0; l < 256; ++l)
    S.palette[l] = palette[4 * l] | palette[4 * l + 1] << 8 | palette[4 * l + 2] << 16 | (uint32_t)palette[4 * l + 3] << 24;
  for (int f = 0; f < 6; ++f) {
    if (!(shade[f] >= 0.f && shade[f] <= 1.f)) return SO_ERR_INVALID_ARG;
    S.shade[f] = shade[f];
  }
  S.background = background[0] | background[1] << 8 | background[2] << 16;
  const dim3 grid((unsigned)ceil_div64(img_w, kVisTile), (unsigned)ceil_div64(img_h, kVisTile), (unsigned)K);
  voxel_render_kernel<<<grid, kVisBlock, 0, (cudaStream_t)stream>>>(G, cams, img_h, img_w, S, rgb, voxel, face, dist);
  note_launch(1);
  return check_launch();
}

extern "C" int so_voxel_faces_count(const uint8_t* labels, int32_t H, int32_t W, int32_t D, const uint8_t* drawn, int32_t* counts,
                                    void* stream) {
  const float origin[3] = {0.f, 0.f, 0.f};
  VoxelGridDev G;
  int rc = make_voxel_grid(labels, H, W, D, origin, 1.f, G);
  if (rc) return rc;
  if (!drawn || !counts || !aligned(counts, 4)) return SO_ERR_INVALID_ARG;
  const int64_t n = (int64_t)H * W * D;
  voxel_faces_count_kernel<<<(unsigned)ceil_div64(n, kFaceBlock), kFaceBlock, 0, (cudaStream_t)stream>>>(G, make_drawn(drawn), counts);
  note_launch(1);
  return check_launch();
}

extern "C" int so_voxel_faces_emit(const uint8_t* labels, int32_t H, int32_t W, int32_t D, const float* origin, float voxel_size,
                                   const uint8_t* drawn, const int32_t* scans, int64_t n_faces, float* vertices, int32_t* faces,
                                   float* normals, uint8_t* sem, void* stream) {
  VoxelGridDev G;
  int rc = make_voxel_grid(labels, H, W, D, origin, voxel_size, G);
  if (rc) return rc;
  if (!drawn || !scans || !vertices || !faces || !normals || n_faces < 1) return SO_ERR_INVALID_ARG;
  if (!aligned(scans, 4) || !aligned(vertices, 4) || !aligned(faces, 4) || !aligned(normals, 4)) return SO_ERR_INVALID_ARG;
  if (4 * n_faces >= (int64_t)1 << 31) return SO_ERR_UNSUPPORTED;   // int32 vertex ids
  const int64_t n = (int64_t)H * W * D;
  voxel_faces_emit_kernel<<<(unsigned)ceil_div64(n, kFaceBlock), kFaceBlock, 0, (cudaStream_t)stream>>>(
      G, make_drawn(drawn), scans, (int)n_faces, vertices, faces, normals, sem);
  note_launch(1);
  return check_launch();
}
