// The uniform lattice of NeuSHead.get_uniform_sdf (neus_head.py:265-293) and its values, shared by the occupancy labels
// (occupancy.cu) and the surface extraction (mesh.cu).  A lattice value is the field query of so_field_query at the
// lattice point (same device functions, same operands); the sources that include this header are built with render.cu's
// flags so it also rounds the same way.
#pragma once
#include "render_common.cuh"

namespace so {

struct LatticeDev {
  const float *xs, *ys, *zs;  // lattice axes in metres: W = nx (x), H = ny (y), D = nz (z)
  int nx, ny, nz;
};

__device__ __forceinline__ Taps lattice_taps(const VolumeDev& V, const LatticeDev& L, int iy, int ix, int iz) {
  float kh, kw, kd;
  float gh = axis_m2g(V.ax[0], __ldg(L.ys + iy), kh);
  float gw = axis_m2g(V.ax[1], __ldg(L.xs + ix), kw);
  float gd = axis_m2g(V.ax[2], __ldg(L.zs + iz), kd);
  return make_taps(V, gh, gw, gd);
}

__device__ __forceinline__ float tap_sdf(const VolumeDev& V, const Taps& t) {
  float s, dgh, dgw, dgd;
  gather_sdf(V, t, s, dgh, dgw, dgd);
  return s;
}

}  // namespace so
