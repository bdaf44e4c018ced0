"""Oracle: marching cubes in numpy / fp64 on a given lattice (test infrastructure).

The reference has no surface extraction; this restates the rule of so_mesh_count / so_mesh_emit with the case table that
selfocc_b200/mc_table.py generates, in the same vertex and face order, so the device mesh can be compared index for index:
* point p = (iy, ix, iz) of the [ny, nx, nz] lattice, index (iy * nx + ix) * nz + iz, is inside when sdf <= thresh and
  owns its +x, +y, +z edges; vertices in ascending owner index, then axis, at p_a + t (p_b - p_a),
  t = (thresh - s_a) / (s_b - s_a);
* cell p has corner k at p + (k & 1, (k >> 1) & 1, (k >> 2) & 1) in (x, y, z); faces in ascending cell index, then in
  table order.
"""
import numpy as np

from selfocc_b200 import mc_table

_MASKS, _TRIS, _MAX_TRI = mc_table.tables()
_TRI = np.full((256, _MAX_TRI, 3), -1, dtype=np.int64)
for _c, _t in enumerate(_TRIS):
    if _t:
        _TRI[_c, :len(_t)] = _t
_NTRI = np.array([len(t) for t in _TRIS], dtype=np.int64)
_EDGE_CORNER = np.array(mc_table.EDGE_CORNER, dtype=np.int64)
_POPC = np.array([bin(i).count('1') for i in range(8)], dtype=np.int64)


def marching_cubes_ref(sdf, xs, ys, zs, thresh=0.0):
    """sdf [ny, nx, nz] lattice values, axes xs [nx], ys [ny], zs [nz] -> (vertices fp64 [V, 3], faces int64 [F, 3])."""
    s = np.asarray(sdf, dtype=np.float64)
    ny, nx, nz = s.shape
    axes = [np.asarray(a, dtype=np.float64) for a in (xs, ys, zs)]
    ins = s <= thresh
    cross = np.zeros((ny, nx, nz, 3), dtype=bool)
    cross[:, :-1, :, 0] = ins[:, :-1] != ins[:, 1:]
    cross[:-1, :, :, 1] = ins[:-1] != ins[1:]
    cross[:, :, :-1, 2] = ins[:, :, :-1] != ins[:, :, 1:]
    cross = cross.reshape(-1, 3)
    mask = cross[:, 0] | (cross[:, 1].astype(np.int64) << 1) | (cross[:, 2].astype(np.int64) << 2)
    cnt = _POPC[mask]
    base = np.cumsum(cnt) - cnt
    # vertices: (owner, axis) pairs in row-major order = ascending owner, then axis
    p, a = np.nonzero(cross)
    iy, ix, iz = np.unravel_index(p, (ny, nx, nz))
    idx = [ix, iy, iz]
    step = np.array([nz, nx * nz, 1])
    sa = s.reshape(-1)[p]
    sb = s.reshape(-1)[p + step[a]]
    t = (thresh - sa) / (sb - sa)
    verts = np.stack([axes[k][idx[k]] for k in range(3)], -1)
    for k in range(3):
        on = a == k
        verts[on, k] = verts[on, k] + t[on] * (axes[k][idx[k][on] + 1] - verts[on, k])
    # faces: cells in ascending index
    cy, cx, cz = np.meshgrid(np.arange(ny - 1), np.arange(nx - 1), np.arange(nz - 1), indexing='ij')
    cells = ((cy * nx + cx) * nz + cz).reshape(-1)
    flat = ins.reshape(-1)
    case = np.zeros(cells.shape, dtype=np.int64)
    for k in range(8):
        case |= flat[cells + (k & 1) * nz + ((k >> 1) & 1) * nx * nz + ((k >> 2) & 1)].astype(np.int64) << k
    keep = _NTRI[case] > 0
    cells, case = cells[keep], case[keep]
    e = _TRI[case]                                               # [n_cells, max_tri, 3]
    valid = e[..., 0] >= 0
    e = np.where(e < 0, 0, e)
    c = _EDGE_CORNER[e]
    q = cells[:, None, None] + (c & 1) * nz + ((c >> 1) & 1) * nx * nz + ((c >> 2) & 1)
    ax = e >> 2
    mq = mask[q]
    vid = base[q] + _POPC[mq & ((1 << ax) - 1)]
    faces = vid[valid]
    return verts, faces.reshape(-1, 3)
