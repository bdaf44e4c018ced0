"""CPU: the marching-cubes case table (selfocc_b200/mc_table.py -> csrc/mc_table.cuh), the fp64 oracle's meshes (closed,
oriented 2-manifolds; sphere and torus topology, area and orientation) and the C ABI's refusals of so_mesh_count /
so_mesh_emit."""
import ctypes as C
import os
import numpy as np
import pytest

from oracle.mesh import marching_cubes_ref
from selfocc_b200 import mc_table

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, '..', 'selfocc_b200', 'csrc', 'mc_table.cuh')


def test_table_header_regenerates_byte_for_byte():
    with open(HEADER) as f:
        assert f.read() == mc_table.header()


def test_every_case_triangulates_exactly_its_crossing_edges():
    masks, tris, max_tri = mc_table.tables()
    assert max_tri == 5
    for case in range(256):
        crossing = {e for e in range(12) if (masks[case] >> e) & 1}
        used = {e for t in tris[case] for e in t}
        assert used == crossing, case
        assert all(len(set(t)) == 3 for t in tris[case]), case
    assert tris[0] == [] and tris[255] == []


def _edges(faces):
    f = np.asarray(faces)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def _check_closed_oriented(verts, faces):
    """Every directed edge occurs once and its reverse once: each undirected edge is shared by exactly two faces with
    opposite directions.  Every vertex is used."""
    d = _edges(faces)
    key = d[:, 0] * len(verts) + d[:, 1]
    rkey = d[:, 1] * len(verts) + d[:, 0]
    assert np.unique(key).size == key.size, 'a directed edge is used twice'
    assert np.array_equal(np.sort(key), np.sort(rkey)), 'an edge without its reverse'
    assert np.array_equal(np.unique(faces), np.arange(len(verts)))


def _euler(verts, faces):
    d = _edges(faces)
    e = np.unique(np.sort(d, 1), axis=0).shape[0]
    return len(verts) - e + len(faces)


def _lattice(n, lo=-1.0, hi=1.0):
    ax = np.linspace(lo, hi, n)
    y, x, z = np.meshgrid(ax, ax, ax, indexing='ij')       # [ny, nx, nz] layout
    return ax, x, y, z


@pytest.mark.parametrize('seed', range(6))
def test_random_lattices_give_closed_oriented_manifolds(seed):
    """Random signs (including many ambiguous faces) inside, the border outside; exact threshold hits included."""
    rng = np.random.default_rng(seed)
    ny, nx, nz = rng.integers(4, 12, size=3)
    s = rng.standard_normal((ny, nx, nz))
    s[rng.random(s.shape) < 0.05] = 0.0                    # on the threshold: inside
    s[0], s[-1], s[:, 0], s[:, -1], s[:, :, 0], s[:, :, -1] = 1.0, 1.0, 1.0, 1.0, 1.0, 1.0
    v, f = marching_cubes_ref(s, np.arange(nx), np.arange(ny), np.arange(nz))
    assert len(f) > 0
    _check_closed_oriented(v, f)
    # a vertex on a lattice edge exactly where the labels differ at its ends
    assert len(v) == sum(int(((s[tuple(sl_a)] <= 0) != (s[tuple(sl_b)] <= 0)).sum()) for sl_a, sl_b in (
        ([slice(None), slice(None, -1)], [slice(None), slice(1, None)]),
        ([slice(None, -1)], [slice(1, None)]),
        ([slice(None), slice(None), slice(None, -1)], [slice(None), slice(None), slice(1, None)])))


def _face_normals(v, f):
    return np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])


def test_sphere_is_closed_with_genus_0_the_right_area_and_outward_faces():
    ax, x, y, z = _lattice(101, -1.0, 1.0)
    r = 0.7
    s = np.sqrt((x - 0.013) ** 2 + (y + 0.021) ** 2 + (z - 0.007) ** 2) - r
    v, f = marching_cubes_ref(s, ax, ax, ax)
    _check_closed_oriented(v, f)
    assert _euler(v, f) == 2
    n = _face_normals(v, f)
    area = 0.5 * np.linalg.norm(n, axis=1).sum()
    assert abs(area / (4 * np.pi * r * r) - 1) < 0.01
    centroid = v[f].mean(1) - np.array([0.013, -0.021, 0.007])
    assert (np.einsum('ij,ij->i', n, centroid) > 0).all()
    # vertices lie on the sphere to within the interpolation error of a chord
    assert np.abs(np.linalg.norm(v - np.array([0.013, -0.021, 0.007]), axis=1) - r).max() < (ax[1] - ax[0]) ** 2


def test_torus_has_euler_characteristic_0():
    ax, x, y, z = _lattice(81, -1.0, 1.0)
    R, r = 0.55, 0.22
    s = np.sqrt((np.sqrt(x ** 2 + y ** 2) - R) ** 2 + z ** 2) - r
    v, f = marching_cubes_ref(s, ax, ax, ax)
    _check_closed_oriented(v, f)
    assert _euler(v, f) == 0


def test_vertex_order_is_owner_then_axis():
    s = np.ones((3, 3, 3))
    s[1, 1, 1] = -1.0
    ax = np.arange(3.0)
    v, f = marching_cubes_ref(s, ax, ax, ax)
    # owners in ascending (iy, ix, iz): (0, 1, 1) +y, (1, 0, 1) +x, (1, 1, 0) +z, then the centre's +x, +y, +z
    assert len(v) == 6 and len(f) == 8
    assert np.allclose(v, [[1, 0.5, 1], [0.5, 1, 1], [1, 1, 0.5], [1.5, 1, 1], [1, 1.5, 1], [1, 1, 1.5]])
    _check_closed_oriented(v, f)
    assert _euler(v, f) == 2


def test_mesh_entry_points_refuse_bad_arguments_before_any_cuda_call():
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    assert lib.so_abi_version() == 10
    N, one = None, C.c_void_p(16)
    d = _lib.VolumeDesc()
    d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch = 9, 9, 5, 8, 24, 24
    for i in range(3):
        d.axis[i].range0, d.axis[i].size0 = 1.0, 4.0
    D = C.byref(d)
    lat = lambda nx=4, ny=4, nz=4: (one, nx, one, ny, one, nz)
    assert lib.so_mesh_count(N, D, *lat(), 0.0, one, one, N) == -1                 # no volume
    assert lib.so_mesh_count(one, None, *lat(), 0.0, one, one, N) == -1            # no descriptor
    assert lib.so_mesh_count(one, D, *lat(), 0.0, N, one, N) == -1                 # no counts
    assert lib.so_mesh_count(one, D, *lat(), 0.0, one, N, N) == -1                 # no edge mask
    assert lib.so_mesh_count(one, D, N, 4, one, 4, one, 4, 0.0, one, one, N) == -1  # no axis
    for bad in (dict(nx=1), dict(ny=1), dict(nz=1), dict(nx=0)):                   # an axis shorter than 2
        assert lib.so_mesh_count(one, D, *lat(**bad), 0.0, one, one, N) == -1
        assert lib.so_mesh_emit(one, D, *lat(**bad), 0.0, one, one, 10, 10, one, one, N) == -1
    assert lib.so_mesh_count(one, D, *lat(2048, 2048, 512), 0.0, one, one, N) == -2   # 2^31 lattice points
    assert lib.so_mesh_emit(one, D, *lat(2048, 2048, 512), 0.0, one, one, 10, 10, one, one, N) == -2
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, N, one, 10, 10, one, one, N) == -1    # no scans
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, one, N, 10, 10, one, one, N) == -1    # no edge mask
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, one, one, 10, 10, N, one, N) == -1    # no vertices
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, one, one, 10, 10, one, N, N) == -1    # no faces
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, one, one, -1, 10, one, one, N) == -1  # negative totals
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, one, one, 10, -1, one, one, N) == -1
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, one, one, 2 ** 31, 10, one, one, N) == -2   # vertex ids beyond int32
    assert lib.so_mesh_emit(one, D, *lat(), 0.0, one, one, 10, 2 ** 31, one, one, N) == -2


RGB3 = np.array([[255, 0, 0], [100, 150, 245], [0, 175, 0]], dtype=np.uint8)


# uint8 RGB; an int64 RGBA table of 0..255 values, the kind vis_3d.py builds; 0..1 floats
@pytest.mark.parametrize('cmap', [RGB3, np.concatenate([RGB3, np.full((3, 1), 255)], 1).astype(np.int64), RGB3 / 255.0],
                         ids=['uint8_rgb', 'int64_rgba', 'float_rgb'])
def test_write_ply_round_trips(tmp_path, cmap):
    import torch
    from selfocc_b200.mesh import write_ply
    ax, x, y, z = _lattice(11, -1.0, 1.0)
    v, f = marching_cubes_ref(np.sqrt(x ** 2 + y ** 2 + z ** 2) - 0.6, ax, ax, ax)
    nrm = v / np.linalg.norm(v, axis=1, keepdims=True)
    sem = np.arange(len(v)) % 3
    mesh = {'vertices': torch.tensor(v, dtype=torch.float32), 'faces': torch.tensor(f, dtype=torch.int32),
            'normals': torch.tensor(nrm, dtype=torch.float32), 'sem': torch.tensor(sem, dtype=torch.uint8)}
    path = str(tmp_path / 'm.ply')
    write_ply(path, mesh, colormap=cmap)
    data = open(path, 'rb').read()
    end = data.index(b'end_header\n') + len(b'end_header\n')
    head = data[:end].decode('ascii').split('\n')
    assert head[:3] == ['ply', 'format binary_little_endian 1.0', 'element vertex %d' % len(v)]
    assert 'element face %d' % len(f) in head and 'property list uchar int vertex_indices' in head
    vt = np.dtype([(k, '<f4') for k in ('x', 'y', 'z', 'nx', 'ny', 'nz')] + [(k, 'u1') for k in ('red', 'green', 'blue')])
    va = np.frombuffer(data, vt, len(v), end)
    fa = np.frombuffer(data, np.dtype([('n', 'u1'), ('v', '<i4', (3,))]), len(f), end + vt.itemsize * len(v))
    assert end + vt.itemsize * len(v) + fa.itemsize * len(f) == len(data)
    assert np.array_equal(np.stack([va['x'], va['y'], va['z']], 1), v.astype(np.float32))
    assert np.array_equal(np.stack([va['nx'], va['ny'], va['nz']], 1), nrm.astype(np.float32))
    assert np.array_equal(np.stack([va['red'], va['green'], va['blue']], 1), RGB3[sem])
    assert (fa['n'] == 3).all() and np.array_equal(fa['v'], f)
