"""CPU: the voxel-cube picture's oracle, cameras, palettes, grid layout and face mesh (oracle/voxel_vis.py,
selfocc_b200/voxel_vis.py), PNG writing, and the argument checks of so_voxel_render / so_voxel_faces_*."""
import ctypes as C
import math
import os
import struct
import zlib
import numpy as np
import pytest
import torch

from oracle import voxel_vis as ref
from selfocc_b200 import voxel_vis as vv

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = np.load(os.path.join(HERE, 'golden', 'reference_golden_vis.npz'))
DRAWN = vv.drawn_table().astype(bool)


def _dda(labels, origin, vs, o, d, near, far, drawn):
    """An independent fp64 DDA: Amanatides-Woo with accumulated tMax += tDelta, one ray at a time."""
    H, W, D = labels.shape
    n = (W, H, D)
    org = np.asarray(origin, dtype=np.float64)
    t0, t1, axis0 = near, far, -1
    for a in range(3):
        lo, hi = org[a], org[a] + n[a] * vs
        if d[a] == 0:
            if not lo <= o[a] <= hi:
                return -1, -1
            continue
        ta, tb = sorted(((lo - o[a]) / d[a], (hi - o[a]) / d[a]))
        if ta > t0:
            t0, axis0 = ta, a
        t1 = min(t1, tb)
    if t0 > t1:
        return -1, -1
    p = o + t0 * d
    cell = [min(max(int(math.floor((p[a] - org[a]) / vs)), 0), n[a] - 1) for a in range(3)]
    step = [int(np.sign(d[a])) for a in range(3)]
    if axis0 >= 0:
        cell[axis0] = 0 if step[axis0] > 0 else n[axis0] - 1
    tmax = [math.inf if step[a] == 0 else (org[a] + (cell[a] + (step[a] > 0)) * vs - o[a]) / d[a] for a in range(3)]
    tdelta = [math.inf if step[a] == 0 else vs / abs(d[a]) for a in range(3)]
    face = -1 if axis0 < 0 else 2 * axis0 + (step[axis0] < 0)
    while True:
        if face >= 0 and drawn[labels[cell[1], cell[0], cell[2]]]:
            return (cell[1] * W + cell[0]) * D + cell[2], face
        a = int(np.argmin(tmax))
        if tmax[a] > t1:
            return -1, -1
        cell[a] += step[a]
        if not 0 <= cell[a] < n[a]:
            return -1, -1
        face = 2 * a + (step[a] < 0)
        tmax[a] += tdelta[a]


def _random_grid(rng, shape, p):
    lab = rng.integers(1, 17, size=shape).astype(np.uint8)
    lab[rng.random(shape) > p] = 0
    lab[rng.random(shape) < 0.02] = 200                     # >= 100: never drawn
    return lab


@pytest.mark.parametrize('seed', range(4))
def test_oracle_slab_test_equals_independent_dda(seed):
    rng = np.random.default_rng(seed)
    shape = (7, 6, 5)
    lab = _random_grid(rng, shape, 0.25)
    origin, vs = (-1.3, 0.7, -0.4), 0.37
    centre = np.asarray(origin) + 0.5 * vs * np.array([shape[1], shape[0], shape[2]])
    n_px = 0
    for k in range(4):
        if k == 3:                                          # a camera inside the grid
            pos = centre + rng.normal(size=3) * 0.3
        else:
            pos = centre + rng.normal(size=3) * 3.0 + np.array([0, 0, 2.0])
        cam = vv.look_at(pos, centre + rng.normal(size=3) * 0.2, (0, 0, 1), 50.0, (24, 32),
                         (0.01 if k != 1 else 2.5, 30.0 if k != 2 else 3.0))
        o, d, near, far = ref.rays_from_rows(cam.row()[None].astype(np.float32), (24, 32))
        o, d = o[0], d[0].reshape(-1, 3)
        vox, face, t = ref.render_ref(lab, origin, vs, o, d, near[0], far[0], DRAWN)
        got = np.array([_dda(lab, origin, vs, o, d[i], near[0], far[0], DRAWN) for i in range(len(d))])
        bad = (got[:, 0] != vox) | (got[:, 1] != face)
        tie = ref.ties(lab, origin, vs, o, d, near[0], far[0], got[:, 0], got[:, 1], vox, face, t)
        assert not (bad & ~tie).any(), np.flatnonzero(bad & ~tie)[:10]
        assert (bad & tie).sum() <= 2
        n_px += (vox >= 0).sum()
    assert n_px > 500


def test_oracle_covers_rays_starting_inside_drawn_voxels():
    """A solid block with the camera inside it: the first voxel entered past near, never the one holding the camera."""
    lab = np.ones((4, 4, 4), np.uint8)
    origin, vs = (0.0, 0.0, 0.0), 1.0
    o = np.array([1.5, 1.5, 1.5])
    d = np.array([[1.0, 0.0, 0.0], [0.3, 0.2, 1.0], [-1.0, 0.1, 0.05]])
    vox, face, t = ref.render_ref(lab, origin, vs, o, d, 0.0, 10.0, DRAWN)
    assert vox[0] == (1 * 4 + 2) * 4 + 1 and face[0] == 0 and t[0] == pytest.approx(0.5)
    assert (vox >= 0).all()
    for i in range(3):
        assert vox[i] == _dda(lab, origin, vs, o, d[i], 0.0, 10.0, DRAWN)[0]


def test_vis3d_nuscenes_preset_is_vtks_elevation_sequence():
    assert list(GOLD['cam_elevations']) == [5, 5, -5]
    pos, fp, up = GOLD['cam_position'], GOLD['cam_focal_point'], GOLD['cam_view_up']
    for deg in GOLD['cam_elevations']:
        pos, up = ref.elevation(pos, fp, up, deg)
    cam = vv.VIS3D_NUSCENES
    assert np.allclose(cam.position, pos, rtol=0, atol=1e-12)
    assert np.allclose(cam.view_up, up, rtol=0, atol=1e-14)
    assert np.array_equal(cam.focal_point, GOLD['cam_focal_point'])
    assert cam.view_angle == GOLD['cam_view_angle'] and cam.clip == tuple(GOLD['cam_clip'])
    assert cam.image_size == (1440, 2560)
    # Elevation(5) Elevation(5) Elevation(-5) about the focal point: one net 5 degree rotation, distance kept
    r0 = GOLD['cam_position'] - GOLD['cam_focal_point']
    r1 = cam.position - cam.focal_point
    assert np.linalg.norm(r1) == pytest.approx(np.linalg.norm(r0), rel=1e-14)
    assert math.degrees(math.acos(r0 @ r1 / (np.linalg.norm(r0) * np.linalg.norm(r1)))) == pytest.approx(5.0, abs=1e-9)
    assert r1[2] > r0[2]                                            # elevation raises the camera


@pytest.mark.parametrize('which', ['nuscenes', 'kitti', 'random'])
def test_camera_rays_equal_vtk_unprojection(which):
    rng = np.random.default_rng(3)
    if which == 'nuscenes':
        cam = vv.VIS3D_NUSCENES.resized((36, 64))
    elif which == 'kitti':
        cam = vv.kitti_camera(dict(cam_positions=[[0.7, -20.0, 9.0]], focal_positions=[[0.7, -19.1, 8.6]]), (45, 80))
        assert cam.view_angle == 41.0 and cam.clip == (0.01, 300.0)
    else:
        cam = vv.look_at(rng.normal(size=3) * 30, rng.normal(size=3), (0.1, 0.2, 1.0), 23.0, (50, 30), (0.5, 90.0))
    o, d = ref.camera_rays(cam.position, cam.focal_point, cam.view_up, cam.view_angle, cam.image_size, cam.clip)
    row = cam.row()
    o2, d2, near, far = ref.rays_from_rows(row[None], cam.image_size)
    assert np.array_equal(o2[0], cam.position) and (near[0], far[0]) == cam.clip
    assert np.abs(d2[0] - d).max() < 1e-9 * np.abs(d).max()


def test_palettes_equal_the_reference_tables():
    assert int(GOLD['sem_vmin']) == 1 and int(GOLD['sem_vmax_nuscenes']) == 16 and int(GOLD['sem_vmax_kitti']) == 19
    assert np.array_equal(np.array(vv.NUSCENES_COLORS, np.uint8), GOLD['nuscenes_colors'])
    assert np.array_equal(np.array(vv.KITTI_COLORS, np.uint8), GOLD['kitti_colors'])
    lo, hi = int(GOLD['drawn_lo']), int(GOLD['drawn_hi'])
    l = np.arange(256)
    for pal, table in ((vv.NUSCENES_PALETTE, GOLD['nuscenes_colors']),
                       (vv.KITTI_PALETTE, np.concatenate([GOLD['kitti_colors'], np.full((19, 1), 255, np.uint8)], 1))):
        n = len(table)
        assert pal.shape == (256, 4) and pal.dtype == np.uint8
        assert np.array_equal(pal[:, 3] != 0, (l > lo) & (l < hi))
        # VTK's lookup of scalar l in [vmin, vmax] = [1, n] over n entries: floor((l - 1) / (n - 1) * n), clamped
        row = np.clip(np.floor((l - 1) / (n - 1) * n), 0, n - 1).astype(int)
        drawn = (l > lo) & (l < hi)
        assert np.array_equal(pal[drawn, :3], table[row[drawn], :3])
    j = vv.jet(1, 16)
    assert np.array_equal(j[:, 3] != 0, (l > lo) & (l < hi))
    assert tuple(j[1, :3]) == (0, 0, 128) and tuple(j[16, :3]) == (128, 0, 0)      # dark blue .. dark red
    assert 6 <= 1 + int(np.argmax(j[1:17, 1])) <= 11 and j[1:17, 1].max() == 255   # green at mid-height


def test_voxel_layout_is_get_grid_coords_and_the_flattening_of_vis_3d():
    """vis_3d.py pairs get_grid_coords(voxels.shape)[n] with voxels.reshape(-1)[n]; on a square grid voxel [h, w, d] is
    drawn centred at (w + 1/2, h + 1/2, d + 1/2) * res: the first array axis runs along y."""
    dims, res = tuple(GOLD['grid_dims']), GOLD['grid_res'].astype(np.float32)
    assert dims[0] == dims[1]
    coords = GOLD['grid_coords']
    H, W, D = dims
    n = np.arange(H * W * D)
    h, w, d = n // (W * D), (n // D) % W, n % D                   # voxels.reshape(-1)[n] = voxels[h, w, d]
    origin = (0.0, 0.0, 0.0)
    lo, hi = ref._boxes(dims, origin, float(res[0]), n)
    assert np.allclose((lo + hi) / 2, coords, atol=1e-6)
    assert np.allclose(coords[:, 0], (w + 0.5) * res[0], atol=1e-6) and np.allclose(coords[:, 1], (h + 0.5) * res[1], atol=1e-6)


def _weld(m):
    v = m['vertices']
    _, inv = np.unique(v, axis=0, return_inverse=True)
    return inv.reshape(-1)[m['faces']], inv.max() + 1


def _directed_edges(f):
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def _components(f, nv):
    parent = np.arange(nv)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in _directed_edges(f):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[ra] = rb
    roots = np.array([find(x) for x in np.unique(f)])
    return len(np.unique(roots))


def _check_closed_oriented(f):
    e = _directed_edges(f)
    fwd = {tuple(x) for x in e.tolist()}
    assert len(fwd) == len(e), 'an edge is used twice in the same direction: inconsistent orientation'
    assert all((b, a) in fwd for a, b in fwd), 'an edge has no opposite: the surface is open'


def _euler(f):
    e = _directed_edges(f)
    return len(np.unique(f)) - len(e) // 2 + len(f)


@pytest.mark.parametrize('box', [(1, 1, 1), (2, 3, 4), (5, 1, 2)])
def test_face_mesh_of_a_box(box):
    a, b, c = box
    lab = np.zeros((a + 2, b + 2, c + 2), np.uint8)
    lab[1:1 + a, 1:1 + b, 1:1 + c] = 7
    m = ref.faces_ref(lab, (0.5, -1.0, 2.0), 0.25, DRAWN)
    assert len(m['faces']) == 4 * (a * b + b * c + c * a)
    if box == (1, 1, 1):
        assert len(m['faces']) == 12
    f, nv = _weld(m)
    _check_closed_oriented(f)
    assert _euler(f) == 2 and _components(f, nv) == 1
    assert (m['sem'] == 7).all()
    _check_outward(m)


def _check_outward(m):
    v = m['vertices'].astype(np.float64)
    f = m['faces']
    n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (np.einsum('ij,ij->i', n, m['normals'][f[:, 0]]) > 0).all()
    assert np.array_equal(np.abs(m['normals']).sum(1), np.ones(len(v), np.float32))


def test_face_mesh_of_separate_boxes_and_a_random_grid():
    lab = np.zeros((6, 9, 5), np.uint8)
    lab[1:3, 1:4, 1:3] = 3
    lab[3:5, 6:8, 2:4] = 12                                   # a second component
    m = ref.faces_ref(lab, (0, 0, 0), 1.0, DRAWN)
    f, nv = _weld(m)
    _check_closed_oriented(f)
    assert _components(f, nv) == 2 and _euler(f) == 4
    # random grids: every edge still pairs with an opposite edge (closed, oriented), faces point out, grid borders close
    rng = np.random.default_rng(0)
    lab = _random_grid(rng, (6, 7, 5), 0.5)
    m = ref.faces_ref(lab, (-1, 2, 0.5), 0.4, DRAWN)
    e = _directed_edges(_weld(m)[0])
    fwd, bwd = np.unique(e, axis=0, return_counts=True), np.unique(e[:, ::-1], axis=0, return_counts=True)
    assert np.array_equal(fwd[0], bwd[0]) and np.array_equal(fwd[1], bwd[1])
    _check_outward(m)
    # exposed faces counted directly
    dv = DRAWN[lab]
    p = np.pad(dv, 1)
    n_exp = sum((dv & ~np.roll(p, s, ax)[1:-1, 1:-1, 1:-1]).sum() for ax in range(3) for s in (1, -1))
    assert len(m['faces']) == 2 * n_exp


def _read_png(path):
    data = open(path, 'rb').read()
    assert data[:8] == b'\x89PNG\r\n\x1a\n'
    pos, idat, hdr = 8, b'', None
    while pos < len(data):
        n, = struct.unpack('>I', data[pos:pos + 4])
        tag, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack('>I', data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(tag + body) & 0xffffffff
        if tag == b'IHDR':
            hdr = struct.unpack('>IIBBBBB', body)
        elif tag == b'IDAT':
            idat += body
        pos += 12 + n
    w, h, depth, ctype = hdr[:4]
    assert depth == 8 and ctype == 2
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 3 * w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, 3)


def test_write_png_round_trips(tmp_path):
    img = np.random.default_rng(1).integers(0, 256, size=(37, 53, 3), dtype=np.uint8)
    vv.write_png(str(tmp_path / 'a.png'), img)
    assert np.array_equal(_read_png(str(tmp_path / 'a.png')), img)
    vv.write_png(str(tmp_path / 'b.png'), torch.from_numpy(img))
    assert open(tmp_path / 'a.png', 'rb').read() == open(tmp_path / 'b.png', 'rb').read()


def test_height_labels_and_from_img2lidar():
    occ = torch.zeros(3, 4, 6, dtype=torch.uint8)
    occ[1, 2] = 1
    occ[0, 0, 2] = 5
    h = vv.height_labels(occ, cap=2)
    assert h.dtype == torch.uint8
    assert h[1, 2].tolist() == [1, 2, 3, 4, 0, 0] and h[0, 0, 2] == 3 and int(h.sum()) == 13
    # the frame's cameras: a lidar point at depth t along pixel (u + 1/2, v + 1/2) of the output image
    K = np.array([[400.0, 0, 320.0], [0, 400.0, 180.0], [0, 0, 1.0]])
    l2c = np.eye(4)
    l2c[:3, :3] = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]])      # camera looking along lidar +x
    l2c[:3, 3] = [0.1, 1.5, -0.3]
    l2i = np.eye(4)
    l2i[:3, :4] = K @ l2c[:3, :4]
    i2l = np.linalg.inv(l2i)
    rows = vv.from_img2lidar(torch.tensor(i2l[None]), (360, 640), out_size=(90, 160), clip=(0.5, 80.0))
    assert rows.shape == (1, 16) and rows.dtype == torch.float32
    o, d, near, far = ref.rays_from_rows(rows.numpy().astype(np.float64), (90, 160))
    u, v, t = 17, 60, 12.5
    p = o[0] + t * d[0, v, u]
    q = l2i @ np.append(p, 1.0)
    assert q[2] == pytest.approx(t, rel=1e-6)
    assert q[0] / q[2] == pytest.approx((u + 0.5) * 4.0, rel=1e-6) and q[1] / q[2] == pytest.approx((v + 0.5) * 4.0, rel=1e-6)
    assert (near[0], far[0]) == (0.5, 80.0)


def test_entry_points_refuse_bad_arguments_without_a_gpu():
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N, one = None, C.c_void_p(16)
    org = (C.c_float * 3)(0, 0, 0)
    pal = np.zeros((256, 4), np.uint8)
    sh = np.array(vv.SHADE, np.float32)
    bg = np.array([255, 255, 255], np.uint8)
    P, S, B = (a.ctypes.data_as(C.c_void_p) for a in (pal, sh, bg))
    r = lib.so_voxel_render
    assert r(N, 4, 4, 4, org, 0.4, one, 2, 8, 8, P, S, B, one, N, N, N, N) == -1                 # no labels
    assert r(one, 4, 4, 4, N, 0.4, one, 2, 8, 8, P, S, B, one, N, N, N, N) == -1                  # no origin
    assert r(one, 0, 4, 4, org, 0.4, one, 2, 8, 8, P, S, B, one, N, N, N, N) == -1                # H = 0
    assert r(one, 4, 4, 4, org, 0.0, one, 2, 8, 8, P, S, B, one, N, N, N, N) == -1                # voxel size 0
    assert r(one, 4, 4, 4, org, float('inf'), one, 2, 8, 8, P, S, B, one, N, N, N, N) == -1
    assert r(one, 4, 4, 4, org, 0.4, N, 2, 8, 8, P, S, B, one, N, N, N, N) == -1                  # no cameras
    assert r(one, 4, 4, 4, org, 0.4, one, 0, 8, 8, P, S, B, one, N, N, N, N) == -1                # K = 0
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 0, 8, P, S, B, one, N, N, N, N) == -1                # empty image
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 8, 8, N, S, B, one, N, N, N, N) == -1                # no palette
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 8, 8, P, N, B, one, N, N, N, N) == -1
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 8, 8, P, S, N, one, N, N, N, N) == -1
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 8, 8, P, S, B, N, N, N, N, N) == -1                  # no output at all
    assert r(one, 4, 4, 4, org, 0.4, C.c_void_p(24), 2, 8, 8, P, S, B, one, N, N, N, N) == -1     # cameras not 16-byte aligned
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 8, 8, P, S, B, N, C.c_void_p(18), N, N, N) == -1     # voxel not 4-byte aligned
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 8, 8, P, S, B, N, N, N, C.c_void_p(18), N) == -1     # dist not 4-byte aligned
    bad = np.array([0.8, 0.8, 0.65, 0.65, 0.5, 1.5], np.float32)
    assert r(one, 4, 4, 4, org, 0.4, one, 2, 8, 8, P, bad.ctypes.data_as(C.c_void_p), B, one, N, N, N, N) == -1
    assert r(one, 4, 4, 4, org, 0.4, one, 70000, 8, 8, P, S, B, one, N, N, N, N) == -2            # K beyond the grid
    assert r(one, 40000, 40000, 4, org, 0.4, one, 2, 8, 8, P, S, B, one, N, N, N, N) == -2        # >= 2^31 voxels
    dr = vv.drawn_table()
    DR = dr.ctypes.data_as(C.c_void_p)
    cnt = lib.so_voxel_faces_count
    assert cnt(N, 4, 4, 4, DR, one, N) == -1 and cnt(one, 4, 4, 4, N, one, N) == -1 and cnt(one, 4, 4, 4, DR, N, N) == -1
    assert cnt(one, 4, -1, 4, DR, one, N) == -1 and cnt(one, 4, 4, 4, DR, C.c_void_p(18), N) == -1
    assert cnt(one, 40000, 40000, 4, DR, one, N) == -2
    em = lib.so_voxel_faces_emit
    assert em(one, 4, 4, 4, org, 0.4, DR, one, 0, one, one, one, N, N) == -1                      # no faces
    assert em(one, 4, 4, 4, org, 0.4, DR, N, 5, one, one, one, N, N) == -1                        # no scans
    assert em(one, 4, 4, 4, org, 0.4, DR, one, 5, N, one, one, N, N) == -1
    assert em(one, 4, 4, 4, org, 0.4, DR, one, 5, one, N, one, N, N) == -1
    assert em(one, 4, 4, 4, org, 0.4, DR, one, 5, one, one, N, N, N) == -1
    assert em(one, 4, 4, 4, org, -0.4, DR, one, 5, one, one, one, N, N) == -1
    assert em(one, 4, 4, 4, org, 0.4, DR, one, 5, C.c_void_p(18), one, one, N, N) == -1
    assert em(one, 4, 4, 4, org, 0.4, DR, one, 1 << 29, one, one, one, N, N) == -2                # vertex ids beyond int32


def test_python_entry_points_refuse_cpu_tensors_and_device_tables():
    lab = torch.zeros(4, 4, 4, dtype=torch.uint8)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        vv.render_voxels(lab, (0, 0, 0), 0.4, vv.VIS3D_NUSCENES, (8, 8), vv.NUSCENES_PALETTE)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        vv.voxel_mesh(lab, (0, 0, 0), 0.4)
    with pytest.raises(ValueError):
        vv.drawn_table(np.zeros((255, 4), np.uint8))
