"""GPU: the voxel-cube picture (so_voxel_render through voxel_vis.render_voxels and NeuSHead.render_occupancy) against the
fp64 slab-test oracle (oracle/voxel_vis.py) on every pixel: analytic scenes, a random grid and labels from
head.occupancy on the Occ3D grid (points=) and the KITTI lattice, seen from the vis_3d presets, the frame's own cameras
and random look-ats.  Hit voxel and face equal the oracle's except counted ties; the colour equals the palette-and-shade
rule exactly.  Also: K cameras in one launch equal K launches, bit-identical reruns, no host synchronisation, and
voxel_mesh equal to the oracle's faces with a PLY that loads back."""
import json
import os
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import voxel_vis as ref
from selfocc_b200 import mesh as mesh_mod, synth, voxel_vis as vv
from selfocc_b200 import occupancy as occ_mod
from selfocc_b200.registry import build_head
import selfocc_b200.segmentor  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_model_cfgs.json')))
OCC3D_ORIGIN, OCC3D_VS = (-40.0, -40.0, -1.0), 0.4


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _check(tag, labels, origin, vs, cameras, image_size, palette, shade=vv.SHADE, background=vv.BACKGROUND, min_hits=1):
    """Render on the device, run the oracle on every pixel of every camera, and hold the device to it."""
    out = vv.render_voxels(labels, origin, vs, cameras, image_size, palette, shade=shade, background=background,
                           want=('rgb', 'voxel', 'face', 'dist'))
    if isinstance(cameras, (list, tuple)) and isinstance(cameras[0], vv.Camera):
        cameras = [c.resized(image_size) for c in cameras]
    rows = vv.camera_rows(cameras, labels.device).cpu().numpy()
    lab = labels.cpu().numpy()
    drawn = np.asarray(palette)[:, 3] != 0
    o, d, near, far = ref.rays_from_rows(rows, image_size)
    n_px = n_tie = n_hit = 0
    for k in range(rows.shape[0]):
        dk = d[k].reshape(-1, 3)
        vox, face, t = ref.render_ref(lab, origin, vs, o[k], dk, near[k], far[k], drawn)
        gv = out['voxel'][k].reshape(-1).cpu().numpy().astype(np.int64)
        gf = out['face'][k].reshape(-1).cpu().numpy().astype(np.int64)
        bad = (gv != vox) | (gf != face)
        tie = ref.ties(lab, origin, vs, o[k], dk, near[k], far[k], gv, gf, vox, face, t)
        assert not (bad & ~tie).any(), (tag, k, np.flatnonzero(bad & ~tie)[:8], gv[bad & ~tie][:8], vox[bad & ~tie][:8])
        n_tie += int((bad & tie).sum())
        n_px += dk.shape[0]
        n_hit += int((gv >= 0).sum())
        # given the device's hit: its colour by the rule, its depth the fp64 entry rounded to fp32
        rgb = ref.shade_rgb(lab, gv, gf, palette, shade, background)
        assert np.array_equal(out['rgb'][k].reshape(-1, 3).cpu().numpy(), rgb), (tag, k)
        dist = out['dist'][k].reshape(-1).cpu().numpy()
        hit = gv >= 0
        assert np.isinf(dist[~hit]).all() and (gf[~hit] == -1).all()
        te = ref.voxel_entry(lab.shape, origin, vs, o[k], dk, gv)[0]
        assert np.allclose(dist[hit], te[hit], rtol=1e-6, atol=0), tag
    print('%s: %d pixels, %d hit, %d ties' % (tag, n_px, n_hit, n_tie))
    assert n_tie <= 1e-4 * n_px, (tag, n_tie, n_px)
    assert n_hit >= min_hits, tag
    return out


def _random_look_ats(rng, centre, radius, n, image_size, clip=(0.01, 300.0)):
    cams = []
    for _ in range(n):
        dirn = rng.normal(size=3)
        dirn[2] = abs(dirn[2]) + 0.3
        pos = centre + radius * dirn / np.linalg.norm(dirn)
        cams.append(vv.look_at(pos, centre + rng.normal(size=3), (0, 0, 1), rng.uniform(25, 60), image_size, clip))
    return cams


def _grid_centre(shape, origin, vs):
    return np.asarray(origin) + 0.5 * vs * np.array([shape[1], shape[0], shape[2]])


# ----------------------------------------------------------------------------------------------------- analytic scenes
def _analytic(kind, dev):
    shape = (12, 10, 6)
    lab = np.zeros(shape, np.uint8)
    if kind == 'one_voxel':
        lab[5, 4, 2] = 3
    elif kind == 'checkerboard':
        h, w, d = np.meshgrid(*[np.arange(s) for s in shape], indexing='ij')
        lab[:] = np.where((h + w + d) % 2 == 0, 1 + (h + 2 * w + 3 * d) % 16, 0)
    elif kind == 'slab':
        lab[:, :, 1:3] = 11
        lab[2:5, 3:7, 3] = 200                              # >= 100: not drawn
    elif kind == 'empty':
        lab[:] = 0
        lab[0, 0, 0] = 150
    return torch.from_numpy(lab).to(dev)


@pytest.mark.parametrize('kind', ['one_voxel', 'checkerboard', 'slab', 'empty'])
def test_analytic_scenes_match_oracle(kind):
    dev = _dev()
    lab = _analytic(kind, dev)
    origin, vs = (-1.7, 0.3, -0.9), 0.5
    centre = _grid_centre(lab.shape, origin, vs)
    cams = _random_look_ats(np.random.default_rng(1), centre, 9.0, 3, (40, 56))
    out = _check(kind, lab, origin, vs, cams, (40, 56), vv.NUSCENES_PALETTE, min_hits=0 if kind == 'empty' else 10)
    if kind == 'empty':
        assert (out['rgb'] == 255).all() and (out['voxel'] == -1).all()


def test_camera_inside_grid_axis_parallel_rays_and_clipping():
    dev = _dev()
    rng = np.random.default_rng(2)
    shape = (16, 14, 8)
    lab_np = np.where(rng.random(shape) < 0.15, rng.integers(1, 17, shape), 0).astype(np.uint8)
    lab = torch.from_numpy(lab_np).to(dev)
    origin, vs = (0.0, 0.0, 0.0), 1.0
    centre = _grid_centre(shape, origin, vs) + np.array([0.31, -0.27, 0.13])
    # inside the grid, rows built so the pixel-centre rays of row 15 and column 15 of a 31 x 31 image have exact zero
    # components (s a power of two): along +x, along -y and straight down
    s = 1.0 / 16
    dirs = [((0, 0, 1), (s, 0, -15.5 * s), (0, -s, 15.5 * s)),
            ((s, 0, -15.5 * s), (0, 0, -1), (0, -s, 15.5 * s)),
            ((s, 0, -15.5 * s), (0, -s, 15.5 * s), (0, 0, -1))]
    rows = np.array([np.concatenate([centre, np.array(M, dtype=np.float64).reshape(-1), [0.01, 100.0, 0, 0]])
                     for M in dirs])
    _check('inside/axis', lab, origin, vs, rows, (31, 31), vv.NUSCENES_PALETTE, min_hits=100)
    o, d, _, _ = ref.rays_from_rows(rows.astype(np.float32), (31, 31))
    assert (d[:, 15, :] == 0).sum() >= 3 * 31 and (d[:, 15, 15] == 0).sum() == 6
    # near / far clipping cut through the grid
    cams = [vv.look_at(centre + np.array([-20.0, 3.0, 9.0]), centre, (0, 0, 1), 40.0, (31, 31), (17.3, 24.1)),
            vv.look_at(centre + np.array([4.0, 18.0, 12.0]), centre, (0, 0, 1), 50.0, (31, 31), (0.01, 19.7))]
    _check('clip', lab, origin, vs, cams, (31, 31), vv.NUSCENES_PALETTE, min_hits=100)


def test_random_grid_64x64x16():
    dev = _dev()
    rng = np.random.default_rng(3)
    shape = (64, 64, 16)
    lab_np = np.where(rng.random(shape) < 0.2, rng.integers(1, 17, shape), 0).astype(np.uint8)
    lab = torch.from_numpy(lab_np).to(dev)
    origin, vs = (-12.8, -12.8, -2.0), 0.4
    centre = _grid_centre(shape, origin, vs)
    cams = _random_look_ats(rng, centre, 35.0, 2, (45, 80)) + [vv.VIS3D_NUSCENES]
    _check('random64', lab, origin, vs, cams, (45, 80), vv.NUSCENES_PALETTE, shade=(0.9, 0.7, 0.6, 0.55, 0.3, 1.0),
           background=(10, 20, 30), min_hits=1000)


# ----------------------------------------------------------------------------------------------------- the model
def _head(kind, dev, occupied=0.3):
    cfg = CFGS['nuscenes/nuscenes_occ.py' if kind == 'nusc' else 'kitti/kitti_occ.py']['head']
    over = {} if kind == 'nusc' else dict(color_dims=3 + 19, return_sem=True)
    head = build_head(dict(cfg, return_second_grad=False, **over)).eval().to(dev)
    f = head.model.field
    cf = 1 + f.color_dims
    rep = [p[None].to(dev) for p in synth.random_planes(f.mapping, 96, scale=1.0, seed=5)]
    w1, b1, w2, b2 = synth.random_mlp(96, f.density_net[3].out_features, seed=2)
    with torch.no_grad():
        for lin, w, b in ((f.density_net[1], w1, b1), (f.density_net[3], w2, b2)):
            lin.weight.copy_(w); lin.bias.copy_(b)
        head.prepare(rep)
        q = torch.quantile(f.vol_sdf[..., :f.desc.Z].flatten()[::7], occupied)
        f.density_net[3].bias[::cf] -= q
        head.prepare(rep)                               # decode again with the shifted bias
    return head, cfg['roi_aabb']


def test_occ3d_labels_from_the_model():
    dev = _dev()
    head, aabb = _head('nusc', dev)
    pts = occ_mod.occ3d_lidar_points(torch.eye(4), dev)
    l2i, i2l = synth.camera_rig(f=633.0, cx=400.0, cy=225.0)
    own = vv.from_img2lidar(torch.tensor(i2l, device=dev), (450, 800), out_size=(18, 32), clip=(0.05, 120.0))
    out, labels = head.render_occupancy(aabb, 0.4, 0.0, own, (18, 32), vv.NUSCENES_PALETTE, lut=occ_mod.OPENSEED2NUSCENES,
                                        points=pts, want=('rgb', 'voxel'))
    ref_labels = head.occupancy(aabb, 0.4, 0.0, lut=occ_mod.OPENSEED2NUSCENES, points=pts)['sem'].permute(1, 0, 2)
    assert torch.equal(labels, ref_labels) and labels.shape == (200, 200, 16)
    assert labels.unique().numel() > 4
    _check('occ3d/own', labels, OCC3D_ORIGIN, OCC3D_VS, own, (18, 32), vv.NUSCENES_PALETTE, min_hits=500)
    rng = np.random.default_rng(4)
    views = [vv.VIS3D_NUSCENES] + _random_look_ats(rng, np.array([0.0, 0.0, 2.2]), 60.0, 1, (27, 48))
    _check('occ3d/views', labels, OCC3D_ORIGIN, OCC3D_VS, views, (27, 48), vv.NUSCENES_PALETTE, min_hits=500)
    # the frame's cameras through the head's wrapper equal render_voxels on its labels
    again = vv.render_voxels(labels, OCC3D_ORIGIN, OCC3D_VS, own, (18, 32), vv.NUSCENES_PALETTE, want=('rgb', 'voxel'))
    assert torch.equal(again['rgb'], out['rgb']) and torch.equal(again['voxel'], out['voxel'])


def test_kitti_lattice_from_the_model():
    dev = _dev()
    head, aabb = _head('kitti', dev)
    occ = head.occupancy(aabb, 0.2, 0.0, lut=occ_mod.CITYSCAPES2SEMANTICKITTI)
    labels = occ['sem']
    assert labels.shape == (256, 256, 32)
    metas = dict(cam_positions=[[0.3, -6.0, 9.0]], focal_positions=[[0.3, 8.0, 1.0]])
    views = [vv.kitti_camera(metas)] + _random_look_ats(np.random.default_rng(5), np.array([0.0, 25.6, 1.2]), 45.0, 1,
                                                        (27, 48))
    out = _check('kitti', labels, tuple(aabb[:3]), 0.2, views, (18, 32), vv.KITTI_PALETTE, min_hits=200)
    # the non-semantic branch: height labels under jet
    hl = vv.height_labels(occ['occ'], cap=4)
    _check('kitti/height', hl, tuple(aabb[:3]), 0.2, views[:1], (18, 32), vv.jet(1, 28), min_hits=100)
    w, _ = head.render_occupancy(aabb, 0.2, 0.0, views, (18, 32), vv.KITTI_PALETTE, lut=occ_mod.CITYSCAPES2SEMANTICKITTI)
    assert torch.equal(w['rgb'], out['rgb'])


# ----------------------------------------------------------------------------------------------------- launch properties
def _scene(dev):
    rng = np.random.default_rng(6)
    shape = (200, 200, 16)
    lab = torch.from_numpy(np.where(rng.random(shape) < 0.1, rng.integers(1, 17, shape), 0).astype(np.uint8)).to(dev)
    cams = [vv.VIS3D_NUSCENES] + _random_look_ats(rng, np.array([0.0, 0.0, 2.0]), 70.0, 5, (1, 1))
    return lab, cams


def test_k_cameras_in_one_launch_equal_k_launches_and_reruns_are_bit_identical():
    dev = _dev()
    lab, cams = _scene(dev)
    size = (144, 256)
    want = ('rgb', 'voxel', 'face', 'dist')
    allk = vv.render_voxels(lab, OCC3D_ORIGIN, OCC3D_VS, cams, size, vv.NUSCENES_PALETTE, want=want)
    for k, c in enumerate(cams):
        one = vv.render_voxels(lab, OCC3D_ORIGIN, OCC3D_VS, [c], size, vv.NUSCENES_PALETTE, want=want)
        for key in want:
            assert torch.equal(one[key][0], allk[key][k]), (k, key)
    again = vv.render_voxels(lab, OCC3D_ORIGIN, OCC3D_VS, cams, size, vv.NUSCENES_PALETTE, want=want)
    for key in want:
        assert torch.equal(again[key], allk[key]), key
    # outputs asked for alone equal the full set
    rgb = vv.render_voxels(lab, OCC3D_ORIGIN, OCC3D_VS, cams, size, vv.NUSCENES_PALETTE)
    assert set(rgb) == {'rgb'} and torch.equal(rgb['rgb'], allk['rgb'])
    assert (allk['voxel'] >= 0).float().mean() > 0.05


def test_no_host_synchronisation():
    dev = _dev()
    lab, cams = _scene(dev)
    l2i, i2l = synth.camera_rig(f=633.0, cx=400.0, cy=225.0)
    M = torch.tensor(i2l, device=dev)
    vv.render_voxels(lab, OCC3D_ORIGIN, OCC3D_VS, cams, (72, 128), vv.NUSCENES_PALETTE)       # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        a = vv.render_voxels(lab, OCC3D_ORIGIN, OCC3D_VS, cams, (72, 128), vv.NUSCENES_PALETTE, want=('rgb', 'dist'))
        own = vv.from_img2lidar(M, (450, 800), out_size=(45, 80))
        b = vv.render_voxels(lab, OCC3D_ORIGIN, OCC3D_VS, own, (45, 80), vv.NUSCENES_PALETTE, want=('rgb', 'voxel', 'face'))
    finally:
        torch.cuda.set_sync_debug_mode('default')
    torch.cuda.synchronize()
    assert a['rgb'].shape == (len(cams), 72, 128, 3) and b['voxel'].shape == (6, 45, 80)


# ----------------------------------------------------------------------------------------------------- the face mesh
@pytest.mark.parametrize('palette', [None, 'nusc'])
def test_voxel_mesh_equals_oracle_faces_and_writes_a_ply(palette, tmp_path):
    dev = _dev()
    rng = np.random.default_rng(7)
    shape = (40, 48, 16)
    lab_np = np.where(rng.random(shape) < 0.3, rng.integers(1, 20, shape), 0).astype(np.uint8)
    lab_np[rng.random(shape) < 0.02] = 180
    lab = torch.from_numpy(lab_np).to(dev)
    pal = vv.NUSCENES_PALETTE if palette else None
    origin, vs = (-9.6, -8.0, -1.0), 0.4
    m = vv.voxel_mesh(lab, origin, vs, palette=pal)
    r = ref.faces_ref(lab_np, origin, vs, vv.drawn_table(pal).astype(bool))
    assert len(r['faces']) > 10000
    assert np.array_equal(m['vertices'].cpu().numpy(), r['vertices'])
    assert np.array_equal(m['faces'].cpu().numpy(), r['faces'])
    assert np.array_equal(m['normals'].cpu().numpy(), r['normals'])
    assert np.array_equal(m['sem'].cpu().numpy(), r['sem'])
    again = vv.voxel_mesh(lab, origin, vs, palette=pal)
    assert all(torch.equal(again[k], m[k]) for k in m)
    path = str(tmp_path / 'voxels.ply')
    mesh_mod.write_ply(path, m, colormap=vv.NUSCENES_PALETTE)
    data = open(path, 'rb').read()
    head = data[:data.index(b'end_header\n') + len(b'end_header\n')].decode()
    nv = int(head.split('element vertex ')[1].split()[0])
    nf = int(head.split('element face ')[1].split()[0])
    assert nv == m['vertices'].shape[0] and nf == m['faces'].shape[0]
    assert len(data) == len(head) + nv * (6 * 4 + 3) + nf * (1 + 3 * 4)


def test_empty_volume_gives_an_empty_mesh():
    dev = _dev()
    m = vv.voxel_mesh(torch.zeros(8, 8, 4, dtype=torch.uint8, device=dev), (0, 0, 0), 0.5)
    assert m['vertices'].shape == (0, 3) and m['faces'].shape == (0, 3) and m['sem'].shape == (0,)
