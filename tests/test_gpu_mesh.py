"""GPU: the surface of the decoded field (so_mesh_count / so_mesh_emit through NeuSHead.mesh) against the fp64 oracle
(oracle/mesh.py) run on forward_occ's sdf, index for index, at the nuScenes-occ, KITTI-occ and BEV (tpv=False) geometries
and on an analytic scene; vertices against head.occupancy's labels; attributes against the field query; determinism, one
host synchronisation per call, and the empty surface."""
import json
import os
import warnings
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle.mesh import marching_cubes_ref
from selfocc_b200 import _lib, mesh as mesh_mod, ops, synth
from selfocc_b200 import occupancy as occ_mod
from selfocc_b200.mapping import GridMeterMapping
from selfocc_b200.registry import build_head
import selfocc_b200.segmentor  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_model_cfgs.json')))
BEV_HEAD = json.load(open(os.path.join(HERE, 'golden', 'reference_model_cfgs_bev.json')))['nuscenes/nuscenes_occ_bev.py']['head']
EPS32 = float(torch.finfo(torch.float32).eps)

# kind -> (head config, overrides, resolution, lut)
CASES = {
    'nusc_occ': (CFGS['nuscenes/nuscenes_occ.py']['head'], {}, 0.4, occ_mod.OPENSEED2NUSCENES),
    # kitti_occ.py decodes colour only; with 19 Cityscapes logits its lattice labels go through cityscapes2semantickitti
    'kitti_occ': (CFGS['kitti/kitti_occ.py']['head'], dict(color_dims=3 + 19, return_sem=True), 0.2,
                  occ_mod.CITYSCAPES2SEMANTICKITTI),
    'bev': (BEV_HEAD, {}, 0.4, occ_mod.OPENSEED2NUSCENES),
}


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _head(kind, dev, occupied=0.3):
    """A head of the config with a random decoder, its sdf bias shifted so that ``occupied`` of the voxels are inside.
    -> (head, representation, aabb, resolution, lut)"""
    cfg, over, res, lut = CASES[kind]
    head = build_head(dict(cfg, return_second_grad=False, **over)).eval().to(dev)
    f = head.model.field
    m = f.mapping
    cf = 1 + f.color_dims
    if f.tpv:
        rep = [p[None].to(dev) for p in synth.random_planes(m, 96, scale=1.0, seed=5)]
    else:
        rep = torch.randn(1, m.size_h * m.size_w, 96, generator=torch.Generator().manual_seed(5)).to(dev)
    w1, b1, w2, b2 = synth.random_mlp(96, f.density_net[3].out_features, seed=2)
    with torch.no_grad():
        for lin, w, b in ((f.density_net[1], w1, b1), (f.density_net[3], w2, b2)):
            lin.weight.copy_(w); lin.bias.copy_(b)
        head.prepare(rep)
        q = torch.quantile(f.vol_sdf[..., :f.desc.Z].flatten()[::7], occupied)
        f.density_net[3].bias[::cf] -= q                # the sdf row (TPV) or the sdf column of every z (BEV)
    return head, rep, cfg['roi_aabb'], res, lut


def _check_against_oracle(tag, vertices, faces, sdf, axes, thresh, res):
    """faces torch.equal to the oracle's on the same lattice values; vertices within 1e-5 of a cell plus the fp32 rounding
    of the coordinate itself."""
    v_ref, f_ref = marching_cubes_ref(sdf.cpu().double().numpy(), *[a.cpu().double().numpy() for a in axes], thresh=thresh)
    print('%s: %d vertices, %d faces' % (tag, len(v_ref), len(f_ref)))
    assert len(f_ref) > 1000
    assert torch.equal(faces.cpu(), torch.from_numpy(f_ref).to(torch.int32)), tag
    v_ref = torch.from_numpy(v_ref)
    err = (vertices.cpu().double() - v_ref).abs()
    assert (err <= 1e-5 * res + 2 * EPS32 * v_ref.abs()).all(), (tag, err.max().item())


@pytest.mark.parametrize('kind', list(CASES))
def test_mesh_matches_oracle_occupancy_and_field_query(kind):
    dev = _dev()
    head, rep, aabb, res, lut = _head(kind, dev)
    thresh = 0.0
    out = head.forward_occ(rep, aabb=aabb, resolution=res)
    m = head.mesh(aabb, res, thresh=thresh, lut=lut)
    f = head.model.field
    axes = occ_mod.lattice_axes(aabb, res, dev)
    assert m['vertices'].dtype == torch.float32 and m['faces'].dtype == torch.int32
    _check_against_oracle(kind, m['vertices'], m['faces'], out['sdf'], axes, thresh, res)

    # a vertex on a lattice edge if and only if head.occupancy's labels differ at its ends, in owner-then-axis order
    occ = head.occupancy(aabb, res, thresh=thresh)['occ'].bool()
    ny, nx, nz = occ.shape
    cross = torch.zeros(ny, nx, nz, 3, dtype=torch.bool, device=dev)
    cross[:, :-1, :, 0] = occ[:, :-1] != occ[:, 1:]
    cross[:-1, :, :, 1] = occ[:-1] != occ[1:]
    cross[:, :, :-1, 2] = occ[:, :, :-1] != occ[:, :, 1:]
    p, a = torch.nonzero(cross.reshape(-1, 3), as_tuple=True)
    assert p.numel() == m['vertices'].shape[0]
    iy, ix, iz = p // (nx * nz), (p // nz) % nx, p % nz
    lo = torch.stack([axes[0][ix], axes[1][iy], axes[2][iz]], -1)
    hi = torch.stack([axes[0][(ix + 1).clamp(max=nx - 1)], axes[1][(iy + 1).clamp(max=ny - 1)],
                      axes[2][(iz + 1).clamp(max=nz - 1)]], -1)
    v = m['vertices']
    along = F.one_hot(a, 3).bool()
    assert torch.equal(v[~along], lo[~along])
    va, la, ha = v[along], lo[along], hi[along]
    assert ((va >= la) & (va <= ha)).all()

    # attributes: the field query at the vertices
    _, grad, feat = ops.field_query(f.vol_sdf, f.vol_feat, f.desc, v, want_grad=True, want_feat=True)
    assert torch.equal(m['normals'], F.normalize(grad, dim=-1))
    n_sem = f.color_dims - 3
    assert torch.equal(m['sem'], torch.tensor(lut, dtype=torch.uint8, device=dev)[torch.argmax(feat[:, 3:3 + n_sem], -1)])
    assert torch.equal(m['rgb'], (feat[:, :3] * mesh_mod.SH_C0 + 0.5).clamp_min(0.0))
    assert m['sem'].unique().numel() > 4

    # bit-identical reruns, with and without the decode
    for again in (head.mesh(aabb, res, thresh=thresh, lut=lut), head.mesh(aabb, res, thresh=thresh, lut=lut, representation=rep)):
        assert set(again) == set(m)
        for k in m:
            assert torch.equal(again[k], m[k]), k


def test_analytic_scene_matches_oracle_and_has_outward_faces():
    """The ground plane, spheres and box of synth.analytic_sdf_volume on the nuScenes-occ volume, meshed at 0.2 m."""
    dev = _dev()
    cfg = CFGS['nuscenes/nuscenes_occ.py']['head']
    m = GridMeterMapping(**cfg['mapping_args'])
    desc = m.volume_desc(0)
    vs = synth.pack_sdf_volume(synth.analytic_sdf_volume(m), desc.zpitch).to(dev)
    aabb, res = cfg['roi_aabb'], 0.2
    axes = occ_mod.lattice_axes(aabb, res, dev)
    xs, ys, zs = axes
    ny, nx, nz = len(ys), len(xs), len(zs)
    xyz = torch.stack([xs[None, :, None].expand(ny, nx, nz), ys[:, None, None].expand(ny, nx, nz),
                       zs[None, None, :].expand(ny, nx, nz)], -1).reshape(-1, 3).contiguous()
    sdf = ops.field_query(vs, None, desc, xyz)[0].reshape(ny, nx, nz)        # forward_occ's lattice values
    v, f = mesh_mod.marching_cubes(vs, desc, axes, 0.0)
    _check_against_oracle('analytic', v, f, sdf, axes, 0.0, res)
    # faces point up the field gradient (out of the solids) wherever the face has an area
    fl = f.long()
    n = torch.cross(v[fl[:, 1]] - v[fl[:, 0]], v[fl[:, 2]] - v[fl[:, 0]], dim=-1)
    area = n.norm(dim=-1)
    g = ops.field_query(vs, None, desc, v[fl].mean(1).contiguous(), want_grad=True)[1]
    big = area > 1e-3 * res * res
    assert ((n[big] * g[big]).sum(-1) > 0).float().mean() > 0.999


def test_one_synchronisation_per_call():
    dev = _dev()
    head, rep, aabb, res, lut = _head('nusc_occ', dev)
    head.mesh(aabb, res, lut=lut)                  # warm-up: the LUT's one-time upload
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            m = head.mesh(aabb, res, lut=lut, representation=rep)
        finally:
            torch.cuda.set_sync_debug_mode('default')
    syncs = [x for x in w if 'called a synchronizing CUDA operation' in str(x.message)]
    assert len(syncs) == 1, [str(x.message) for x in syncs]
    assert m['faces'].shape[0] > 0


@pytest.mark.parametrize('thresh', [-1e9, 1e9])
def test_empty_surface_gives_empty_outputs_and_no_emit_pass(thresh):
    dev = _dev()
    head, rep, aabb, res, lut = _head('nusc_occ', dev)
    n0 = _lib.launch_count()
    m = head.mesh(aabb, res, thresh=thresh, lut=lut)
    assert _lib.launch_count() - n0 == 1                # the count pass only
    assert m['vertices'].shape == (0, 3) and m['faces'].shape == (0, 3) and m['normals'].shape == (0, 3)
    assert m['sem'].shape == (0,) and m['rgb'].shape == (0, 3)
