"""GPU parity of the inference render against the fp64 oracle at every shipped TPV head's geometry: each head's mapping,
ROI, S = 256, image size and eval ray grid (strided to a few thousand rays), the camera rigs of test_gpu_train_parity.py,
the random background every shipped head renders with, and the kernel instantiation each head runs in production:

  nuScenes_depth        render_packed_kernel<false, false, 32, 257 * 32>   compile-time pitches, fp32 element index
  nuScenes_novel_depth  render_packed_kernel<true, false, 31, 257 * 31>
  nuScenes_occ          render_infer_kernel<true, true, true>              the plain kernel, 21 semantic classes
  KITTI_occ             render_packed_kernel<true, false, 0, 0>            zpitch 40: pitches from the descriptor
  KITTI_novel_depth     render_packed_kernel<true, false, 0, 0>
  KITTI_raw_depth       render_packed_kernel<false, false, 0, 0>

Per case (analytic scene / tensor-core-decoded scene, inv_s = e, e^3, e^6.5, random background, plus white on one colour
head):
  (a) packed heads: the production launch against the probe launch (render_packed_kernel<RGB, true, 0, 0>) on every output:
      bit for bit on the rays of warps that never reach the early exit, within the exit's tail bound on the others;
  (b) the probe against the fp64 oracle with the three-part rule of oracle/parity.py, max_depth, rgb and semantics included;
  (c) nuScenes_occ has no probe: the plain kernel samples at the coordinates of march_padded, so the probe of a depth-only
      pack of the same sdf volume gives its coordinates, and (b) holds at them;
and once per head (d) NeuSHead.render against the direct launch (bit for bit) and against the oracle.

Every case asserts what it exercised: warps on the interior loop and on march_padded, warps that took the early exit (analytic
scene, sharpest inv_s), rays whose colour the random background changes, and saturated (clamped) colour channels.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from selfocc_b200 import synth
from selfocc_b200.mapping import GridMeterMapping

ROOT = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(ROOT, 'golden', 'reference_model_cfgs.json')))
S = 256
INV_S = (math.e, math.e ** 3, math.e ** 6.5)
EXIT_T, EXIT_EVERY, WARP = 1e-9, 4, 32          # render_fast.cu: SO_RF_EXIT_T, SO_RF_EXIT_EVERY; one warp = 32 launch rays
EPS32 = float(torch.finfo(torch.float32).eps)
# colour features f ~ N(1.5, 2.5^2): C0 f + 1/2 ~ N(0.92, 0.7^2) leaves [0, 1] on both sides, so the colour relu and the
# eval clamp both act
FEAT_SCALE, FEAT_OFFSET = 2.5, 1.5

# name -> (config, ray stride into the config's eval ray grid)
HEADS = {
    'nuScenes_depth': ('nuscenes/nuscenes_depth.py', 15),
    'nuScenes_novel_depth': ('nuscenes/nuscenes_novel_depth.py', 15),
    'nuScenes_occ': ('nuscenes/nuscenes_occ.py', 15),
    'KITTI_occ': ('kitti/kitti_occ.py', 5),
    'KITTI_novel_depth': ('kitti/kitti_novel_depth.py', 5),
    'KITTI_raw_depth': ('kitti_raw/kitti_raw_depth.py', 3),
}
WHITE_HEAD = 'nuScenes_novel_depth'


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def _setup(name, full=False):
    """(head config, img2lidar [N, 4, 4] fp32, pixel table [R, 2]).  The rig of test_gpu_train_parity.py plus one
    camera 7.3 m up, above every ROI, looking at the horizon.  Each shipped ROI is exactly the volume's extent, so only a ray
    that misses the ROI samples outside the volume (at the camera: the collider's near is 0 at inference); the warps that
    hold such rays take march_padded.  full: the whole eval ray grid (NeuSHead.render's), else every stride-th ray."""
    from oracle import rays as orays
    cfg_name, stride = HEADS[name]
    head = CFGS[cfg_name]['head']
    img_h, img_w = head['ray_img_size']
    if cfg_name.startswith('nuscenes'):
        lens = dict(f=1266.0 * img_w / 1600, cx=img_w / 2, cy=img_h / 2)
        _, i2l = synth.camera_rig(**lens)
    else:
        lens = dict(f=721.5, cx=img_w / 2, cy=img_h / 2)
        _, i2l = synth.camera_rig((0.,), height=1.65, radius=0.0, **lens)
    # its position lies inside no cell face of any shipped grid (a sample on a face may change cells under rounding)
    _, up = synth.camera_rig((10.,), height=7.3, radius=0.7, **lens)
    i2l = torch.tensor(np.concatenate([i2l, up]), dtype=torch.float32)
    pix = orays.fixed_ray_grid(head['ray_number'], head['ray_img_size'])
    return head, i2l, (pix if full else pix[::stride].contiguous())


def _decoder(m, n_feat, seed=0):
    """Random TPV planes and decode MLP on the device: a free-space field (sdf 1.3 +- 0.2), the kind of frame the bench
    renders.  Planes of unit scale decode to white noise of 0.6 per voxel, where the fp32 rounding of the sample
    coordinates alone (~1e-5 grid units, no cell change) moves low-accumulation depths by up to 1.5e-3 at inv_s = e^6.5,
    beyond what the independent comparison attributes.  The colour rows of the last layer get the gain and offset of the
    analytic scene's features."""
    dev = _dev()
    planes = [p.to(dev) for p in synth.random_planes(m, 96, scale=0.3, seed=seed)]
    w1, b1, w2, b2 = synth.random_mlp(96, 1 + n_feat, seed=seed)
    if n_feat:
        w2[1:4] *= FEAT_SCALE
        b2[1:4] = FEAT_SCALE * b2[1:4] + FEAT_OFFSET
    return planes, [t.to(dev) for t in (w1, b1, w2, b2)]


def _oracle_volume(planes, mlp, m):
    """fp64 decode of the planes, slab by slab on the device -> [Cf, H, W, Z]."""
    from oracle import decode_parity as dp
    v = dp.decode_slabwise(*[p.double() for p in planes], (m.size_h, m.size_w, m.size_d), *[t.double() for t in mlp])
    return v.permute(3, 0, 1, 2).contiguous()


def _volume(head, scene, seed=0):
    """-> (vol_sdf, vol_feat, desc, fp64 volume [Cf, H, W, Z] on the device)."""
    from selfocc_b200 import ops
    dev = _dev()
    m, n_feat = GridMeterMapping(**head['mapping_args']), head['color_dims']
    desc = m.volume_desc(n_feat)
    if scene == 'analytic':                 # ground plane, spheres and a box: rays terminate, warps take the early exit
        sdf = synth.analytic_sdf_volume(m, noise=0.02, seed=seed)
        feat = None
        if n_feat:
            feat = FEAT_SCALE * torch.randn(n_feat, *sdf.shape, generator=torch.Generator().manual_seed(seed + 1))
            feat[:3] += FEAT_OFFSET
        vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
        vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev) if n_feat else None
        vol64 = (sdf[None] if feat is None else torch.cat([sdf[None], feat], 0)).double().to(dev)
    else:                                   # random planes through the wgmma decode
        planes, mlp = _decoder(m, n_feat, seed)
        vs, vf = ops.tpv_decode(*planes, *mlp, desc)
        vol64 = _oracle_volume(planes, mlp, m)
    return vs, vf, desc, vol64


def _warps(x, n):
    """[n, ...] per ray -> [n_warps, 32, ...]: the kernel's lanes past the last ray repeat the last ray."""
    nw = (n + WARP - 1) // WARP
    idx = torch.arange(nw * WARP, device=x.device).clamp(max=n - 1)
    return x[idx].reshape(nw, WARP, *x.shape[1:])


def _warp_paths(grid, desc):
    """Per warp: True where render_packed_kernel takes the interior loop.  The kernel decides per ray from the cells of its
    first and last sample (the probe's coordinates are the kernel's own fp32 values); one ray outside sends its warp to
    march_padded."""
    n = grid.shape[0]
    top = torch.tensor([desc.H - 2, desc.W - 2, desc.Z - 2], dtype=grid.dtype, device=grid.device)
    ends = grid[:, [0, -1]].floor()
    inside = ((ends >= 0) & (ends <= top)).all(-1).all(-1)
    return _warps(inside, n).all(-1)


def _exit_warps(weights, interior):
    """From the fp64 weights at the kernel's coordinates: (warps that certainly stop marching early, warps that certainly
    march to the end).  T_{s+1} = (1 + 1e-7) T_s - w_s; the kernel votes after every 4th sample and stops once every lane's
    T < 1e-9.  A factor 100 either side of the threshold covers the difference between the kernel's fp32 T and this one."""
    n = weights.numel() // S
    w = weights.reshape(n, S).double()
    p = (1.0 + 1e-7) ** torch.arange(1, S + 1, dtype=torch.float64, device=w.device)
    T = p * (1.0 - torch.cumsum(w / p, -1))                     # T after sample s, [n, S]
    votes = T[:, EXIT_EVERY - 1:S - 1:EXIT_EVERY]                 # votes before the last sample
    tmax = _warps(votes, n).amax(1)                               # [n_warps, votes]
    early = interior & (tmax < 0.01 * EXIT_T).any(-1)
    never = ~interior | (tmax >= 100 * EXIT_T).all(-1)
    return early, never


def _tail_close(a, b):
    """The early exit drops a tail of weight < 1e-9 (render_fast.cu header): < 1e-9 relative, in fp32 at most a rounding step
    of the last additions."""
    a, b = a.double(), b.double()
    return (a - b).abs() <= EXIT_T * b.abs().clamp_min(1.0) + 2 * EPS32 * b.abs()


def _ray_mask(warp_mask, n):
    return warp_mask[:, None].expand(-1, WARP).reshape(-1)[:n]


def _render_case(name, head, scene, vol, i2l, pix, inv_s, bkgd, seed):
    """One (head, scene, inv_s, background) case: launches, the three-part oracle report and the edge-case counts."""
    dev = _dev()
    from oracle import rays as orays
    from oracle.mapping import GridMeterMappingRef
    from oracle.parity import render_parity
    from selfocc_b200 import ops
    vs, vf, desc, vol64 = vol
    n_feat, aabb = head['color_dims'], head['roi_aabb']
    n_cam, n_pix = i2l.shape[0], pix.shape[0]
    n = n_cam * n_pix
    want = ['depth', 'max_depth', 'max_idx', 'acc', 'normal_vis'] + (['rgb'] if n_feat else []) + (['sem'] if n_feat > 3 else [])
    g = torch.Generator().manual_seed(100 + seed)
    bk = torch.rand(n, 3, generator=g).to(dev) if (bkgd == 'random' and n_feat) else None
    params = ops.make_render_params(aabb, S, inv_s, bkgd=bkgd)
    cams, pixd = i2l.to(dev), pix.to(dev)

    def launch(vf_, desc_, want_, pack=None, probe=False, begin=0, count=None, bk_=bk):
        rays = ops.make_ray_desc(n_cam, n_pix=n_pix, ray_begin=begin, ray_count=count)
        return ops.render_infer(vs, vf_, desc_, cams, rays, params, pix=pixd, bkgd_rand=bk_, want=want_, pack=pack,
                                probe_grid=probe)

    packed = n_feat <= 3
    if packed:
        pack = ops.render_pack(vs, vf, desc)
        assert pack is not None
        prod = launch(vf, desc, want, pack=pack)
        probe = launch(vf, desc, want, pack=pack, probe=True)
        got = probe
    else:
        # (c) the plain kernel, and the sample coordinates of a depth-only pack of the same sdf volume
        assert ops.render_pack(vs, vf, desc) is None
        prod = launch(vf, desc, want)
        desc0 = GridMeterMapping(**head['mapping_args']).volume_desc(0)
        grid = launch(None, desc0, ['depth'], pack=ops.render_pack(vs, None, desc0), probe=True, bk_=None)['grid']
        got = dict(prod, grid=grid)
    origin, direction = orays.img2lidar_rays(i2l[None], pix)
    refs = {}
    kw = dict(bkgd=bkgd, bkgd_rand=bk) if bk is not None else dict(bkgd=bkgd)
    rep = render_parity(got, vol64, GridMeterMappingRef(**head['mapping_args']), origin, direction, aabb, inv_s, S,
                        color_dims=n_feat, max_flip_frac=0.04 if name.startswith('KITTI') else 0.02, refs=refs,
                        abs_rel_flip_rays=False, **kw)
    tag = '%s/%s inv_s=%.1f bkgd=%s' % (name, scene, inv_s, bkgd)
    b, ind = rep['same_cells'], rep['independent']
    print('%s: %d rays; geometry %.2e grid units; same cells: depth %.2e rel, max_depth %.2e rel, acc %.2e, normal %.2e, '
          'rgb %.2e, sem %.2e; max_idx mismatches %d (ties %d); independent: %d rays with a cell flip, %d over tol, '
          'abs_rel %.2e (%.2e without the flip rays), acc median %.3f'
          % (tag, n, rep['geometry']['max_abs_grid_units'], b['depth_max_rel'], b.get('max_depth_max_rel', 0.0),
             b['acc_max_abs'], b['normal_max_abs'], b.get('rgb_max_abs', 0.0), b.get('sem_max_abs', 0.0),
             b['max_idx']['mismatch'], b['max_idx']['tie_rays'], ind['rays_with_cell_flip'], ind['rays_over_tol'],
             ind['abs_rel'], ind['abs_rel_no_flip_rays'], ind['acc_median']))
    if not rep['ok']:
        print(tag, json.dumps(rep))
    assert rep['ok'], tag

    # which paths the case exercised
    interior = _warp_paths(got['grid'], desc)
    early, never = _exit_warps(refs['same_cells']['weights'], interior)
    counts = dict(interior_warps=int(interior.sum()), padded_warps=int((~interior).sum()),
                  exit_warps=int(early.sum()) if packed else 0)
    assert counts['interior_warps'] > 0 and counts['padded_warps'] > 0, (tag, counts)
    if packed and scene == 'analytic' and inv_s == _f32(INV_S[-1]):
        assert counts['exit_warps'] > 0, (tag, counts)
    if n_feat:
        rgb, acc = got['rgb'], got['acc']
        counts['saturated_channels'] = int((rgb == 1.0).sum())      # asserted over the head's cases by the caller
        if bk is not None:
            counts['rays_acc_below_half'] = int((acc < 0.5).sum())
            assert counts['rays_acc_below_half'] > 0, (tag, 'the random background changes no ray')

    # (a) production launch vs probe launch
    if packed:
        same = _ray_mask(never, n)
        diffs = {}
        for k in want:
            a, p = prod[k], probe[k]
            assert torch.equal(a[same], p[same]), (tag, k, 'production and probe launches differ on warps without an exit')
            if k in ('max_idx', 'max_depth'):
                assert torch.equal(a, p), (tag, k)
            else:
                assert _tail_close(a, p).all(), (tag, k, float((a.double() - p.double()).abs().max()))
            diffs[k] = float((a.double() - p.double()).abs().max())
        counts['bit_equal_rays'] = int(same.sum())
        print('%s: production vs probe max |diff| %s' % (tag, ' '.join('%s %.1e' % kv for kv in diffs.items())))

    # the background row of a launch-local ray: a slice launch with its own rows equals the whole launch's rows (the slice
    # starts and ends on a warp boundary, so every warp holds the same rays, votes alike and takes the same path)
    if bk is not None:
        b0, c = WARP * (n // (3 * WARP)), WARP * (n // (2 * WARP))
        part = launch(vf, desc, ['rgb'], pack=pack if packed else None, begin=b0, count=c, bk_=bk[b0:b0 + c].contiguous())
        assert torch.equal(part['rgb'], prod['rgb'][b0:b0 + c]), tag
    print('%s: %s' % (tag, counts))
    return rep, counts


@pytest.mark.parametrize('scene', ['analytic', 'decoded'])
@pytest.mark.parametrize('name', list(HEADS))
def test_inference_render_at_shipped_geometry(name, scene):
    """(a) - (c) for one head and scene at the three sharpnesses, random background (and white on one colour head)."""
    _dev()
    head, i2l, pix = _setup(name)
    vol = _volume(head, scene)
    cases = [(inv_s, 'random') for inv_s in INV_S] + ([(INV_S[1], 'white')] if name == WHITE_HEAD else [])
    saturated = 0
    for i, (inv_s, bkgd) in enumerate(cases):
        _, counts = _render_case(name, head, scene, vol, i2l, pix, _f32(inv_s), bkgd, seed=i)
        saturated += counts.get('saturated_channels', 0)
    # the eval clamp engaged (a colour channel above 1 was clamped) in some case; on the free-space decoded scene at a sharp
    # inv_s the accumulation is ~0.003 and colour is the background's
    assert saturated > 0 or not head['color_dims'], (name, scene, 'the eval clamp never engaged')


@pytest.mark.parametrize('name', list(HEADS))
def test_neus_head_render_at_shipped_geometry(name, monkeypatch):
    """(d) NeuSHead built from the head's config, prepared on decoded planes, rendering its eval ray grid: equal bit for bit
    to the direct launch it stands for (background redrawn from the same seed; the second render reuses the cached pack),
    and within the oracle gate."""
    dev = _dev()
    from oracle import rays as orays
    from oracle.mapping import GridMeterMappingRef
    from oracle.parity import render_parity
    from selfocc_b200 import ops
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    monkeypatch.setenv('eval', 'true')                    # the fixed eval ray grid
    cfg, i2l, pix = _setup(name, full=True)
    head = build_head(cfg).to(dev).eval()
    f = head.model.field
    m = f.mapping
    n_feat = cfg['color_dims']
    planes, mlp = _decoder(m, n_feat, seed=1)
    with torch.no_grad():
        for lin, w, bias in ((f.density_net[1], mlp[0], mlp[1]), (f.density_net[3], mlp[2], mlp[3])):
            lin.weight.copy_(w)
            lin.bias.copy_(bias)
        f.deviation_network.variance.fill_(0.3)          # inv_s = e^3
    head.prepare([p[None] for p in planes])
    metas = [dict(temImg2lidar=list(i2l.double().numpy()))]
    torch.manual_seed(7)
    out = head.render(metas=metas)
    torch.manual_seed(7)
    again = head.render(metas=metas)
    n_cam, n_pix = i2l.shape[0], pix.shape[0]
    n = n_cam * n_pix
    has_rgb = n_feat >= 3
    torch.manual_seed(7)
    bk = torch.rand(n, 3, device=dev) if (cfg['render_bkgd'] == 'random' and has_rgb) else None
    ny, nx = cfg['ray_number']
    img_h, img_w = cfg['ray_img_size']
    rays = ops.make_ray_desc(n_cam, grid=(ny, nx, 1.0 * img_w / nx, 0.0, 1.0 * img_h / ny, 0.0))
    params = head._params(False)
    want = ['depth', 'acc', 'normal_vis', 'max_depth', 'max_idx'] + (['rgb'] if has_rgb else []) + (['sem'] if head.return_sem else [])
    cams = i2l.to(dev)
    direct = ops.render_infer(f.vol_sdf, f.vol_feat, f.desc, cams, rays, params, bkgd_rand=bk, want=want,
                              pack=ops.render_pack(f.vol_sdf, f.vol_feat, f.desc))
    got = dict(depth=out['ms_depths'][0].reshape(n), acc=out['ms_accs'][0].reshape(n), normal_vis=out['vis_normal'][0].reshape(n, 3))
    if has_rgb:
        got['rgb'] = out['ms_colors'][0].reshape(n, 3)
    if head.return_sem:
        got['sem'] = out['sem'][0].reshape(n, -1)
        assert got['sem'].shape[1] == n_feat - 3
    for k, v in got.items():
        assert torch.equal(v, direct[k]), (name, k, 'NeuSHead.render differs from the direct launch')
    for a, b in ((again['ms_depths'], out['ms_depths']), (again['ms_accs'], out['ms_accs']), (again['ms_colors'], out['ms_colors'])):
        assert torch.equal(a[0], b[0]), (name, 'the second render (cached pack) differs')
    # the oracle gate on the module's outputs; max_idx / max_depth from the direct launch, coordinates from the probe
    packed = f.render_pack() is not None
    desc_p = f.desc if packed else m.volume_desc(0)
    vf_p = f.vol_feat if packed else None
    probe = ops.render_infer(f.vol_sdf, vf_p, desc_p, cams, rays, params, bkgd_rand=bk if packed else None,
                             want=('depth',), pack=ops.render_pack(f.vol_sdf, vf_p, desc_p), probe_grid=True)
    got.update(max_idx=direct['max_idx'], max_depth=direct['max_depth'], grid=probe['grid'])
    vol64 = _oracle_volume(planes, [t.detach() for t in (f.density_net[1].weight, f.density_net[1].bias,
                                                         f.density_net[3].weight, f.density_net[3].bias)], m)
    origin, direction = orays.img2lidar_rays(i2l[None], pix)
    kw = dict(bkgd='random', bkgd_rand=bk) if bk is not None else {}
    rep = render_parity(got, vol64, GridMeterMappingRef(**cfg['mapping_args']), origin, direction, cfg['roi_aabb'], params.inv_s, S,
                        color_dims=n_feat, max_flip_frac=0.04 if name.startswith('KITTI') else 0.02, abs_rel_flip_rays=False, **kw)
    print('NeuSHead.render %s (%d rays, inv_s %.2f): %s' % (name, n, params.inv_s, rep))
    assert rep['ok'], rep
