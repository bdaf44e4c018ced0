"""GPU parity of the training-form render (forward AND backward) against the differentiable fp64 oracle at the shipped
configs' geometry, with the three-part rule of oracle/train_parity.py; the sample probe against the forward; the field-query
backward, alone and through NeuSHead's uniform sdf; ray-sharded launches against the unsharded one; and a small matrix of
edge cases (H != W, ring mapping, ray-count tails, rays that miss the AABB, the generic semantic path)."""
import json
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

from selfocc_b200 import synth
from selfocc_b200.mapping import GridMeterMapping

ROOT = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(ROOT, 'golden', 'reference_model_cfgs.json')))
S_SHIPPED = 256
# inv_s = exp(10 variance): beta_init 0.1 (the start of training), e^3, and a sharp surface (e^6.5 ~ 665, an assumed value)
INV_S = (math.e, math.e ** 3, math.e ** 6.5)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


# name -> (config, decoded feature channels besides sdf, ray stride into the config's fixed ray grid)
SHIPPED = {
    'nuScenes_occ': ('nuscenes/nuscenes_occ.py', 24, 15),            # semantic path <true, 24>
    'nuScenes_novel_depth': ('nuscenes/nuscenes_novel_depth.py', 3, 15),   # fwd5, const pitch <32, 257 * 32>
    'nuScenes_depth': ('nuscenes/nuscenes_depth.py', 0, 15),         # fwd5, const pitch, depth only
    'KITTI_occ': ('kitti/kitti_occ.py', 3, 5),                       # h_half, zpitch 40: generic-pitch fwd5
    'KITTI_raw_depth': ('kitti_raw/kitti_raw_depth.py', 0, 3),
}


def _shipped_setup(name):
    from oracle import rays as orays
    cfg_name, n_feat, stride = SHIPPED[name]
    head = CFGS[cfg_name]['head']
    margs, aabb = head['mapping_args'], head['roi_aabb']
    img_h, img_w = head['ray_img_size']
    if cfg_name.startswith('nuscenes'):
        _, i2l = synth.camera_rig(f=1266.0 * img_w / 1600, cx=img_w / 2, cy=img_h / 2)
    else:
        _, i2l = synth.camera_rig((0.,), f=721.5, cx=img_w / 2, cy=img_h / 2, height=1.65, radius=0.0)
    pix = orays.fixed_ray_grid(head['ray_number'], head['ray_img_size'])[::stride].contiguous()
    return margs, aabb, n_feat, torch.tensor(i2l, dtype=torch.float32), pix


def _volume(m, n_feat, scene, seed=0):
    """[H,W,Z] sdf and [n_feat,H,W,Z] features: the analytic scene (rays terminate on ground / spheres / a box) or random
    TPV planes through the wgmma decode."""
    dev = _dev()
    g = torch.Generator().manual_seed(seed)
    if scene == 'analytic':
        sdf = synth.analytic_sdf_volume(m, noise=0.02, seed=seed)
        feat = 0.7 * torch.randn(n_feat, *sdf.shape, generator=g) if n_feat else None
        return sdf, feat
    from selfocc_b200 import ops
    planes = [p.to(dev) for p in synth.random_planes(m, 96, scale=1.0, seed=seed)]
    mlp = [p.to(dev) for p in synth.random_mlp(96, 1 + n_feat, seed=seed)]
    desc = m.volume_desc(n_feat)
    vs, vf = ops.tpv_decode(*planes, *mlp, desc)
    sdf = vs[..., :m.size_d].cpu()
    feat = vf[..., :n_feat].permute(3, 0, 1, 2).cpu() if n_feat else None
    return sdf.contiguous(), feat


def _run_case(m, mref, aabb, sdf, feat, i2l, pix, inv_s, S, seed=0, jitter=True, ray_begin=0, ray_count=None, tag='',
              max_flip_frac=0.02):
    """Kernel forward + probes + backward with flip-masked cotangents, then the fp64 oracle report."""
    dev = _dev()
    from oracle import rays as orays, train_parity as tp
    from selfocc_b200 import ops
    g = torch.Generator().manual_seed(seed + 7)
    n_feat = 0 if feat is None else feat.shape[0]
    n_cam, n_pix = i2l.shape[0], pix.shape[0]
    total = n_cam * n_pix
    n = total - ray_begin if ray_count is None else ray_count
    inv_s = _f32(inv_s)
    jit = torch.rand(total, S + 1, generator=g) if jitter else None
    bk = torch.rand(n, 3, generator=g) if n_feat else None          # per launched ray (jitter rows are per global ray)
    desc = m.volume_desc(n_feat)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev).requires_grad_(True)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev).requires_grad_(True) if n_feat else None
    invs = torch.tensor([inv_s], device=dev, requires_grad=True)
    want = ['depth', 'acc', 'fars', 'max_depth', 'weights', 'ts', 'deltas', 'eik_grad', 'sample_sdf']
    want += (['rgb'] if n_feat >= 3 else []) + (['sem'] if n_feat > 3 else [])
    rays = ops.make_ray_desc(n_cam, n_pix=n_pix, ray_begin=ray_begin, ray_count=n)
    params = ops.make_render_params(aabb, S, inv_s, training=True, bkgd='random')
    cfg = dict(desc=desc, cam_mats=i2l.to(dev), rays=rays, params=params, pix=pix.to(dev), want=want,
               jitter=jit.to(dev) if jit is not None else None, bkgd_rand=bk.to(dev) if bk is not None else None)
    res = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vs, vf, invs, cfg)))
    gf = ops.render_train_probe(desc, cfg['cam_mats'], rays, params, pix=cfg['pix'], jitter=cfg['jitter'])
    # fp64 rays and sample geometry
    origin, direction = orays.img2lidar_rays(i2l[None], pix)
    o, d, nrm = (t.to(dev) for t in orays.flatten_rays(origin.double(), direction.double()))
    sl = slice(ray_begin, ray_begin + n)
    o, d, nrm = o[sl], d[sl], nrm[sl]
    j64 = jit[sl].double().to(dev) if jit is not None else None
    bk64 = bk.double().to(dev) if bk is not None else None
    g64, _ = tp.sample_geometry(mref, o, d, aabb, S, j64)
    _check_probe_against_forward(m, gf, res, o, d, nrm)
    flip = tp.flip_rays(gf, g64)
    cot = {k: torch.randn(res[k].shape, generator=g).to(dev) for k in tp.DIFF if k in want}
    for t in cot.values():
        t[flip] = 0
    sum((res[k] * c).sum() for k, c in cot.items()).backward()
    gvol = vs.grad[..., :m.size_d][None]
    if n_feat:
        gvol = torch.cat([gvol, vf.grad[..., :n_feat].permute(3, 0, 1, 2)], 0)
    vol64 = (sdf[None] if feat is None else torch.cat([sdf[None], feat], 0)).double().to(dev)
    got = {k: res[k].detach() for k in want}
    rep = tp.train_parity(got, {'vol': gvol, 'inv_s': invs.grad.item()}, {k: c.double() for k, c in cot.items()}, vol64, mref,
                          o, d, nrm, aabb, inv_s, S, gf, jitter=j64, color_dims=3 if n_feat else 0, bkgd_rand=bk64,
                          max_flip_frac=max_flip_frac)
    print(tp.format_report(tag, rep))
    return rep, res, gf, cfg, (vs, vf, invs)


def _check_probe_against_forward(m, grid, res, o, d, nrm):
    """Ties the probe to what the forward computed: on an affine map each grid coordinate is k0 (o + t d - start) + offset
    along its axis, so the probe's coordinates, mapped back through the axis with the largest |k0 d|, give the ray length
    of the sample; it must equal the forward's ts * |dir| within the rounding of the fp32 coordinate and of ts."""
    if any(m._ax[k]['size'][1] > 0 for k in 'hwd'):
        return
    ax = [m._ax[k] for k in 'hwd']
    k0 = torch.tensor([a['size'][0] / a['rng'][0] for a in ax], dtype=torch.float64, device=o.device)
    start = torch.tensor([a['start'] for a in ax], dtype=torch.float64, device=o.device)
    off = torch.tensor([a['offset'] for a in ax], dtype=torch.float64, device=o.device)
    oo, dd = o[:, [1, 0, 2]], d[:, [1, 0, 2]]                    # (h, w, d) axes take metre (y, x, z)
    slope = k0 * dd                                                # d grid / d t per axis, [n, 3]
    a = slope.abs().argmax(-1)
    n, S = grid.shape[:2]
    g = grid.double().gather(2, a[:, None, None].expand(n, S, 1))[..., 0]
    pick = lambda t: t.gather(1, a[:, None])
    t_probe = ((g - pick(off[None].expand(n, 3))) / pick(k0[None].expand(n, 3)) + pick(start[None].expand(n, 3)) - pick(oo)) / pick(dd)
    t_fwd = res['ts'].detach().double().reshape(n, S) * nrm
    eps = float(torch.finfo(torch.float32).eps)
    bound = 4 * eps * (g.abs() + 1) / pick(slope).abs() + 4 * eps * t_fwd.abs() + 1e-6 * t_fwd.abs()
    miss = (t_probe - t_fwd).abs() > bound
    assert not miss.any(), 'probe coordinates do not reproduce the forward ts on %d samples' % int(miss.sum())


@pytest.mark.parametrize('scene', ['analytic', 'planes'])
@pytest.mark.parametrize('name', list(SHIPPED))
def test_train_parity_at_shipped_geometry(name, scene):
    """Every shipped training config's volume, channel count and kernel path at S = 256 with jitter and random background,
    on a strided subset of its ray grid, at three sharpnesses: the fp64 oracle gate, and the forward / backward probes."""
    dev = _dev()
    from oracle.mapping import GridMeterMappingRef
    from selfocc_b200 import ops, _lib
    margs, aabb, n_feat, i2l, pix = _shipped_setup(name)
    m, mref = GridMeterMapping(**margs), GridMeterMappingRef(**margs)
    sdf, feat = _volume(m, n_feat, scene)
    # flip rays per ray grow with the faces a ray crosses: the 2 % bound of the inference gate is set on nuScenes' 2.5 cells
    # per metre; KITTI's grid has 5 cells per metre along h and w
    flip_frac = 0.04 if name.startswith('KITTI') else 0.02
    reps = []
    for i, inv_s in enumerate(INV_S):
        rep, res, gf, cfg, (vs, vf, invs) = _run_case(m, mref, aabb, sdf, feat, i2l, pix, inv_s, S_SHIPPED, seed=i,
                                                      tag='%s/%s' % (name, scene), max_flip_frac=flip_frac)
        reps.append(rep)
        if n_feat <= 3:
            # the batched forward and the one-ray-per-warp forward share the sample arithmetic: bit-identical geometry
            lib = _lib.load()
            try:
                lib.so_render_train_force_fwd32(1)
                one = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vs.detach(), None if vf is None else vf.detach(),
                                                                                             invs.detach(), cfg)))
            finally:
                lib.so_render_train_force_fwd32(0)
            for k in ('ts', 'deltas', 'fars'):
                assert torch.equal(one[k], res[k].detach()), k
    print('peak memory %.2f GB' % (torch.cuda.max_memory_allocated() / 2 ** 30))
    assert all(r['ok'] for r in reps)


# ---- small edge matrix --------------------------------------------------------------------------------------------------
def _small(kind):
    """(mapping args, aabb): H != W, or a ring mapping (size1 > 0: the non-affine metre->grid map, one-ray-per-warp path)."""
    if kind == 'ring':
        return dict(nonlinear_mode='linear', h_size=[6, 3], h_range=[8.0, 4.8], h_half=False, w_size=[6, 3], w_range=[8.0, 4.8],
                    w_half=False, d_size=[6, 0], d_range=[-2.0, 3.0, 3.0]), [-12.8, -12.8, -2.0, 12.8, 12.8, 3.0]
    return dict(nonlinear_mode='linear', h_size=[12, 0], h_range=[12.8, 0], h_half=False, w_size=[7, 0], w_range=[8.0, 0],
                w_half=False, d_size=[6, 0], d_range=[-2.0, 3.0, 3.0]), [-8.0, -12.8, -2.0, 8.0, 12.8, 3.0]


def _small_rig(n_cam=2, miss=False):
    _, i2l = synth.camera_rig(synth.NUSC_YAWS[:n_cam], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    i2l = torch.tensor(i2l, dtype=torch.float32)
    if miss:        # a camera 10 m above the box looking at the horizon: most of its rays never enter the AABB
        _, up = synth.camera_rig((90.,), f=126.6, cx=80., cy=45., height=10.0, radius=0.2)
        i2l = torch.cat([i2l, torch.tensor(up, dtype=torch.float32)], 0)
    return i2l


@pytest.mark.parametrize('case', ['h_ne_w', 'ring', 'rays1', 'rays3', 'rays5', 'rays33', 'miss_aabb'])
def test_train_parity_edge_cases(case):
    _dev()
    from oracle import rays as orays
    from oracle.mapping import GridMeterMappingRef
    margs, aabb = _small('ring' if case == 'ring' else 'h_ne_w')
    m, mref = GridMeterMapping(**margs), GridMeterMappingRef(**margs)
    assert (m.size_h != m.size_w) or case == 'ring'
    sdf = synth.analytic_sdf_volume(m, ground_z=-1.0, spheres=((3., 5., 0., 1.5),), boxes=(), noise=0.05, seed=1)
    feat = torch.randn(3, *sdf.shape, generator=torch.Generator().manual_seed(4))
    i2l = _small_rig(miss=case == 'miss_aabb')
    pix = orays.fixed_ray_grid([5, 7], [90, 160])
    kw = {}
    S = 64
    if case.startswith('rays'):     # the batched forward (S a multiple of 32 U) with batch and warp tails
        S, kw = 128, dict(ray_begin=3, ray_count=int(case[4:]))
    if case == 'miss_aabb':         # the missing camera's zero-length samples sit on the AABB face: its rays may flip cells
        kw = dict(max_flip_frac=1.0 / 3.0)
    for inv_s in (12.0, INV_S[2]):
        rep, _, _, _, _ = _run_case(m, mref, aabb, sdf, feat, i2l, pix, inv_s, S, tag=case, **kw)
        assert rep['ok']


def test_train_generic_semantic_path_matches_the_24_channel_path():
    """so_render_train_force_sem_generic(1) on a 24-channel volume (the generic runtime-channel-count path) against the
    vectorised default, forward and backward, and both against the fp64 oracle."""
    _dev()
    from oracle import rays as orays
    from oracle.mapping import GridMeterMappingRef
    from selfocc_b200 import _lib
    margs, aabb = _small('h_ne_w')
    m, mref = GridMeterMapping(**margs), GridMeterMappingRef(**margs)
    sdf = synth.analytic_sdf_volume(m, ground_z=-1.0, spheres=((3., 5., 0., 1.5),), boxes=(), noise=0.05, seed=1)
    feat = torch.randn(24, *sdf.shape, generator=torch.Generator().manual_seed(4))
    i2l, pix = _small_rig(), orays.fixed_ray_grid([5, 7], [90, 160])
    lib = _lib.load()
    out = {}
    for generic in (0, 1):
        try:
            lib.so_render_train_force_sem_generic(generic)
            rep, res, _, _, (vs, vf, invs) = _run_case(m, mref, aabb, sdf, feat, i2l, pix, 20.0, 64, tag='sem generic=%d' % generic)
        finally:
            lib.so_render_train_force_sem_generic(0)
        assert rep['ok']
        out[generic] = ({k: v.detach() for k, v in res.items()}, vs.grad.clone(), vf.grad.clone(), invs.grad.clone())
    a, b = out[0], out[1]
    for k in ('weights', 'ts', 'deltas', 'eik_grad', 'sample_sdf', 'depth', 'acc', 'fars', 'max_depth'):
        assert torch.equal(a[0][k], b[0][k]), k
    assert torch.allclose(a[0]['rgb'], b[0]['rgb'], atol=1e-6) and torch.allclose(a[0]['sem'], b[0]['sem'], atol=1e-6)
    assert torch.allclose(a[1], b[1], atol=1e-5 * max(1.0, a[1].abs().max().item()))
    assert torch.allclose(a[2], b[2], atol=1e-5 * max(1.0, a[2].abs().max().item()))
    assert torch.allclose(a[3], b[3], rtol=1e-4)


# ---- field-query backward -----------------------------------------------------------------------------------------------
def _field_points(m, mref, n, g):
    """inside, outside (zero padding), exactly on the volume's boundary faces, and within 1e-6 grid units of interior faces."""
    H, W, Z = m.size_h, m.size_w, m.size_d
    def to_m(gr):
        return mref.grid2meter(gr.double()).float()
    gin = torch.rand(n, 3, generator=g) * torch.tensor([H - 1., W - 1., Z - 1.])
    gout = torch.rand(n // 4, 3, generator=g) * torch.tensor([H + 3., W + 3., Z + 3.]) - 2.0
    gbd = torch.rand(n // 4, 3, generator=g) * torch.tensor([H - 1., W - 1., Z - 1.])
    ax = torch.randint(0, 3, (n // 4,), generator=g)
    gbd[torch.arange(n // 4), ax] = torch.where(torch.rand(n // 4, generator=g) < 0.5, 0.0, torch.tensor([H - 1., W - 1., Z - 1.])[ax])
    gnf = torch.rand(n // 4, 3, generator=g) * torch.tensor([H - 1., W - 1., Z - 1.])
    ax = torch.randint(0, 3, (n // 4,), generator=g)
    gnf[torch.arange(n // 4), ax] = gnf[torch.arange(n // 4), ax].round() + 1e-6 * (torch.rand(n // 4, generator=g) - 0.5)
    return torch.cat([to_m(gin), to_m(gout), to_m(gbd), to_m(gnf)]).contiguous()


@pytest.mark.parametrize('cots', [('sdf',), ('grad',), ('feat',), ('sdf', 'grad', 'feat')])
@pytest.mark.parametrize('geom', ['kitti_h_half', 'h_ne_w', 'ring'])
def test_field_query_backward_matches_fp64_autograd(geom, cots):
    """FieldQueryFunction (so_field_query_backward) w.r.t. vol_sdf and vol_feat vs fp64 autograd of field_query_manual.  The
    analytic position gradient jumps across cell faces, so its cotangent is zeroed (on both sides) for points whose fp64
    grid coordinate lies within 1e-4 of a face (boundary faces included); the value and feature cotangents are continuous there and stay."""
    dev = _dev()
    from oracle import render as orender
    from oracle.mapping import GridMeterMappingRef
    from selfocc_b200 import ops
    margs = CFGS['kitti/kitti_occ.py']['head']['mapping_args'] if geom == 'kitti_h_half' else _small(geom.replace('h_ne_w', 'x'))[0]
    m, mref = GridMeterMapping(**margs), GridMeterMappingRef(**margs)
    g = torch.Generator().manual_seed(11)
    n_feat = 4
    sdf = torch.randn(m.size_h, m.size_w, m.size_d, generator=g)
    feat = torch.randn(n_feat, *sdf.shape, generator=g)
    x = _field_points(m, mref, 4000, g)
    n = x.shape[0]
    gr64 = mref.meter2grid(x.double(), False)
    near = ((gr64 - gr64.round()).abs() < 1e-4).any(-1)     # incl. boundary points that fp32 rounding put just outside
    assert near.sum() > n // 8
    c = {'sdf': torch.randn(n, generator=g), 'grad': torch.randn(n, 3, generator=g), 'feat': torch.randn(n, n_feat, generator=g)}
    c['grad'][near] = 0
    c = {k: (v if k in cots else torch.zeros_like(v)) for k, v in c.items()}
    vol64 = torch.cat([sdf[None], feat], 0).double().requires_grad_(True)
    h, grad = orender.field_query_manual(vol64, mref, x.double())
    ((h[:, 0] * c['sdf'].double()).sum() + (grad * c['grad'].double()).sum() + (h[:, 1:] * c['feat'].double()).sum()).backward()
    desc = m.volume_desc(n_feat)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev).requires_grad_(True)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev).requires_grad_(True)
    s, gk, fk = ops.FieldQueryFunction.apply(vs, vf, desc, x.to(dev), True, True)
    ((s * c['sdf'].to(dev)).sum() + (gk * c['grad'].to(dev)).sum() + (fk * c['feat'].to(dev)).sum()).backward()
    gs_ref, gf_ref = vol64.grad[0], vol64.grad[1:]
    gs, gf = vs.grad[..., :m.size_d].cpu().double(), vf.grad[..., :n_feat].permute(3, 0, 1, 2).cpu().double()
    es = (gs - gs_ref).abs().max().item() / max(1.0, gs_ref.abs().max().item())
    ef = (gf - gf_ref).abs().max().item() / max(1.0, gf_ref.abs().max().item())
    print('field query backward %s %s: d/d vol_sdf %.2e, d/d vol_feat %.2e (rel to max)' % (geom, '+'.join(cots), es, ef))
    assert es < 2e-5 and ef < 2e-5
    if 'sdf' in cots or 'grad' in cots:
        assert gs_ref.abs().max() > 0
    if 'feat' in cots:
        assert gf_ref.abs().max() > 0
    else:
        assert gf.abs().max() == 0


# ---- ray sharding --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['nuScenes_occ', 'nuScenes_novel_depth'])
def test_ray_sharded_launches_equal_the_unsharded_launch(name):
    """head.ray_shard: rank r renders the r-th contiguous slice (dist.ray_slice) of every camera's pixel rays as a pixel-table
    launch with the matching jitter and background rows.  Per-ray and per-sample forward outputs equal the same rays of the
    unsharded launch bit for bit; the summed shard gradients equal the unsharded gradient within fp32 atomics."""
    dev = _dev()
    from selfocc_b200 import ops
    from selfocc_b200.dist import ray_slice
    margs, aabb, n_feat, i2l, pix = _shipped_setup(name)
    m = GridMeterMapping(**margs)
    sdf, feat = _volume(m, n_feat, 'analytic')
    g = torch.Generator().manual_seed(3)
    n_cam, n_pix, S = i2l.shape[0], pix.shape[0], S_SHIPPED
    desc = m.volume_desc(n_feat)
    vs0 = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    vf0 = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev) if n_feat else None
    jit = torch.rand(n_cam, n_pix, S + 1, generator=g).to(dev)
    bk = torch.rand(n_cam, n_pix, 3, generator=g).to(dev)
    want = ['depth', 'acc', 'fars', 'max_depth', 'weights', 'ts', 'deltas', 'eik_grad', 'sample_sdf', 'rgb'] + (['sem'] if n_feat > 3 else [])
    params = ops.make_render_params(aabb, S, _f32(math.e ** 3), training=True, bkgd='random')
    cot = {k: None for k in ('depth', 'acc', 'weights', 'eik_grad', 'sample_sdf', 'rgb', 'sem') if k in want}

    def launch(b, c):
        vs, vf = vs0.clone().requires_grad_(True), vf0.clone().requires_grad_(True)
        invs = torch.tensor([params.inv_s], device=dev, requires_grad=True)
        cfg = dict(desc=desc, cam_mats=i2l.to(dev), rays=ops.make_ray_desc(n_cam, n_pix=c), params=params,
                   pix=pix[b:b + c].contiguous().to(dev), jitter=jit[:, b:b + c].reshape(-1, S + 1).contiguous(),
                   bkgd_rand=bk[:, b:b + c].reshape(-1, 3).contiguous(), want=want)
        res = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vs, vf, invs, cfg)))
        res = {k: res[k].reshape(n_cam, c, *res[k].shape[1:]) for k in want}
        for k in cot:
            if cot[k] is None:
                cot[k] = torch.randn(res[k].shape, generator=torch.Generator().manual_seed(len(k))).to(dev)
        sum((res[k] * cot[k][:, b:b + c]).sum() for k in cot).backward()
        return {k: v.detach() for k, v in res.items()}, vs.grad, vf.grad, invs.grad

    full, gs_full, gf_full, gi_full = launch(0, n_pix)
    for world in (2, 3):
        gs, gf, gi = torch.zeros_like(gs_full), torch.zeros_like(gf_full), torch.zeros_like(gi_full)
        for r in range(world):
            b, c = ray_slice(n_pix, world, r)
            part, a, f, i = launch(b, c)
            for k in want:
                assert torch.equal(part[k], full[k][:, b:b + c]), (world, r, k)
            gs, gf, gi = gs + a, gf + f, gi + i
        for a, b in ((gs, gs_full), (gf, gf_full)):
            err = (a - b).abs().max().item() / max(1.0, b.abs().max().item())
            print('%s ray shards %d: summed gradient rel-to-max err %.2e' % (name, world, err))
            assert err < 1e-5
        assert abs(gi.item() - gi_full.item()) <= 1e-4 * max(1.0, abs(gi_full.item()))


# ---- NeuSHead uniform sdf (kitti_occ trains with return_uniform_sdf=True) ----------------------------------------------
def test_head_uniform_sdf_gradient_reaches_the_planes_like_the_oracle():
    """NeuSHead.forward(return_uniform_sdf=True) with an explicit lattice jitter: uniform_sdf and its gradient w.r.t. the
    three TPV planes and the decode MLP against fp64 autograd of the oracle decode (tpv_decode_ref) plus field query
    (field_query_manual) at the same points, on the KITTI half-axis mapping at a reduced size."""
    dev = _dev()
    from selfocc_b200 import configs
    from selfocc_b200.head_train import uniform_lattice_train
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    from oracle import render as orender
    from oracle.mapping import GridMeterMappingRef
    torch.manual_seed(0)
    margs = dict(nonlinear_mode='linear', h_size=[16, 0], h_range=[12.8, 0], h_half=True, w_size=[8, 0], w_range=[6.4, 0],
                 w_half=False, d_size=[8, 0], d_range=[-2.0, 4.4, 4.4])
    rng = [-6.4, 0.0, -2.0, 6.4, 12.8, 4.4]
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=1, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=32, ray_number=(4, 6), ray_img_size=(90, 160), color_dims=3,
                                  render_bkgd='random')
    cfg['head'].update(return_uniform_sdf=True, resolution=0.4)
    head = build_head(cfg['head']).to(dev).train()
    l2i, i2l = synth.camera_rig((0.,), f=126.6, cx=80., cy=45., height=1.65, radius=0.0)
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(90, 160))]
    m = GridMeterMapping(**margs)
    H, W, Z = m.size_h, m.size_w, m.size_d
    planes = [(0.5 * torch.randn(1, k, 96, device=dev)).requires_grad_(True) for k in (H * W, Z * H, W * Z)]
    lat = uniform_lattice_train(head, dev)
    g = torch.Generator().manual_seed(6)
    shift = torch.rand(lat.numel() // 3, 3, generator=g).to(dev)
    out = head(representation=planes, metas=metas, jitter=torch.rand(24, 33, device=dev), bkgd_rand=torch.rand(24, 3, device=dev),
               uniform_shift=shift)
    us = out['uniform_sdf']
    assert us.shape == lat.shape[:3]
    c = torch.randn(us.shape, generator=g).to(dev)
    f = head.model.field
    params = [planes[0], planes[1], planes[2], f.density_net[1].weight, f.density_net[1].bias, f.density_net[3].weight,
              f.density_net[3].bias]
    got = torch.autograd.grad((us * c).sum(), params)
    # oracle: fp64 decode of the same planes and MLP, queried at the same fp32 points
    ins = [p.detach().cpu().double().requires_grad_(True) for p in params]
    vol = orender.tpv_decode_ref(ins[0][0], ins[1][0], ins[2][0], (H, W, Z), *ins[3:])
    xyz = (lat.flatten(0, 2) + shift * head.resolution).cpu()
    h, _ = orender.field_query_manual(vol, GridMeterMappingRef(**margs), xyz.double())
    sdf64 = h[:, 0].reshape(us.shape)
    err_v = (us.detach().cpu().double() - sdf64.detach()).abs().max().item()
    ref = torch.autograd.grad((sdf64 * c.cpu().double()).sum(), ins)
    print('uniform sdf: value max abs err %.2e' % err_v)
    assert err_v < 1e-4 * max(1.0, sdf64.abs().max().item())
    for name, a, b in zip(('tpv_hw', 'tpv_zh', 'tpv_wz', 'w1', 'b1', 'w2', 'b2'), got, ref):
        err = (a.cpu().double().reshape(b.shape) - b).abs().max().item() / (b.abs().max().item() + 1e-12)
        print('uniform sdf: d/d %s rel-to-max err %.2e' % (name, err))
        assert err < 2e-4, (name, err)
