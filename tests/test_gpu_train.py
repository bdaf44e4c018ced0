"""GPU parity of the training-form render (forward outputs + backward) and of NeuSHead.forward vs the oracle."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from selfocc_b200 import synth, configs
from selfocc_b200.mapping import GridMeterMapping


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _oracle_train(vol, mref, i2l, pix, aabb, inv_s, S, jitter, training, color_dims, bkgd_rand):
    from oracle import rays as orays, render as orender
    origin, direction = orays.img2lidar_rays(i2l[None], pix)
    o, d, nrm = orays.flatten_rays(origin.double(), direction.double())
    out = orender.neus_render_chunk(vol, mref, o, d, nrm, aabb, inv_s, S=S, near_plane=0.0, training=training, jitter=jitter,
                                    color_dims=color_dims, bkgd='random' if bkgd_rand is not None else 'white',
                                    bkgd_rand=bkgd_rand, differentiable=True)
    out['ts'] = (out['starts'] + out['ends']) / 2 / nrm
    out['deltas'] = (out['ends'] - out['starts']) / nrm
    return out


@pytest.mark.parametrize('n_feat,S,use_jitter', [(0, 64, False), (0, 48, True), (7, 40, True),
                                                 (0, 128, True), (0, 256, False), (3, 128, True),
                                                 (24, 64, True), (24, 40, False)])   # 24: the vectorised rgb + 21-class path (nuscenes_occ.py:350)
def test_render_train_forward_backward(n_feat, S, use_jitter):
    dev = _dev()
    from oracle.mapping import GridMeterMappingRef
    from oracle import rays as orays
    from selfocc_b200 import ops
    g = torch.Generator().manual_seed(3)
    margs, aabb = synth.small_mapping(10, 6)
    m, mref = GridMeterMapping(**margs), GridMeterMappingRef(**margs)
    sdf = synth.analytic_sdf_volume(m, ground_z=-1.0, spheres=((3., 5., 0., 1.5),), boxes=(), noise=0.05, seed=1)
    feat = torch.randn(n_feat, *sdf.shape, generator=g) if n_feat else None
    _, i2l = synth.camera_rig(synth.NUSC_YAWS[:2], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    i2l = torch.tensor(i2l, dtype=torch.float32)
    ny, nx = 5, 7
    pix = orays.fixed_ray_grid([ny, nx], [90, 160])
    n = 2 * ny * nx
    jitter = torch.rand(n, S + 1, generator=g) if use_jitter else None
    bk = torch.rand(n, 3, generator=g) if n_feat else None
    inv_s0 = 12.0
    # ---- oracle (fp64, differentiable through the manual field query)
    vol64 = (sdf[None] if feat is None else torch.cat([sdf[None], feat], 0)).double().requires_grad_(True)
    invs64 = torch.tensor(inv_s0, dtype=torch.float64, requires_grad=True)
    ref = _oracle_train(vol64, mref, i2l, pix, aabb, invs64, S, jitter.double() if use_jitter else None, True,
                        3 if n_feat else 0, bk.double() if bk is not None else None)
    # ---- kernel
    desc = m.volume_desc(n_feat)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev).requires_grad_(True)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev).requires_grad_(True) if n_feat else None
    invs = torch.tensor([inv_s0], device=dev, requires_grad=True)
    want = ['depth', 'acc', 'fars', 'max_depth', 'weights', 'ts', 'deltas', 'eik_grad', 'sample_sdf'] + (['rgb'] if n_feat else []) + (['sem'] if n_feat > 3 else [])
    cfg = dict(desc=desc, cam_mats=i2l.to(dev), rays=ops.make_ray_desc(2, grid=(ny, nx, 160 / nx, 0., 90 / ny, 0.)),
               params=ops.make_render_params(aabb, S, inv_s0, training=True, bkgd='random' if n_feat else 'white'),
               jitter=jitter.to(dev) if use_jitter else None, bkgd_rand=bk.to(dev) if bk is not None else None, want=want)
    res = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vs, vf, invs, cfg)))
    cmp = lambda a, b, atol, rtol=1e-4: torch.allclose(a.detach().cpu(), b.detach().float().reshape(a.shape), atol=atol, rtol=rtol)
    assert cmp(res['weights'], ref['weights'], 2e-6)
    assert cmp(res['ts'], ref['ts'], 1e-5, 1e-5) and cmp(res['deltas'], ref['deltas'], 4e-6, 1e-4)   # difference of two fp32 edges up to ~20 m: 2 ulp(20 m) absolute
    assert cmp(res['eik_grad'], ref['eik_grad'], 2e-5) and cmp(res['sample_sdf'], ref['sdf'], 2e-5)
    assert cmp(res['depth'], ref['depth'], 1e-5) and cmp(res['acc'], ref['accumulation'], 2e-5)
    assert cmp(res['fars'], ref['fars'], 1e-5)
    if n_feat:
        assert cmp(res['rgb'], ref['rgb'], 5e-5)
    if n_feat > 3:
        assert cmp(res['sem'], ref['sem'], 5e-5)
    # ---- backward with random cotangents on every differentiable output
    keys = [('depth', 'depth'), ('acc', 'accumulation'), ('weights', 'weights'), ('eik_grad', 'eik_grad'), ('sample_sdf', 'sdf')]
    if n_feat:
        keys += [('rgb', 'rgb')] + ([('sem', 'sem')] if n_feat > 3 else [])
    cot = {k: torch.randn(res[k].shape, generator=g) for k, _ in keys}
    loss = sum((res[k] * cot[k].to(dev)).sum() for k, _ in keys)
    loss.backward()
    loss64 = sum((ref[rk].reshape(cot[k].shape) * cot[k].double()).sum() for k, rk in keys)
    loss64.backward()
    gv = vs.grad[..., :m.size_d].cpu()
    gref = vol64.grad[0].float()
    scale = gref.abs().max().item()
    err = (gv - gref).abs().max().item()
    print('train bwd: d/d(vol sdf) max abs err %.3e (max |g| %.3e); d/d(inv_s) %.6e vs %.6e' % (
        err, scale, invs.grad.item(), invs64.grad.item()))
    assert err < 1e-3 * max(scale, 1.0)     # fp32 atomics over hundreds of signed per-sample terms per voxel
    # a scalar that sums thousands of signed fp32 terms: 2e-3 relative
    assert abs(invs.grad.item() - invs64.grad.item()) < 2e-3 * max(1.0, abs(invs64.grad.item()))
    if n_feat:
        gf = vf.grad[..., :n_feat].cpu().permute(3, 0, 1, 2)
        assert torch.allclose(gf, vol64.grad[1:].float(), atol=2e-4 * max(1.0, vol64.grad[1:].abs().max().item()))


@pytest.mark.parametrize('n_feat', [0, 3])
def test_render_train_forward_batched_kernel_matches_one_ray_per_warp_kernel(n_feat):
    """The two forward kernels on cfg-5-like geometry (const-pitch specialisation, 256 samples): identical per-sample
    arithmetic -> per-sample tensors equal to rounding; the z-pair repack changes loads only -> bit-identical."""
    dev = _dev()
    from selfocc_b200 import ops, _lib
    margs = dict(synth.NUSC_MAPPING, d_size=[24, 0], d_range=[-4.0, 4.0, 4.0])
    aabb = [-51.2, -51.2, -4.0, 51.2, 51.2, 4.0]
    m = GridMeterMapping(**margs)
    desc = m.volume_desc(n_feat)
    g = torch.Generator().manual_seed(5)
    vs = synth.pack_sdf_volume(synth.analytic_sdf_volume(m, noise=0.02), desc.zpitch).to(dev)
    vf = (0.5 * torch.randn(desc.H, desc.W, desc.Z, desc.feat_pitch, generator=g)).to(dev) if n_feat else None
    _, i2l = synth.camera_rig()
    ny, nx, S = 12, 25, 256
    n = 6 * ny * nx
    want = ['depth', 'acc', 'fars', 'max_depth', 'weights', 'ts', 'deltas', 'eik_grad', 'sample_sdf'] + (['rgb'] if n_feat else [])
    cfg = dict(desc=desc, cam_mats=torch.tensor(i2l, dtype=torch.float32, device=dev),
               rays=ops.make_ray_desc(6, grid=(ny, nx, 64.0, 3.0, 64.0, 5.0)),
               params=ops.make_render_params(aabb, S, 20.0, training=True, bkgd='random' if n_feat else 'white'),
               jitter=torch.rand(n, S + 1, generator=g).to(dev), bkgd_rand=torch.rand(n, 3, generator=g).to(dev) if n_feat else None,
               want=want)
    invs = torch.tensor([20.0], device=dev)
    run = lambda c: dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vs, vf, invs, c)))
    lib = _lib.load()
    try:
        lib.so_render_train_force_fwd32(1)
        a = run(cfg)
    finally:
        lib.so_render_train_force_fwd32(0)
    b = run(cfg)
    c = run(dict(cfg, zpair=False))
    for k in want:
        assert torch.equal(b[k], c[k]), k
    for k in ('ts', 'deltas', 'eik_grad', 'sample_sdf', 'fars'):
        assert torch.allclose(a[k], b[k], rtol=1e-6, atol=1e-7), k
    assert torch.allclose(a['weights'], b['weights'], rtol=2e-5, atol=1e-7)
    for k in ('depth', 'acc') + (('rgb',) if n_feat else ()):
        assert torch.allclose(a[k], b[k], rtol=1e-5, atol=1e-6), k
    assert (a['max_depth'] != b['max_depth']).float().mean().item() < 1e-3     # ties broken by 1-ulp weight differences


def test_head_forward_training_outputs_and_grads():
    """NeuSHead.forward (neus_head.py:473-713): output dict contract + gradients reach the TPV planes and the MLP."""
    dev = _dev()
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    from oracle.mapping import GridMeterMappingRef
    from oracle import render as orender, rays as orays
    torch.manual_seed(0)
    margs, rng = synth.small_mapping(8, 4, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=32, ray_number=(4, 6), ray_img_size=(90, 160), color_dims=7,
                                  return_sem=True, render_bkgd='random')
    head = build_head(cfg['head']).to(dev).train()
    with torch.no_grad():
        head.model.field.deviation_network.variance.fill_(0.25)
    l2i, i2l = synth.camera_rig(f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(90, 160))]
    H, W, Z = 17, 17, 5
    planes = [(0.5 * torch.randn(1, n, 96, device=dev)).requires_grad_(True) for n in (H * W, Z * H, W * Z)]
    n = 6 * 24
    jitter = torch.rand(n, 33, device=dev)
    bk = torch.rand(n, 3, device=dev)
    out = head(representation=planes, metas=metas, jitter=jitter, bkgd_rand=bk)
    for k in ('ms_depths', 'ms_colors', 'ms_accs', 'ms_fars', 'ms_rays', 'origin', 'direction', 'direction_norm', 'ray_indices',
              'weights', 'ts', 'deltas', 'eik_grad', 'uniform_sdf', 'ms_max_depths', 'sem'):
        assert k in out, k
    assert out['ms_depths'][0].shape == (1, 6, 24) and out['ms_colors'][0].shape == (1, 6, 24, 3)
    assert len(out['weights']) == 6 and out['weights'][0].shape == (24 * 32,)
    assert torch.equal(out['ray_indices'][0], torch.arange(24, device=dev).repeat_interleave(32))
    assert out['eik_grad'].shape == (n, 32, 3)
    # oracle forward on the same planes / jitter
    f = head.model.field
    w1, b1, w2, b2 = (t.detach().cpu().double() for t in (f.density_net[1].weight, f.density_net[1].bias,
                                                         f.density_net[3].weight, f.density_net[3].bias))
    mref = GridMeterMappingRef(**margs)
    vol = orender.tpv_decode_ref(*[p[0].detach().cpu().double() for p in planes], (H, W, Z), w1, b1, w2, b2)
    origin, direction = orays.img2lidar_rays(torch.tensor(i2l, dtype=torch.float32)[None], orays.fixed_ray_grid([4, 6], [90, 160]))
    o, d, nrm = orays.flatten_rays(origin.double(), direction.double())
    ref = orender.neus_render_chunk(vol, mref, o, d, nrm, rng, float(f.deviation_network.get_variance()), S=32, training=True,
                                    jitter=jitter.cpu().double(), color_dims=3, bkgd='random', bkgd_rand=bk.cpu().double())
    assert torch.allclose(out['ms_depths'][0].detach().cpu().reshape(-1), ref['depth'].float(), rtol=1e-4, atol=1e-5)
    assert torch.allclose(torch.cat(out['weights']).detach().cpu(), ref['weights'].float().reshape(-1), atol=3e-6)
    assert torch.allclose(out['ms_colors'][0].detach().cpu().reshape(-1, 3), ref['rgb'].float(), atol=5e-5)
    loss = out['ms_depths'][0].mean() + torch.cat(out['weights']).pow(2).sum() + (out['eik_grad'].norm(dim=-1) - 1).pow(2).mean() \
        + out['ms_colors'][0].mean() + out['sem'][0].pow(2).mean()
    loss.backward()
    for p in planes:
        assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0
    assert f.density_net[1].weight.grad.abs().sum() > 0 and f.deviation_network.variance.grad is not None


def test_second_grad_matches_double_backward_of_the_oracle_field():
    """B8 `second_grad` (opt-in declared assumption, so_field_second_grad): row sums of the Hessian of the trilinear field
    = torch.autograd.grad(grad_sdf.sum(), x) of the oracle's explicit 8-corner field query; backward is exact because the
    output is linear in the volume."""
    dev = _dev()
    from oracle.mapping import GridMeterMappingRef
    from oracle import render as orender
    from selfocc_b200 import ops
    g = torch.Generator().manual_seed(5)
    margs, aabb = synth.small_mapping(10, 6)
    m, mref = GridMeterMapping(**margs), GridMeterMappingRef(**margs)
    sdf = torch.randn(m.size_h, m.size_w, m.size_d, generator=g)
    lo, hi = torch.tensor(aabb[:3]) - 0.8, torch.tensor(aabb[3:]) + 0.8          # some points outside: zeros padding
    x = lo + (hi - lo) * torch.rand(4000, 3, generator=g)
    x64 = x.double().requires_grad_(True)
    vol64 = sdf[None].double().requires_grad_(True)
    _, grad_chk = orender.field_query_manual(vol64, mref, x64)
    _, grad = _manual_grad_of_x(vol64, mref, x64)                  # same gradient, fractions kept differentiable w.r.t. x
    assert torch.allclose(grad, grad_chk)
    sg_ref = torch.autograd.grad(grad.sum(), x64, create_graph=True)[0]
    desc = m.volume_desc(0)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev).requires_grad_(True)
    sg = ops.FieldSecondGradFunction.apply(vs, desc, x.to(dev).contiguous())
    assert torch.allclose(sg.detach().cpu().double(), sg_ref.detach(), atol=2e-4, rtol=1e-4)
    # backward: d (sum c * second_grad) / d volume
    c = torch.randn(4000, 3, generator=g)
    (sg * c.to(dev)).sum().backward()
    gv_ref = torch.autograd.grad((sg_ref * c.double()).sum(), vol64)[0][0]
    assert torch.allclose(vs.grad[..., :m.size_d].cpu().double(), gv_ref, atol=2e-3, rtol=1e-4)


def _manual_grad_of_x(vol, mapping, x):
    """field_query_manual with the fractions kept differentiable w.r.t. x (meter2grid is piecewise linear in x)."""
    Cf, H, W, Z = vol.shape
    g = mapping.meter2grid(x, False)
    gh, gw, gd = g[:, 0], g[:, 1], g[:, 2]
    h0, w0, z0 = gh.detach().floor(), gw.detach().floor(), gd.detach().floor()
    fh, fw, fz = gh - h0, gw - w0, gd - z0
    h0, w0, z0 = h0.long(), w0.long(), z0.long()
    dgh = dgw = dgd = 0
    for dh in (0, 1):
        for dw in (0, 1):
            for dz in (0, 1):
                hh, ww, zz = h0 + dh, w0 + dw, z0 + dz
                ok = ((hh >= 0) & (hh < H) & (ww >= 0) & (ww < W) & (zz >= 0) & (zz < Z)).to(vol.dtype)
                v = vol[0, hh.clamp(0, H - 1), ww.clamp(0, W - 1), zz.clamp(0, Z - 1)] * ok
                wh, w_w, wz = (fh if dh else 1 - fh), (fw if dw else 1 - fw), (fz if dz else 1 - fz)
                dgh = dgh + (1.0 if dh else -1.0) * w_w * wz * v
                dgw = dgw + wh * (1.0 if dw else -1.0) * wz * v
                dgd = dgd + wh * w_w * (1.0 if dz else -1.0) * v
    xr = x.detach().clone().requires_grad_(True)
    slopes = torch.autograd.grad(mapping.meter2grid(xr, False).sum(), xr)[0]
    return None, torch.stack([dgw * slopes[:, 0], dgh * slopes[:, 1], dgd * slopes[:, 2]], -1)


def test_head_forward_with_the_shipped_occ_config_options():
    """config/nuscenes/nuscenes_occ.py:321-322,350: return_second_grad=True, return_sem=True, color_dims=24 -- the training
    forward refuses without the opt-in and runs (all outputs finite, gradients reach the planes) with it."""
    dev = _dev()
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    margs, rng = synth.small_mapping(8, 4, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=64, ray_number=(6, 8), ray_img_size=(90, 160), color_dims=24,
                                  return_sem=True, ray_sample_mode='cellular')
    cfg['head'].update(return_second_grad=True, return_uniform_sdf=True)
    model = build_head(cfg).to(dev).train()
    l2i, i2l = synth.camera_rig(f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(90, 160))]
    planes = [p.detach().clone().requires_grad_(True) for p in (model.lifter.tpv_hw, model.lifter.tpv_zh, model.lifter.tpv_wz)]
    with pytest.raises(NotImplementedError):
        model.head(representation=planes, metas=metas)
    model.head.second_grad_assumption = True
    out = model.head(representation=planes, metas=metas)
    assert out['second_grad'].shape == (6 * 48, 64, 3) and torch.isfinite(out['second_grad']).all()
    assert out['sem'][0].shape[-1] == 21
    loss = out['second_grad'].abs().mean() + out['ms_depths'][0].mean() + out['sem'][0].sum() * 1e-3
    loss.backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().sum() > 0 for p in planes)


@pytest.mark.parametrize('n_feat,hw,d,slab', [(0, 12, 6, 5), (3, 9, 5, 32), (24, 7, 4, 3)])
def test_decode_backward_native_matches_oracle_autograd(n_feat, hw, d, slab, monkeypatch):
    """TPVDecodeFunction.backward, native slab path (wgmma GEMMs + so_tpv_decode_bwd_*): gradients of every plane and
    MLP parameter vs fp64 autograd through the oracle's decode (oracle/render.py:tpv_decode_ref), with several ragged slabs;
    the torch/cuBLAS restatement of the same slab (_backward_torch) must agree as well."""
    dev = _dev()
    from oracle import render as orender
    from selfocc_b200 import ops
    margs, _ = synth.small_mapping(hw, d)
    m = GridMeterMapping(**margs)
    H, W, Z, C = m.size_h, m.size_w, m.size_d, 96
    planes = synth.random_planes(m, C, scale=1.0, seed=4)
    mlp = synth.random_mlp(C, 1 + n_feat, seed=4)
    desc = m.volume_desc(n_feat)
    g = torch.Generator().manual_seed(9)
    g_sdf = torch.randn(H, W, Z, generator=g)
    g_feat = torch.randn(H, W, Z, max(n_feat, 1), generator=g)

    ins64 = [t.double().requires_grad_(True) for t in (*planes, *mlp)]
    ref = orender.tpv_decode_ref(*ins64[:3], (H, W, Z), *ins64[3:])            # [Cf, H, W, Z]
    loss = (ref[0] * g_sdf.double()).sum()
    if n_feat:
        loss = loss + (ref[1:].permute(1, 2, 3, 0) * g_feat.double()).sum()
    gref = torch.autograd.grad(loss, ins64)

    def run(mode):
        if mode == 'torch':
            monkeypatch.setattr(ops.TPVDecodeFunction, '_backward_native', ops.TPVDecodeFunction._backward_torch)
        monkeypatch.setattr(ops.TPVDecodeFunction, 'SLAB_ROWS', slab)
        ins = [t.to(dev).requires_grad_(True) for t in (*planes, *mlp)]
        vs, vf = ops.TPVDecodeFunction.apply(*ins, desc)
        l = (vs[..., :Z] * g_sdf.to(dev)).sum()
        if n_feat:
            l = l + (vf[..., :n_feat] * g_feat.to(dev)).sum()
        return [t.cpu() for t in torch.autograd.grad(l, ins)]

    names = ('tpv_hw', 'tpv_zh', 'tpv_wz', 'w1', 'b1', 'w2', 'b2')
    for mode in ('native', 'torch'):
        got = run(mode)
        for n, a, b in zip(names, got, gref):
            scale = b.abs().max().item() + 1e-12
            err = (a.double() - b).abs().max().item() / scale
            print('decode backward (%s) %s rel-to-max err %.2e' % (mode, n, err))
            assert err < 2e-4, (mode, n, err)
