"""GPU parity: fused render / decode / field-query kernels (through the C ABI) vs the CPU oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from selfocc_b200 import synth
from selfocc_b200.mapping import GridMeterMapping


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _scene(hw=16, d=8, n_feat=0, noise=0.05, seed=0):
    from oracle.mapping import GridMeterMappingRef
    margs, aabb = synth.small_mapping(hw, d)
    m = GridMeterMapping(**margs)
    mref = GridMeterMappingRef(**margs)
    sdf = synth.analytic_sdf_volume(m, ground_z=-1.0, spheres=((3., 5., 0., 1.5), (-4., 2., -0.2, 1.0)),
                                    boxes=((-2., 8., -1., 1.5, 1., 1.),), noise=noise, seed=seed)
    gen = torch.Generator().manual_seed(seed + 7)
    feat = torch.randn(n_feat, *sdf.shape, generator=gen) if n_feat else None
    vol_ref = sdf[None] if feat is None else torch.cat([sdf[None], feat], 0)
    return m, mref, aabb, sdf, feat, vol_ref


def _cams(n=3, scale_hw=(90, 160)):
    l2i, i2l = synth.camera_rig(synth.NUSC_YAWS[:n], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    return torch.tensor(l2i, dtype=torch.float32), torch.tensor(i2l, dtype=torch.float32)


@pytest.mark.parametrize('anchor_mid,batch,n_feat', [(True, 0, 0), (False, 700, 0), (True, 1000, 3), (True, 0, 8)])
def test_render_infer_matches_oracle(anchor_mid, batch, n_feat):
    dev = _dev()
    from oracle import rays as orays, render as orender
    from selfocc_b200 import ops
    m, mref, aabb, sdf, feat, vol_ref = _scene(n_feat=n_feat)
    _, i2l = _cams(3)
    ny, nx, ih, iw = 18, 32, 90, 160
    pix = orays.fixed_ray_grid([ny, nx], [ih, iw])
    origin, direction = orays.img2lidar_rays(i2l[None], pix)
    inv_s = 20.0
    S = 64
    ref = orender.head_render_ref(vol_ref, mref, origin, direction, aabb, inv_s, batch=batch, S=S,
                                  anchor='mid' if anchor_mid else 'start', color_dims=3 if n_feat else 0, bkgd='white')
    ref64 = orender.head_render_ref(vol_ref.double(), _M64(mref), origin.double(), direction.double(), aabb, inv_s,
                                    batch=batch, S=S, anchor='mid' if anchor_mid else 'start',
                                    color_dims=3 if n_feat else 0, bkgd='white')
    desc = m.volume_desc(n_feat)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev) if n_feat else None
    rd = ops.make_ray_desc(3, grid=(ny, nx, iw / nx, 0.0, ih / ny, 0.0), chunk_len=_chunk_len(3 * ny * nx, batch))
    pr = ops.make_render_params(aabb, S, inv_s, anchor_mid=anchor_mid, bkgd='white')
    want = ['depth', 'max_depth', 'max_idx', 'acc', 'normal_vis'] + (['rgb'] if n_feat else []) + (['sem'] if n_feat > 3 else [])
    out = ops.render_infer(vs, vf, desc, i2l.to(dev), rd, pr, want=want)
    out = {k: v.cpu() for k, v in out.items()}
    n = 3 * ny * nx
    d_ref, d64 = ref['depth'].reshape(n), ref64['depth'].reshape(n).float()
    rel32 = ((out['depth'] - d_ref).abs() / d_ref.abs().clamp_min(1e-6)).max().item()
    rel64 = ((out['depth'] - d64).abs() / d64.abs().clamp_min(1e-6)).max().item()
    o64 = ((d_ref - d64).abs() / d64.abs().clamp_min(1e-6)).max().item()
    print('depth max rel err: vs fp32 oracle %.3e, vs fp64 oracle %.3e (fp32 oracle vs fp64 %.3e)' % (rel32, rel64, o64))
    assert rel64 < 1e-4, 'rendered depth must be within 1e-4 relative of the fp64 oracle (north_star tolerance)'
    assert rel32 < 1e-4 + o64   # the fp32 oracle is itself only o64-close to fp64 (cancellation in Phi(prev)-Phi(next))
    assert torch.allclose(out['acc'], ref64['acc'].reshape(n).float(), atol=2e-5, rtol=1e-4)
    assert torch.allclose(out['normal_vis'], ref64['vis_normal'].reshape(n, 3).float(), atol=5e-5)
    # bit-exact sample indices: argmax must equal the fp64 oracle's wherever the oracle's top-2 gap is not a near-tie
    idx64 = ref64['max_idx'].reshape(n)
    w, dl = ref64['weights'].reshape(n, S), ref64['deltas'].reshape(n, S)
    score = w / dl.clamp_min(torch.finfo(torch.float32).eps)
    top2 = score.topk(2, -1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-5 * top2[:, 0].abs().clamp_min(1e-30)
    print('argmax: %.1f%% of rays have a clear (non-tie) maximum; kernel == fp64 oracle on %.2f%% of all rays' % (
        100 * clear.float().mean().item(), 100 * (out['max_idx'] == idx64).float().mean().item()))
    assert clear.float().mean() > 0.5
    assert torch.equal(out['max_idx'][clear], idx64[clear])
    agree = out['max_idx'] == idx64
    assert torch.allclose(out['max_depth'][agree], ref64['max_depth'].reshape(n)[agree].float(), rtol=1e-5, atol=1e-6)
    # near-ties may pick the neighbouring candidate; the score there must be within rounding of the maximum
    bad = ~agree
    if bad.any():
        got = score[bad].gather(1, out['max_idx'][bad][:, None])[:, 0]
        assert torch.allclose(got, top2[bad, 0], rtol=1e-4)
    if n_feat:
        assert torch.allclose(out['rgb'], ref64['rgb'].reshape(n, 3).float(), atol=5e-5)
    if n_feat > 3:
        assert torch.allclose(out['sem'], ref64['sem'].reshape(n, -1).float(), atol=5e-5)


def _chunk_len(total, batch):
    import math
    if batch <= 0:
        return 0
    chunks = int(math.ceil(total / batch))
    return int(math.ceil(total / chunks))  # torch.chunk size


class _M64:
    """fp64 view of the oracle mapping (same arithmetic, double inputs)."""
    def __init__(self, m):
        self.m = m
    def meter2grid(self, x, normalize=False):
        return self.m.meter2grid(x, normalize)


def test_ray_sharding_is_order_preserving():
    dev = _dev()
    from selfocc_b200 import ops
    m, _, aabb, sdf, _, _ = _scene()
    _, i2l = _cams(3)
    desc = m.volume_desc(0)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    ny, nx = 10, 16
    pr = ops.make_render_params(aabb, 32, 15.0)
    full = ops.render_infer(vs, None, desc, i2l.to(dev), ops.make_ray_desc(3, grid=(ny, nx, 10., 0., 9., 0.), chunk_len=100),
                            pr, want=('depth', 'max_idx'))
    total = 3 * ny * nx
    parts = []
    for b, e in ((0, 131), (131, 300), (300, total)):
        rd = ops.make_ray_desc(3, grid=(ny, nx, 10., 0., 9., 0.), ray_begin=b, ray_count=e - b, chunk_len=100)
        parts.append(ops.render_infer(vs, None, desc, i2l.to(dev), rd, pr, want=('depth', 'max_idx')))
    assert torch.equal(torch.cat([p['depth'] for p in parts]), full['depth'])
    assert torch.equal(torch.cat([p['max_idx'] for p in parts]), full['max_idx'])


def test_pixel_table_equals_in_kernel_grid():
    dev = _dev()
    from oracle import rays as orays
    from selfocc_b200 import ops
    m, _, aabb, sdf, _, _ = _scene()
    _, i2l = _cams(2)
    desc = m.volume_desc(0)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    pr = ops.make_render_params(aabb, 32, 15.0)
    u4 = np.array([0.3, 0.7, 0.2, 0.9])
    pix = orays.cellular_ray_grid([6, 10], [90, 160], u4, ray_upper_crop=8)
    xm, ym = 160 / 10, (90 - 8) / 6
    xd, yd = u4[0] * (xm - 1) + 1, u4[1] * (ym - 1) + 1
    grid = (6, 10, xd, u4[2] * (160 - 10 * xd), yd, u4[3] * (90 - 8 - 6 * yd) + 8)
    a = ops.render_infer(vs, None, desc, i2l.to(dev), ops.make_ray_desc(2, n_pix=60), pr, pix=pix.to(dev), want=('depth',))
    b = ops.render_infer(vs, None, desc, i2l.to(dev), ops.make_ray_desc(2, grid=grid), pr, want=('depth',))
    assert torch.allclose(a['depth'], b['depth'], rtol=1e-5)


@pytest.mark.parametrize('C,n_feat,hw,d', [(96, 0, 12, 6), (96, 24, 8, 5), (32, 3, 6, 4), (128, 0, 5, 9)])
def test_tpv_decode_matches_oracle(C, n_feat, hw, d):
    dev = _dev()
    from oracle import render as orender
    from selfocc_b200 import ops
    margs, _ = synth.small_mapping(hw, d)
    m = GridMeterMapping(**margs)
    planes = synth.random_planes(m, C, scale=1.0, seed=3)
    w1, b1, w2, b2 = synth.random_mlp(C, 1 + n_feat, seed=3)
    ref = orender.tpv_decode_ref(*[p.double() for p in planes], (m.size_h, m.size_w, m.size_d), w1.double(), b1.double(),
                                 w2.double(), b2.double()).float()
    desc = m.volume_desc(n_feat)
    vs, vf = ops.tpv_decode(*[p.to(dev) for p in planes], w1.to(dev), b1.to(dev), w2.to(dev), b2.to(dev), desc)
    vs, vf = vs.cpu(), (vf.cpu() if vf is not None else None)
    assert torch.all(vs[..., m.size_d:] == 0)
    err = (vs[..., :m.size_d] - ref[0]).abs().max().item()
    print('decode sdf max abs err %.3e (|sdf| max %.2f)' % (err, ref[0].abs().max().item()))
    assert err < 2e-5 * max(1.0, ref[0].abs().max().item())
    if n_feat:
        assert torch.allclose(vf[..., :n_feat], ref[1:].permute(1, 2, 3, 0), atol=5e-5, rtol=1e-5)


def test_field_query_and_uniform_lattice():
    dev = _dev()
    from oracle import render as orender
    from selfocc_b200 import ops
    m, mref, aabb, sdf, feat, vol_ref = _scene(n_feat=5)
    desc = m.volume_desc(5)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev)
    # lattice that pokes outside the volume to exercise zero padding
    big = [aabb[0] - 1.0, aabb[1] - 1.0, aabb[2] - 0.5, aabb[3] + 1.0, aabb[4] + 1.0, aabb[5] + 0.5]
    xyz = orender.uniform_lattice(big, 0.9)
    h_ref, g_ref = orender.field_query_ref(vol_ref.double(), mref, xyz.reshape(-1, 3).double())
    s, g, f = ops.field_query(vs, vf, desc, xyz.reshape(-1, 3).contiguous().to(dev), want_grad=True, want_feat=True)
    assert torch.allclose(s.cpu(), h_ref[:, 0].float(), atol=2e-5)
    assert torch.allclose(f.cpu(), h_ref[:, 1:].float(), atol=2e-5)
    # gradients agree except exactly on cell faces (measure zero for this lattice)
    assert torch.allclose(g.cpu(), g_ref.float(), atol=2e-4)
