"""GPU, BASELINE.json full sizes: size-independent properties (the oracle cannot run these sizes in seconds)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from selfocc_b200 import synth
from selfocc_b200.mapping import GridMeterMapping


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def test_render_cfg2_properties_sharding_and_chunking():
    """configs[1]: 6 x 450 x 800 rays x 256 samples over a 257 x 257 x 31 volume."""
    dev = _dev()
    from selfocc_b200 import ops
    m = GridMeterMapping(**synth.NUSC_MAPPING)
    desc = m.volume_desc(0)
    sdf = synth.analytic_sdf_volume(m, noise=0.02)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    _, i2l = synth.camera_rig()
    cams = torch.tensor(i2l, dtype=torch.float32, device=dev)
    ny, nx, S = 450, 800, 256
    total = 6 * ny * nx
    pr = ops.make_render_params(synth.NUSC_RANGE, S, 20.0)
    grid = (ny, nx, 1600 / nx, 0.0, 900 / ny, 0.0)
    want = ('depth', 'max_depth', 'max_idx', 'acc', 'normal_vis')
    full = ops.render_infer(vs, None, desc, cams, ops.make_ray_desc(6, grid=grid), pr, want=want)
    for k in want:
        assert torch.isfinite(full[k].float()).all(), k
    assert full['acc'].min() >= 0 and full['acc'].max() <= 1 + 1e-4
    assert full['depth'].min() >= 0 and full['max_depth'].min() >= 0
    assert full['max_idx'].min() >= 0 and full['max_idx'].max() < S
    assert (full['normal_vis'] >= -1e-4).all() and (full['normal_vis'] <= 1 + 1e-4).all()
    # the analytic scene has a ground plane 2.5 m under the cameras: most downward rays must terminate (acc ~ 1)
    assert (full['acc'] > 0.99).float().mean() > 0.3
    # ray sharding over 8 "ranks": concatenation is bit-identical to the single launch
    from selfocc_b200.dist import ray_slice
    parts = []
    for r in range(8):
        b, c = ray_slice(total, 8, r)
        parts.append(ops.render_infer(vs, None, desc, cams, ops.make_ray_desc(6, grid=grid, ray_begin=b, ray_count=c), pr,
                                      want=('depth', 'max_idx')))
    assert torch.equal(torch.cat([p['depth'] for p in parts]), full['depth'])
    assert torch.equal(torch.cat([p['max_idx'] for p in parts]), full['max_idx'])
    # the reference's --batch 90000 chunking only changes the clip bounds: everything but clipped depths is identical
    chunked = ops.render_infer(vs, None, desc, cams, ops.make_ray_desc(6, grid=grid, chunk_len=90000), pr, want=('depth', 'acc', 'max_idx'))
    assert torch.equal(chunked['acc'], full['acc']) and torch.equal(chunked['max_idx'], full['max_idx'])
    same = chunked['depth'] == full['depth']
    assert same.float().mean() > 0.95 and (full['acc'][~same] < 1e-3).all()
    # empty slice: a valid no-op
    empty = ops.render_infer(vs, None, desc, cams, ops.make_ray_desc(6, grid=grid, ray_begin=total, ray_count=0), pr, want=('depth',))
    assert empty['depth'].numel() == 0


def test_cross_attention_core_is_linear_in_value_at_cfg2_size():
    """A7 at configs[1] sizes (66 049 hw queries x 8-point pillars, 6 cameras, 29 750 pixels x 6 heads x 16)."""
    dev = _dev()
    from selfocc_b200 import ops
    g = torch.Generator(device='cpu').manual_seed(0)
    shapes = [(112, 200), (56, 100), (28, 50), (14, 25)]
    Nv = sum(h * w for h, w in shapes)
    ss = torch.tensor(shapes, dtype=torch.int64, device=dev)
    lsi = torch.cat([ss.new_zeros(1), ss.prod(1).cumsum(0)[:-1]])
    Q, Hd, L, D, N = 66049, 6, 4, 8, 6
    v1 = torch.randn(N, Nv, Hd, 16, device=dev)
    v2 = torch.randn(N, Nv, Hd, 16, device=dev)
    off = 3.0 * torch.randn(Q, Hd, L, D, 2, device=dev)
    lg = torch.randn(Q, Hd, L, D, device=dev)
    uv = torch.rand(N, Q, D, 2, device=dev) * 1.2 - 0.1
    vis = (torch.rand(N, Q, device=dev) < 0.3).to(torch.uint8)
    f = lambda v: ops.tpv_cross_attn_forward(v, ss, lsi, off, lg, uv, vis)
    a, b, c = f(v1), f(v2), f(2.0 * v1 - 0.5 * v2)
    assert torch.isfinite(c).all()
    assert torch.allclose(c, 2.0 * a - 0.5 * b, atol=2e-4, rtol=1e-4)
    none_visible = vis.sum(0) == 0
    assert none_visible.any() and (a[none_visible] == 0).all()          # queries seen by no camera get exactly 0


def test_projection_gemm_at_full_size_matches_cublas_fp32():
    dev = _dev()
    from selfocc_b200 import ops
    x = torch.randn(6 * 29750, 96, device=dev)
    w = 0.1 * torch.randn(288, 96, device=dev)
    b = torch.randn(288, device=dev)
    hi, lo = ops.split_tf32(w)
    y = ops.linear_3xtf32(x, hi, lo, b)
    ref = torch.nn.functional.linear(x.double(), w.double(), b.double())
    assert (y.double() - ref).abs().max().item() < 5e-5


# ---------------------------------------------------------------------------------------------------------------------
# Parity gate at BASELINE sizes (VERDICT r1 item 1): the 257 x 257 x 31 volume, S = 256, the 6-camera 900 x 1600 rig, on
# a strided sub-grid of the cfg-2 (450 x 800) / cfg-3 (900 x 1600) ray grids, fp64 oracle as the checker.
# See oracle/parity.py for what (a) geometry / (b) same cells / (c) independent mean and why the split is needed.
def _fullsize_volume(scene, color_dims, dev):
    """-> (vol_sdf, vol_feat, desc, vol64 [Cf,H,W,Z], oracle mapping)"""
    from oracle.mapping import GridMeterMappingRef
    from oracle import render as orender
    from selfocc_b200 import ops
    m = GridMeterMapping(**synth.NUSC_MAPPING)
    mref = GridMeterMappingRef(**synth.NUSC_MAPPING)
    desc = m.volume_desc(color_dims)
    H, W, Z = m.size_h, m.size_w, m.size_d
    if scene == 'analytic':                    # SURVEY 8d: ground plane + spheres + a box (rays terminate: acc ~ 1)
        sdf = synth.analytic_sdf_volume(m, noise=0.02)
        feat = torch.randn(color_dims, H, W, Z, generator=torch.Generator().manual_seed(3)) if color_dims else None
        vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
        vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev) if color_dims else None
        vol64 = (sdf[None] if feat is None else torch.cat([sdf[None], feat], 0)).double()
    else:                                      # 'decoded': unit-variance planes (what the encoder's LayerNorm emits) through
        planes = synth.random_planes(m, 96, scale=1.0, seed=5)     # the tensor-core decode kernel -- the bench's scene type
        w1, b1, w2, b2 = synth.random_mlp(96, 1 + color_dims, seed=2)
        vs, vf = ops.tpv_decode(*[p.to(dev) for p in planes], w1.to(dev), b1.to(dev), w2.to(dev), b2.to(dev), desc)
        vol64 = orender.tpv_decode_ref(*[p.double() for p in planes], (H, W, Z), w1.double(), b1.double(), w2.double(), b2.double())
    return vs, vf, desc, vol64, mref


@pytest.mark.parametrize('cfg,scene,color_dims', [(2, 'analytic', 0), (2, 'decoded', 0), (3, 'analytic', 3), (3, 'decoded', 3),
                                                  (3, 'decoded', 0)])
def test_render_parity_gate_at_baseline_size(cfg, scene, color_dims):
    dev = _dev()
    import numpy as np
    from oracle import rays as orays
    from oracle.parity import render_parity
    from selfocc_b200 import ops
    vs, vf, desc, vol64, mref = _fullsize_volume(scene, color_dims, dev)
    _, i2l = synth.camera_rig()
    cams = torch.tensor(i2l, dtype=torch.float32)
    # every 25th (cfg 2) / 50th (cfg 3) ray of the configuration's own pixel grid, all 6 cameras: 18 x 32 rays per camera
    full = {2: (450, 800), 3: (900, 1600)}[cfg]
    stride = {2: 25, 3: 50}[cfg]
    ny, nx = full[0] // stride, full[1] // stride
    sx, sy = 1600.0 / full[1] * stride, 900.0 / full[0] * stride
    grid = (ny, nx, sx, 0.0, sy, 0.0)
    pix = torch.stack([(torch.arange(nx, dtype=torch.float) * sx)[None, :].expand(ny, -1),
                       (torch.arange(ny, dtype=torch.float) * sy)[:, None].expand(-1, nx)], -1).flatten(0, 1)
    origin, direction = orays.img2lidar_rays(cams[None], pix)
    S, inv_s = 256, float(np.exp(3.0))
    pr = ops.make_render_params(synth.NUSC_RANGE, S, inv_s, bkgd='white')
    pack = ops.render_pack(vs, vf, desc)
    want = ['depth', 'max_depth', 'max_idx', 'acc', 'normal_vis'] + (['rgb'] if color_dims else [])
    got = ops.render_infer(vs, vf, desc, cams.to(dev), ops.make_ray_desc(6, grid=grid), pr, want=want, pack=pack, probe_grid=True)
    prod = ops.render_infer(vs, vf, desc, cams.to(dev), ops.make_ray_desc(6, grid=grid), pr, want=want, pack=pack)
    got = {k: v.cpu() for k, v in got.items()}
    torch.set_num_threads(max(torch.get_num_threads(), 8))
    rep = render_parity(got, vol64, mref, origin, direction, synth.NUSC_RANGE, inv_s, S, color_dims=color_dims, bkgd='white')
    print('cfg %d %s color_dims=%d: %s' % (cfg, scene, color_dims, rep))
    assert rep['ok'], rep
    # the production launch (early exit on) equals the probe launch
    assert torch.allclose(prod['depth'].cpu(), got['depth'], rtol=2e-6, atol=0) and torch.equal(prod['max_idx'].cpu(), got['max_idx'])
    # and the plain (unpacked) kernel passes the independent comparison to the same standard on the rays without a cell flip
    plain = ops.render_infer(vs, vf, desc, cams.to(dev), ops.make_ray_desc(6, grid=grid), pr, want=('depth',))
    rel = ((plain['depth'].cpu() - got['depth']).abs() / got['depth'].abs().clamp_min(1e-6))
    assert (rel > 1e-4).float().mean() < 0.02
