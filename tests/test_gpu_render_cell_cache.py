"""GPU parity of the packed render kernel's per-lane cell cache (a lane reuses the last cell's corners while it stays in
that cell) against the plain render_infer_kernel, at both extremes: dense sampling, where lanes sit in one cell for many
samples, and sparse sampling, where the cell changes on (almost) every sample.  Also checks the colour pack's contents."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from selfocc_b200 import synth
from test_gpu_render import _dev, _scene, _cams

C0 = 0.28209479177387814


def _render(n_feat, S):
    dev = _dev()
    from selfocc_b200 import ops
    m, _, aabb, sdf, feat, _ = _scene(n_feat=n_feat)
    _, i2l = _cams(3)
    ny, nx, ih, iw = 18, 32, 90, 160
    desc = m.volume_desc(n_feat)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev) if n_feat else None
    pack = ops.render_pack(vs, vf, desc)
    rd = ops.make_ray_desc(3, grid=(ny, nx, iw / nx, 0.0, ih / ny, 0.0))
    pr = ops.make_render_params(aabb, S, 20.0, bkgd='white')
    want = ['depth', 'max_depth', 'max_idx', 'acc', 'normal_vis'] + (['rgb'] if n_feat else [])
    plain = ops.render_infer(vs, vf, desc, i2l.to(dev), rd, pr, want=want)
    packed = ops.render_infer(vs, vf, desc, i2l.to(dev), rd, pr, want=want, pack=pack)
    probed = ops.render_infer(vs, vf, desc, i2l.to(dev), rd, pr, want=('depth',), pack=pack, probe_grid=True)
    cpu = lambda d: {k: v.cpu() for k, v in d.items()}
    return cpu(plain), cpu(packed), probed['grid'].cpu()


def _same_cell_fraction(grid):
    """Share of sample steps (s - 1 -> s) whose trilinear cell is unchanged, over all rays."""
    cell = torch.floor(grid)
    return (cell[:, 1:] == cell[:, :-1]).all(-1).float().mean().item()


@pytest.mark.parametrize('n_feat', [0, 3])
@pytest.mark.parametrize('S,dense', [(1024, True), (4, False)])
def test_cell_cache_matches_plain_kernel(n_feat, S, dense):
    plain, packed, grid = _render(n_feat, S)
    same = _same_cell_fraction(grid)
    if dense:
        assert same > 0.8, same          # lanes stay in one cell for many samples: the cached corners are reused
    else:
        assert same < 0.5, same          # the cell changes on most samples: the lanes reload
    rel = ((packed['depth'] - plain['depth']).abs() / plain['depth'].abs().clamp_min(1e-6)).max().item()
    assert rel < 2e-5, rel
    assert torch.allclose(packed['acc'], plain['acc'], atol=5e-6)
    assert torch.allclose(packed['normal_vis'], plain['normal_vis'], atol=2e-5)
    agree = packed['max_idx'] == plain['max_idx']
    assert agree.float().mean() > 0.995
    assert torch.allclose(packed['max_depth'][agree], plain['max_depth'][agree], rtol=1e-6)
    if n_feat:
        assert torch.allclose(packed['rgb'], plain['rgb'], atol=2e-5)


def test_colour_pack_holds_the_sh0_colour_and_the_raw_sdf():
    dev = _dev()
    from selfocc_b200 import ops
    m, _, _, sdf, feat, _ = _scene(n_feat=3)
    desc = m.volume_desc(3)
    vs = synth.pack_sdf_volume(sdf, desc.zpitch).to(dev)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev)
    pack = ops.render_pack(vs, vf, desc).cpu().view(desc.H, desc.W, desc.Z, 4)
    assert torch.equal(pack[..., 3], sdf.float())
    want = (C0 * feat.double() + 0.5).permute(1, 2, 3, 0)
    assert (pack[..., :3].double() - want).abs().max().item() <= 2.5e-7
