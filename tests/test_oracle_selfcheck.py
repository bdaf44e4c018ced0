"""CPU: analytic self-checks of the (unpinned) parts of the oracle (SURVEY.md 8c iii)."""
import math
import pytest
import torch
from oracle.mapping import GridMeterMappingRef
from oracle import render as orender, lifting as ol, rays as orays
from selfocc_b200 import synth


def _map(hw=10, d=6):
    margs, aabb = synth.small_mapping(hw, d)
    return GridMeterMappingRef(**margs), aabb


def test_manual_field_query_equals_grid_sample():
    m, aabb = _map()
    g = torch.Generator().manual_seed(0)
    vol = torch.randn(4, m.size_h, m.size_w, m.size_d, generator=g, dtype=torch.float64)
    x = (torch.rand(500, 3, generator=g, dtype=torch.float64) - 0.5) * torch.tensor([30., 30., 7.]) + torch.tensor([0., 0., 0.5])
    h1, g1 = orender.field_query_ref(vol, m, x)
    h2, g2 = orender.field_query_manual(vol, m, x)
    assert torch.allclose(h1, h2, atol=1e-10) and torch.allclose(g1, g2, atol=1e-9)


def test_planar_sdf_renders_plane_depth():
    """sdf = z - z0 (exactly representable by trilinear interpolation): as inv_s grows the rendered depth tends to
    the camera-z depth of the plane hit, and normals to +z."""
    m, aabb = _map(16, 8)
    H, W, Z = m.size_h, m.size_w, m.size_d
    g = torch.stack(torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64),
                                   torch.arange(Z, dtype=torch.float64), indexing='ij'), -1)
    z0 = -1.0
    vol = (m.grid2meter(g)[..., 2] - z0)[None]
    l2i, i2l = synth.camera_rig((0.,), f=126.6, cx=80., cy=45., height=0.5, radius=0.0)
    pix = torch.tensor([[80., 70.], [60., 80.], [100., 85.]])
    origin, direction = orays.img2lidar_rays(torch.tensor(i2l, dtype=torch.float64)[None].float(), pix)
    out = orender.head_render_ref(vol, m, origin.double(), direction.double(), aabb, inv_s=400.0, S=2048)
    # analytic: ray o + t*dir (dir has camera depth 1) hits z = z0 at t = (z0 - o_z) / dir_z
    t_hit = (z0 - origin[0, 0, 2].double()) / direction[0, 0, :, 2].double()
    # the +1e-5 in the alpha formula leaks ~1e-5 of weight per sample in front of the surface: a known ~0.5% pull
    assert torch.allclose(out['depth'][0, 0], t_hit, rtol=1e-2)
    assert (out['depth'][0, 0] < t_hit).all()
    assert torch.allclose(out['vis_normal'][0, 0], torch.tensor([0.5, 0.5, 1.0], dtype=torch.float64).expand(3, 3), atol=2e-2)
    assert torch.allclose(out['acc'][0, 0], torch.ones(3, dtype=torch.float64), atol=2e-3)


def test_msda_integer_centres_and_uniform_weights():
    shapes = [(4, 6)]
    value = torch.arange(24 * 2 * 4, dtype=torch.float64).reshape(1, 24, 2, 4)
    loc = torch.tensor([(2 + 0.5) / 6, (1 + 0.5) / 4], dtype=torch.float64).reshape(1, 1, 1, 1, 1, 2).repeat(1, 1, 2, 1, 1, 1)
    out = ol.msda_ref(value, shapes, loc, torch.ones(1, 1, 2, 1, 1, dtype=torch.float64))
    assert torch.equal(out.view(2, 4), value[0, 1 * 6 + 2])
    # a location on the border between 4 pixels averages them
    loc2 = torch.tensor([3.0 / 6, 2.0 / 4], dtype=torch.float64).reshape(1, 1, 1, 1, 1, 2).repeat(1, 1, 2, 1, 1, 1)
    out2 = ol.msda_ref(value, shapes, loc2, torch.ones(1, 1, 2, 1, 1, dtype=torch.float64))
    exp = (value[0, 1 * 6 + 2] + value[0, 1 * 6 + 3] + value[0, 2 * 6 + 2] + value[0, 2 * 6 + 3]) / 4
    assert torch.allclose(out2.view(2, 4), exp)


def test_point_sampling_identity_camera():
    """lidar2img = identity: uv = (x/z/w, y/z/h), mask = in front & inside the unit square."""
    ref = torch.tensor([[[0.5, 0.25, 1.0], [2.0, 1.0, 4.0], [1.0, 1.0, -1.0], [3.0, 0.1, 1.0]]]).reshape(1, 1, 4, 3)
    uv, mask = ol.point_sampling_ref(ref, torch.eye(4)[None, None], (1.0, 2.0))
    assert torch.allclose(uv[0, 0, :, 0], torch.tensor([[0.25, 0.25], [0.25, 0.25], [1.0 / 1e-5 / 2, 1.0 / 1e-5], [1.5, 0.1]]))
    assert mask[0, 0, :, 0].tolist() == [True, True, False, False]


def test_max_depth_first_maximum():
    w = torch.tensor([[0.1, 0.4, 0.4, 0.1]])
    ts = torch.tensor([[1., 2., 3., 4.]])
    d = torch.full((1, 4), 0.5)
    md, idx = orender.max_depth_ref(w, ts, d)
    assert idx.item() == 1 and md.item() == 2.0


def test_train_parity_reproduces_itself_and_masks_exactly_the_flip_rays():
    """oracle/train_parity.py on the oracle's own fp64 results: with its own coordinates as the kernel's probe the same-cells
    run reproduces the independent one exactly (outputs and gradients) and every tolerance keeps its unscaled value;
    flip_rays flags exactly the rays with a sample moved into another cell (a move inside the cell is not a flip), and a
    cotangent left on a flagged ray is refused."""
    from oracle import train_parity as tp
    m, aabb = _map(10, 6)
    g = torch.Generator().manual_seed(2)
    sdf = synth.analytic_sdf_volume(m, ground_z=-1.0, spheres=((3., 5., 0., 1.5),), boxes=(), noise=0.05, seed=1)
    vol = torch.cat([sdf[None], torch.randn(4, *sdf.shape, generator=g)], 0).double()
    _, i2l = synth.camera_rig(synth.NUSC_YAWS[:2], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    origin, direction = orays.img2lidar_rays(torch.tensor(i2l, dtype=torch.float32)[None], orays.fixed_ray_grid([3, 4], [90, 160]))
    o, d, nrm = orays.flatten_rays(origin.double(), direction.double())
    n, S = o.shape[0], 32
    jitter = torch.rand(n, S + 1, generator=g, dtype=torch.float64)
    bk = torch.rand(n, 3, generator=g, dtype=torch.float64)
    g64, clip = tp.sample_geometry(m, o, d, aabb, S, jitter)
    moved = g64.clone()
    moved[1, 7, 0] = moved[1, 7, 0].floor() + 1.5          # next cell along h
    moved[4, 20, 2] = moved[4, 20, 2].floor() - 0.5        # previous cell along d
    moved[6, 3, 1] = moved[6, 3, 1].floor() + 0.25         # same cell
    flip = tp.flip_rays(g64, moved)
    assert flip.nonzero()[:, 0].tolist() == [1, 4]
    shapes = dict(depth=(n,), acc=(n,), weights=(n, S), eik_grad=(n, S, 3), sample_sdf=(n, S), rgb=(n, 3), sem=(n, 1))
    cot = {k: torch.randn(s, generator=g, dtype=torch.float64) for k, s in shapes.items()}
    for t in cot.values():
        t[flip] = 0
    got, gvol, ginv, _ = tp.oracle_train(vol, m, o, d, nrm, aabb, 12.0, S, cot, jitter=jitter, color_dims=3, bkgd_rand=bk,
                                         depth_clip=clip, chunk=5)
    whole, gvol1, ginv1, _ = tp.oracle_train(vol, m, o, d, nrm, aabb, 12.0, S, cot, jitter=jitter, color_dims=3, bkgd_rand=bk, chunk=n)
    assert torch.equal(got['depth'], whole['depth']) and torch.allclose(gvol, gvol1, atol=1e-12)   # chunking keeps the batch clip
    assert torch.allclose(ginv, ginv1, rtol=1e-12)
    rep = tp.train_parity(got, {'vol': gvol, 'inv_s': ginv}, cot, vol, m, o, d, nrm, aabb, 12.0, S, g64, jitter=jitter,
                          color_dims=3, bkgd_rand=bk, chunk=5)
    print(tp.format_report('selfcheck', rep))
    assert rep['ok'] and rep['geometry']['max_abs_grid_units'] == 0 and rep['independent']['rays_with_cell_flip'] == 0
    assert rep['kappa']['same_cells'] == 1.0 and rep['kappa']['independent'] == 1.0
    for part in ('same_cells', 'independent'):
        assert all(v[1] == 0 for v in rep[part].values() if isinstance(v, tuple)), rep[part]
    # the kernel's probe (here: the moved coordinates) flags the same rays, whose cotangents must be zero
    cot['weights'][1, 0] = 1.0
    with pytest.raises(AssertionError, match='not zero on a flip ray'):
        tp.train_parity(got, {'vol': gvol, 'inv_s': ginv}, cot, vol, m, o, d, nrm, aabb, 12.0, S, moved, jitter=jitter,
                        color_dims=3, bkgd_rand=bk, chunk=5)


def _random_bkgd_scene(n_feat=7):
    """Small analytic scene with 3 colour + (n_feat - 3) semantic channels, 2 cameras x 3 x 4 rays, one background row per ray."""
    m, aabb = _map(10, 6)
    g = torch.Generator().manual_seed(3)
    sdf = synth.analytic_sdf_volume(m, ground_z=-1.0, spheres=((3., 5., 0., 1.5),), boxes=(), noise=0.05, seed=1)
    vol = torch.cat([sdf[None], 2.5 * torch.randn(n_feat, *sdf.shape, generator=g)], 0).double()
    _, i2l = synth.camera_rig(synth.NUSC_YAWS[:2], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    origin, direction = orays.img2lidar_rays(torch.tensor(i2l, dtype=torch.float32)[None], orays.fixed_ray_grid([3, 4], [90, 160]))
    bk = torch.rand(origin.shape[1] * direction.shape[2], 3, generator=g, dtype=torch.float64)
    return m, aabb, vol, origin, direction, bk


def test_render_parity_passes_the_oracle_itself_and_gates_max_depth_rgb_and_semantics():
    """oracle/parity.py on the fp64 oracle's own outputs, its grid as the probe, random background: every comparison is at
    rounding level and the report is ok.  Each planted error in max_depth, in rgb (the background of the next ray) and in
    one semantic channel fails the report."""
    from oracle.parity import render_parity
    m, aabb, vol, origin, direction, bk = _random_bkgd_scene()
    S, inv_s = 32, 12.0
    kw = dict(color_dims=7, bkgd='random', bkgd_rand=bk)
    ref = orender.head_render_ref(vol, m, origin.double(), direction.double(), aabb, inv_s, S=S, **kw)
    n = bk.shape[0]
    got = dict(depth=ref['depth'].reshape(n), acc=ref['acc'].reshape(n), max_idx=ref['max_idx'].reshape(n),
               max_depth=ref['max_depth'].reshape(n), grid=ref['grid'].reshape(n, S, 3), rgb=ref['rgb'].reshape(n, 3),
               normal_vis=ref['vis_normal'].reshape(n, 3), sem=ref['sem'].reshape(n, -1))
    assert got['sem'].shape == (n, 4) and (ref['acc'] < 0.5).any()
    rep = render_parity(got, vol, m, origin, direction, aabb, inv_s, S, **kw)
    print(rep)
    b = rep['same_cells']
    assert rep['ok'] and rep['geometry']['max_abs_grid_units'] == 0 and rep['independent']['rays_with_cell_flip'] == 0
    for k in ('depth_max_rel', 'acc_max_abs', 'max_depth_max_rel', 'normal_max_abs', 'rgb_max_abs', 'sem_max_abs'):
        assert b[k] < 1e-12, (k, b[k])
    low = (ref['acc'].reshape(n) < 0.5).nonzero()[0, 0]
    bad_bk = got['rgb'].clone()
    bad_bk[low] += (bk[(low + 1) % n] - bk[low]) * (1 - got['acc'][low])
    for k, v in (('max_depth', got['max_depth'] * (1 + 2e-5)), ('rgb', bad_bk), ('sem', got['sem'] + 2e-4 * (torch.arange(4) == 2))):
        assert not render_parity(dict(got, **{k: v}), vol, m, origin, direction, aabb, inv_s, S, **kw)['ok'], k


def test_chunked_random_background_render_equals_the_per_chunk_restatement():
    """head_render_ref with batch > 0 hands every chunk the background rows of its own rays (torch.chunk sizes)."""
    m, aabb, vol, origin, direction, bk = _random_bkgd_scene()
    S, inv_s, batch = 32, 12.0, 7
    out = orender.head_render_ref(vol, m, origin.double(), direction.double(), aabb, inv_s, batch=batch, S=S, color_dims=7,
                                  bkgd='random', bkgd_rand=bk)
    o, d, nrm = orays.flatten_rays(origin.double(), direction.double())
    n = orays.num_chunks(o.shape[0], batch)
    assert n == 4
    parts = [orender.neus_render_chunk(vol, m, oc, dc, nc, aabb, inv_s, S=S, color_dims=7, bkgd='random', bkgd_rand=bc)
             for oc, dc, nc, bc in zip(torch.chunk(o, n), torch.chunk(d, n), torch.chunk(nrm, n), torch.chunk(bk, n))]
    for k, pk in (('rgb', 'rgb'), ('depth', 'depth'), ('sem', 'sem')):
        assert torch.equal(out[k].reshape(o.shape[0], -1), torch.cat([p[pk] for p in parts]).reshape(o.shape[0], -1)), k


def test_slabwise_decode_equals_the_whole_volume_oracle_and_its_autograd():
    """oracle/decode_parity.py restates tpv_decode_ref slab by slab (ragged last slab, H != W): same volume, same gradients
    of every plane and MLP tensor, fp64, 1e-12; and its per-slice and per-bucket error reports on planted errors."""
    from oracle import decode_parity as dp
    g = torch.Generator().manual_seed(5)
    H, W, Z, C, n_out = 11, 6, 5, 32, 4
    planes = [torch.randn(n, C, generator=g, dtype=torch.float64) for n in (H * W, Z * H, W * Z)]
    mlp = [t.double() for t in synth.random_mlp(C, n_out, seed=5)]
    cot = torch.randn(H, W, Z, n_out, generator=g, dtype=torch.float64)
    ins = [t.clone().requires_grad_(True) for t in (*planes, *mlp)]
    ref = orender.tpv_decode_ref(*ins[:3], (H, W, Z), *ins[3:]).permute(1, 2, 3, 0)       # [H, W, Z, n_out]
    gref = torch.autograd.grad((ref * cot).sum(), ins)
    for slab in (3, 4, 11, 32):
        vol = dp.decode_slabwise(*planes, (H, W, Z), *mlp, slab=slab)
        assert vol.shape == ref.shape and (vol - ref.detach()).abs().max() < 1e-12
        grads, b1_mass = dp.decode_grads_slabwise(*planes, (H, W, Z), *mlp, cot, slab=slab)
        for name, a, b in zip(dp.GRAD_NAMES, grads, gref):
            assert a.shape == b.shape and (a - b).abs().max() < 1e-12 * max(1.0, b.abs().max().item()), (slab, name)
        # the un-cancelled sum behind d/d b1: the same gradient with every voxel's term taken positive
        assert (b1_mass >= gref[4].abs() * (1 - 1e-12)).all() and b1_mass.max() > 3 * gref[4].abs().max()
    f = dp.preactivation(*planes, (H, W, Z), 2, 5)
    assert f.shape == (3, W, Z, C)
    assert f[1, 4, 3, 7] == planes[0].view(H, W, C)[3, 4, 7] + planes[1].view(Z, H, C)[3, 3, 7] + planes[2].view(W, Z, C)[4, 3, 7]
    # slice_errors: an error planted in one small column is invisible relative to the tensor's max-abs, not to its own slice
    w = torch.ones(4, 3, dtype=torch.float64)
    w[:, 1] = 1e-6
    bad = w.clone()
    bad[2, 1] = 2e-6
    assert (bad - w).abs().max() / w.abs().max() < 1e-5
    assert dp.slice_errors(bad, w, 1).tolist() == [0.0, 1.0, 0.0]
    assert dp.slice_errors(torch.ones(3, dtype=torch.float64), torch.tensor([2.0, 0.0, 1.0], dtype=torch.float64), 0).tolist() == [0.5, 0.0, 0.0]
    # bucket_errors: the relative error is taken per element, inside the bucket of its pre-activation
    pre = torch.tensor([-13.0, -9.0, -9.5, 1.0, 25.0], dtype=torch.float64)
    val = torch.nn.functional.softplus(pre)
    rows = dp.bucket_errors(val * torch.tensor([1.5, 1.0, 1.01, 1.0, 1.0], dtype=torch.float64), val, pre)
    assert [r[0] for r in rows] == [0, 1, 2, 0, 0, 1, 1]
    assert abs(rows[1][2] - 0.5) < 1e-12 and abs(rows[2][2] - 0.01) < 1e-12 and rows[5][2] == 0 and rows[6][1] == 0
