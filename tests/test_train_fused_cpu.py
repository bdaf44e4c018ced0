"""The fused training objective off the GPU: the argument checks of so_render_train_objective_forward / _backward (every
case fails or returns before any launch: the ray count is 0), and which objectives fuse_objective accepts."""
import ctypes as C
import json
import os
from types import SimpleNamespace

import pytest

from test_render_args_cpu import ONE, _desc, _params, _rays

HERE = os.path.dirname(os.path.abspath(__file__))
CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))
INVALID, UNSUPPORTED = -1, -2


def _objective(**kw):
    from selfocc_b200 import _lib
    ob = _lib.ObjectiveDesc()
    ob.reproj_mode, ob.eikonal = 0, 1
    ob.pix = ob.img2prev = ob.img2next = ob.curr_imgs = ob.prev_imgs = ob.next_imgs = 16
    ob.img_h, ob.img_w, ob.size_h, ob.size_w = 96, 200, 768.0, 1600.0
    ob.workspace, ob.workspace_bytes = 16, 0
    for k, v in kw.items():
        setattr(ob, k, v)
    return ob


def _fwd(lib, ob=None, rd=None, pr=None, stats=ONE, colours=None, mean=ONE):
    ob = _objective() if ob is None else ob
    rd, pr = _rays(**(rd or {})), _params(**(pr or {}))
    n = None
    return lib.so_render_train_objective_forward(ONE, n, C.byref(_desc()), ONE, n, C.byref(rd), C.byref(pr), n, n,
                                                 None if ob == 'null' else C.byref(ob), n, n, n, n, n, n, n, n, n, n, n,
                                                 stats, colours, mean, ONE, n, n)


def _bwd(lib, ob=None, rd=None, pr=None, stats=ONE, g_stats=ONE, g_mean=ONE, g_inv_s=None):
    ob = _objective() if ob is None else ob
    rd, pr = _rays(**(rd or {})), _params(**(pr or {}))
    n = None
    return lib.so_render_train_objective_backward(ONE, n, C.byref(_desc()), ONE, n, C.byref(rd), C.byref(pr), n, n,
                                                  None if ob == 'null' else C.byref(ob), n, n, n, n, stats, g_stats, g_mean,
                                                  ONE, n, g_inv_s, ONE, n)


@pytest.fixture(scope='module')
def lib():
    from selfocc_b200 import _lib
    return _lib.load()


def test_valid_calls_without_rays_return_ok(lib):
    assert _fwd(lib) == 0
    assert _bwd(lib) == 0
    assert _bwd(lib, g_inv_s=ONE) == 0
    assert _fwd(lib, _objective(reproj_mode=-1), stats=None) == 0         # eikonal only
    assert _bwd(lib, _objective(reproj_mode=-1, eikonal=0), stats=None, g_stats=None, g_mean=None) == 0
    assert _fwd(lib, _objective(reproj_mode=1, eikonal=0), mean=None) == 0


@pytest.mark.parametrize('case, code', [
    (dict(ob='null'), INVALID),
    (dict(ob=dict(reproj_mode=2)), INVALID),
    (dict(ob=dict(eikonal=2)), INVALID),
    (dict(ob=dict(pix=0)), INVALID),
    (dict(ob=dict(img2next=0)), INVALID),
    (dict(ob=dict(prev_imgs=0)), INVALID),
    (dict(ob=dict(curr_imgs=18)), INVALID),                     # misaligned float operand
    (dict(ob=dict(img_h=0)), INVALID),
    (dict(ob=dict(size_w=0.0)), INVALID),
    (dict(ob=dict(size_h=float('inf'))), INVALID),
    (dict(ob=dict(img_h=50000, img_w=50000)), UNSUPPORTED),
    (dict(stats=None), INVALID),
    (dict(mean=None), INVALID),
    (dict(ob=dict(workspace=0)), INVALID),
    (dict(ob=dict(workspace=20)), INVALID),                     # not 8-byte aligned
    (dict(ob=dict(workspace_bytes=8 * 3), rd=dict(ray_count=4)), INVALID),
    (dict(pr=dict(num_samples=512)), UNSUPPORTED),              # S <= 256, the training render's bound
    (dict(pr=dict(num_samples=0)), INVALID),
    (dict(rd=dict(ray_count=5)), INVALID),                      # beyond n_cam * rays_per_cam
])
def test_forward_refuses_bad_arguments(lib, case, code):
    case = dict(case)
    if 'ob' in case and case['ob'] != 'null':
        case['ob'] = _objective(**case['ob'])
    assert _fwd(lib, **case) == code


@pytest.mark.parametrize('case, code', [
    (dict(ob='null'), INVALID),
    (dict(ob=dict(reproj_mode=-2)), INVALID),
    (dict(ob=dict(next_imgs=0)), INVALID),
    (dict(ob=dict(img_w=-1)), INVALID),
    (dict(stats=None), INVALID),
    (dict(g_stats=None), INVALID),
    (dict(g_mean=C.c_void_p(18)), INVALID),
    (dict(g_inv_s=ONE, ob=dict(workspace=0)), INVALID),         # the per-ray inv_s values need the workspace
    (dict(g_inv_s=ONE, ob=dict(workspace_bytes=8 * 3), rd=dict(ray_count=4)), INVALID),
    (dict(pr=dict(num_samples=300)), UNSUPPORTED),
])
def test_backward_refuses_bad_arguments(lib, case, code):
    case = dict(case)
    if 'ob' in case and case['ob'] != 'null':
        case['ob'] = _objective(**case['ob'])
    assert _bwd(lib, **case) == code


# ------------------------------------------------------------------------------------------------ fuse_objective
def _head(two_split=False, sample_sdf=False):
    return SimpleNamespace(two_split=two_split, img2lidar=SimpleNamespace(two_split=True), return_sample_sdf=sample_sdf,
                           fused_objective=None)


def _multiloss(cfgs):
    from selfocc_b200.loss import MultiLoss
    return MultiLoss(cfgs)


@pytest.mark.parametrize('name', sorted(CFGS))
def test_every_shipped_objective_can_be_fused(name):
    from selfocc_b200.loss import fuse_objective
    cfgs = CFGS[name]['loss_cfgs']
    head = _head()
    rec = fuse_objective(head, _multiloss(cfgs))
    reproj = next(c for c in cfgs if c['type'].startswith('ReprojLoss'))
    assert head.fused_objective is rec
    assert rec == dict(mode='combine' if reproj['type'] == 'ReprojLossMonoMultiNewCombine' else 'multi_new',
                       img_size=tuple(reproj['img_size']), eikonal=any(c['type'] == 'EikonalLoss' for c in cfgs))


R_COMBINE = dict(type='ReprojLossMonoMultiNewCombine', img_size=[768, 1600], ray_resize=[48, 100])
R_MULTI = dict(type='ReprojLossMonoMultiNew', img_size=[768, 1600], ray_resize=[48, 100])
EIK = dict(type='EikonalLoss', weight=0.1)
DEFAULT_IN = {k: k for k in ('curr_imgs', 'prev_imgs', 'next_imgs', 'ray_indices', 'weights', 'ts', 'metas', 'ms_rays')}


@pytest.mark.parametrize('cfgs, head', [
    ([R_COMBINE, R_MULTI, EIK], {}),                                                        # two reprojection terms
    ([R_COMBINE, EIK, EIK], {}),                                                            # two eikonal terms
    ([dict(R_COMBINE, input_dict=dict(DEFAULT_IN, deltas='deltas')), EIK], {}),            # deltas input
    ([dict(R_MULTI, input_dict=dict(DEFAULT_IN, weights='other_weights')), EIK], {}),      # weights from elsewhere
    ([R_COMBINE, dict(EIK, input_dict={'eik_grad': 'second_grad'})], {}),                   # eikonal of another tensor
    ([R_COMBINE, EIK, dict(type='SecondGradLoss', input_dict={'second_grad': 'eik_grad'})], {}),   # another per-sample reader
    ([R_COMBINE, EIK], dict(two_split=True)),
    ([R_COMBINE, EIK], dict(sample_sdf=True)),
])
def test_fuse_objective_refuses_unsupported_objectives(cfgs, head):
    from selfocc_b200.loss import fuse_objective
    h = _head(**head)
    with pytest.raises(NotImplementedError):
        fuse_objective(h, _multiloss(cfgs))
    assert h.fused_objective is None


def test_objective_without_per_sample_terms_fuses_to_nothing():
    from selfocc_b200.loss import fuse_objective
    assert fuse_objective(_head(), _multiloss([dict(type='SecondGradLoss')])) == dict(mode=None, img_size=None, eikonal=False)


# ------------------------------------------------------------------------------------------------ fp64 objective oracle
def _tiny_objective_scene(mode):
    """2 cameras x 4 x 3 rays x 16 samples on a small analytic volume with 3 colour channels, the temporal rig of the
    cameras and textured neighbour frames: (render args, objective, cotangents)."""
    import torch
    from oracle import rays as orays
    from oracle.mapping import GridMeterMappingRef
    from selfocc_b200 import synth
    margs, aabb = synth.small_mapping(10, 6, rng=20.0, z0=-2.0, z1=4.0)
    m = GridMeterMappingRef(**margs)
    g = torch.Generator().manual_seed(3)
    sdf = synth.analytic_sdf_volume(m, noise=0.02, seed=2)
    vol = torch.cat([sdf[None], 0.7 * torch.randn(3, *sdf.shape, generator=g)]).double()
    yaws = synth.NUSC_YAWS[:2]
    _, i2l = synth.camera_rig(yaws, f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    prev, nxt = synth.temporal_rig(yaws, f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    pix = orays.fixed_ray_grid([3, 4], [90, 160]) + 0.37
    origin, direction = orays.img2lidar_rays(torch.tensor(i2l, dtype=torch.float32)[None], pix)
    o, d, nrm = orays.flatten_rays(origin.double(), direction.double())
    n, S, R = o.shape[0], 16, pix.shape[0]
    imgs = synth.textured_images(6, 30, 50, seed=4).double().reshape(3, 2, 3, 30, 50)
    obj = dict(mode=mode, eikonal=True, images=tuple(imgs), img2prev=torch.from_numpy(prev), img2next=torch.from_numpy(nxt),
               img_size=(90, 160), cam=torch.arange(2).repeat_interleave(R), pix=pix.double().repeat(2, 1))
    sets = 1 if mode == 'combine' else 2
    cot = dict(depth=torch.randn(n, generator=g, dtype=torch.float64), acc=torch.randn(n, generator=g, dtype=torch.float64),
               rgb=torch.randn(n, 3, generator=g, dtype=torch.float64),
               reproj_stats=torch.randn(n, 6 * sets, generator=g, dtype=torch.float64), eikonal_mean=torch.tensor(0.7))
    jitter = torch.rand(n, S + 1, generator=g, dtype=torch.float64)
    bk = torch.rand(n, 3, generator=g, dtype=torch.float64)
    return dict(vol=vol, m=m, o=o, d=d, nrm=nrm, aabb=aabb, S=S, R=R, jitter=jitter, bk=bk), obj, cot


@pytest.mark.parametrize('mode', ['combine', 'multi_new'])
def test_objective_oracle_equals_render_then_statistics_then_eikonal(mode):
    """oracle.train_objective's chunked composition (chunks of 5 rays: they straddle the camera boundary) equals the
    plain fp64 render of every ray at once followed by ray_stats_ref and eikonal_ref: outputs and d/d volume, d/d inv_s."""
    import torch
    from oracle import losses as olosses, render as orender, reproj as oreproj, train_parity as tp
    from oracle.train_objective import oracle_objective
    sc, obj, cot = _tiny_objective_scene(mode)
    o, d, nrm, S, R, inv_s = sc['o'], sc['d'], sc['nrm'], sc['S'], sc['R'], 20.0
    _, clip = tp.sample_geometry(sc['m'], o, d, sc['aabb'], S, sc['jitter'])
    got, g_vol, g_inv, _ = oracle_objective(sc['vol'], sc['m'], o, d, nrm, sc['aabb'], inv_s, S, cot, obj, jitter=sc['jitter'],
                                            color_dims=3, bkgd_rand=sc['bk'], depth_clip=clip, chunk=5)
    vol = sc['vol'].clone().requires_grad_(True)
    invs = torch.tensor(inv_s, dtype=torch.float64, requires_grad=True)
    r = orender.neus_render_chunk(vol, sc['m'], o, d, nrm, sc['aabb'], invs, S=S, training=True, jitter=sc['jitter'],
                                  color_dims=3, bkgd='random', bkgd_rand=sc['bk'], differentiable=True, depth_clip=clip)
    ts = (r['starts'] + r['ends']) / 2 / nrm
    w = r['weights']
    stats, cols = oreproj.ray_stats_ref(mode, *obj['images'], list(w.reshape(2, R * S)), list(ts.reshape(2, R * S)),
                                        obj['img2prev'], obj['img2next'], obj['pix'][:R], obj['img_size'])
    eik = olosses.eikonal_ref(r['eik_grad'])
    loss = (r['depth'] * cot['depth']).sum() + (r['accumulation'] * cot['acc']).sum() + (r['rgb'] * cot['rgb']).sum() + \
        (stats.reshape(-1, stats.shape[-1]) * cot['reproj_stats']).sum() + eik * cot['eikonal_mean']
    ref_vol, ref_inv = torch.autograd.grad(loss, [vol, invs])
    assert (stats[..., 5::6] == 1).any() and (stats[..., 0] > 1e-3).any()        # the scene exercises the reprojection
    close = lambda a, b: torch.allclose(a, b.detach().reshape(a.shape), rtol=1e-10, atol=1e-12)
    assert close(got['reproj_stats'], stats) and close(got['reproj_colours'], cols)
    assert close(got['eikonal_mean'], eik) and close(got['depth'], r['depth']) and close(got['rgb'], r['rgb'])
    assert close(g_vol, ref_vol) and close(g_inv, ref_inv)
    assert ref_vol.abs().max() > 0 and ref_inv.abs() > 0
    # the valid-sample counts: the W column of the statistics at unit weights
    ones, _ = oreproj.ray_stats_ref(mode, *obj['images'], list(torch.ones(2, R * S, dtype=torch.float64)), list(ts.reshape(2, R * S)),
                                    obj['img2prev'], obj['img2next'], obj['pix'][:R], obj['img_size'])
    assert torch.equal(got['reproj_valid'], ones.reshape(2 * R, -1)[:, 0::6])


def test_reproj_guard_flags_samples_on_an_image_bound_or_at_zero_depth():
    """With img2prev = img2next = identity a sample (u t, v t, t, 1) reprojects to pixel (u, v) at depth t."""
    import torch
    from oracle.train_objective import reproj_guard_rays, GUARD_PX, GUARD_Z
    eye = torch.eye(4, dtype=torch.float64)[None]
    pix = torch.tensor([[50., 40.], [0.0, 40.], [160. - GUARD_PX / 2, 40.], [50., 90.], [50., 40.], [50., 40.], [0.01, 89.9]],
                       dtype=torch.float64)
    ts = torch.tensor([[1., 2., 3.]] * 7, dtype=torch.float64)
    ts[4, 1] = GUARD_Z / 2                  # a sample at (almost) zero depth in the other frame
    ts[5, 2] = -3.0                         # behind the other camera: invalid whatever its pixel, never ambiguous
    bad = reproj_guard_rays(ts, torch.zeros(7, dtype=torch.long), pix, eye, eye, (90, 160))
    assert bad.tolist() == [False, True, True, True, True, False, False]
