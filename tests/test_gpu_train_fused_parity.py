"""GPU parity of the training render with the objective fused in (ops.RenderTrainObjectiveFunction:
so_render_train_objective_forward / _backward) against the fp64 composition of oracle/train_objective.py -- the chunked
training render, the reprojection statistics (oracle/reproj.py) and the eikonal mean (oracle/losses.py) -- forward and
backward, with the three-part rule of oracle/train_parity.py.

Cotangents are random on every output and zero on rays with a cell flip; the reproj_stats cotangent is also zero on rays
with a sample in the reprojection guard band (oracle.train_objective.reproj_guard_rays).  kappa is measured on each case
from the per-sample tensors of the plain training render of the same launch (RenderTrainFunction: the same kernels with
the objective off; its per-ray outputs must equal the fused launch's bit for bit).

Each case names the kernel instantiation it runs, from the dispatch of render_train.cu (render_train_forward_obj /
render_train_backward_obj): fwd5<HAS_RGB, PAIR, ZP, WZP, OBJ> (ZP, WZP = 32, 257 * 32: the constant-pitch build for
zpitch 32 and W 257; 0, 0: the generic pitch), fwd<HAS_RGB, SEM, FAST, OBJ> and bwd<HAS_RGB, SEM, FAST, OBJ>, with OBJ one of
kObjNoReproj (eikonal only), kObjCombine, kObjMultiNew."""
import json
import math
import os
import sys

import pytest
import torch

from selfocc_b200 import synth
from selfocc_b200.mapping import GridMeterMapping

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_gpu_train_parity import CFGS, INV_S, S_SHIPPED, _check_probe_against_forward, _f32, _small, _volume  # noqa: E402

LOSS_CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))
OBJ_NAME = {None: 'kObjNoReproj', 'combine': 'kObjCombine', 'multi_new': 'kObjMultiNew'}


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


# ---- geometry -------------------------------------------------------------------------------------------------------------
def _rig(kind, img_size, n_cam=2, miss=False, blind_last=False):
    """(img2lidar, img2prevImg, img2nextImg) fp32 [N,4,4] of the cameras and their temporal neighbours (synth.temporal_rig:
    0.5 m and 1 degree of ego motion).  miss: a third camera 10 m above the small box looking at the horizon.  blind_last:
    the last camera's neighbour matrices shifted by 1.5 / 0.4 of the image along x / y (as tests/test_gpu_reproj_loss.py):
    its bottom rays have no valid sample in the next frame; the previous frame sees none of its samples."""
    h, w = img_size
    if kind == 'nusc':
        rigs = [(synth.NUSC_YAWS, dict(f=1266.0 * w / 1600, cx=w / 2, cy=h / 2))]
    elif kind == 'kitti':
        rigs = [((0.,), dict(f=721.5, cx=w / 2, cy=h / 2, height=1.65, radius=0.0))]
    else:
        rigs = [(synth.NUSC_YAWS[:n_cam], dict(f=126.6, cx=80., cy=45., height=0.5, radius=0.2))]
        if miss:
            rigs.append(((90.,), dict(f=126.6, cx=80., cy=45., height=10.0, radius=0.2)))
    mats = [[], [], []]
    for yaws, kw in rigs:
        _, i2l = synth.camera_rig(yaws, **kw)
        prev, nxt = synth.temporal_rig(yaws, **kw)
        for lst, a in zip(mats, (i2l, prev, nxt)):
            lst.append(torch.tensor(a, dtype=torch.float64))
    i2l, prev, nxt = (torch.cat(x) for x in mats)
    if blind_last:
        prev[-1, 0] += 1.5 * w * prev[-1, 2]
        nxt[-1, 1] += 0.4 * h * nxt[-1, 2]
    return i2l.float(), prev.float(), nxt.float()


def _shipped_geo(cfg_name, stride, scene, n_feat):
    """A shipped config's mapping, ROI, rig (loss img_size = the head's ray_img_size), strided ray grid and volume."""
    from oracle import rays as orays
    from oracle.mapping import GridMeterMappingRef
    head = CFGS[cfg_name]['head']
    margs, aabb = head['mapping_args'], head['roi_aabb']
    i2l, prev, nxt = _rig('nusc' if cfg_name.startswith('nuscenes') else 'kitti', head['ray_img_size'])
    pix = orays.fixed_ray_grid(head['ray_number'], head['ray_img_size'])[::stride].contiguous()
    m = GridMeterMapping(**margs)
    sdf, feat = _volume(m, n_feat, scene)
    ih, iw = (96, 200) if cfg_name.startswith('nuscenes') else (88, 304)
    return dict(m=m, mref=GridMeterMappingRef(**margs), aabb=aabb, sdf=sdf, feat=feat, i2l=i2l, prev=prev, nxt=nxt, pix=pix,
                img_size=tuple(head['ray_img_size']), img_hw=(ih, iw))


def _small_geo(kind, n_feat, miss=False, blind_last=False):
    """The small edge geometries of tests/test_gpu_train_parity.py (H != W or the ring mapping, 2 cameras, 5 x 7 rays of a
    90 x 160 image) with 3 or 24 feature channels or none."""
    from oracle import rays as orays
    from oracle.mapping import GridMeterMappingRef
    margs, aabb = _small(kind)
    m = GridMeterMapping(**margs)
    sdf = synth.analytic_sdf_volume(m, ground_z=-1.0, spheres=((3., 5., 0., 1.5),), boxes=(), noise=0.05, seed=1)
    feat = torch.randn(n_feat, *sdf.shape, generator=torch.Generator().manual_seed(4)) if n_feat else None
    i2l, prev, nxt = _rig('small', (90, 160), miss=miss, blind_last=blind_last)
    return dict(m=m, mref=GridMeterMappingRef(**margs), aabb=aabb, sdf=sdf, feat=feat, i2l=i2l, prev=prev, nxt=nxt,
                pix=orays.fixed_ray_grid([5, 7], [90, 160]), img_size=(90, 160), img_hw=(30, 54))


def _objective(geo, mode, eikonal, dev, loss_pix=None, seed=5):
    ob = dict(mode=mode, eikonal=eikonal)
    if mode is not None:
        n_cam = geo['i2l'].shape[0]
        imgs = synth.textured_images(3 * n_cam, *geo['img_hw'], seed=seed).reshape(3, n_cam, 3, *geo['img_hw']).to(dev)
        lp = geo['pix'] if loss_pix is None else loss_pix
        ob.update(pix=lp.float().contiguous().to(dev), img2prev=geo['prev'].to(dev).contiguous(),
                  img2next=geo['nxt'].to(dev).contiguous(), images=tuple(imgs[i].contiguous() for i in range(3)),
                  img_size=geo['img_size'])
    return ob


# ---- one case -------------------------------------------------------------------------------------------------------------
def _launch(geo, ob, S, inv_s, jit, bk, ray_begin=0, ray_count=None, zpair=True):
    """RenderTrainObjectiveFunction on the geometry -> (outputs dict, leaves (vs, vf, invs), cfg)."""
    from selfocc_b200 import ops
    dev = _dev()
    feat = geo['feat']
    n_feat = 0 if feat is None else feat.shape[0]
    n_cam, n_pix = geo['i2l'].shape[0], geo['pix'].shape[0]
    n = n_cam * n_pix - ray_begin if ray_count is None else ray_count
    desc = geo['m'].volume_desc(n_feat)
    vs = synth.pack_sdf_volume(geo['sdf'], desc.zpitch).to(dev).requires_grad_(True)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev).requires_grad_(True) if n_feat else None
    invs = torch.tensor([inv_s], device=dev, requires_grad=True)
    want = ['depth', 'acc', 'fars', 'max_depth', 'ts', 'deltas'] + (['rgb'] if n_feat >= 3 else []) + (['sem'] if n_feat > 3 else [])
    cfg = dict(desc=desc, cam_mats=geo['i2l'].to(dev), rays=ops.make_ray_desc(n_cam, n_pix=n_pix, ray_begin=ray_begin, ray_count=n),
               params=ops.make_render_params(geo['aabb'], S, inv_s, training=True, bkgd='random'), pix=geo['pix'].to(dev),
               want=want, jitter=jit.to(dev), bkgd_rand=None if bk is None else bk.to(dev), zpair=zpair)
    res = dict(zip(ops.RenderTrainObjectiveFunction.ORDER, ops.RenderTrainObjectiveFunction.apply(vs, vf, invs, dict(cfg, objective=ob))))
    return res, (vs, vf, invs), cfg


# Guard rays may be 1 % of a case, ten times the 0.1 % of tests/test_gpu_reproj_loss.py's head test: a ray here reprojects
# 2 x 256 samples (there 2 x 32), so it meets the guard band about 16 times as often.  Measured on the H100: at most 19 of
# 2090 rays (KITTI occ at e^6.5, 0.91 %), 13 of 1920 on nuScenes (0.68 %), 1 of 480 on the matrix's nuScenes volume and
# none on the small geometries.
def _run_case(geo, inv_s, S, mode, eikonal=True, seed=0, ray_begin=0, ray_count=None, zpair=True, loss_pix=None, tag='',
              max_flip_frac=0.02, max_guard_frac=0.01):
    """Fused forward + backward with flip- and guard-masked random cotangents, the plain render's per-sample tensors, the
    probe, then the fp64 report of oracle.train_objective.objective_parity -> (report, outputs, d/d inv_s, flip rays)."""
    dev = _dev()
    from oracle import rays as orays, train_parity as tp, train_objective as tob
    from selfocc_b200 import ops
    g = torch.Generator().manual_seed(seed + 7)
    feat = geo['feat']
    n_feat = 0 if feat is None else feat.shape[0]
    n_cam, n_pix = geo['i2l'].shape[0], geo['pix'].shape[0]
    total = n_cam * n_pix
    n = total - ray_begin if ray_count is None else ray_count
    sl = slice(ray_begin, ray_begin + n)
    inv_s = _f32(inv_s)
    jit = torch.rand(total, S + 1, generator=g)
    bk = torch.rand(n, 3, generator=g) if n_feat else None
    ob = _objective(geo, mode, eikonal, dev, loss_pix, seed=seed + 5)
    res, (vs, vf, invs), cfg = _launch(geo, ob, S, inv_s, jit, bk, ray_begin, ray_count, zpair)
    # the plain training render of the same launch: per-ray outputs bit-identical, per-sample tensors for kappa
    plain_want = cfg['want'] + ['weights', 'eik_grad', 'sample_sdf']
    plain = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(
        vs.detach(), None if vf is None else vf.detach(), invs.detach(), dict(cfg, want=plain_want))))
    for k in cfg['want']:
        assert torch.equal(res[k], plain[k]), k
    gf = ops.render_train_probe(cfg['desc'], cfg['cam_mats'], cfg['rays'], cfg['params'], pix=cfg['pix'], jitter=cfg['jitter'])
    origin, direction = orays.img2lidar_rays(geo['i2l'][None], geo['pix'])
    o, d, nrm = (t.to(dev)[sl] for t in orays.flatten_rays(origin.double(), direction.double()))
    _check_probe_against_forward(geo['m'], gf, plain, o, d, nrm)
    j64 = jit[sl].double().to(dev)
    g64, _ = tp.sample_geometry(geo['mref'], o, d, geo['aabb'], S, j64)
    flip = tp.flip_rays(gf, g64)
    cam = (torch.arange(total, device=dev) // n_pix)[sl]
    lp = (geo['pix'] if loss_pix is None else loss_pix).double().to(dev).repeat(n_cam, 1)[sl]
    obj64 = dict(mode=mode, eikonal=eikonal)
    guard = torch.zeros(n, dtype=torch.bool, device=dev)
    if mode is not None:
        obj64.update(images=tuple(t.double() for t in ob['images']), img2prev=ob['img2prev'].double(),
                     img2next=ob['img2next'].double(), img_size=geo['img_size'], cam=cam, pix=lp)
        guard = tob.reproj_guard_rays(res['ts'], cam, lp, obj64['img2prev'], obj64['img2next'], geo['img_size'])
    cot = {k: torch.randn(res[k].shape, generator=g).to(dev) for k in ('depth', 'acc', 'rgb', 'sem') if k in cfg['want']}
    # depth = sum w mid / acc: on a ray that hits nothing acc is the S * 1e-5 of alpha's leak term, and d depth / d w = (mid -
    # depth) / acc turns the ~1e-7 absolute fp32 error of the leak weights (fast logistics, 1 - pa) into a gradient error that
    # no relative bar on the volume gradient absorbs (measured on the H100: 2 % of a voxel's gradient on the small volume's
    # far faces at S = 128).  The depth cotangent is scaled by the ray's acc on both sides, which takes out the 1 / acc;
    # tests/test_gpu_train_parity.py gates the plain depth cotangent, where unit per-sample cotangents set the scale
    cot['depth'] *= res['acc'].detach()
    if mode is not None:
        cot['reproj_stats'] = torch.randn(res['reproj_stats'].shape, generator=g).to(dev)
        cot['reproj_stats'][guard] = 0
    if eikonal:
        cot['eikonal_mean'] = torch.tensor(0.7, device=dev)
    for k, t in cot.items():
        if t.dim():
            t[flip] = 0
    torch.autograd.backward([res[k] for k in cot], [cot[k] for k in cot])
    gvol = vs.grad[..., :geo['m'].size_d][None]
    if n_feat:
        gvol = torch.cat([gvol, vf.grad[..., :n_feat].permute(3, 0, 1, 2)], 0)
    got = {k: res[k].detach() for k in cfg['want'] + [k for k in ('reproj_stats', 'reproj_colours', 'eikonal_mean') if res[k].numel()]}
    got.update({k: plain[k] for k in ('weights', 'eik_grad', 'sample_sdf')})
    vol64 = (geo['sdf'][None] if feat is None else torch.cat([geo['sdf'][None], feat], 0)).double().to(dev)
    rep = tob.objective_parity(got, {'vol': gvol, 'inv_s': invs.grad.item()}, {k: c.double() for k, c in cot.items()}, vol64,
                               geo['mref'], o, d, nrm, geo['aabb'], inv_s, S, gf, obj64, jitter=j64,
                               color_dims=3 if n_feat else 0, bkgd_rand=None if bk is None else bk.double().to(dev),
                               max_flip_frac=max_flip_frac, max_guard_frac=max_guard_frac)
    print(tob.format_report(tag, rep))
    return rep, res, invs.grad.clone(), flip


# ---- shipped geometry -----------------------------------------------------------------------------------------------------
# config -> (decoded feature channels besides sdf, ray stride into the config's fixed ray grid, instantiation run)
SHIPPED = {
    'nuscenes/nuscenes_occ.py': (24, 15, 'fwd<true, 24, true, kObjCombine>, bwd<true, 24, true, kObjCombine>'),
    'nuscenes/nuscenes_novel_depth.py': (3, 15, 'fwd5<true, true, 32, 257 * 32, kObjCombine>, bwd<true, 0, true, kObjCombine>'),
    'nuscenes/nuscenes_depth.py': (0, 15, 'fwd5<false, true, 32, 257 * 32, kObjCombine>, bwd<false, 0, true, kObjCombine>'),
    'kitti/kitti_occ.py': (3, 5, 'fwd5<true, true, 0, 0, kObjMultiNew>, bwd<true, 0, true, kObjMultiNew>'),
    'kitti/kitti_novel_depth.py': (3, 5, 'fwd5<true, true, 0, 0, kObjMultiNew>, bwd<true, 0, true, kObjMultiNew>'),
    'kitti_raw/kitti_raw_depth.py': (0, 3, 'fwd5<false, true, 0, 0, kObjMultiNew>, bwd<false, 0, true, kObjMultiNew>'),
}


def _shipped_objective(cfg_name):
    cfgs = LOSS_CFGS[cfg_name]['loss_cfgs']
    reproj = next(c for c in cfgs if c['type'].startswith('ReprojLoss'))
    mode = 'combine' if reproj['type'] == 'ReprojLossMonoMultiNewCombine' else 'multi_new'
    return mode, any(c['type'] == 'EikonalLoss' for c in cfgs), reproj


@pytest.mark.parametrize('scene', ['analytic', 'planes'])
@pytest.mark.parametrize('cfg_name', list(SHIPPED))
def test_fused_objective_parity_at_shipped_geometry(cfg_name, scene):
    """Every shipped objective on its config's volume, channel count, rig and loss image size, at S = 256 with jitter and
    a random background, on a strided subset of the ray grid, at three sharpnesses."""
    n_feat, stride, inst = SHIPPED[cfg_name]
    mode, eikonal, reproj = _shipped_objective(cfg_name)
    geo = _shipped_geo(cfg_name, stride, scene, n_feat)
    assert tuple(reproj['img_size']) == geo['img_size']
    # KITTI's grid has 5 cells per metre along h and w: twice the flip rays of nuScenes (tests/test_gpu_train_parity.py)
    flip_frac = 0.04 if cfg_name.startswith('kitti') else 0.02
    reps = []
    for i, inv_s in enumerate(INV_S):
        rep, res, _, _ = _run_case(geo, inv_s, S_SHIPPED, mode, eikonal, seed=i, tag='%s/%s %s' % (cfg_name, scene, inst),
                                max_flip_frac=flip_frac)
        reps.append(rep)
        # the geometry exercises the reprojection: valid and invalid directions (nuScenes: 2 rays whose samples all leave
        # both neighbour frames; KITTI: about 110 of 2090 x 2 directions), weight on the valid samples
        anys = res['reproj_stats'][:, 5::6]
        print('%s/%s: directions without a valid sample %d of %d' % (cfg_name, scene, int((anys == 0).sum()), anys.numel()))
        assert (anys == 1).float().mean().item() > 0.1 and (anys == 0).any() and (res['reproj_stats'][:, 0] > 0.1).any()
    assert all(r['ok'] for r in reps)


# ---- instantiation matrix -------------------------------------------------------------------------------------------------
# path -> (geometry, feature channels, forced switch, zpair, the instantiations it runs for OBJ)
PATHS = {
    'fwd5_const_pitch_pair_rgb': ('nusc', 3, None, True, 'fwd5<true, true, 32, 257 * 32, OBJ>, bwd<true, 0, true, OBJ>'),
    'fwd5_const_pitch_nopair_depth': ('nusc', 0, None, False, 'fwd5<false, false, 32, 257 * 32, OBJ>, bwd<false, 0, true, OBJ>'),
    'fwd5_generic_pitch_pair_depth': ('h_ne_w', 0, None, True, 'fwd5<false, true, 0, 0, OBJ>, bwd<false, 0, true, OBJ>'),
    'fwd5_generic_pitch_nopair_rgb': ('h_ne_w', 3, None, False, 'fwd5<true, false, 0, 0, OBJ>, bwd<true, 0, true, OBJ>'),
    'fwd_sem24_fast': ('h_ne_w', 24, None, True, 'fwd<true, 24, true, OBJ>, bwd<true, 24, true, OBJ>'),
    'fwd_sem_generic_fast': ('h_ne_w', 24, 'sem_generic', True, 'fwd<true, 1, true, OBJ>, bwd<true, 1, true, OBJ>'),
    'fwd_rgb_fast': ('h_ne_w', 3, 'fwd32', True, 'fwd<true, 0, true, OBJ>, bwd<true, 0, true, OBJ>'),
    'fwd_depth_fast': ('h_ne_w', 0, 'fwd32', True, 'fwd<false, 0, true, OBJ>, bwd<false, 0, true, OBJ>'),
    'fwd_sem24_ring': ('ring', 24, None, True, 'fwd<true, 24, false, OBJ>, bwd<true, 24, false, OBJ>'),
    'fwd_sem_generic_ring': ('ring', 24, 'sem_generic', True, 'fwd<true, 1, false, OBJ>, bwd<true, 1, false, OBJ>'),
    'fwd_rgb_ring': ('ring', 3, None, True, 'fwd<true, 0, false, OBJ>, bwd<true, 0, false, OBJ>'),
    'fwd_depth_ring': ('ring', 0, None, True, 'fwd<false, 0, false, OBJ>, bwd<false, 0, false, OBJ>'),
}
# objective -> (mode, eikonal): every OBJ value, and the eikonal term off once
OBJECTIVES = {'eikonal_only': (None, True), 'combine': ('combine', True), 'multi_new_without_eikonal': ('multi_new', False)}


@pytest.mark.parametrize('objective', list(OBJECTIVES))
@pytest.mark.parametrize('path', list(PATHS))
def test_fused_objective_parity_on_every_kernel_instantiation(path, objective):
    """Every OBJ value through every forward family (fwd5 with and without colour, z-pair and constant pitch; fwd with
    SEM 0 / 1 / 24, affine and ring mapping) and the backward, reached through so_render_train_force_fwd32,
    so_render_train_force_sem_generic, zpair=False and the ring mapping."""
    _dev()
    from selfocc_b200 import _lib
    kind, n_feat, force, zpair, inst = PATHS[path]
    mode, eikonal = OBJECTIVES[objective]
    if kind == 'nusc':      # the nuScenes novel-depth volume (zpitch 32, W 257) on every 60th ray
        geo, S = _shipped_geo('nuscenes/nuscenes_novel_depth.py', 60, 'analytic', n_feat), S_SHIPPED
    else:                   # S = 128: the batched forward applies on the affine map (S / 32 a multiple of its 4 chunks)
        geo, S = _small_geo(kind, n_feat), 128 if kind == 'h_ne_w' else 64
    lib = _lib.load()
    hook = {'fwd32': lib.so_render_train_force_fwd32, 'sem_generic': lib.so_render_train_force_sem_generic}.get(force)
    try:
        if hook:
            hook(1)
        rep, _, _, _ = _run_case(geo, 20.0, S, mode, eikonal, zpair=zpair, tag='%s %s' % (path, inst.replace('OBJ', OBJ_NAME[mode])))
    finally:
        if hook:
            hook(0)
    assert rep['ok']


# ---- edge rays ------------------------------------------------------------------------------------------------------------
def _edge_loss_pix(pix, img_size):
    """Loss pixels on the image bounds: u = 0, W - 1, W and v = 0, H on the first rays of every camera."""
    h, w = img_size
    lp = pix.clone()
    lp[0, 0], lp[1, 0], lp[2, 0], lp[3, 1], lp[4, 1] = 0.0, w - 1.0, float(w), 0.0, float(h)
    return lp


# the window of masked weight sums W for the `flat` case: well inside (0, eps), away from both ends by a factor of 3, so that
# fp32 and fp64 take the same branch and the backward's g / eps carries a weight the comparison can see
FLAT_W = (3e-9, 4e-8)


def _flat_loss_pix(geo, S, inv_s, seed=0):
    """Loss pixels for the `flat` backward (ObjBwd: W < eps with valid samples, d loss / d w = g / eps (x - 0)): with the loss
    pixel near the image's left or right edge, the next frame's 0.5 m of forward motion moves a ray's near samples out of
    the image and keeps its far ones, so its valid samples start at a depth t* that grows as the pixel nears the edge.  For
    every pixel of the grid, the u (v kept) at which the fp64 oracle's next-frame W of some camera's ray falls in FLAT_W:
    all of that ray's valid samples lie past its surface, where the transmittance is ~1e-8.  Pixels without one keep u."""
    from oracle import rays as orays, render as orender, train_parity as tp
    dev = _dev()
    g = torch.Generator().manual_seed(seed + 7)          # the jitter _run_case draws for this seed
    n_cam, n_pix = geo['i2l'].shape[0], geo['pix'].shape[0]
    jit = torch.rand(n_cam * n_pix, S + 1, generator=g).double().to(dev)
    origin, direction = orays.img2lidar_rays(geo['i2l'][None], geo['pix'])
    o, d, nrm = (t.to(dev) for t in orays.flatten_rays(origin.double(), direction.double()))
    _, clip = tp.sample_geometry(geo['mref'], o, d, geo['aabb'], S, jit)
    vol = geo['sdf'][None].double().to(dev)
    r = orender.neus_render_chunk(vol, geo['mref'], o, d, nrm, geo['aabb'], torch.tensor(_f32(inv_s), dtype=torch.float64), S=S,
                                  training=True, jitter=jit, depth_clip=clip)
    w, t = r['weights'].reshape(n_cam, n_pix, 1, S), ((r['starts'] + r['ends']) / 2 / nrm).reshape(n_cam, n_pix, 1, S)
    h, wd = geo['img_size']
    us = torch.cat([torch.linspace(0.05, 24.0, 480), torch.linspace(wd - 24.0, wd - 0.05, 480)]).double().to(dev)
    shape = (n_cam, n_pix, len(us), S)
    u = us[None, None, :, None].expand(shape)
    v = geo['pix'][:, 1].double().to(dev)[None, :, None, None].expand(shape)
    tt = t.expand(shape)
    c = torch.stack([u * tt, v * tt, tt, torch.ones_like(tt)], -1)          # (u t, v t, t, 1) per camera, pixel, u, sample
    q = torch.einsum('nij,npusj->npusi', geo['nxt'].double().to(dev), c)
    z = q[..., 2]
    x, y = q[..., 0] / z.clamp_min(1e-5), q[..., 1] / z.clamp_min(1e-5)
    valid = (z > 0) & (x > 0) & (x < wd) & (y > 0) & (y < h)
    W = (w * valid).sum(-1)                                                  # [n_cam, n_pix, U]
    ok = ((W > FLAT_W[0]) & (W < FLAT_W[1])).any(0)                          # [n_pix, U]
    lp = geo['pix'].clone()
    for i in ok.any(-1).nonzero()[:, 0].tolist():
        lp[i, 0] = float(us[ok[i].nonzero()[0, 0]])
    return lp


@pytest.mark.parametrize('mode', ['combine', 'multi_new'])
@pytest.mark.parametrize('case', ['rays1', 'rays3', 'rays5', 'rays33', 'miss_aabb', 'loss_pix_on_bounds', 'no_valid_sample', 'flat'])
def test_fused_objective_parity_on_edge_rays(case, mode):
    """Ray-count tails of the batched forward (a partial batch of 4 rays and of a warp), the camera whose rays miss the
    AABB (zero-length samples), loss pixels on the image bounds, a camera whose neighbour frames see none of some rays'
    samples (any = 0, W = 0: the `flat` backward, with no sample for it to act on), and directions whose only valid
    samples lie behind the surface (0 < W < eps with valid samples: the `flat` backward's g / eps and zero mean act)."""
    _dev()
    geo = _small_geo('h_ne_w', 3, miss=case == 'miss_aabb', blind_last=case == 'no_valid_sample')
    S, kw = 64, {}
    if case.startswith('rays'):         # fwd5<true, true, 0, 0, OBJ> with batch and warp tails
        S, kw = 128, dict(ray_begin=3, ray_count=int(case[4:]))
    if case == 'miss_aabb':             # the missing camera's zero-length samples sit on the AABB face: its rays may flip cells
        kw = dict(max_flip_frac=1.0 / 3.0)
    if case == 'loss_pix_on_bounds':
        kw = dict(loss_pix=_edge_loss_pix(geo['pix'], geo['img_size']))
    for i, inv_s in enumerate((12.0, INV_S[1], INV_S[2]) if case == 'flat' else (12.0, INV_S[2])):
        if case == 'flat':
            kw = dict(loss_pix=_flat_loss_pix(geo, S, inv_s, seed=i), seed=i)
        rep, res, _, flip = _run_case(geo, inv_s, S, mode, tag='%s/%s' % (case, mode), **kw)
        st = res['reproj_stats']
        W, anys = st[:, 0::6], st[:, 5::6]
        sub_eps = (W > 0) & (W < 1.1920928955078125e-07) & (anys == 1)
        flat = sub_eps.any(-1)
        print('%s/%s inv_s %.4g: directions without a valid sample %d, valid with 0 < W < eps %d (W %s), on rays with a '
              'nonzero cotangent %d' % (case, mode, inv_s, int((anys == 0).sum()), int(sub_eps.sum()),
                                        ['%.2e' % x for x in W[sub_eps][:8].tolist()], int((flat & ~flip).sum())))
        if case == 'no_valid_sample':
            assert (anys == 0).any() and (anys == 1).any()
        if case == 'miss_aabb':         # the missing camera keeps rays whose cotangents are not zeroed
            n_pix = geo['pix'].shape[0]
            print('miss_aabb: missing camera flip rays %d of %d' % (int(flip[-n_pix:].sum()), n_pix))
            assert (~flip[-n_pix:]).sum() >= n_pix // 2
        if case == 'flat' and mode == 'multi_new':      # combine merges the previous frame, which sees the near samples
            assert (flat & ~flip).any()
        assert rep['ok']


# ---- ray-sharded launches and determinism ---------------------------------------------------------------------------------
@pytest.mark.parametrize('cfg_name', ['kitti/kitti_occ.py', 'nuscenes/nuscenes_novel_depth.py'])
def test_ray_sharded_fused_launches_equal_the_unsharded_launch(cfg_name):
    """ray_begin / ray_count launches with shard boundaries inside a camera: per-ray outputs and the reproj_stats /
    reproj_colours rows equal the same rows of the unsharded launch bit for bit; the shards' eikonal means weighted by their
    sample counts equal the unsharded mean within 1e-6 relative."""
    dev = _dev()
    n_feat, stride, _ = SHIPPED[cfg_name]
    mode, _, _ = _shipped_objective(cfg_name)
    geo = _shipped_geo(cfg_name, stride, 'analytic', n_feat)
    S, inv_s = S_SHIPPED, _f32(math.e ** 3)
    n_pix = geo['pix'].shape[0]
    total = geo['i2l'].shape[0] * n_pix
    g = torch.Generator().manual_seed(3)
    jit, bk = torch.rand(total, S + 1, generator=g), torch.rand(total, 3, generator=g)
    ob = _objective(geo, mode, True, dev)
    keys = ('depth', 'acc', 'fars', 'max_depth', 'rgb', 'ts', 'deltas', 'reproj_stats', 'reproj_colours')
    with torch.no_grad():
        full, _, _ = _launch(geo, ob, S, inv_s, jit, bk)
        cuts = [0, n_pix // 3 + 7, n_pix + n_pix // 2 + 1 if total > n_pix else 2 * n_pix // 3 + 1, total]
        assert all(c % n_pix for c in cuts[1:-1])                          # every boundary inside a camera
        eik = 0.0
        for b, e in zip(cuts[:-1], cuts[1:]):
            part, _, _ = _launch(geo, ob, S, inv_s, jit, bk[b:e].contiguous(), ray_begin=b, ray_count=e - b)
            for k in keys:
                assert torch.equal(part[k], full[k][b:e]), (k, b, e)
            eik += part['eikonal_mean'].double().item() * (e - b) * S
    ref = full['eikonal_mean'].double().item()
    print('%s: shards %s, weighted eikonal mean rel err %.2e' % (cfg_name, cuts, abs(eik / (total * S) - ref) / ref))
    assert abs(eik / (total * S) - ref) <= 1e-6 * abs(ref)


def test_fused_inv_s_gradient_is_bitwise_deterministic_and_within_the_parity_bar():
    """d/d inv_s is summed from the fp64 per-ray partials in ray order: a rerun gives the same bits; the first run is
    within the train-parity bar of the fp64 composition."""
    geo = _shipped_geo('nuscenes/nuscenes_novel_depth.py', 30, 'planes', 3)
    runs = [_run_case(geo, INV_S[1], S_SHIPPED, 'combine', seed=4, tag='determinism run %d' % i) for i in range(2)]
    assert torch.equal(runs[0][2], runs[1][2])
    for rep, _, _, _ in runs:
        assert rep['same_cells']['grad_inv_s'][0] <= 1.0 and rep['ok']


# ---- the objective end to end ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('cfg_name', ['nuscenes/nuscenes_novel_depth.py', 'kitti_raw/kitti_raw_depth.py'])
def test_fused_objective_loss_end_to_end_matches_the_oracle(cfg_name):
    """The full ray grid of one config per mode through the config's ReprojLoss* (SSIM and automask on) and EikonalLoss
    modules on the fused outputs, against loss_from_stats_ref on the fp64 composition at the kernel's sample coordinates
    and ts (same cells: no flip rays) plus eikonal_ref.  The loss values, and d/d volume, d/d inv_s of the
    objective's backward with d loss / d stats zeroed on guard rays and automask near-ties (relative gap < 1e-6, as
    tests/test_gpu_reproj_loss.py) on both sides.  RenderTrainObjectiveFunction is called directly and its outputs packed
    into the modules' inputs as the head's fused step packs them (head_train.py: reproj_stats / reproj_colours as
    [num_cams, R, ...], curr_imgs [1, num_cams, 3, H, W]); the head's own fused step is compared with its unfused step in
    tests/test_gpu_train_fused.py, not with the oracle."""
    dev = _dev()
    from oracle import rays as orays, reproj as oreproj, train_parity as tp, train_objective as tob
    from selfocc_b200 import ops
    from selfocc_b200.loss import EikonalLoss, ReprojLossMonoMultiNew, ReprojLossMonoMultiNewCombine
    n_feat = SHIPPED[cfg_name][0]
    mode, _, rcfg = _shipped_objective(cfg_name)
    eik_w = next(c for c in LOSS_CFGS[cfg_name]['loss_cfgs'] if c['type'] == 'EikonalLoss').get('weight', 1.0)
    geo = _shipped_geo(cfg_name, 1, 'analytic', n_feat)
    n_cam, R = geo['i2l'].shape[0], geo['pix'].shape[0]
    n, S, inv_s = n_cam * R, S_SHIPPED, _f32(math.e ** 3)
    g = torch.Generator().manual_seed(9)
    jit, bk = torch.rand(n, S + 1, generator=g), (torch.rand(n, 3, generator=g) if n_feat else None)
    ob = _objective(geo, mode, True, dev)
    res, (vs, vf, invs), cfg = _launch(geo, ob, S, inv_s, jit, bk)
    cls = ReprojLossMonoMultiNewCombine if mode == 'combine' else ReprojLossMonoMultiNew
    rl = cls(**{k: v for k, v in rcfg.items() if k != 'type'})
    el = EikonalLoss(weight=eik_w)
    stats_k = res['reproj_stats'].reshape(n_cam, R, -1)
    inputs = dict(reproj_stats=stats_k, reproj_colours=res['reproj_colours'].reshape(n_cam, R, 9),
                  curr_imgs=ob['images'][0][None], eikonal_mean=res['eikonal_mean'])
    l_rep = rl(inputs)
    loss_k = l_rep + el(inputs)
    gst_k, = torch.autograd.grad(l_rep, stats_k, retain_graph=True)        # d loss / d stats, masked below
    # the fp64 composition at the kernel's coordinates and ts: forward for the statistics, tail, then its backward
    gf = ops.render_train_probe(cfg['desc'], cfg['cam_mats'], cfg['rays'], cfg['params'], pix=cfg['pix'], jitter=cfg['jitter'])
    origin, direction = orays.img2lidar_rays(geo['i2l'][None], geo['pix'])
    o, d, nrm = (t.to(dev) for t in orays.flatten_rays(origin.double(), direction.double()))
    _, clip = tp.sample_geometry(geo['mref'], o, d, geo['aabb'], S, jit.double().to(dev))
    cam = torch.arange(n, device=dev) // R
    obj64 = dict(mode=mode, eikonal=True, images=tuple(t.double() for t in ob['images']), img2prev=ob['img2prev'].double(),
                 img2next=ob['img2next'].double(), img_size=geo['img_size'], cam=cam, pix=geo['pix'].double().to(dev).repeat(n_cam, 1),
                 ts=res['ts'].detach().double())
    vol64 = (geo['sdf'][None] if geo['feat'] is None else torch.cat([geo['sdf'][None], geo['feat']], 0)).double().to(dev)
    kw = dict(jitter=jit.double().to(dev), color_dims=3 if n_feat else 0, bkgd_rand=None if bk is None else bk.double().to(dev),
              depth_clip=clip, grid_override=gf.double())
    fwd, _, _, _ = tob.oracle_objective(vol64, geo['mref'], o, d, nrm, geo['aabb'], inv_s, S, {}, obj64, **kw)
    st_o = fwd['reproj_stats'].reshape(n_cam, R, -1).requires_grad_(True)
    l_rep_o, cands = oreproj.loss_from_stats_ref(mode, st_o, fwd['reproj_colours'].reshape(n_cam, R, 9), rcfg['ray_resize'],
                                                 rcfg.get('no_ssim', False), rcfg.get('no_automask', False))
    l_rep_o = rcfg.get('weight', 1.0) * l_rep_o
    gst_o, = torch.autograd.grad(l_rep_o, st_o)
    loss_o = l_rep_o.item() + eik_w * float(fwd["eikonal_mean"])
    srt = cands.detach().sort(dim=-1).values
    tie = (((srt[..., 1] - srt[..., 0]).abs() <= 1e-6 * srt[..., 0].abs()) & (srt[..., 0] < 1e3)).reshape(n)
    guard = tob.reproj_guard_rays(res['ts'], cam, obj64['pix'], obj64['img2prev'], obj64['img2next'], geo['img_size'])
    drop = tie | guard
    assert drop.float().mean().item() < 0.01, (int(tie.sum()), int(guard.sum()))
    gk, go = gst_k.reshape(n, -1).clone(), gst_o.reshape(n, -1).clone()
    gk[drop], go[drop] = 0, 0
    # kappa from the plain render's per-sample tensors (chunked: the full grid's per-sample tensors are large)
    plain = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(
        vs.detach(), None if vf is None else vf.detach(), invs.detach(), dict(cfg, want=['weights', 'eik_grad', 'sample_sdf', 'deltas']))))
    kappa = max(1.0, inv_s * tp.alpha_arg_error(plain, {'sample_sdf': fwd['sample_sdf'], 'eik_grad': fwd['eik_grad'],
                                                         'deltas': fwd['deltas']}, d, nrm) / tp.A0)
    del plain
    torch.autograd.backward([res['reproj_stats'], res['eikonal_mean']], [gk.float(), torch.tensor(eik_w, device=dev)])
    _, g_vol, g_inv, mass = tob.oracle_objective(vol64, geo['mref'], o, d, nrm, geo['aabb'], inv_s, S,
                                                 {'reproj_stats': go, 'eikonal_mean': torch.tensor(eik_w)}, obj64, **kw)
    e_loss = abs(loss_k.item() - loss_o) / (1e-5 * kappa * abs(loss_o))
    gs = vs.grad[..., :geo['m'].size_d].double()
    # the train-parity bars relative to each gradient's own max: d loss / d volume is ~1e-5 here, the floor of 1 would be vacuous
    e_sdf = (gs - g_vol[0]).abs().max().item() / (1e-3 * kappa * g_vol[0].abs().max().item())
    e_feat = 0.0
    if n_feat:          # no colour term in the objective: both gradients are exactly zero
        gfe = vf.grad[..., :n_feat].permute(3, 0, 1, 2).double()
        e_feat = float('inf') if gfe.abs().max().item() or g_vol[1:].abs().max().item() else 0.0
    gi, gi_o = invs.grad.item(), float(g_inv)
    e_inv = abs(gi - gi_o) / (2e-3 * kappa * abs(gi_o) + 2.0 ** -13 * mass)
    print('%s end to end (%s): rays %d kappa %.3g | loss %.6g vs %.6g | ties %d guard %d | worst ratio to bar: loss %.2g, '
          'd/d vol_sdf %.2g, d/d vol_feat %.2g, d/d inv_s %.2g (%.4g vs %.4g)' % (
              cfg_name, OBJ_NAME[mode], n, kappa, loss_k.item(), loss_o, int(tie.sum()), int(guard.sum()), e_loss, e_sdf, e_feat,
              e_inv, gi, gi_o))
    assert max(e_loss, e_sdf, e_feat, e_inv) <= 1.0
