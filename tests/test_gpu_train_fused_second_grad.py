"""GPU: SecondGradLoss fused into the training render (so_objective_desc.second_grad, ops.RenderTrainObjectiveFunction's
second_grad_mean, loss.fuse_objective(..., second_grad=True)).

1. fp64 gate: the fused second_grad_mean and its gradient w.r.t. vol_sdf against oracle/second_grad.py at the kernel's own
   fp32 sample points (ops.render_train_probe), at the volume and ray geometry of the five configs that train
   SecondGradLoss, at three sharpnesses, on every OBJ value and kernel family, with edge rays, both sample anchors and
   ray-sharded launches.  Mean: 1e-6 relative (the eikonal mean's bar).  Gradient: 1e-5 of its max-abs per voxel, plus
   twice the contribution of the elements whose fp64 value is too close to 0 for fp32 to hold its sign (the oracle's
   `bound`: about 0.4 % of the elements at the shipped geometry).
2. The end-to-end step against the unfused step at nuscenes_occ's objective, sharded steps, the term switched off,
   determinism, host syncs and what forward_train no longer allocates."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from selfocc_b200 import synth
from selfocc_b200.mapping import GridMeterMapping

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_gpu_train_parity import CFGS as MODEL_CFGS, INV_S, S_SHIPPED, _f32, _volume  # noqa: E402
from test_gpu_train_fused_parity import PATHS, OBJ_NAME, _rig, _small_geo, _objective, _shipped_objective  # noqa: E402

BEV_CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_model_cfgs_bev.json')))
HEADS = dict({k: v['head'] for k, v in MODEL_CFGS.items()}, **{k: v['head'] for k, v in BEV_CFGS.items()})
# config -> (decoded feature channels besides sdf, ray stride into the config's fixed ray grid)
SG_SHIPPED = {
    'nuscenes/nuscenes_occ.py': (24, 15),
    'nuscenes/nuscenes_occ_bev.py': (24, 15),
    'nuscenes/nuscenes_novel_depth.py': (3, 15),
    'kitti/kitti_occ.py': (3, 5),
    'kitti/kitti_novel_depth.py': (3, 5),
}
G_MEAN = 0.7


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _geo(cfg_name, stride, n_feat, scene='analytic'):
    """A config's mapping, ROI, rig (loss img_size = the head's ray_img_size), strided ray grid and volume."""
    from oracle import rays as orays
    head = HEADS[cfg_name]
    i2l, prev, nxt = _rig('nusc' if cfg_name.startswith('nuscenes') else 'kitti', head['ray_img_size'])
    m = GridMeterMapping(**head['mapping_args'])
    sdf, feat = _volume(m, n_feat, scene)
    ih, iw = (96, 200) if cfg_name.startswith('nuscenes') else (88, 304)
    return dict(m=m, aabb=head['roi_aabb'], sdf=sdf, feat=feat, i2l=i2l, prev=prev, nxt=nxt,
                pix=orays.fixed_ray_grid(head['ray_number'], head['ray_img_size'])[::stride].contiguous(),
                img_size=tuple(head['ray_img_size']), img_hw=(ih, iw))


def _axes(desc):
    """(offset, size0, k0, k1) of each axis as the kernels hold them (fp32 slopes)."""
    out = []
    for a in desc.axis:
        f = lambda x: torch.tensor(x, dtype=torch.float32)
        k0 = float(f(a.size0) / f(a.range0))
        k1 = float(f(a.size1) / f(a.range1)) if a.size1 > 0 and a.range1 > 0 else 0.0
        out.append((a.offset, a.size0, k0, k1))
    return out


def _launch(geo, ob, S, inv_s, seed, ray_begin=0, ray_count=None, zpair=True, anchor_mid=True):
    """RenderTrainObjectiveFunction on the geometry -> (outputs, leaves (vs, vf, invs), cfg)."""
    from selfocc_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(seed + 7)
    feat = geo['feat']
    n_feat = 0 if feat is None else feat.shape[0]
    n_cam, n_pix = geo['i2l'].shape[0], geo['pix'].shape[0]
    n = n_cam * n_pix - ray_begin if ray_count is None else ray_count
    jit = torch.rand(n_cam * n_pix, S + 1, generator=g)
    bk = torch.rand(n, 3, generator=g) if n_feat else None
    desc = geo['m'].volume_desc(n_feat)
    vs = synth.pack_sdf_volume(geo['sdf'], desc.zpitch).to(dev).requires_grad_(True)
    vf = synth.pack_feat_volume(feat, desc.feat_pitch).to(dev).requires_grad_(True) if n_feat else None
    invs = torch.tensor([inv_s], device=dev, requires_grad=True)
    want = ['depth', 'acc', 'fars', 'max_depth'] + (['rgb'] if n_feat >= 3 else []) + (['sem'] if n_feat > 3 else [])
    cfg = dict(desc=desc, cam_mats=geo['i2l'].to(dev), rays=ops.make_ray_desc(n_cam, n_pix=n_pix, ray_begin=ray_begin, ray_count=n),
               params=ops.make_render_params(geo['aabb'], S, inv_s, training=True, bkgd='random', anchor_mid=anchor_mid),
               pix=geo['pix'].to(dev), want=want, jitter=jit.to(dev), bkgd_rand=None if bk is None else bk.to(dev), zpair=zpair)
    res = dict(zip(ops.RenderTrainObjectiveFunction.ORDER,
                   ops.RenderTrainObjectiveFunction.apply(vs, vf, invs, dict(cfg, objective=ob))))
    return res, (vs, vf, invs), cfg


def _gate(geo, S, inv_s, mode, eikonal, seed=0, tag='', **kw):
    """Fused forward, backward of G_MEAN * second_grad_mean alone, and the fp64 oracle at the probe's points -> report."""
    from oracle.second_grad import axis_slopes, second_grad_mean_ref
    from selfocc_b200 import ops
    dev = _dev()
    inv_s = _f32(inv_s)
    ob = dict(_objective(geo, mode, eikonal, dev, seed=seed + 5), second_grad=True)
    res, (vs, vf, invs), cfg = _launch(geo, ob, S, inv_s, seed, **kw)
    # the per-ray outputs are the plain training render's, bit for bit
    plain = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(
        vs.detach(), None if vf is None else vf.detach(), invs.detach(), cfg)))
    for k in cfg['want']:
        assert torch.equal(res[k], plain[k]), k
    torch.autograd.backward([res['second_grad_mean']], [torch.tensor(G_MEAN, device=dev)])
    grid = ops.render_train_probe(cfg['desc'], cfg['cam_mats'], cfg['rays'], cfg['params'], pix=cfg['pix'],
                                  jitter=cfg['jitter']).reshape(-1, 3).double()
    Z = geo['m'].size_d
    vol64 = geo['sdf'].double().to(dev)
    mean, gref, bound, n_amb = second_grad_mean_ref(vol64, grid, axis_slopes(grid, _axes(cfg['desc'])), G_MEAN)
    got_mean = res['second_grad_mean'].item()
    got_g = vs.grad[..., :Z].double()
    err = (got_g - gref).abs()
    bar = 1e-5 * gref.abs().max().item()
    worst = (err - bound).max().item()
    rel_mean = abs(got_mean - mean.item()) / mean.item()
    print('%s: mean %.6e rel err %.2e; grad max err %.2e (bar %.2e), max err beyond bound %.2e; ambiguous elements %d of %d'
          % (tag, mean.item(), rel_mean, err.max().item(), bar, worst, n_amb, grid.numel()))
    assert mean.item() > 0 and gref.abs().max().item() > 0
    assert rel_mean <= 1e-6, (tag, got_mean, mean.item())
    assert worst <= bar, tag
    assert n_amb <= 0.05 * grid.numel(), tag
    return res, vs.grad.clone(), invs.grad


@pytest.mark.parametrize('inv_s', INV_S)
@pytest.mark.parametrize('cfg_name', list(SG_SHIPPED))
def test_fused_second_grad_parity_at_shipped_geometry(cfg_name, inv_s):
    n_feat, stride = SG_SHIPPED[cfg_name]
    mode, eikonal, _ = _shipped_objective(cfg_name)
    _gate(_geo(cfg_name, stride, n_feat), S_SHIPPED, inv_s, mode, eikonal, tag='%s inv_s %.1f' % (cfg_name, inv_s))


OBJECTIVES = {'second_grad_only': (None, False), 'eikonal': (None, True), 'combine': ('combine', True),
              'multi_new_without_eikonal': ('multi_new', False)}


@pytest.mark.parametrize('objective', list(OBJECTIVES))
@pytest.mark.parametrize('path', list(PATHS))
def test_fused_second_grad_parity_on_every_kernel_instantiation(path, objective):
    """The instantiation matrix of test_gpu_train_fused_parity.py (fwd5 / fwd families, affine and ring maps, forced
    switches) with every OBJ value and the term alone; the small geometries' rays leave the volume (zero padding)."""
    _dev()
    from selfocc_b200 import _lib
    kind, n_feat, force, zpair, inst = PATHS[path]
    mode, eikonal = OBJECTIVES[objective]
    if kind == 'nusc':
        geo, S = _geo('nuscenes/nuscenes_novel_depth.py', 60, n_feat), S_SHIPPED
    else:
        geo, S = _small_geo(kind, n_feat), 128 if kind == 'h_ne_w' else 64
    lib = _lib.load()
    hook = {'fwd32': lib.so_render_train_force_fwd32, 'sem_generic': lib.so_render_train_force_sem_generic}.get(force)
    try:
        if hook:
            hook(1)
        _gate(geo, S, 20.0, mode, eikonal, zpair=zpair, tag='%s %s' % (path, inst.replace('OBJ', OBJ_NAME[mode])))
    finally:
        if hook:
            hook(0)


@pytest.mark.parametrize('kind', ['h_ne_w', 'ring'])
def test_fused_second_grad_parity_with_the_start_anchor(kind):
    """sample_anchor='start': the query point is the bin's start (the one-ray-per-warp path)."""
    _gate(_small_geo(kind, 3), 64, 20.0, 'combine', True, anchor_mid=False, tag='%s start anchor' % kind)


def test_ray_sharded_launches_give_the_unsharded_sums():
    """Launches over [ray_begin, ray_begin + count): each passes the gate, and count-weighted means add up to the whole."""
    geo = _geo('nuscenes/nuscenes_occ.py', 15, 24)
    n = geo['i2l'].shape[0] * geo['pix'].shape[0]
    full, _, _ = _gate(geo, S_SHIPPED, 20.0, 'combine', True, tag='whole')
    parts = [(0, 700), (700, n - 1400), (n - 700, 700)]
    tot = 0.0
    for b, c in parts:
        res, _, _ = _gate(geo, S_SHIPPED, 20.0, 'combine', True, ray_begin=b, ray_count=c, tag='rays [%d, %d)' % (b, b + c))
        tot += res['second_grad_mean'].double().item() * c
    assert abs(tot / n - full['second_grad_mean'].item()) <= 1e-6 * full['second_grad_mean'].item()


def test_the_term_off_leaves_the_objective_unchanged_and_is_deterministic():
    """second_grad off and on: every other output bit-identical, d/d inv_s bit-identical (per-ray values summed in ray
    order), the volume gradients within the atomics' reordering.  Two identical fused launches: the same second_grad_mean
    bit for bit, and the term's volume gradient within the atomics' reordering (its corner gradients join the render's
    float-atomic scatter).  A launch and its backward never sync with the host."""
    from test_gpu_train_fused import _cotangents, _geometry, _max_rel
    from selfocc_b200 import ops
    dev = _dev()
    vs0, vf0, cfg, ob, shape = _geometry(dev, 'shipped', 24)
    cot = _cotangents(cfg, shape, 'combine', dev)
    g_mean = torch.tensor(G_MEAN, device=dev)            # made before sync debug mode: a host-to-device copy synchronises

    def run(sg, g_sg=None):
        vs, vf = vs0.clone().requires_grad_(True), vf0.clone().requires_grad_(True)
        invs = torch.full((1,), 20.0, device=dev, requires_grad=True)
        res = dict(zip(ops.RenderTrainObjectiveFunction.ORDER, ops.RenderTrainObjectiveFunction.apply(
            vs, vf, invs, dict(cfg, objective=dict(ob, mode='combine', second_grad=sg)))))
        outs = [res[k] for k in cot] + ([res['second_grad_mean']] if g_sg is not None else [])
        cots = [cot[k] for k in cot] + ([g_sg] if g_sg is not None else [])
        grads = torch.autograd.grad(outs, [vs, invs, vf], cots)
        return res, grads
    off, g_off = run(False)
    on, g_on = run(True)
    assert off['second_grad_mean'].numel() == 0 and on['second_grad_mean'].numel() == 1
    for k in ops.RenderTrainObjectiveFunction.ORDER[:-1]:
        assert torch.equal(off[k], on[k]), k
    assert torch.equal(g_off[1], g_on[1])
    assert _max_rel(g_on[0], g_off[0]) <= 1e-6 and _max_rel(g_on[2], g_off[2]) <= 1e-6
    a, ga = run(True, g_mean)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        b, gb = run(True, g_mean)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(a['second_grad_mean'], b['second_grad_mean'])
    assert torch.equal(ga[1], gb[1])
    assert (ga[0] - g_on[0]).abs().max().item() > 0                 # the term adds a volume gradient
    assert _max_rel(gb[0], ga[0]) <= 1e-6 and _max_rel(gb[2], ga[2]) <= 1e-6


# ------------------------------------------------------------------------------------------------ end to end
def _nuscenes_occ():
    from test_gpu_ray_shard import small_training_model
    dev = _dev()
    model, ml, feats, metas, imgs = small_training_model(dev)
    assert any(type(t).__name__ == 'SecondGradLoss' for t in ml.losses) and model.head.return_second_grad
    return model, ml, feats, metas, imgs


def test_fused_second_grad_step_equals_unfused_step(monkeypatch):
    """nuscenes_occ's objective end to end through MultiLoss: the per-ray outputs bit-identical, every term and the total
    as the unfused step's, and every parameter and FPN-feature gradient within the bar of test_gpu_train_fused.py.

    SecondGradLoss is the exception to 1e-6: the unfused step queries second_grad at positions rebuilt in torch (origin +
    direction * ts * |dir|, metres), the fused one at the render's own fp32 grid coordinates (g0 + dg * t).  The two round
    differently, and a sample within ~1e-6 of a cell face can land in the neighbouring cell, whose second derivatives are
    another cell's: the term moves by that sample's share of the mean.  Measured on an H100: 6.8e-7 of the term, inside the
    1e-6 bar of every term."""
    from test_gpu_train_fused import _step
    from selfocc_b200.loss import fuse_objective
    from selfocc_b200 import ops
    model, ml, feats, metas, imgs = _nuscenes_occ()
    feats = [f.clone().requires_grad_(True) for f in feats]
    params = [p for p in model.parameters() if p.requires_grad] + feats
    tot1, ref, inp1 = _step(model, ml, feats, metas, imgs)
    ref_g = torch.autograd.grad(tot1, params, allow_unused=True)
    per_ray = {k: [t.detach() for t in inp1[k]] for k in ('ms_depths', 'ms_accs', 'ms_colors', 'sem')}
    assert inp1['second_grad'].shape[-1] == 3
    del inp1
    tot1b, _, _ = _step(model, ml, feats, metas, imgs)
    spread = [None if b is None else (a - b).abs().max().item()
              for a, b in zip(torch.autograd.grad(tot1b, params, allow_unused=True), ref_g)]
    rec = fuse_objective(model.head, ml, second_grad=True)
    assert rec['second_grad'] is True
    calls = []
    apply = ops.RenderTrainObjectiveFunction.apply

    def spy(*a):
        calls.append(sorted(a[3]['want']))
        return apply(*a)

    def no_field_pass(*a):
        raise AssertionError('the fused step runs no separate second-grad field pass')
    monkeypatch.setattr(ops.RenderTrainObjectiveFunction, 'apply', spy)
    monkeypatch.setattr(ops.FieldSecondGradFunction, 'apply', no_field_pass)
    try:
        tot2, got, inp = _step(model, ml, feats, metas, imgs)
        got_g = torch.autograd.grad(tot2, params, allow_unused=True)
    finally:
        monkeypatch.undo()
        model.head.fused_objective = None
    # nothing per sample: the render was asked for per-ray outputs only, and no [rays, S, .] tensor reaches the outputs
    assert calls == [['acc', 'depth', 'fars', 'rgb', 'sem']], calls
    assert not any(k in inp for k in ('weights', 'ts', 'deltas', 'eik_grad', 'second_grad'))
    assert inp['second_grad_mean'].dim() == 0
    for k, v in per_ray.items():
        for a, b in zip(inp[k], v):
            assert torch.equal(a, b), k
    assert list(got) == list(ref)
    d_sg = abs(got['SecondGradLoss'].item() - ref['SecondGradLoss'].item())
    print('SecondGradLoss fused %.9e unfused %.9e rel %.2e; total rel %.2e' % (
        got['SecondGradLoss'].item(), ref['SecondGradLoss'].item(), d_sg / abs(ref['SecondGradLoss'].item()),
        abs(tot2.item() - tot1.item()) / abs(tot1.item())))
    for k in ref:
        assert abs(got[k].item() - ref[k].item()) <= 1e-6 * abs(ref[k].item()), (k, got[k].item(), ref[k].item())
    assert abs(tot2.item() - tot1.item()) <= 1e-6 * abs(tot1.item())
    for i, (a, b) in enumerate(zip(got_g, ref_g)):
        assert (a is None) == (b is None), i
        if b is not None:
            err, scale = (a - b).abs().max().item(), b.abs().max().item()
            assert err <= max(1e-5 * scale, 3 * spread[i]), (i, err, scale, spread[i])


@pytest.mark.parametrize('world', [2, 3])
def test_fused_second_grad_ray_sharded_step_equals_fused_step(world):
    from test_gpu_ray_shard import _check_values
    from test_gpu_train_fused import _step
    from test_ray_shard_cpu import emulated_ranks
    from selfocc_b200.loss import fuse_objective
    model, ml, feats, metas, imgs = _nuscenes_occ()
    params = [p for p in model.parameters() if p.requires_grad]
    fuse_objective(model.head, ml, second_grad=True)
    try:
        tot1, ref, _ = _step(model, ml, feats, metas, imgs)
        ref_g = torch.autograd.grad(tot1, params, allow_unused=True)
        inputs = [_step(model, ml, feats, metas, imgs, shard=(r, world)) for r in range(world)]
        assert all('second_grad_mean' in inp and 'second_grad' not in inp for inp in inputs)
        res = emulated_ranks(ml, inputs, world)
    finally:
        model.head.fused_objective = None
    for tot_r, d in res:
        _check_values(ref, d)
        assert abs(tot_r.item() - tot1.item()) <= 1e-6 * abs(tot1.item())
    grads = [torch.autograd.grad(t, params, allow_unused=True) for t, _ in res]
    for i, g1 in enumerate(ref_g):
        if g1 is None:
            continue
        g = torch.stack([gr[i] for gr in grads]).mean(0)  # what DDP's gradient mean gives
        assert (g - g1).abs().max().item() <= 1e-5 * g1.abs().max().item(), i


def test_fused_second_grad_decode_sharded_step_equals_unsharded():
    from test_gpu_decode_shard import _check_grads, _check_values, _tpv_case, decode_sharded_grads, unsharded
    from selfocc_b200.loss import fuse_objective
    dev = _dev()
    model, ml, feats, metas, imgs = _tpv_case(dev, sparsity=False)
    assert model.head.return_second_grad
    fuse_objective(model.head, ml, second_grad=True)
    try:
        ref, ref_g = unsharded(model, ml, feats, metas, imgs)
        ds, got = decode_sharded_grads(model, ml, feats, metas, imgs, 2)
    finally:
        model.head.fused_objective = None
    for d in ds:
        _check_values(ref, d)
    _check_grads(got, ref_g)


def test_fused_second_grad_loss_never_syncs_with_the_host():
    """The fused render's second_grad_mean through SecondGradLoss, forward and backward, under sync debug mode 'error'."""
    from test_gpu_train_fused import _geometry
    from selfocc_b200 import ops
    from selfocc_b200.loss import SecondGradLoss
    dev = _dev()
    vs, vf, cfg, ob, _ = _geometry(dev, 'shipped', 24)
    vs = vs.clone().requires_grad_(True)
    invs = torch.full((1,), 20.0, device=dev, requires_grad=True)
    term = SecondGradLoss(weight=0.01)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        res = dict(zip(ops.RenderTrainObjectiveFunction.ORDER, ops.RenderTrainObjectiveFunction.apply(
            vs, vf, invs, dict(cfg, objective=dict(ob, mode=None, eikonal=False, second_grad=True)))))
        loss = term(res)
        loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert vs.grad.abs().max().item() > 0
    np.testing.assert_allclose(loss.item(), 0.01 * res['second_grad_mean'].item(), rtol=1e-7)
