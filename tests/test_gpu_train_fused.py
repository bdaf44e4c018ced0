"""GPU: the training render with the objective's per-sample terms fused in (so_render_train_objective_forward / _backward,
ops.RenderTrainObjectiveFunction, loss.fuse_objective) against the unfused step it replaces: the training render's
per-sample tensors fed to the reprojection statistics and the eikonal sample mean.

Per-ray outputs are the same kernels' and must be bit-identical; the statistics and the eikonal mean sum the same
per-sample values in another order (1e-6); gradients are atomically accumulated on both sides (1e-5 of each tensor's
max-abs)."""
import os
import sys

import numpy as np
import pytest
import torch

from selfocc_b200 import synth
from selfocc_b200.dist import ray_slice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_gpu_ray_shard import CFGS, _build, _check_values, small_training_model  # noqa: E402
from test_ray_shard_cpu import emulated_ranks  # noqa: E402


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


# ------------------------------------------------------------------------------------------------ kernel level
def _geometry(dev, size, n_feat, seed=0):
    """(cfg of RenderTrainFunction, objective operands) at the small or the shipped geometry (6 cameras x 48 x 100 rays x
    256 samples on the nuScenes volume), jitter and a random background on."""
    from selfocc_b200 import ops
    from selfocc_b200.mapping import GridMeterMapping
    g = torch.Generator().manual_seed(seed)
    if size == 'shipped':
        margs, aabb, (ny, nx), S = dict(synth.NUSC_MAPPING, d_size=[24, 0], d_range=[-4.0, 4.0, 4.0]), \
            [-51.2, -51.2, -4.0, 51.2, 51.2, 4.0], (48, 100), 256
    else:
        margs, rng = synth.small_mapping(16, 8, rng=20.0, z0=-2.0, z1=4.0)
        aabb, (ny, nx), S = rng, (6, 10), 64
    m = GridMeterMapping(**margs)
    desc = m.volume_desc(n_feat)
    vs = synth.pack_sdf_volume(synth.analytic_sdf_volume(m, noise=0.02), desc.zpitch).to(dev)
    vf = (0.5 * torch.randn(desc.H, desc.W, desc.Z, desc.feat_pitch, generator=g)).to(dev) if n_feat else None
    _, i2l = synth.camera_rig()
    R, n = ny * nx, 6 * ny * nx
    ys, xs = torch.meshgrid(torch.arange(ny), torch.arange(nx), indexing='ij')
    pix = torch.stack([(xs.flatten() + torch.rand(R, generator=g)) * (1600 / nx),
                       (ys.flatten() + torch.rand(R, generator=g)) * (768 / ny)], -1).to(dev)
    want = ['depth', 'acc', 'fars', 'max_depth', 'rgb'] + (['sem'] if n_feat > 3 else [])
    cfg = dict(desc=desc, cam_mats=torch.tensor(i2l, dtype=torch.float32, device=dev), rays=ops.make_ray_desc(6, n_pix=R),
               params=ops.make_render_params(aabb, S, 20.0, training=True, bkgd='random'), pix=pix,
               jitter=torch.rand(n, S + 1, generator=g).to(dev), bkgd_rand=torch.rand(n, 3, generator=g).to(dev), want=want)
    prev, nxt = synth.temporal_rig()
    imgs = synth.textured_images(18, 96, 200, seed=seed + 5).reshape(3, 6, 3, 96, 200).to(dev)
    ob = dict(pix=pix, img2prev=torch.tensor(prev, dtype=torch.float32, device=dev).reshape(-1, 4, 4)[:6].contiguous(),
              img2next=torch.tensor(nxt, dtype=torch.float32, device=dev).reshape(-1, 4, 4)[:6].contiguous(),
              images=tuple(imgs[i].contiguous() for i in range(3)), img_size=(768, 1600), eikonal=True)
    return vs, vf, cfg, ob, (6, R, S)


def _unfused(vs, vf, cfg, ob, shape, mode, cot):
    """RenderTrainFunction -> ReprojStatsFunction + SampleMeanFunction(eikonal): outputs and gradients."""
    from selfocc_b200 import ops
    N, R, S = shape
    vs, vf = vs.clone().requires_grad_(True), None if vf is None else vf.clone().requires_grad_(True)
    invs = torch.full((1,), 20.0, device=vs.device, requires_grad=True)
    want = cfg['want'] + ['weights', 'ts', 'eik_grad']
    res = dict(zip(ops.RenderTrainFunction.ORDER, ops.RenderTrainFunction.apply(vs, vf, invs, dict(cfg, want=want))))
    rc = dict(mode=mode, shape=shape, ts=res['ts'].reshape(N, R * S), deltas=None, pix=ob['pix'], img2prev=ob['img2prev'],
              img2next=ob['img2next'], images=ob['images'], img_size=ob['img_size'])
    stats, colours = ops.ReprojStatsFunction.apply(rc, *res['weights'].reshape(N, R * S).unbind(0))
    eik = ops.SampleMeanFunction.apply(res['eik_grad'], 'eikonal')
    out = {k: res[k] for k in cfg['want']}
    out.update(reproj_stats=stats.reshape(N * R, -1), reproj_colours=colours.reshape(N * R, 9), eikonal_mean=eik)
    return out, _grads(out, cot, vs, vf, invs)


def _fused(vs, vf, cfg, ob, mode, cot):
    from selfocc_b200 import ops
    vs, vf = vs.clone().requires_grad_(True), None if vf is None else vf.clone().requires_grad_(True)
    invs = torch.full((1,), 20.0, device=vs.device, requires_grad=True)
    res = dict(zip(ops.RenderTrainObjectiveFunction.ORDER,
                   ops.RenderTrainObjectiveFunction.apply(vs, vf, invs, dict(cfg, objective=dict(ob, mode=mode)))))
    out = {k: res[k] for k in cfg['want'] + ['reproj_stats', 'reproj_colours', 'eikonal_mean']}
    return out, _grads(out, cot, vs, vf, invs)


def _cotangents(cfg, shape, mode, dev, seed=1):
    g = torch.Generator().manual_seed(seed)
    n = shape[0] * shape[1]
    sets = 1 if mode == 'combine' else 2
    cot = dict(depth=torch.randn(n, generator=g) * 0.01, acc=torch.randn(n, generator=g) * 0.01, rgb=torch.randn(n, 3, generator=g) * 0.01,
               sem=torch.randn(n, 21, generator=g) * 0.01, reproj_stats=torch.randn(n, 6 * sets, generator=g) * 0.01,
               eikonal_mean=torch.tensor(0.7))
    return {k: v.to(dev) for k, v in cot.items() if k in cfg['want'] or k in ('reproj_stats', 'eikonal_mean')}


def _grads(out, cot, vs, vf, invs):
    loss = sum((out[k] * cot[k]).sum() for k in cot)
    leaves = [vs, invs] + ([vf] if vf is not None else [])
    return torch.autograd.grad(loss, leaves)


def _max_rel(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.mark.parametrize('size, n_feat', [('small', 24), ('small', 3), ('shipped', 24), ('shipped', 3)])
@pytest.mark.parametrize('mode', ['combine', 'multi_new'])
def test_fused_render_equals_unfused_render_and_loss_kernels(size, n_feat, mode):
    dev = _dev()
    vs, vf, cfg, ob, shape = _geometry(dev, size, n_feat)
    cot = _cotangents(cfg, shape, mode, dev)
    ref, ref_g = _unfused(vs, vf, cfg, ob, shape, mode, cot)
    got, got_g = _fused(vs, vf, cfg, ob, mode, cot)
    for k in cfg['want']:
        assert torch.equal(got[k], ref[k]), k
    assert torch.equal(got['reproj_stats'][:, 5::6], ref['reproj_stats'][:, 5::6])        # the `any` flags
    assert (got['reproj_stats'] - ref['reproj_stats']).abs().max().item() <= 1e-6 * max(1.0, ref['reproj_stats'].abs().max().item())
    assert (got['reproj_colours'] - ref['reproj_colours']).abs().max().item() <= 1e-6
    assert abs(got['eikonal_mean'].item() - ref['eikonal_mean'].item()) <= 1e-6 * abs(ref['eikonal_mean'].item())
    assert ref['reproj_stats'][:, 5].mean().item() > 0.1              # the geometry exercises the reprojection
    for name, a, b in zip(('vol_sdf', 'inv_s', 'vol_feat'), got_g, ref_g):
        assert _max_rel(a, b) <= 1e-5, (name, _max_rel(a, b))


def test_fused_render_is_deterministic_and_never_syncs_with_the_host():
    dev = _dev()
    vs, vf, cfg, ob, shape = _geometry(dev, 'shipped', 24)
    cot = _cotangents(cfg, shape, 'combine', dev)
    a, ag = _fused(vs, vf, cfg, ob, 'combine', cot)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        b, bg = _fused(vs, vf, cfg, ob, 'combine', cot)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    # inv_s: per-ray values summed in ray order -> bitwise; the volume gradients are scattered with atomics (the training
    # render's contract), so only their summation order varies
    assert torch.equal(ag[1], bg[1])
    for x, y in (ag[0], bg[0]), (ag[2], bg[2]):
        assert _max_rel(x, y) <= 1e-6


def test_fused_step_drops_the_per_sample_tensors_from_peak_memory():
    dev = _dev()
    vs, vf, cfg, ob, shape = _geometry(dev, 'shipped', 3)
    cot = _cotangents(cfg, shape, 'combine', dev)
    peaks = {}
    for name, run in (('unfused', lambda: _unfused(vs, vf, cfg, ob, shape, 'combine', cot)),
                      ('fused', lambda: _fused(vs, vf, cfg, ob, 'combine', cot))):
        run()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        run()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() - base
    n, S = shape[0] * shape[1], shape[2]
    per_sample = n * S * 4 * (1 + 1 + 3)            # weights, ts and eik_grad, which the unfused step allocates
    assert peaks['unfused'] - peaks['fused'] >= per_sample, peaks


# ------------------------------------------------------------------------------------------------ end to end
def _step(model, ml, feats, metas, imgs, shard=None, seed=0):
    """One training forward (torch and numpy seeded as train.py seeds every rank) with the images as model kwargs, then
    the objective -> (total, loss_dict, inputs)."""
    torch.manual_seed(seed)
    np.random.seed(seed)
    model.head.ray_shard = shard
    out = model(ms_img_feats=feats, metas=metas, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2])
    inputs = dict(out, color_imgs=imgs[3])
    if shard is not None:
        return inputs
    tot, d = ml(inputs)
    return tot, d, inputs


def _objective_cfgs(name):
    """The shipped objective at the test model's ray grid (6 x 48 x 100)."""
    cfgs = []
    for c in CFGS[name]['loss_cfgs']:
        c = dict(c)
        if 'ray_resize' in c:
            c['ray_resize'] = [48, 100]
        cfgs.append(c)
    return dict(type='MultiLoss', loss_cfgs=cfgs)


@pytest.mark.parametrize('name', sorted(CFGS))
def test_shipped_objective_fused_step_equals_unfused_step(name):
    from selfocc_b200.loss import fuse_objective
    dev = _dev()
    model, _, feats, metas, imgs = small_training_model(dev)
    ml = _build(_objective_cfgs(name))
    model.head.return_uniform_sdf = any(c['type'] == 'SoftSparsityLoss' for c in CFGS[name]['loss_cfgs'])
    params = [p for p in model.parameters() if p.requires_grad]
    tot1, ref, inp = _step(model, ml, feats, metas, imgs)
    ref_g = torch.autograd.grad(tot1, params, allow_unused=True)
    assert 'weights' in inp and 'reproj_stats' not in inp
    del inp
    # the unfused step once more: its own run-to-run spread per gradient tensor.  The volume gradients are scattered with
    # float atomics, and a tensor such as the decode's sdf bias is a sum over the whole volume in which the gradient-of-sdf
    # terms cancel exactly, so its value moves with the atomics' order by more than 1e-5 of itself
    tot1b, _, _ = _step(model, ml, feats, metas, imgs)
    spread = [None if b is None else (a - b).abs().max().item()
              for a, b in zip(torch.autograd.grad(tot1b, params, allow_unused=True), ref_g)]
    fuse_objective(model.head, ml)
    try:
        tot2, got, inp = _step(model, ml, feats, metas, imgs)
        assert not any(k in inp for k in ('weights', 'ts', 'deltas', 'eik_grad'))
        got_g = torch.autograd.grad(tot2, params, allow_unused=True)
    finally:
        model.head.fused_objective = None
    assert list(got) == list(ref)
    for k in ref:
        assert abs(got[k].item() - ref[k].item()) <= 1e-6 * abs(ref[k].item()), (name, k, got[k].item(), ref[k].item())
    assert abs(tot2.item() - tot1.item()) <= 1e-6 * abs(tot1.item())
    for i, (a, b) in enumerate(zip(got_g, ref_g)):
        assert (a is None) == (b is None), i
        if b is not None:
            err, scale = (a - b).abs().max().item(), b.abs().max().item()
            assert err <= max(1e-5 * scale, 3 * spread[i]), (name, i, err, scale, spread[i])


@pytest.mark.parametrize('world', [2, 3])
def test_fused_ray_sharded_step_equals_fused_step(world):
    from selfocc_b200.loss import fuse_objective
    dev = _dev()
    model, ml, feats, metas, imgs = small_training_model(dev)
    params = [p for p in model.parameters() if p.requires_grad]
    fuse_objective(model.head, ml)
    tot1, ref, _ = _step(model, ml, feats, metas, imgs)
    ref_g = torch.autograd.grad(tot1, params, allow_unused=True)
    inputs = [_step(model, ml, feats, metas, imgs, shard=(r, world)) for r in range(world)]
    assert all(inp['ray_shard'] == (r, world, 4800) and inp['reproj_stats'].shape[1] == ray_slice(4800, world, r)[1]
               for r, inp in enumerate(inputs))
    res = emulated_ranks(ml, inputs, world)
    for tot_r, d in res:
        _check_values(ref, d)
        assert abs(tot_r.item() - tot1.item()) <= 1e-6 * abs(tot1.item())
    grads = [torch.autograd.grad(t, params, allow_unused=True) for t, _ in res]
    for i, g1 in enumerate(ref_g):
        if g1 is None:
            continue
        g = torch.stack([gr[i] for gr in grads]).mean(0)  # what DDP's gradient mean gives
        assert (g - g1).abs().max().item() <= 1e-5 * g1.abs().max().item(), i
