"""GPU: ray-sharded training of the shipped objectives (MultiLoss with inputs['ray_shard'], NeuSHead under head.ray_shard).
Ranks are emulated one after the other on one GPU (test_ray_shard_cpu.emulated_ranks: the collective hands each rank every
rank's payload); the torchrun test runs DDP over NCCL when the machine has >= 2 GPUs and skips otherwise.

Per-ray terms gather per-ray kernel outputs (row-independent) and run the same tail on the same tensors, so their values
are bit-identical to the unsharded objective; the per-sample means combine the ranks' sums in fp64 (1e-6 relative)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from selfocc_b200 import synth
from selfocc_b200.dist import ray_slice

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from test_ray_shard_cpu import emulated_ranks  # noqa: E402

CFGS = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))
SAMPLE_MEANS = ('EikonalLoss', 'SecondGradLoss')


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _build(cfg):
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss  # noqa: F401
    return LOSSES.build(cfg)


def _case(loss_cfgs, dev, S=32, seed=0):
    """Synthetic inputs of one shipped objective at its ray grid (6 cameras), as test_gpu_losses.objective_inputs builds
    nuscenes_occ's.  Per-ray leaves are kept with an explicit ray axis: name -> (tensor, ray axis)."""
    rr = next(c['ray_resize'] for c in loss_cfgs if 'ray_resize' in c)
    img = next(c['img_size'] for c in loss_cfgs if 'img_size' in c)
    g = torch.Generator().manual_seed(seed)
    n, R, C = 6, rr[0] * rr[1], 17
    ys, xs = torch.meshgrid(torch.arange(rr[0]), torch.arange(rr[1]), indexing='ij')
    rays = torch.stack([(xs.flatten() + torch.rand(R, generator=g)) * (img[1] / rr[1]),
                        (ys.flatten() + torch.rand(R, generator=g)) * (img[0] / rr[0])], -1)
    prev, nxt = synth.temporal_rig()
    imgs = synth.textured_images(4 * n, 96, 200, seed=seed + 5).reshape(4, 1, n, 3, 96, 200).to(dev)
    lab = torch.randint(0, C, (n, img[0], img[1]), generator=g).to(torch.uint8).numpy()
    leaves = dict(weights=(torch.rand(n, R, S, generator=g) / S, 1), colors=(torch.rand(1, n, R, 3, generator=g), 2),
                  depths=(1 + 40 * torch.rand(1, n, R, generator=g), 2),
                  sem=(torch.softmax(3 * torch.randn(1, n, R, C, generator=g), -1), 2),
                  eik=(torch.randn(n, R, S, 3, generator=g) * 0.6, 1), sg=(torch.randn(n, R, S, 3, generator=g), 1),
                  usdf=(torch.randn(24, 24, 4, generator=g), None))
    leaves = {k: (v.to(dev), a) for k, (v, a) in leaves.items()}
    fixed = dict(curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], rays=rays.to(dev),
                 ts=(0.5 + 40 * torch.rand(n, R, S, generator=g)).sort(-1).values.to(dev),
                 metas=[dict(img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                             img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev), sem=lab)])
    return leaves, fixed, R


def _inputs(own, fixed, b, c):
    """The objective's inputs from the leaves of the rays [b, b + c) (own: name -> leaf)."""
    n, S = own['weights'].shape[0], own['weights'].shape[2]
    dev = own['weights'].device
    return dict(curr_imgs=fixed['curr_imgs'], prev_imgs=fixed['prev_imgs'], next_imgs=fixed['next_imgs'],
                color_imgs=fixed['color_imgs'], metas=fixed['metas'], ms_rays=fixed['rays'][b:b + c],
                weights=list(own['weights'].reshape(n, -1).unbind(0)),
                ts=list(fixed['ts'][:, b:b + c].reshape(n, -1).unbind(0)),
                ray_indices=[torch.arange(c, device=dev).repeat_interleave(S)] * n,
                ms_colors=[own['colors']], ms_depths=[own['depths']], sem=[own['sem']],
                eik_grad=own['eik'].reshape(-1, S, 3), second_grad=own['sg'].reshape(-1, S, 3), uniform_sdf=own['usdf'])


def _rank_leaves(leaves, b, c):
    return {k: (v.narrow(a, b, c) if a is not None else v).detach().clone().requires_grad_(True) for k, (v, a) in leaves.items()}


def _check_values(ref, d, exact=True):
    assert list(d) == list(ref)
    for k in ref:
        if k in SAMPLE_MEANS or not exact:
            assert abs(d[k].item() - ref[k].item()) <= 1e-6 * abs(ref[k].item()), (k, d[k].item(), ref[k].item())
        else:
            assert torch.equal(d[k], ref[k]), (k, d[k].item(), ref[k].item())


@pytest.mark.parametrize('name', sorted(CFGS))
def test_shipped_objective_on_emulated_ranks_equals_unsharded(name):
    dev = _dev()
    ml = _build(CFGS[name])
    leaves, fixed, R = _case(CFGS[name]['loss_cfgs'], dev)
    full = _rank_leaves(leaves, 0, R)
    tot, ref = ml(_inputs(full, fixed, 0, R))
    used = [k for k, v in full.items() if v.requires_grad]
    ref_g = dict(zip(used, torch.autograd.grad(tot, [full[k] for k in used], allow_unused=True)))
    for world in (2, 3, 8):
        own = [_rank_leaves(leaves, *ray_slice(R, world, r)) for r in range(world)]
        inputs = [dict(_inputs(o, fixed, *ray_slice(R, world, r)), ray_shard=(r, world, R)) for r, o in enumerate(own)]
        res = emulated_ranks(ml, inputs, world)
        for tot_r, d in res:
            _check_values(ref, d)
            assert abs(tot_r.item() - tot.item()) <= 1e-6 * abs(tot.item())
        got = [dict(zip(used, torch.autograd.grad(t, [o[k] for k in used], allow_unused=True))) for (t, _), o in zip(res, own)]
        for k in used:
            if ref_g[k] is None:
                assert all(g[k] is None for g in got), k
                continue
            a = leaves[k][1]
            g = torch.stack([gr[k] for gr in got]).mean(0) if a is None else torch.cat([gr[k] / world for gr in got], a)
            assert (g - ref_g[k]).abs().max().item() <= 1e-6 * ref_g[k].abs().max().item(), (name, world, k)


def test_sharded_objective_never_syncs_with_the_host():
    dev = _dev()
    ml = _build(CFGS['nuscenes/nuscenes_occ.py'])
    leaves, fixed, R = _case(CFGS['nuscenes/nuscenes_occ.py']['loss_cfgs'], dev)
    own = [_rank_leaves(leaves, *ray_slice(R, 2, r)) for r in range(2)]
    inputs = [dict(_inputs(o, fixed, *ray_slice(R, 2, r)), ray_shard=(r, 2, R)) for r, o in enumerate(own)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        res = emulated_ranks(ml, inputs, 2)
        grads = [torch.autograd.grad(t, list(o.values()), allow_unused=True) for (t, _), o in zip(res, own)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(g is None or torch.isfinite(g).all() for gs in grads for g in gs)
    assert all(sum(g is not None for g in gs) == 5 for gs in grads)       # weights, colours, semantics, eik_grad, second_grad


# ---------------------------------------------------------------------------------------------------------- end to end
def small_training_model(dev):
    """lifter + encoder + NeuSHead at a small TPV, nuscenes_occ's head (24 colour dims, semantics, second grad), encoder
    dropout 0.1, the cellular ray sampler and a random background; its objective, features, metas and images."""
    from selfocc_b200 import configs
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    torch.manual_seed(0)
    margs, rng = synth.small_mapping(16, 8, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=32, ray_number=(48, 100), ray_img_size=(768, 1600),
                                  color_dims=24, return_sem=True, return_max_depth=False, ray_sample_mode='cellular',
                                  render_bkgd='random', dropout=0.1)
    cfg['head'].update(return_second_grad=True, second_grad_assumption=True)
    model = build_head(cfg)
    model.encoder.init_weights()
    with torch.no_grad():
        model.head.model.field.deviation_network.variance.fill_(0.25)
    model.train().to(dev)
    l2i, i2l = synth.camera_rig()
    prev, nxt = synth.temporal_rig()
    lab = torch.randint(0, 17, (6, 768, 1600), generator=torch.Generator().manual_seed(2)).to(torch.uint8).numpy()
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(768, 1600), sem=lab,
                  img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                  img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))]
    g = torch.Generator().manual_seed(1)
    feats = [torch.randn(1, 6, 96, h, w, generator=g).to(dev) for h, w in synth.fpn_level_shapes(768, 1600)]
    imgs = synth.textured_images(24, 192, 400, seed=3).reshape(4, 1, 6, 3, 192, 400).to(dev)
    return model, _build(CFGS['nuscenes/nuscenes_occ.py']), feats, metas, imgs


def forward_step(model, feats, metas, imgs, shard=None, seed=0):
    """One training forward with torch and numpy seeded as train.py seeds every rank -> (representation, objective inputs)."""
    torch.manual_seed(seed)
    np.random.seed(seed)
    model.head.ray_shard = shard
    r = model.lifter(ms_img_feats=feats)
    rep = model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)['representation']
    out = model.head(representation=rep, metas=metas)
    return rep, dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas)


@pytest.mark.parametrize('world', [2, 3])
def test_sharded_training_step_end_to_end_equals_unsharded(world):
    dev = _dev()
    model, ml, feats, metas, imgs = small_training_model(dev)
    params = [p for p in model.parameters() if p.requires_grad]
    rep1, inp1 = forward_step(model, feats, metas, imgs)
    tot1, ref = ml(inp1)
    ref_g = torch.autograd.grad(tot1, params, allow_unused=True)
    del inp1
    reps, inputs = zip(*[forward_step(model, feats, metas, imgs, shard=(r, world)) for r in range(world)])
    for rep in reps:                                       # the same dropout masks: every rank lifts the same frame
        assert all(torch.equal(a, b) for a, b in zip(rep, rep1))
    assert all(inp['ray_shard'] == (r, world, 4800) for r, inp in enumerate(inputs))
    res = emulated_ranks(ml, list(inputs), world)
    for tot_r, d in res:
        _check_values(ref, d)
    grads = [torch.autograd.grad(t, params, allow_unused=True) for t, _ in res]
    for i, g1 in enumerate(ref_g):
        if g1 is None:
            continue
        g = torch.stack([gr[i] for gr in grads]).mean(0)  # what DDP's gradient mean gives
        assert (g - g1).abs().max().item() <= 1e-5 * g1.abs().max().item(), i


WORKER = r'''
import os, sys
import torch, torch.distributed as dist
sys.path.insert(0, %r); sys.path.insert(0, %r)
from test_gpu_ray_shard import small_training_model, forward_step
rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
dist.init_process_group('nccl', device_id=dev)
model, ml, feats, metas, imgs = small_training_model(dev)
net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], broadcast_buffers=False)


def step(feats, metas, shard):
    _, inputs = forward_step(model, feats, metas, imgs, shard=shard)
    return inputs
model.forward = step                                       # DDP sees one module call per step
tot, d = ml(net(feats, metas, (rank, world)))
tot.backward()
vals = torch.stack(list(d.values()))
hi, lo = vals.clone(), vals.clone()
dist.all_reduce(hi, op=dist.ReduceOp.MAX)
dist.all_reduce(lo, op=dist.ReduceOp.MIN)
ok = torch.equal(hi, lo)
params = [p for p in model.parameters() if p.requires_grad]
ddp = [None if p.grad is None else p.grad.clone() for p in params]
if rank == 0:                                              # the unsharded step on one GPU, on a model built the same way
    model1, ml1, _, _, _ = small_training_model(dev)
    _, inputs1 = forward_step(model1, feats, metas, imgs)
    tot1, d1 = ml1(inputs1)
    tot1.backward()
    ok = ok and all(torch.equal(d[k], d1[k]) or abs(d[k].item() - d1[k].item()) <= 1e-6 * abs(d1[k].item()) for k in d1)
    for g, p in zip(ddp, [p for p in model1.parameters() if p.requires_grad]):
        if p.grad is not None:
            ok = ok and g is not None and (g - p.grad).abs().max().item() <= 1e-5 * p.grad.abs().max().item()
flag = torch.tensor([int(bool(ok))], device=dev)
dist.all_reduce(flag, op=dist.ReduceOp.MIN)
if rank == 0:
    print('SHARD_OK' if int(flag) == 1 else 'SHARD_MISMATCH', world)
dist.destroy_process_group()
'''


def test_ray_sharded_training_step_over_nccl_with_ddp(tmp_path):
    """Needs >= 2 GPUs: DDP + NCCL, every rank reports the same loss_dict, and the DDP-averaged gradients equal the
    unsharded step's computed on rank 0."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip('needs >= 2 GPUs')
    n = 3 if torch.cuda.device_count() >= 3 else 2
    script = tmp_path / 'worker.py'
    script.write_text(WORKER % (ROOT, HERE))
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(n), '--master-addr',
                        '127.0.0.1', '--master-port', '29761', str(script)], capture_output=True, text=True, timeout=900)
    assert 'SHARD_OK %d' % n in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
