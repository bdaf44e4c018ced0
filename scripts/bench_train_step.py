"""One full training-form step of the hot path at BASELINE configs[4] sizes (fp32); under torchrun the step is RAY-SHARDED:
every rank lifts the same frame, renders its slice of each camera's rays (head.ray_shard) and DDP averages the gradients.
    python scripts/bench_train_step.py [--profile]
    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 scripts/bench_train_step.py
Single GPU:
lifter -> encoder (autograd path: the fused self- and image cross-attention cores with their backward kernels, projections
forward and input gradient on the wgmma GEMM, weight gradients on cuBLAS) -> NeuSHead.forward (fused decode forward,
training-form render kernels) -> toy loss on depth / weights / eik_grad / rgb -> backward to every parameter.  Prints one
JSON line (ms per step, device timed; peak device memory of the timed steps).  nuScenes_occ geometry: TPV 257x257x25,
6 cams x 48x100 rays.
    --loss reproj: the toy loss's weights term is replaced by ReprojLossMonoMultiNewCombine (the nuScenes configs' objective,
    SSIM + automask) on seeded textured 768x1600 previous / current / next images under a small ego motion (synth).
    --loss shipped: the toy loss is replaced by nuscenes_occ's whole MultiLoss (reprojection, RGBLossMS with SSIM,
    EikonalLoss, SecondGradLoss, SemCELossMS), with the head as that config sets it: color_dims = 24, return_sem, and
    return_second_grad under the declared opt-in assumption (second_grad_assumption=True); seeded synthetic previous /
    current / next / colour images and semantic labels."""
import json, os, sys, time
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from selfocc_b200 import configs, synth, _lib
from selfocc_b200.registry import build_head
import selfocc_b200.segmentor  # noqa

import torch.distributed as dist
rank, world, local = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1)), int(os.environ.get('LOCAL_RANK', 0))
torch.cuda.set_device(local)
dev = torch.device('cuda', local)
if world > 1:
    dist.init_process_group('nccl', device_id=dev)
margs = dict(synth.NUSC_MAPPING, h_size=[128, 0], h_range=[40.0, 0], w_size=[128, 0], w_range=[40.0, 0], d_size=[24, 0], d_range=[-1.0, 5.4, 5.4])
rng = [-40.0, -40.0, -1.0, 40.0, 40.0, 5.4]
loss_mode = sys.argv[sys.argv.index('--loss') + 1] if '--loss' in sys.argv else None
shipped = loss_mode == 'shipped'
cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, ray_number=(48, 100), ray_img_size=(768, 1600), color_dims=24 if shipped else 3,
                              ray_sample_mode='cellular', render_bkgd='random', return_max_depth=False, dropout=0.1, return_sem=shipped)
if shipped:
    cfg['head'].update(return_second_grad=True, second_grad_assumption=True)
torch.manual_seed(0)
model = build_head(cfg)
model.encoder.init_weights()
with torch.no_grad():
    for p in (model.lifter.tpv_hw, model.lifter.tpv_zh, model.lifter.tpv_wz):
        p.mul_(0.1)
    model.head.model.field.deviation_network.variance.fill_(0.3)
model.train().to(dev)
l2i, i2l = synth.camera_rig()
metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(768, 1600))]
g = torch.Generator().manual_seed(1)
feats = [torch.randn(1, 6, 96, h, w, generator=g).to(dev) for h, w in synth.fpn_level_shapes(768, 1600)]
opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
reproj = objective = None
if shipped:
    from bench_train_objective import CFG
    from selfocc_b200.registry import LOSSES
    objective = LOSSES.build(dict(type='MultiLoss', loss_cfgs=CFG))
    prev, nxt = synth.temporal_rig()
    lab = torch.randint(0, 17, (6, 768, 1600), generator=torch.Generator().manual_seed(3)).to(torch.uint8).numpy()
    metas[0].update(img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev), img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev),
                    sem=lab)
    imgs = synth.textured_images(24, 768, 1600, seed=2).reshape(4, 1, 6, 3, 768, 1600).to(dev)
if loss_mode == 'reproj':
    from selfocc_b200.loss import ReprojLossMonoMultiNewCombine
    reproj = ReprojLossMonoMultiNewCombine(img_size=[768, 1600], ray_resize=[48, 100])
    prev, nxt = synth.temporal_rig()
    metas[0].update(img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev), img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))
    imgs = synth.textured_images(18, 768, 1600, seed=2).reshape(3, 1, 6, 3, 768, 1600).to(dev)
net = model
if world > 1:
    model.head.ray_shard = (rank, world)
    net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], broadcast_buffers=False)


class _Step(torch.nn.Module):
    """the whole hot path as ONE forward so that DDP sees a single module call"""
    def forward(self, feats, metas):
        r = model.lifter(ms_img_feats=feats)
        r = model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)
        return model.head(representation=r['representation'], metas=metas)


model.forward = lambda feats, metas: _Step.forward(None, feats, metas)


def step():
    opt.zero_grad(set_to_none=True)
    out = net(feats, metas)
    if objective is not None:
        loss, _ = objective(dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas))
        loss.backward()
        opt.step()
        return loss.detach()
    if reproj is None:
        w_term = torch.cat(out['weights']).pow(2).mean()
    else:
        w_term = reproj(dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], metas=metas))
    loss = out['ms_depths'][0].mean() * 1e-2 + w_term \
        + (out['eik_grad'].norm(dim=-1) - 1).pow(2).mean() * 0.1 + out['ms_colors'][0].mean() * 0.1
    loss.backward()
    opt.step()
    return float(loss.detach()) if False else loss.detach()


for _ in range(2):
    step()
torch.cuda.synchronize()
torch.cuda.reset_peak_memory_stats()
K = 5
a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
l0 = _lib.launch_count()
a.record()
for _ in range(K):
    last = step()
b.record()
torch.cuda.synchronize()
ms = a.elapsed_time(b) / K
peak_gb = torch.cuda.max_memory_allocated() / 2 ** 30
if world > 1:
    t = torch.tensor([ms], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t)
if '--profile' in sys.argv and world == 1:
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    print(prof.key_averages().table(sort_by='cuda_time_total', row_limit=25))
if rank == 0:
  print(json.dumps({'workload': 'nuscenes_occ-like training step, %d GPU(s)%s, fp32, 6x48x100 rays x 256, TPV 257x257x25, colour%s' % (world, ' ray-sharded + DDP' if world > 1 else '', ', reprojection loss' if reproj is not None else ', nuscenes_occ MultiLoss (24 colour dims, semantics, second grad)' if shipped else ''), 'ms_per_step': ms,
                  'rays_per_s': 28800 / (ms * 1e-3), 'library_launches_per_step': (_lib.launch_count() - l0) / K, 'peak_mem_gb': peak_gb,
                  'loss': float(last), 'finite': bool(torch.isfinite(last))}))
if world > 1:
    dist.destroy_process_group()
