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
    current / next / colour images and semantic labels.
Under torchrun both objectives run ray-sharded: MultiLoss gathers the per-ray loss inputs of every rank (one collective per
step), so its terms have the 1-GPU values, and each rank prints its last step's terms.  With --loss reproj the printed total
also holds the toy terms (depth, eikonal and colour means), which stay per-rank means of the rank's own rays and differ
between ranks and from the 1-GPU run; with --loss shipped the total is the MultiLoss total.
    --shard-encoder (under torchrun): the encoder's training pass is query-sharded too (encoder.query_shard, its exchange on
    its own NCCL process group): each rank runs every layer on its 1/world of each plane, one all_gather per layer forward
    and one reduce-scatter per layer backward.
    --emulate-world W (one process): ONE rank's share of a W-rank step with both shardings on one GPU -- rank 0's rows
    through every layer, a local stand-in for the exchange (it fills the other ranks' rows with this rank's buffer and returns
    this rank's own gradient rows, talking to no one), the head on rank 0's ray slice.  Compute per rank, communication
    excluded; the loss value is not the W-rank step's.
    --shard-decode (under torchrun, or with --emulate-world): the head's decode is sharded too (head.decode_shard, its
    exchange on its own NCCL process group; emulated by the same local stand-ins): each rank decodes and backpropagates
    its slab of the volume's h rows, one all_gather of the volume forward and one reduce-scatter of its gradient backward.
    The JSON line then carries the bytes that exchange moves per rank and step (decode_exchange_bytes_per_rank)."""
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
emulate = int(sys.argv[sys.argv.index('--emulate-world') + 1]) if '--emulate-world' in sys.argv else 0
shard_encoder = '--shard-encoder' in sys.argv
shard_decode = '--shard-decode' in sys.argv
if emulate and world > 1:
    raise SystemExit('--emulate-world runs in one process (it emulates one rank of the W-rank step)')
shipped = loss_mode == 'shipped'
cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, ray_number=(48, 100), ray_img_size=(768, 1600), color_dims=24 if shipped else 3,
                              ray_sample_mode='cellular', render_bkgd='random', return_max_depth=False, dropout=0.1, return_sem=shipped)
if shipped:
    cfg['head'].update(return_second_grad=True, second_grad_assumption=True)
torch.manual_seed(0)
np.random.seed(0)                  # every rank must draw the same cellular ray grid (RaySampler.draw uses numpy)
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
    from selfocc_b200.loss import MultiLoss
    # inside a MultiLoss so that a ray-sharded step gathers the per-ray statistics for SSIM over the whole ray grid
    reproj = MultiLoss([dict(type='ReprojLossMonoMultiNewCombine', img_size=[768, 1600], ray_resize=[48, 100])])
    prev, nxt = synth.temporal_rig()
    metas[0].update(img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev), img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))
    imgs = synth.textured_images(18, 768, 1600, seed=2).reshape(3, 1, 6, 3, 768, 1600).to(dev)
net = model
if world > 1:
    model.head.ray_shard = (rank, world)
    if shard_encoder:
        model.encoder.query_shard = (rank, world)
        model.encoder.query_shard_group = dist.new_group(backend='nccl')
    if shard_decode:
        model.head.decode_shard = (rank, world)
        model.head.decode_shard_group = dist.new_group(backend='nccl')
    net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local], broadcast_buffers=False)


def local_gather(out, buf):
    """the stand-in all_gather of --emulate-world: every rank's slot gets this rank's buffer"""
    out.view(emulate, -1).copy_(buf.reshape(1, -1).expand(emulate, -1))


def local_reduce_scatter(out, buf):
    """the stand-in reduce-scatter of --emulate-world: this rank's block of its own gradient"""
    out.copy_(buf.view(emulate, -1)[0].view_as(out))


if emulate:
    model.head.ray_shard = (0, emulate)
    if shard_decode:
        model.head.decode_shard = (0, emulate)
        model.head.decode_shard_collectives = (local_gather, local_reduce_scatter)
    for ml_ in (objective, reproj):
        if ml_ is not None:
            ml_.collective = local_gather


class _Step(torch.nn.Module):
    """the whole hot path as ONE forward so that DDP sees a single module call"""
    def forward(self, feats, metas):
        r = model.lifter(ms_img_feats=feats)
        if emulate:
            rep = model.encoder.forward_query_sharded(r['representation'], feats, metas, 0, emulate, local_gather,
                                                      local_reduce_scatter)
            return model.head(representation=rep, metas=metas)
        r = model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)
        return model.head(representation=r['representation'], metas=metas)


model.forward = lambda feats, metas: _Step.forward(None, feats, metas)


terms = {}


def step():
    opt.zero_grad(set_to_none=True)
    out = net(feats, metas)
    if objective is not None:
        loss, terms_ = objective(dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas))
        terms.update(terms_)
        loss.backward()
        opt.step()
        return loss.detach()
    if reproj is None:
        w_term = torch.cat(out['weights']).pow(2).mean()
    else:
        w_term, terms_ = reproj(dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], metas=metas))
        terms.update(terms_)
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
if world > 1 and terms:            # the last step's loss terms on every rank: ray sharding gives every rank the same values
    print(json.dumps({'rank': rank, 'terms': {k: float(v) for k, v in terms.items()}}), flush=True)
    dist.barrier()
if emulate:
    mode = ', ONE rank of %d emulated (query-%s and ray-sharded): compute per rank, communication excluded' % (
        emulate, ', decode-' if shard_decode else '')
elif world > 1:
    mode = ' ray-sharded%s%s + DDP' % (' + query-sharded encoder' if shard_encoder else '', ' + decode-sharded' if shard_decode else '')
else:
    mode = ''
exchange = {}
if shard_decode and (emulate or world > 1):
    from selfocc_b200.dist import volume_exchange_bytes
    exchange = {'decode_exchange_bytes_per_rank': volume_exchange_bytes(model.head.model.field.desc, emulate or world)}
if rank == 0:
  print(json.dumps({'workload': 'nuscenes_occ-like training step, %d GPU(s)%s, fp32, 6x48x100 rays x 256, TPV 257x257x25, colour%s' % (world, mode, ', reprojection loss' if reproj is not None else ', nuscenes_occ MultiLoss (24 colour dims, semantics, second grad)' if shipped else ''), 'ms_per_step': ms,
                  'rays_per_s': 28800 / (ms * 1e-3), 'library_launches_per_step': (_lib.launch_count() - l0) / K, 'peak_mem_gb': peak_gb,
                  'loss': float(last), 'finite': bool(torch.isfinite(last)), **exchange}))
if world > 1:
    dist.destroy_process_group()
