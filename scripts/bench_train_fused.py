"""One training step with the objective fused into the training render (loss.fuse_objective) against the same step unfused,
alternated in one process, on one GPU:
    python scripts/bench_train_fused.py [--steps K] [--rounds N] [--second-grad]
Two workloads, each at nuScenes sizes (6 cams x 48x100 rays x 256 samples, TPV 257x257x25, fp32):
  shipped : the bench_train_step.py --loss shipped step -- nuscenes_occ's whole MultiLoss (reprojection, RGBLossMS with
            SSIM, EikonalLoss, SecondGradLoss, SemCELossMS), 24 colour dims, semantics, second grad under its opt-in
            assumption;
  depth   : nuscenes_depth's MultiLoss (ReprojLossMonoMultiNewCombine, EikonalLoss, EdgeLoss3DMS), a 3-channel colour head.
Each round runs K unfused steps then K fused steps per workload (device-timed, after warm-up); prints one JSON line per
workload with the per-round ms per step (median), peak device memory of a step and library launches per step, and the
card's name and power limit.
--second-grad: the shipped workload only, alternating three forms: unfused, fused (SecondGradLoss on the head's
second_grad tensor) and fused with second_grad=True (SecondGradLoss's mean taken in the render)."""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
from selfocc_b200 import configs, synth, _lib  # noqa: E402
from selfocc_b200.loss import fuse_objective  # noqa: E402
from selfocc_b200.registry import build_head, LOSSES  # noqa: E402
import selfocc_b200.segmentor  # noqa: F401,E402

K = int(sys.argv[sys.argv.index('--steps') + 1]) if '--steps' in sys.argv else 5
ROUNDS = int(sys.argv[sys.argv.index('--rounds') + 1]) if '--rounds' in sys.argv else 3
SECOND_GRAD = '--second-grad' in sys.argv
dev = torch.device('cuda', 0)
margs = dict(synth.NUSC_MAPPING, h_size=[128, 0], h_range=[40.0, 0], w_size=[128, 0], w_range=[40.0, 0], d_size=[24, 0],
             d_range=[-1.0, 5.4, 5.4])
rng = [-40.0, -40.0, -1.0, 40.0, 40.0, 5.4]
NUSC_DEPTH = [dict(type='ReprojLossMonoMultiNewCombine', img_size=[900, 1600], no_automask=False, no_ssim=False, ray_resize=[48, 100]),
              dict(type='EikonalLoss', weight=0.1),
              dict(type='EdgeLoss3DMS', img_size=[900, 1600], ray_resize=[48, 100], weight=0.01)]


def workload(name):
    shipped = name == 'shipped'
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, ray_number=(48, 100), ray_img_size=(768, 1600),
                                  color_dims=24 if shipped else 3, ray_sample_mode='cellular', render_bkgd='random',
                                  return_max_depth=False, dropout=0.1, return_sem=shipped)
    if shipped:
        cfg['head'].update(return_second_grad=True, second_grad_assumption=True)
    torch.manual_seed(0)
    np.random.seed(0)
    model = build_head(cfg)
    model.encoder.init_weights()
    with torch.no_grad():
        for p in (model.lifter.tpv_hw, model.lifter.tpv_zh, model.lifter.tpv_wz):
            p.mul_(0.1)
        model.head.model.field.deviation_network.variance.fill_(0.3)
    model.train().to(dev)
    l2i, i2l = synth.camera_rig()
    prev, nxt = synth.temporal_rig()
    lab = torch.randint(0, 17, (6, 768, 1600), generator=torch.Generator().manual_seed(3)).to(torch.uint8).numpy()
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=(768, 1600), sem=lab,
                  img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                  img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))]
    g = torch.Generator().manual_seed(1)
    feats = [torch.randn(1, 6, 96, h, w, generator=g).to(dev) for h, w in synth.fpn_level_shapes(768, 1600)]
    imgs = synth.textured_images(24, 768, 1600, seed=2).reshape(4, 1, 6, 3, 768, 1600).to(dev)
    if shipped:
        from bench_train_objective import CFG
        objective = LOSSES.build(dict(type='MultiLoss', loss_cfgs=CFG))
    else:
        objective = LOSSES.build(dict(type='MultiLoss', loss_cfgs=NUSC_DEPTH))
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
    recs = {False: None, True: fuse_objective(model.head, objective)}
    if shipped:
        recs['sg'] = fuse_objective(model.head, objective, second_grad=True)

    def step(fused):
        model.head.fused_objective = recs[fused]
        opt.zero_grad(set_to_none=True)
        out = model(ms_img_feats=feats, metas=metas, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2])
        loss, _ = objective(dict(out, color_imgs=imgs[3]))
        loss.backward()
        opt.step()
        return loss.detach()

    return step


def measure(step, fused):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    l0 = _lib.launch_count()
    a.record()
    for _ in range(K):
        last = step(fused)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / K, (torch.cuda.max_memory_allocated() - base) / 2 ** 30, (_lib.launch_count() - l0) / K, float(last)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0)


def main():
    forms = ((False, 'unfused'), (True, 'fused')) + ((('sg', 'fused_second_grad'),) if SECOND_GRAD else ())
    for name in ('shipped',) if SECOND_GRAD else ('shipped', 'depth'):
        step = workload(name)
        for _ in range(2):                             # warm-up of every form
            for fused, _tag in forms:
                step(fused)
        res = {fused: [] for fused, _tag in forms}
        for _ in range(ROUNDS):
            for fused, _tag in forms:
                res[fused].append(measure(step, fused))
        out = {'workload': 'nuscenes %s training step, 1 GPU, fp32, 6x48x100 rays x 256, TPV 257x257x25' % name, 'card': card(),
               'steps_per_round': K, 'rounds': ROUNDS}
        for fused, tag in forms:
            r = res[fused]
            out[tag] = {'ms_per_step': float(np.median([x[0] for x in r])), 'ms_per_step_rounds': [round(x[0], 3) for x in r],
                        'ms_per_step_spread': round(max(x[0] for x in r) - min(x[0] for x in r), 3),
                        'peak_step_mem_gb': max(x[1] for x in r), 'library_launches_per_step': r[-1][2], 'loss': r[-1][3]}
        print(json.dumps(out), flush=True)
        del step
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
