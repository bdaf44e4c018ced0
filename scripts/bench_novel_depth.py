"""Novel-view depth evaluation per frame: the reference's per-source loop body (eval_novel_depth.py:159-208, restated in
torch) vs NovelDepthMetric._after_step, both on the depth maps of one render_poses of the frame's S source poses.

  (a) reference: per source pose, the host-to-device copies of its LiDAR arrays, F.grid_sample of the N depth maps, per
      camera the boolean-mask gather (a host sync) and compute_depth_errors_torch, the dict accumulation by
      ceil(distance);
  (b) native:    NovelDepthMetric._after_step: the frame packed into one pinned buffer, one host-to-device copy, one
      so_novel_depth_errors launch, the per-bin index_add_.

Geometries: nuscenes_novel_depth.py (6 cameras, eval ray grid 96 x 200 of --num-rays' default, a nuScenes LiDAR sweep of
34720 points projected into every camera) and kitti_novel_depth.py (camera 0, eval ray grid 176 x 608, 120000 points).
The loader's arrays are synthetic: locations uniform over the image and a little beyond, about a sixth (nuScenes) or a
fifth (KITTI) of the points in front of each camera.  The two paths alternate after warm-up on the same frames; reported per
geometry: median host wall time per frame step (ending in a device synchronise), the render_poses time beside it, host
synchronisations per step (torch.cuda sync-debug warnings) and the largest relative difference of the two paths' per-bin
sums.  The card's name and power limit are read in the same run.  Prints one JSON line per geometry.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch
import torch.nn.functional as F

KITTI_MAPPING = dict(nonlinear_mode='linear', h_size=[256, 0], h_range=[51.2, 0], h_half=True, w_size=[128, 0],
                     w_range=[25.6, 0], w_half=False, d_size=[32, 0], d_range=[-2.0, 4.4, 4.4])   # config/kitti/kitti_novel_depth.py
GEOMETRIES = {
    # cameras, eval ray grid, image size, LiDAR points per source, fraction in front of a camera
    'nuscenes_novel_depth': dict(N=6, rays=(96, 200), img=(768, 1600), points=34720, visible=1 / 6),
    'kitti_novel_depth': dict(N=1, rays=(176, 608), img=(370, 1216), points=120000, visible=0.2),
}


def _setup(g, dev, sources):
    from selfocc_b200 import configs, synth
    from selfocc_b200.mapping import GridMeterMapping
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    nusc = g['N'] == 6
    margs = synth.NUSC_MAPPING if nusc else KITTI_MAPPING
    rng = synth.NUSC_RANGE if nusc else [-25.6, 0.0, -2.0, 25.6, 51.2, 4.4]
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=g['N'], num_layers=1, num_samples=256,
                                  ray_number=g['rays'], ray_img_size=g['img'], color_dims=3, render_bkgd='random')
    head = build_head(cfg).head.eval()
    w1, b1, w2, b2 = synth.random_mlp(96, 4, seed=2)
    with torch.no_grad():
        f = head.model.field
        for lin, w, b in ((f.density_net[1], w1, b1), (f.density_net[3], w2, b2)):
            lin.weight.copy_(w); lin.bias.copy_(b)
        head.to(dev)
        head.prepare([p[None].to(dev) for p in synth.random_planes(GridMeterMapping(**margs), 96, scale=0.3, seed=5)])
    h, w = g['img']
    if nusc:
        _, i2l = synth.camera_rig(f=1266.0 * w / 1600, cx=w / 2, cy=h / 2)
    else:
        _, i2l = synth.camera_rig((0.,), f=721.5, cx=w / 2, cy=h / 2, height=1.65, radius=0.0)
    poses = []
    for s in range(sources):
        T = np.eye(4); T[0, 3] = 2.0 * (s - sources / 2); T[1, 3] = 0.3 * s
        poses.append([T @ np.asarray(m) for m in i2l])
    return head, poses


def _frame(g, sources, seed):
    """Loader-shaped metas of one frame (float64 locations / depths, bool masks) with source distances in (0, 10)."""
    r = np.random.default_rng(seed)
    N, n = g['N'], g['points']
    meta = dict(depth_loc=[], depth_gt=[], depth_mask=[], frame_dists=list(r.random(sources) * 10))
    for _ in range(sources):
        loc = r.random((N, n, 2)) * 1.1 - 0.05
        meta['depth_loc'].append(loc)
        meta['depth_gt'].append(r.random((N, n)) * 79 + 1.0)
        meta['depth_mask'].append((r.random((N, n)) < g['visible']) & (loc > 0).all(-1) & (loc < 1).all(-1))
    return meta


def step_reference(maps, meta, agg, n_frames):
    """eval_novel_depth.py:159-208 after the render: one source pose at a time."""
    for s, dist in enumerate(meta['frame_dists']):
        loc = maps.new_tensor(meta['depth_loc'][s])
        gt = maps.new_tensor(meta['depth_gt'][s])
        mask = torch.from_numpy(meta['depth_mask'][s]).cuda()
        N = gt.shape[0]
        pred = F.grid_sample(maps[s][:, None], loc[:, None] * 2 - 1, mode='bilinear', padding_mode='border',
                             align_corners=True).reshape(N, -1)
        cams = []
        for c in range(N):
            g, p = gt[c][mask[c]], pred[c][mask[c]]
            p[p < 1e-3] = 1e-3
            p[p > 80] = 80
            th = torch.maximum(g / p, p / g)
            cams.append(torch.stack([torch.mean(torch.abs(g - p) / g), torch.mean((g - p) ** 2 / g),
                                     torch.sqrt(((g - p) ** 2).mean()), torch.sqrt(((torch.log(g) - torch.log(p)) ** 2).mean()),
                                     (th < 1.25).float().mean(), (th < 1.25 ** 2).float().mean(), (th < 1.25 ** 3).float().mean()]))
        cams = torch.stack(cams)
        k = math.ceil(dist)
        if k not in agg:
            agg[k], n_frames[k] = cams, torch.ones(1, dtype=torch.int, device=maps.device)
        else:
            agg[k] += cams
            n_frames[k] += 1


def _timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return sum(1 for x in w if 'synchroniz' in str(x.message).lower())


def _card():
    name, power = torch.cuda.get_device_name(0), None
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(', ')
        name, power = q[0], float(q[1])
    except Exception:
        pass
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--sources', type=int, default=4, help='source poses per frame')
    ap.add_argument('--only', default=None, help='comma-separated geometries')
    ap.add_argument('--out', default=None, help='also write the JSON lines to this file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_novel_depth.py measures on the GPU; no CUDA device found')
    from selfocc_b200.metric import NovelDepthMetric
    dev = torch.device('cuda:0')
    card, power = _card()
    lines = []
    for name, g in GEOMETRIES.items():
        if args.only and name not in args.only.split(','):
            continue
        head, poses = _setup(g, dev, args.sources)
        metas = [[dict(_frame(g, args.sources, seed=f), temImg2lidars=poses)] for f in range(4)]
        S, N, (h, w) = args.sources, g['N'], g['rays']
        metric = NovelDepthMetric(num_cams=N, max_distance=10)
        agg, n_frames = {}, {}
        with torch.no_grad():
            maps = head.render_poses(metas=metas[0])['ms_depths'][0].reshape(S, N, h, w)
            for i in range(args.warmup):
                step_reference(maps, metas[i % 4][0], {}, {})
                metric._after_step(metas[i % 4], maps)
            t = {'ref': [], 'nat': [], 'render': []}
            metric._reset()
            for i in range(args.frames):
                m = metas[i % 4]
                t['render'].append(_timed(lambda: head.render_poses(metas=m)))
                t['ref'].append(_timed(lambda: step_reference(maps, m[0], agg, n_frames)))
                t['nat'].append(_timed(lambda: metric._after_step(m, maps)))
            sync_ref, sync_nat = _syncs(lambda: step_reference(maps, metas[0][0], {}, {})), _syncs(lambda: metric._after_step(metas[0], maps))
        metric._reset()
        with torch.no_grad():
            agg, n_frames = {}, {}
            for i in range(args.frames):
                step_reference(maps, metas[i % 4][0], agg, n_frames)
                metric._after_step(metas[i % 4], maps)
        got, got_n = metric.as_dicts()
        as_t = lambda v: torch.as_tensor(v, dtype=torch.float64).cpu().reshape(-1, 7)
        rel = max(float(((as_t(got[k]) - as_t(agg[k])).abs() / as_t(agg[k]).abs().clamp_min(1e-6)).max()) for k in agg)
        same_bins = sorted(got) == sorted(agg) and all(int(got_n[k] if N == 1 else got_n[k][0]) == int(n_frames[k]) for k in agg)
        med = lambda k: statistics.median(t[k])
        visible = float(np.mean([m.sum() / m.shape[0] for m in metas[0][0]['depth_mask']]))
        res = dict(bench='novel_depth', geometry=name, card=card, power_limit_w=power, cameras=N, ray_grid=[h, w], sources=S,
                   lidar_points_per_source=g['points'], masked_points_per_camera=round(visible), frames=args.frames,
                   ref_step_ms=round(med('ref'), 3), native_step_ms=round(med('nat'), 3),
                   speedup=round(med('ref') / med('nat'), 2), render_poses_ms=round(med('render'), 3),
                   ref_host_syncs=sync_ref, native_host_syncs=sync_nat, same_bins_and_counts=bool(same_bins),
                   max_rel_diff=rel)
        line = json.dumps(res)
        print(line, flush=True)
        lines.append(line)
        del head, maps, metric
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write('\n'.join(lines) + '\n')


if __name__ == '__main__':
    main()
