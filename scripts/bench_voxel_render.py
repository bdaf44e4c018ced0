"""Time the voxel-cube picture on one GPU: so_voxel_render on the Occ3D 200 x 200 x 16 grid and the KITTI 256 x 256 x 32
lattice at 2560 x 1440, one view and 8 views per launch, and head.occupancy -> render end to end; and the fp64 oracle's
CPU time at a reduced size for scale.

    python scripts/bench_voxel_render.py [--iters 20] [--out /tmp/voxel_render/bench.json]

Labels come from head.occupancy of a random-weight head at each config's geometry (about 30 % of the lattice occupied).
Times are CUDA-event means over --iters launches after a warm-up; the card's name and power limit are printed with them.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from selfocc_b200 import occupancy as occ_mod, synth, voxel_vis as vv  # noqa: E402
from selfocc_b200.registry import build_head  # noqa: E402
import selfocc_b200.segmentor  # noqa: F401,E402

CFGS = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'reference_model_cfgs.json')))


def _head(kind, dev, occupied=0.3):
    cfg = CFGS['nuscenes/nuscenes_occ.py' if kind == 'occ3d' else 'kitti/kitti_occ.py']['head']
    over = {} if kind == 'occ3d' else dict(color_dims=3 + 19, return_sem=True)
    head = build_head(dict(cfg, return_second_grad=False, **over)).eval().to(dev)
    f = head.model.field
    rep = [p[None].to(dev) for p in synth.random_planes(f.mapping, 96, scale=1.0, seed=5)]
    w1, b1, w2, b2 = synth.random_mlp(96, f.density_net[3].out_features, seed=2)
    with torch.no_grad():
        for lin, w, b in ((f.density_net[1], w1, b1), (f.density_net[3], w2, b2)):
            lin.weight.copy_(w); lin.bias.copy_(b)
        head.prepare(rep)
        q = torch.quantile(f.vol_sdf[..., :f.desc.Z].flatten()[::7], occupied)
        f.density_net[3].bias[::1 + f.color_dims] -= q
        head.prepare(rep)                               # decode again with the shifted bias
    return head, cfg['roi_aabb']


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def _views(kind, n):
    rng = np.random.default_rng(0)
    first = vv.VIS3D_NUSCENES if kind == 'occ3d' else vv.kitti_camera(
        dict(cam_positions=[[0.3, -6.0, 9.0]], focal_positions=[[0.3, 8.0, 1.0]]))
    cams = [first]
    centre = np.array([0.0, 0.0, 2.0]) if kind == 'occ3d' else np.array([0.0, 25.6, 1.2])
    while len(cams) < n:
        a = rng.uniform(0, 2 * np.pi)
        cams.append(vv.look_at(centre + np.array([60 * np.cos(a), 60 * np.sin(a), 45.0]), centre, (0, 0, 1), 30.0))
    return cams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_voxel_render needs a GPU')
    dev = torch.device('cuda:0')
    try:
        card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True).stdout.strip()
    except OSError:
        card = torch.cuda.get_device_name(0)
    print('device:', card)
    size = vv.IMAGE_SIZE
    res = dict(device=card, image_size=size, iters=args.iters, rows=[])
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    for kind in ('occ3d', 'kitti'):
        head, aabb = _head(kind, dev)
        if kind == 'occ3d':
            pts = occ_mod.occ3d_lidar_points(torch.eye(4), dev)
            occ_args = dict(aabb=aabb, resolution=0.4, thresh=0.0, lut=occ_mod.OPENSEED2NUSCENES, points=pts)
            origin, vs, pal = (-40.0, -40.0, -1.0), 0.4, vv.NUSCENES_PALETTE
        else:
            occ_args = dict(aabb=aabb, resolution=0.2, thresh=0.0, lut=occ_mod.CITYSCAPES2SEMANTICKITTI)
            origin, vs, pal = tuple(aabb[:3]), 0.2, vv.KITTI_PALETTE
        _, labels = head.render_occupancy(cameras=[_views(kind, 1)[0]], image_size=(8, 8), palette=pal, **occ_args)
        drawn = float((torch.as_tensor(vv.drawn_table(pal), device=dev)[labels.long()] != 0).float().mean())
        for n in (1, 8):
            cams = _views(kind, n)
            rows = vv.camera_rows([c.resized(size) for c in cams], dev)
            out = vv.render_voxels(labels, origin, vs, rows, size, pal)
            hit = float((out['rgb'] != 255).any(-1).float().mean())
            t_render = _time(lambda: vv.render_voxels(labels, origin, vs, rows, size, pal), args.iters)
            t_e2e = _time(lambda: head.render_occupancy(cameras=rows, image_size=size, palette=pal, **occ_args), args.iters)
            row = dict(grid=kind, shape=list(labels.shape), drawn_fraction=drawn, views=n, hit_fraction=hit,
                       render_ms=t_render, render_ms_per_view=t_render / n, end_to_end_ms=t_e2e)
            res['rows'].append(row)
            print('%-5s %-13s drawn %.2f  %d view(s) at %dx%d: render %.3f ms (%.3f ms/view), occupancy+render %.3f ms, '
                  '%.0f%% pixels hit' % (kind, tuple(labels.shape), drawn, n, size[1], size[0], t_render, t_render / n,
                                         t_e2e, 100 * hit))
        if args.out:                                    # the first view as a picture, next to the JSON
            vv.write_png(os.path.join(os.path.dirname(os.path.abspath(args.out)), 'voxel_render_%s.png' % kind),
                         vv.render_voxels(labels, origin, vs, _views(kind, 1), size, pal)['rgb'][0])
    # the fp64 oracle at a reduced size, for scale
    from oracle import voxel_vis as ref
    lab = labels.cpu().numpy()
    small = (18, 32)
    o, d, near, far = ref.rays_from_rows(vv.camera_rows([_views('kitti', 1)[0].resized(small)], dev).cpu().numpy(), small)
    t0 = time.perf_counter()
    ref.render_ref(lab, origin, vs, o[0], d[0].reshape(-1, 3), near[0], far[0], vv.drawn_table(pal).astype(bool))
    t_ref = time.perf_counter() - t0
    res['oracle_cpu_s'] = dict(grid='kitti', image_size=small, seconds=t_ref)
    print('fp64 oracle (CPU), kitti grid, one view at %dx%d: %.2f s' % (small[1], small[0], t_ref))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
