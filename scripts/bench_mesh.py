"""Surface extraction per frame: NeuSHead.mesh (marching cubes over the decoded field, vertex normals / semantics / colour)
against forward_occ, the lattice the reference's 3D visualisation (vis_3d.py, vis_3d_scene.py) builds and then draws as
voxels, at the same geometry and resolution.

Geometries: the nuScenes-occ head (config/nuscenes/nuscenes_occ.py: 25 decoded channels = sdf + 3 rgb + 21 logits) at
0.4, 0.2 and 0.1 m, and the KITTI-occ head (config/kitti/kitti_occ.py: sdf + 3 rgb) at 0.2 and 0.1 m, each from random
TPV planes through a decoder whose sdf bias puts 30 % of the voxels inside.  Both calls decode the planes first, as
forward_occ does.  After warm-up the two alternate; reported per geometry: median CUDA-event time per call (and of
marching_cubes alone on the decoded volume: the two passes and the scans, without the decode and the attributes), peak memory
allocated above the inputs (planes and weights), and the mesh's vertex and face counts.  The card's name and power limit
are read in the same run.  Prints one JSON line (and writes it to --out if given).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch

from selfocc_b200 import mesh as mesh_mod, occupancy

CFG_FILE = os.path.join(ROOT, 'tests', 'golden', 'reference_model_cfgs.json')
GEOMETRIES = {'nusc_occ_0.4': ('nuscenes/nuscenes_occ.py', 0.4), 'nusc_occ_0.2': ('nuscenes/nuscenes_occ.py', 0.2),
              'nusc_occ_0.1': ('nuscenes/nuscenes_occ.py', 0.1), 'kitti_occ_0.2': ('kitti/kitti_occ.py', 0.2),
              'kitti_occ_0.1': ('kitti/kitti_occ.py', 0.1)}


def _card():
    name, power = torch.cuda.get_device_name(0), None
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(', ')
        name, power = q[0], float(q[1])
    except Exception:
        pass
    return name, power


def _setup(cfg_name, dev):
    from selfocc_b200 import synth
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    cfg = json.load(open(CFG_FILE))[cfg_name]['head']
    head = build_head(dict(cfg, return_second_grad=False)).eval().to(dev)
    f = head.model.field
    planes = [p[None].to(dev) for p in synth.random_planes(f.mapping, 96, scale=1.0, seed=5)]
    w1, b1, w2, b2 = synth.random_mlp(96, f.density_net[3].out_features, seed=2)
    with torch.no_grad():
        for lin, w, b in ((f.density_net[1], w1, b1), (f.density_net[3], w2, b2)):
            lin.weight.copy_(w); lin.bias.copy_(b)
        head.prepare(planes)
        f.density_net[3].bias[0] -= torch.quantile(f.vol_sdf[..., :f.desc.Z].flatten()[::7], 0.3)
    return head, planes, cfg['roi_aabb']


def _timed(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return out, a.elapsed_time(b), torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--only', default=None, help='comma-separated geometries')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mesh.py measures on the GPU: no CUDA device')
    dev = torch.device('cuda:0')
    card, power = _card()
    res = {'card': card, 'power_limit_w': power, 'iters': args.iters, 'geometries': {}}
    for name, (cfg_name, reso) in GEOMETRIES.items():
        if args.only and name not in args.only.split(','):
            continue
        head, planes, aabb = _setup(cfg_name, dev)
        mesh = lambda: head.mesh(aabb, reso, representation=planes)
        f = head.model.field
        axes = occupancy.lattice_axes(aabb, reso, dev)
        surface = lambda: mesh_mod.marching_cubes(f.vol_sdf, f.desc, axes)       # count + scans + emit, no attributes
        occ = lambda: head.forward_occ(planes, aabb=aabb, resolution=reso)
        with torch.no_grad():
            for _ in range(args.warmup):
                mesh(); occ(); surface()
            tm, to, ts, mm, mo = [], [], [], 0, 0
            for _ in range(args.iters):
                ts.append(_timed(surface)[1])
                out, t, m = _timed(mesh)
                tm.append(t); mm = max(mm, m)
                v, fc = out['vertices'].shape[0], out['faces'].shape[0]
                del out
                out, t, m = _timed(occ)
                to.append(t); mo = max(mo, m)
                lattice = tuple(out['sdf'].shape)
                del out
        res['geometries'][name] = {
            'config': cfg_name, 'resolution_m': reso, 'lattice': lattice, 'channels': 1 + head.model.field.color_dims,
            'mesh_ms': statistics.median(tm), 'marching_cubes_ms': statistics.median(ts), 'mesh_peak_mb': mm / 2 ** 20, 'vertices': v, 'faces': fc,
            'forward_occ_ms': statistics.median(to), 'forward_occ_peak_mb': mo / 2 ** 20}
        del head, planes
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as fh:
            fh.write(line + '\n')


if __name__ == '__main__':
    main()
