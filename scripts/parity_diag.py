#!/usr/bin/env python
"""Where does the depth error at BASELINE size come from?  (VERDICT r1 weak #1: bench parity block max-rel 1.44e-2.)

Renders a strided sub-grid of the bench frame with the CUDA kernels and with the oracle in several
combinations so that a kernel bug, a decode (3xTF32) error and an ill-conditioned ray can be told apart:

  K(tc)    kernel render of the tensor-core-decoded volume          (what bench.py's parity block measured)
  K(simt)  kernel render of the SIMT-decoded volume
  O64      fp64 oracle decode + fp64 oracle render              (the tolerance anchor)
  O64(tc)  fp64 oracle render of the kernel's own decoded volume (isolates the render kernel)
  O32      fp32 oracle decode + render                          (the reference's own arithmetic precision)

Writes gpurun_out/parity_diag.json.  The oracle is the checker here; nothing is timed.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def rel(a, b):
    return ((a - b).abs() / b.abs().clamp_min(1e-6))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='nuscenes_novel_depth_900x1600')
    ap.add_argument('--stride', type=int, default=20)
    ap.add_argument('--scene', default='lifted', choices=['lifted', 'analytic'])
    ap.add_argument('--out', default=os.path.join(ROOT, 'gpurun_out', 'parity_diag.json'))
    a = ap.parse_args()
    from selfocc_b200 import ops, synth, _lib
    from oracle.mapping import GridMeterMappingRef
    from oracle import render as orender, rays as orays
    dev = torch.device('cuda:0')
    lib = _lib.load()
    model, cfg = bench.build_model(a.workload, dev)
    feats, metas, _ = bench.make_frame(a.workload, seed=100)
    feats = [f.to(dev) for f in feats]
    head = model.head
    f = head.model.field
    w = bench.WORKLOADS[a.workload]
    mref = GridMeterMappingRef(**synth.NUSC_MAPPING)
    H, W, Z = mref.size_h, mref.size_w, mref.size_d
    l1, l2 = f.density_net[1], f.density_net[3]
    cpu64 = lambda t: t.detach().cpu().double()
    with torch.no_grad():
        r = model.lifter(ms_img_feats=feats)
        r = model.encoder(representation=r['representation'], ms_img_feats=feats, metas=metas)
        planes = r['representation']
        vols = {}
        for name, simt in (('tc', 0), ('simt', 1)):
            lib.so_tpv_decode_force_simt(simt)
            head.prepare(representation=planes, metas=metas)
            vols[name] = (f.vol_sdf.clone(), None if f.vol_feat is None else f.vol_feat.clone())
        lib.so_tpv_decode_force_simt(0)
    ny, nx = max(w['ray_number'][0] // a.stride, 1), max(w['ray_number'][1] // a.stride, 1)
    H_img, W_img = w['ray_img_size']
    M = head.img2lidar.matrices(metas, dev)[0].contiguous()
    rd = ops.make_ray_desc(M.shape[0], grid=(ny, nx, W_img / nx, 0.0, H_img / ny, 0.0))
    want = ('depth', 'max_idx', 'acc', 'max_depth')
    K = {}
    with torch.no_grad():
        for name in vols:
            K[name] = {k: v.cpu() for k, v in ops.render_infer(vols[name][0], vols[name][1], f.desc, M, rd, head._params(False), want=want).items()}
    torch.set_num_threads(os.cpu_count())
    pl = [cpu64(p[0]) for p in planes]
    wb = [cpu64(t) for t in (l1.weight, l1.bias, l2.weight, l2.bias)]
    vol64 = orender.tpv_decode_ref(pl[0], pl[1], pl[2], (H, W, Z), *wb)
    vol32 = orender.tpv_decode_ref(*[p.float() for p in pl], (H, W, Z), *[t.float() for t in wb])
    vol_tc = vols['tc'][0][..., :Z].cpu().double()[None]          # [1,H,W,Z]
    dec = {'tc_vs_64_max_abs': (vol_tc[0] - vol64[0]).abs().max().item(),
           'simt_vs_64_max_abs': (vols['simt'][0][..., :Z].cpu().double() - vol64[0]).abs().max().item(),
           'o32_vs_64_max_abs': (vol32[0].double() - vol64[0]).abs().max().item(),
           'sdf_abs_max': vol64[0].abs().max().item(), 'sdf_mean': vol64[0].mean().item(), 'sdf_std': vol64[0].std().item()}
    pix = orays.fixed_ray_grid([ny, nx], [H_img, W_img])
    i2l = torch.tensor(np.asarray(metas[0]['img2lidar']), dtype=torch.float32)
    origin, direction = orays.img2lidar_rays(i2l[None], pix)
    inv_s, S, aabb = head._inv_s(), head.num_samples, list(head.aabb)
    O64 = orender.head_render_ref(vol64, mref, origin.double(), direction.double(), aabb, inv_s, S=S)
    O64tc = orender.head_render_ref(vol_tc, mref, origin.double(), direction.double(), aabb, inv_s, S=S)
    O32 = orender.head_render_ref(vol32, mref, origin, direction, aabb, inv_s, S=S)
    flat = lambda d, k: d[k].reshape(-1).double()
    d64, a64 = flat(O64, 'depth'), flat(O64, 'acc')
    res = {'workload': a.workload, 'stride': a.stride, 'rays': int(d64.numel()), 'inv_s': inv_s, 'decode': dec}
    pairs = {'K(tc) vs O64': (K['tc']['depth'].double(), d64), 'K(simt) vs O64': (K['simt']['depth'].double(), d64),
             'K(tc) vs O64(tc)': (K['tc']['depth'].double(), flat(O64tc, 'depth')), 'O32 vs O64': (flat(O32, 'depth'), d64),
             'O64(tc) vs O64': (flat(O64tc, 'depth'), d64)}
    bins = [0, 1e-6, 1e-4, 1e-2, 0.5, 0.99, 2.0]
    for name, (x, y) in pairs.items():
        e = rel(x, y)
        by = {}
        for lo, hi in zip(bins[:-1], bins[1:]):
            m = (a64 >= lo) & (a64 < hi)
            by['acc[%g,%g)' % (lo, hi)] = {'n': int(m.sum()), 'max_rel': float(e[m].max()) if m.any() else None}
        worst = torch.topk(e, 8).indices.tolist()
        res[name] = {'max_rel': float(e.max()), 'n_over_1e-4': int((e > 1e-4).sum()), 'by_acc': by,
                     'worst': [{'ray': i, 'rel': float(e[i]), 'x': float(x[i]), 'y': float(y[i]), 'acc64': float(a64[i]),
                                'idx64': int(O64['max_idx'].reshape(-1)[i])} for i in worst]}
    res['acc'] = {'K(tc) vs O64 max_abs': float((K['tc']['acc'].double() - a64).abs().max()),
                  'O32 vs O64 max_abs': float((flat(O32, 'acc') - a64).abs().max()),
                  'K(tc) vs O64(tc) max_abs': float((K['tc']['acc'].double() - flat(O64tc, 'acc')).abs().max())}
    i64 = O64['max_idx'].reshape(-1)
    res['max_idx'] = {'K(tc)==O64': float((K['tc']['max_idx'] == i64).float().mean()),
                      'K(tc)==O64(tc)': float((K['tc']['max_idx'] == O64tc['max_idx'].reshape(-1)).float().mean()),
                      'O32==O64': float((O32['max_idx'].reshape(-1) == i64).float().mean())}
    # per-sample anatomy of the worst ray of K(tc) vs O64(tc)
    wi = res['K(tc) vs O64(tc)']['worst'][0]['ray']
    ww = O64tc['weights'].reshape(-1, S)[wi]
    res['worst_ray_weights'] = {'ray': wi, 'sum': float(ww.sum()), 'top': [(int(i), float(ww[i])) for i in torch.topk(ww, 6).indices],
                                'sdf_first8': [float(v) for v in O64tc['sdf'].reshape(-1, S)[wi][:8]],
                                'ts_first_last': [float(O64tc['ts'].reshape(-1, S)[wi][0]), float(O64tc['ts'].reshape(-1, S)[wi][-1])]}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    json.dump(res, open(a.out, 'w'), indent=1)
    print(json.dumps({k: (v['max_rel'] if isinstance(v, dict) and 'max_rel' in v else v) for k, v in res.items() if k not in ('worst_ray_weights',)})[:3000])


if __name__ == '__main__':
    main()
