"""Occupancy evaluation per frame: the reference composition vs head.occupancy + the device metrics, at the geometries of
eval_iou.py (Occ3D scene_size 4, OpenOccupancy) and eval_iou_kitti.py (SemanticKITTI), on a decoded synthetic volume of each
config's size.  Prints one JSON line (and writes it to --out if given).

  (a) reference: forward_occ (the whole lattice of field outputs), then the fp32 torch composition of the script
      (threshold, grid_sample / argmax / LUT, crops) and the reference metric classes restated below with their
      host reads (.item() / .tolist() / boolean-mask indexing);
  (b) native:    head.occupancy (byte labels from the decoded volume) + the same crops + selfocc_b200.metric.

The two paths run alternately after warm-up, each frame from the TPV planes (both decode the volume).  Reported per
geometry: median CUDA-event time per frame, host wall time per frame, peak memory allocated above the inputs (the TPV
planes; both paths hold the decoded volume, reported beside it), host
synchronisations per frame (torch.cuda sync-debug warnings) and the agreement of the two paths' labels.  The card's name
and power limit are read in the same run.
"""
import argparse
import json
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
                     w_range=[25.6, 0], w_half=False, d_size=[32, 0], d_range=[-2.0, 4.4, 4.4])   # config/kitti/kitti_occ.py
NUSC_NAMES16 = ['c%d' % i for i in range(16)]


# ---------------------------------------------------------------- reference metric classes (utils/metric_util.py,
# utils/scenerf_metric.py), restated with their per-step host reads; distributed reduction left out (one process)
class RefMeanIoU:
    def __init__(self, class_indices, empty_label):
        self.class_indices, self.empty_label = class_indices, empty_label
        n = len(class_indices) + 1
        self.total_seen, self.total_correct, self.total_positive = (torch.zeros(n).cuda() for _ in range(3))

    def _after_step(self, outputs, targets, mask=None):
        if mask is not None:
            outputs, targets = outputs[mask], targets[mask]
        for i, c in enumerate(self.class_indices):
            self.total_seen[i] += torch.sum(targets == c).item()
            self.total_correct[i] += torch.sum((targets == c) & (outputs == c)).item()
            self.total_positive[i] += torch.sum(outputs == c).item()
        e = self.empty_label
        self.total_seen[-1] += torch.sum(targets != e).item()
        self.total_correct[-1] += torch.sum((targets != e) & (outputs != e)).item()
        self.total_positive[-1] += torch.sum(outputs != e).item()


class RefIoU:
    def __init__(self):
        self.total_seen, self.total_correct, self.total_positive = (torch.zeros(1).cuda() for _ in range(3))

    def _after_step(self, outputs, targets):
        self.total_seen[0] += targets.shape[0]
        self.total_correct[0] += outputs[tuple(targets.transpose(0, 1).tolist())].sum()
        self.total_positive[0] += outputs.sum()


class RefSSC:
    def __init__(self, n_classes):
        self.n = n_classes
        self.tp, self.fp, self.fn = (torch.zeros(1).cuda() for _ in range(3))
        self.tps, self.fps, self.fns = (torch.zeros(n_classes).cuda() for _ in range(3))

    def add_batch(self, y_pred, y_true):
        mask = y_true != 255
        p, t = y_pred.clone(), y_true.clone()
        p[t == 255] = 0
        t[t == 255] = 0
        bp, bt = torch.zeros(p.shape).cuda(), torch.zeros(t.shape).cuda()
        bp[p > 0] = 1
        bt[t > 0] = 1
        bt, bp = bt[mask], bp[mask]
        self.tp += torch.logical_and(bt == 1, bp == 1).sum()
        self.fp += torch.logical_and(bt != 1, bp == 1).sum()
        self.fn += torch.logical_and(bt == 1, bp != 1).sum()
        yt, yp = t[mask], p[mask]
        for j in range(self.n):
            self.tps[j] += torch.logical_and(yt == j, yp == j).sum()
            self.fps[j] += torch.logical_and(yt != j, yp == j).sum()
            self.fns[j] += torch.logical_and(yt == j, yp != j).sum()


# ---------------------------------------------------------------- geometries
def _geometries():
    from selfocc_b200 import synth
    return {
        'occ3d': dict(mapping=synth.NUSC_MAPPING, color_dims=24, aabb=[-40.0, -40.0, -1.0, 40.0, 40.0, 5.4],
                      expansion=[80.0, 80.0, 6.4], resample=True),
        'openoccupancy': dict(mapping=synth.NUSC_MAPPING, color_dims=24, aabb=[-51.2, -51.2, -5, 51.2, 51.2, 3], resample=False),
        'semantickitti': dict(mapping=KITTI_MAPPING, color_dims=3, aabb=[-25.6, 0, -2.0, 25.6, 51.2, 4.4], resample=False),
    }


def _setup(name, g, dev):
    from selfocc_b200 import configs, occupancy as occ_mod, synth
    from selfocc_b200.mapping import GridMeterMapping
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    sem = g['color_dims'] > 3
    cfg = configs.hot_path_config(mapping_args=g['mapping'], pc_range=g['aabb'], num_layers=1, color_dims=g['color_dims'],
                                  return_sem=sem)
    head = build_head(cfg).head.eval()
    m = GridMeterMapping(**g['mapping'])
    w1, b1, w2, b2 = synth.random_mlp(96, 1 + g['color_dims'], seed=2)
    planes = [p[None].to(dev) for p in synth.random_planes(m, 96, scale=1.0, seed=5)]
    with torch.no_grad():
        f = head.model.field
        for lin, w, b in ((f.density_net[1], w1, b1), (f.density_net[3], w2, b2)):
            lin.weight.copy_(w); lin.bias.copy_(b)
        head.to(dev)
        # shift the sdf bias so that 30 % of the voxels are occupied (the random decoder alone puts the whole volume on one
        # side of the surface; a real scene is mostly free space)
        head.prepare(planes)
        f.density_net[3].bias[0] -= torch.quantile(f.vol_sdf[..., :f.desc.Z].flatten()[::7], 0.3)
        head.prepare(planes)
        vol_mib = (f.vol_sdf.numel() + (0 if f.vol_feat is None else f.vol_feat.numel())) * 4 / 2 ** 20
    gen = torch.Generator(device=dev).manual_seed(1)
    xs, ys, zs = occ_mod.lattice_axes(g['aabb'], 0.2)
    shape = (200, 200, 16) if g['resample'] else (len(ys), len(xs), len(zs))
    gt = torch.randint(0, 17, shape, device=dev, generator=gen).to(torch.uint8)
    gt[torch.rand(shape, device=dev, generator=gen) < 0.6] = 0
    data = dict(planes=planes, gt=gt, mask=torch.rand(shape, device=dev, generator=gen) < 0.8, vol_mib=vol_mib)
    if g['resample']:
        a = np.deg2rad(3.0)
        e2l = np.eye(4)
        e2l[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
        e2l[:3, 3] = [0.9, 0.0, 1.8]
        data['e2l'] = torch.tensor(e2l, dtype=torch.float32, device=dev)
    if name == 'semantickitti':
        gt[torch.rand(shape, device=dev, generator=gen) < 0.05] = 255
        k = gt.clone()
        k[k == 255] = 0
        data['points'] = torch.nonzero(k)
    return head, data


def _crop(pred, name):
    if name == 'occ3d':           # eval_iou.py:222-227
        pred[..., 12:] = 0; pred[:6] = 0; pred[-6:] = 0; pred[:, :6] = 0; pred[:, -6:] = 0
    elif name == 'openoccupancy':  # eval_iou.py:253-258
        pred[..., -4:] = 0; pred[..., :5] = 0; pred[:6] = 0; pred[-6:] = 0; pred[:, :6] = 0; pred[:, -6:] = 0
    else:                         # eval_iou_kitti.py:179-183
        pred[..., 28:] = 0; pred[-6:] = 0; pred[:, :6] = 0; pred[:, -6:] = 0
    return pred


def _lut(name):
    from selfocc_b200 import occupancy as occ_mod
    return occ_mod.OPENSEED2NUSCENES if name != 'semantickitti' else None


def frame_reference(name, g, head, data, metrics):
    aabb = g['aabb']
    out = head.forward_occ(data['planes'], aabb=aabb, resolution=0.2)
    pred = (out['sdf'] <= 0.0).to(torch.int)
    sem = None
    if g['resample']:
        from selfocc_b200 import occupancy as occ_mod
        lp = occ_mod.occ3d_lidar_points(data['e2l'], pred.device).reshape(-1, 3)
        for i in range(3):
            lp[:, i] = (lp[:, i] - aabb[i]) / g['expansion'][i]
        lp = lp.reshape(1, 200, 200, 16, 3)
        s = F.grid_sample(out['sdf'][None, None], lp[..., [2, 0, 1]] * 2 - 1, mode='bilinear', align_corners=True)
        pred = (s.squeeze() <= 0.0).to(torch.int)
        lg = F.grid_sample(out['logits'].permute(3, 0, 1, 2)[None], lp[..., [2, 0, 1]] * 2 - 1, mode='bilinear', align_corners=True)
        sem = torch.argmax(lg, dim=1).squeeze()
    elif 'sem' in out:
        sem = out['sem']
    pred = _crop(pred, name)
    if name == 'semantickitti':
        metrics[0]._after_step(pred, data['points'])
        metrics[1].add_batch(pred, data['gt'])
        return pred, None
    lut = torch.tensor(_lut(name), device=pred.device)
    sem = pred * lut[sem.flatten()].reshape(sem.shape)
    gt = data['gt'].to(torch.int)
    metrics[0]._after_step(pred, (gt > 0).to(torch.int), data['mask'])
    metrics[1]._after_step(sem, gt, data['mask'])
    return pred, sem


def frame_native(name, g, head, data, metrics):
    kw = {}
    if g['resample']:
        from selfocc_b200 import occupancy as occ_mod
        kw = dict(points=occ_mod.occ3d_lidar_points(data['e2l'], data['gt'].device), expansion=g['expansion'])
    out = head.occupancy(g['aabb'], 0.2, lut=_lut(name), representation=data['planes'], **kw)
    pred = _crop(out['occ'], name)
    if name == 'semantickitti':
        metrics[0]._after_step(pred, data['points'])
        metrics[1].add_batch(pred, data['gt'])
        return pred, None
    sem = _crop(out['sem'], name)
    metrics[0]._after_step(pred, data['gt'] > 0, data['mask'])
    metrics[1]._after_step(sem, data['gt'], data['mask'])
    return pred, sem


def _metrics(name, native, dev):
    from selfocc_b200 import metric
    if name == 'semantickitti':
        if native:
            m = metric.IoU().to(dev)
            m.reset()
            return [m, metric.SSCMetrics(2)]
        return [RefIoU(), RefSSC(2)]
    if native:
        ms = [metric.MeanIoU([1], 0, ['occupied'], True, 0), metric.MeanIoU(list(range(1, 17)), 0, NUSC_NAMES16, True, 0)]
        for m in ms:
            m.reset()
        return ms
    return [RefMeanIoU([1], 0), RefMeanIoU(list(range(1, 17)), 0)]


def _timed(fn):
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    res = fn()
    e1.record()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3
    return e0.elapsed_time(e1), wall, (torch.cuda.max_memory_allocated() - base) / 2 ** 20, res


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
    ap.add_argument('--frames', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--only', default=None, help='comma-separated geometries')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_occ_eval.py measures on the GPU; no CUDA device found')
    from selfocc_b200.occupancy import lattice_axes as occ_axes
    dev = torch.device('cuda:0')
    card, power = _card()
    res = {'card': card, 'power_limit_w': power, 'frames': args.frames, 'geometries': {}}
    for name, g in _geometries().items():
        if args.only and name not in args.only.split(','):
            continue
        head, data = _setup(name, g, dev)
        ref_m, nat_m = _metrics(name, False, dev), _metrics(name, True, dev)
        ref = lambda: frame_reference(name, g, head, data, ref_m)
        nat = lambda: frame_native(name, g, head, data, nat_m)
        with torch.no_grad():
            for _ in range(args.warmup):
                ref(); nat()
            t = {'ref': [], 'nat': []}
            for _ in range(args.frames):
                for k, fn in (('ref', ref), ('nat', nat)):
                    t[k].append(_timed(fn))
            sync_ref, sync_nat = _syncs(ref), _syncs(nat)
            (pr, sr), (pn, sn) = ref(), nat()
        agree = float((pr.to(torch.uint8) == pn).float().mean())
        if sr is not None:
            agree = min(agree, float((sr.to(torch.uint8) == sn).float().mean()))
        med = lambda k, i: statistics.median(x[i] for x in t[k])
        res['geometries'][name] = dict(
            lattice=[len(occ_axes(g['aabb'], 0.2)[i]) for i in (1, 0, 2)],
            labels=[200, 200, 16] if g['resample'] else None,
            ref_ms=round(med('ref', 0), 3), native_ms=round(med('nat', 0), 3), speedup=round(med('ref', 0) / med('nat', 0), 2),
            ref_wall_ms=round(med('ref', 1), 3), native_wall_ms=round(med('nat', 1), 3),
            ref_peak_mib=round(max(x[2] for x in t['ref']), 1), native_peak_mib=round(max(x[2] for x in t['nat']), 1),
            decoded_volume_mib=round(data['vol_mib'], 1), occupied=round(float(pn.float().mean()), 3),
            ref_host_syncs=sync_ref, native_host_syncs=sync_nat, label_agreement=agree)
        del head, data, ref_m, nat_m
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
