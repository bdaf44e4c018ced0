"""Generate tests/golden/reference_golden_occ.npz from the reference's occupancy metrics.

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored vectors):
    python tests/golden/make_golden_occ.py <path to the SelfOcc checkout>
utils/metric_util.py and utils/scenerf_metric.py are loaded by file path and executed unmodified, with three stand-ins:
an ``mmengine`` module whose MMLogger hands out a standard logger, ``Tensor.cuda`` as the identity (the run is on the CPU)
and a single-process gloo group (IoU._after_epoch and SSCMetrics.get_stats call torch.distributed unconditionally).
"""
import importlib.util
import logging
import os
import sys
import tempfile
import types
import numpy as np
import torch

REF = next((a for a in sys.argv[1:] if not a.startswith('--')), None)   # the SelfOcc checkout (required)
HERE = os.path.dirname(os.path.abspath(__file__))
SHAPE = (40, 40, 8)
STEPS = 2
NUSC_NAMES = ['barrier', 'bicycle', 'bus', 'car', 'construction_vehicle', 'motorcycle', 'pedestrian', 'traffic_cone',
              'trailer', 'truck', 'driveable_surface', 'other_flat', 'sidewalk', 'terrain', 'manmade', 'vegetation']


def inputs(step):
    """Seeded label volumes of one step (shared with tests/test_occupancy_cpu.py through the stored arrays):
    sem_pred / sem_gt 0..16 with out-of-range predictions (17, 20, 200), 255 in the ground truth, class 5 never in the
    ground truth and class 9 never predicted; occ_pred / occ_gt 0/1; mask; kitti_gt 0..19 with 255 (ignored by SSCMetrics);
    nonempty (step 1 only)."""
    g = torch.Generator().manual_seed(100 + step)
    n = int(np.prod(SHAPE))
    sem_gt = torch.randint(0, 17, (n,), generator=g)
    sem_gt[torch.rand(n, generator=g) < 0.45] = 0
    sem_gt[sem_gt == 5] = 6
    sem_gt[torch.rand(n, generator=g) < 0.03] = 255
    keep = torch.rand(n, generator=g) < 0.6
    sem_pred = torch.where(keep, sem_gt, torch.randint(0, 17, (n,), generator=g))
    sem_pred[sem_pred == 255] = 0
    sem_pred[sem_pred == 9] = 10
    odd = torch.rand(n, generator=g)
    sem_pred[odd < 0.01] = 17
    sem_pred[(odd >= 0.01) & (odd < 0.015)] = 20
    sem_pred[(odd >= 0.015) & (odd < 0.02)] = 200
    mask = torch.rand(n, generator=g) < 0.8
    occ_gt = ((sem_gt > 0) & (sem_gt != 255)).to(torch.int)
    occ_pred = torch.where(torch.rand(n, generator=g) < 0.8, occ_gt, 1 - occ_gt).to(torch.int)
    kitti_gt = torch.randint(0, 20, (n,), generator=g).to(torch.uint8)
    kitti_gt[torch.rand(n, generator=g) < 0.5] = 0
    kitti_gt[torch.rand(n, generator=g) < 0.05] = 255
    nonempty = torch.rand(n, generator=g) < 0.7
    r = lambda t: t.reshape(SHAPE)
    return dict(sem_gt=r(sem_gt).to(torch.int64), sem_pred=r(sem_pred).to(torch.int64), mask=r(mask), occ_gt=r(occ_gt),
                occ_pred=r(occ_pred), kitti_gt=r(kitti_gt), nonempty=r(nonempty) if step == 1 else None)


def occ_golden():
    mm = types.ModuleType('mmengine')
    mm.MMLogger = type('MMLogger', (), {'get_instance': staticmethod(lambda name: logging.getLogger(name))})
    sys.modules['mmengine'] = mm
    torch.Tensor.cuda = lambda self, *a, **k: self
    import torch.distributed as dist
    store = tempfile.mktemp(prefix='golden_occ_store')
    dist.init_process_group('gloo', init_method='file://' + store, rank=0, world_size=1)

    def load(rel, name):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    mu = load('utils/metric_util.py', 'ref_metric_util')
    sm = load('utils/scenerf_metric.py', 'ref_scenerf_metric')

    out = {'lut_openseed2nuscenes': mu.openseed2nuscenes(torch.arange(21)).numpy(),
           'lut_cityscapes2semantickitti': mu.cityscapes2semantickitti(torch.arange(19)).numpy()}
    iou1 = mu.MeanIoU([1], 0, ['occupied'], True, 0)
    miou16 = mu.MeanIoU(list(range(1, 17)), 0, NUSC_NAMES, True, 0)
    iou = mu.IoU()
    ssc = sm.SSCMetrics(2)
    for m in (iou1, miou16, iou):
        m.reset()
    for step in range(STEPS):
        x = inputs(step)
        for k, v in x.items():
            if v is not None:
                out['step%d_%s' % (step, k)] = v.numpy()
        iou1._after_step(x['occ_pred'], x['occ_gt'], x['mask'])
        miou16._after_step(x['sem_pred'], x['sem_gt'], x['mask'])
        kitti = x['kitti_gt'].clone()
        kitti[kitti == 255] = 0
        iou._after_step(x['occ_pred'], torch.nonzero(kitti))
        ssc.add_batch(x['occ_pred'], x['kitti_gt'].clone(), x['nonempty'])
    for tag, m in (('miou1', iou1), ('miou16', miou16)):
        miou, occ_iou = m._after_epoch()
        out[tag + '_miou'], out[tag + '_occ_iou'] = np.array(miou), np.array(float(occ_iou))
        for k in ('total_seen', 'total_correct', 'total_positive'):
            out['%s_%s' % (tag, k)] = getattr(m, k).numpy()
    out['iou_iou'] = np.array(iou._after_epoch())
    for k in ('total_seen', 'total_correct', 'total_positive'):
        out['iou_' + k] = getattr(iou, k).numpy()
    stats = ssc.get_stats()
    for k, v in stats.items():
        out['ssc_' + k] = np.asarray(v.numpy() if torch.is_tensor(v) else v, dtype=np.float64)
    for k in ('completion_tp', 'completion_fp', 'completion_fn', 'tps', 'fps', 'fns'):
        out['ssc_' + k] = getattr(ssc, k).numpy()
    dist.destroy_process_group()
    np.savez_compressed(os.path.join(HERE, 'reference_golden_occ.npz'), **out)
    print('wrote occupancy golden:', len(out), 'arrays')


if __name__ == '__main__':
    if REF is None or not os.path.isfile(os.path.join(REF, 'utils', 'scenerf_metric.py')):
        sys.exit('usage: python tests/golden/make_golden_occ.py <path to a huang-yh/SelfOcc checkout>')
    occ_golden()
