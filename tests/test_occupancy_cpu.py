"""CPU: occupancy evaluation pinned to the reference's metric classes (tests/golden/reference_golden_occ.npz) -- the oracle's
counters, the LUTs, the confusion-matrix -> counter derivation of the device metrics, the lattice geometry and the C ABI's
error paths."""
import ctypes as C
import os
import numpy as np
import pytest
import torch

from oracle import occupancy as oocc
from oracle.render import uniform_lattice
from selfocc_b200 import occupancy
from selfocc_b200.metric import counts_from_confusion, iou_score, meaniou_scores, ssc_stats

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_golden_occ.npz'))
STEPS = 2


def _step(s):
    t = lambda k: torch.from_numpy(G['step%d_%s' % (s, k)]) if 'step%d_%s' % (s, k) in G else None
    return {k: t(k) for k in ('sem_gt', 'sem_pred', 'mask', 'occ_gt', 'occ_pred', 'kitti_gt', 'nonempty')}


def _kitti_points(x):
    k = x['kitti_gt'].clone()
    k[k == 255] = 0
    return torch.nonzero(k)


def test_luts_equal_the_reference():
    assert list(G['lut_openseed2nuscenes']) == list(occupancy.OPENSEED2NUSCENES)
    assert list(G['lut_cityscapes2semantickitti']) == list(occupancy.CITYSCAPES2SEMANTICKITTI)


def test_oracle_counters_equal_the_reference():
    m1 = m16 = iou = ssc = None
    add = lambda a, b: b if a is None else tuple(x + y for x, y in zip(a, b))
    for s in range(STEPS):
        x = _step(s)
        m1 = add(m1, oocc.meaniou_counts_ref(x['occ_pred'], x['occ_gt'], x['mask'], [1], 0))
        m16 = add(m16, oocc.meaniou_counts_ref(x['sem_pred'], x['sem_gt'], x['mask'], list(range(1, 17)), 0))
        iou = add(iou, oocc.iou_counts_ref(x['occ_pred'], _kitti_points(x)))
        ssc = add(ssc, oocc.ssc_counts_ref(x['occ_pred'], x['kitti_gt'], 2, x['nonempty']))
    for tag, c in (('miou1', m1), ('miou16', m16)):
        for k, v in zip(('total_seen', 'total_correct', 'total_positive'), c):
            assert np.array_equal(v.numpy(), G['%s_%s' % (tag, k)]), (tag, k)
    for k, v in zip(('total_seen', 'total_correct', 'total_positive'), iou):
        assert v == G['iou_' + k][0], k
    for k, v in zip(('completion_tp', 'completion_fp', 'completion_fn', 'tps', 'fps', 'fns'), ssc):
        assert np.array_equal(np.atleast_1d(np.asarray(v)), G['ssc_' + k]), k


def test_confusion_derivation_reproduces_the_reference_numbers():
    """What the device metrics compute after their confusion kernel, fed a CPU-counted confusion matrix."""
    cm1 = cm16 = cmi = cms = 0
    for s in range(STEPS):
        x = _step(s)
        cm1 = cm1 + oocc.confusion_ref(x['occ_pred'], x['occ_gt'], 2, mask=x['mask'])
        cm16 = cm16 + oocc.confusion_ref(x['sem_pred'], x['sem_gt'], 17, mask=x['mask'])
        occ_gt = torch.zeros_like(x['occ_pred'])
        occ_gt[tuple(_kitti_points(x).t())] = 1
        cmi = cmi + oocc.confusion_ref(x['occ_pred'], occ_gt, 1)
        cms = cms + oocc.confusion_ref(x['occ_pred'], x['kitti_gt'], 2, mask=x['nonempty'], ignore=255)
    for tag, cm, classes in (('miou1', cm1, [1]), ('miou16', cm16, list(range(1, 17)))):
        counts = counts_from_confusion(cm, classes, 0)
        for k, v in zip(('total_seen', 'total_correct', 'total_positive'), counts):
            assert np.array_equal(v.numpy(), G['%s_%s' % (tag, k)]), (tag, k)
        miou, occ_iou = meaniou_scores(*counts)[:2]
        assert miou == pytest.approx(float(G[tag + '_miou']), rel=1e-6)
        assert occ_iou == pytest.approx(float(G[tag + '_occ_iou']), rel=1e-6)
    seen, correct, positive = counts_from_confusion(cmi, [], 0)
    assert [int(seen), int(correct), int(positive)] == [int(G['iou_total_' + k][0]) for k in ('seen', 'correct', 'positive')]
    assert iou_score(seen, correct, positive) == pytest.approx(float(G['iou_iou']), rel=1e-6)
    counts = counts_from_confusion(cms, range(2), 0)
    seen, correct, positive = counts
    assert np.array_equal(correct[:-1].numpy(), G['ssc_tps'])
    assert np.array_equal((positive - correct)[:-1].numpy(), G['ssc_fps'])
    assert np.array_equal((seen - correct)[:-1].numpy(), G['ssc_fns'])
    assert [int(correct[-1]), int(positive[-1] - correct[-1]), int(seen[-1] - correct[-1])] == \
        [int(G['ssc_completion_' + k][0]) for k in ('tp', 'fp', 'fn')]
    st = ssc_stats(*counts)
    for k in ('precision', 'recall', 'iou', 'iou_ssc', 'iou_ssc_mean'):
        assert np.allclose(np.asarray(st[k], dtype=np.float64), G['ssc_' + k], rtol=1e-6, atol=0), k


@pytest.mark.parametrize('aabb,res,shape', [([-40.0, -40.0, -1.0, 40.0, 40.0, 5.4], 0.2, (400, 400, 32)),
                                            ([-51.2, -51.2, -5, 51.2, 51.2, 3], 0.2, (512, 512, 40)),
                                            ([-25.6, 0, -2.0, 25.6, 51.2, 4.4], 0.2, (256, 256, 32))])
def test_lattice_axes_match_get_uniform_sdf(aabb, res, shape):
    """Occ3D (scene_size 4), OpenOccupancy and SemanticKITTI lattices: sizes and coordinates of neus_head.py:266-277."""
    xs, ys, zs = occupancy.lattice_axes(aabb, res)
    assert (len(ys), len(xs), len(zs)) == shape
    xyz = uniform_lattice(aabb, res)
    assert torch.equal(xyz[0, :, 0, 0], xs) and torch.equal(xyz[:, 0, 0, 1], ys) and torch.equal(xyz[0, 0, :, 2], zs)


def test_occupancy_entry_points_reject_bad_arguments_without_a_gpu():
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N, one = None, C.c_void_p(16)
    d = _lib.VolumeDesc()
    d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch = 9, 9, 5, 8, 24, 24
    for i in range(3):
        d.axis[i].range0, d.axis[i].size0 = 1.0, 4.0
    D = C.byref(d)
    lat = lambda nx=4, ny=4, nz=4: (one, nx, one, ny, one, nz)
    assert lib.so_occ_lattice_labels(N, N, D, *lat(), 0.0, 3, 21, N, one, one, N) == -1          # no volume
    assert lib.so_occ_lattice_labels(one, one, D, *lat(), 0.0, 3, 21, N, N, one, N) == -1        # no occ output
    assert lib.so_occ_lattice_labels(one, one, D, *lat(nx=0), 0.0, 3, 21, N, one, one, N) == -1  # empty lattice axis
    assert lib.so_occ_lattice_labels(one, one, None, *lat(), 0.0, 3, 21, N, one, one, N) == -1   # no descriptor
    assert lib.so_occ_lattice_labels(one, N, D, *lat(), 0.0, 3, 21, N, one, one, N) == -1        # semantics, no features
    assert lib.so_occ_lattice_labels(one, one, D, *lat(), 0.0, 4, 21, N, one, one, N) == -1      # channels beyond n_feat
    assert lib.so_occ_lattice_labels(one, one, D, *lat(), 0.0, 3, 0, N, one, one, N) == -1       # no semantic channel
    assert lib.so_occ_lattice_labels(one, one, D, *lat(), 0.0, -1, 21, N, one, one, N) == -1
    assert lib.so_occ_lattice_labels(one, one, D, *lat(2048, 2048, 1024), 0.0, 3, 21, N, one, one, N) == -2   # > 2^31 points
    assert lib.so_occ_sample_labels(one, one, D, *lat(), N, 10, 0.0, 3, 21, N, one, one, N) == -1   # no points
    assert lib.so_occ_sample_labels(one, one, D, *lat(), one, 0, 0.0, 3, 21, N, one, one, N) == -1  # m < 1
    assert lib.so_occ_sample_labels(one, one, D, *lat(), one, 10, 0.0, 3, 22, N, one, one, N) == -1  # channels beyond n_feat
    assert lib.so_occ_confusion(N, one, N, 10, 2, -1, one, N) == -1
    assert lib.so_occ_confusion(one, one, N, 10, 2, -1, N, N) == -1
    assert lib.so_occ_confusion(one, one, N, 0, 2, -1, one, N) == -1          # n < 1
    assert lib.so_occ_confusion(one, one, N, 10, 0, -1, one, N) == -1         # n_cls out of range
    assert lib.so_occ_confusion(one, one, N, 10, 256, -1, one, N) == -1
    assert lib.so_occ_confusion(one, one, N, 10, 2, 256, one, N) == -1        # ignore out of range
    assert lib.so_occ_confusion(one, one, N, 10, 2, -2, one, N) == -1
