"""GPU: occupancy labels from the decoded field (so_occ_lattice_labels / so_occ_sample_labels) against forward_occ's torch
composition and the fp64 oracle, the confusion kernel against an exact count, and the device metrics against the
reference's numbers (tests/golden/reference_golden_occ.npz), with no host synchronisation per frame."""
import os
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from selfocc_b200 import configs, synth
from selfocc_b200 import occupancy as occ_mod
from selfocc_b200.mapping import GridMeterMapping
from selfocc_b200.registry import build_head
import selfocc_b200.segmentor  # noqa: F401

OCC3D_AABB = [-40.0, -40.0, -1.0, 40.0, 40.0, 5.4]       # eval_iou.py scene_size 4
SMALL_MARGS, SMALL_AABB = synth.small_mapping(8, 4, rng=20.0, z0=-2.0, z1=4.0)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _head(kind, dev):
    """'small': the 17 x 17 x 5 test volume with 3 rgb + 4 semantic channels; 'nusc': a decoded nuscenes_occ-size volume
    (257 x 257 x 31, color_dims = 24: 3 rgb + 21 logits).  -> (head, planes [1, n, C] x 3, mapping, aabb, fp64 volume)"""
    from oracle.mapping import GridMeterMappingRef
    from oracle import render as orender
    margs, aabb, cd, seed = (SMALL_MARGS, SMALL_AABB, 7, 11) if kind == 'small' else (synth.NUSC_MAPPING, OCC3D_AABB, 24, 5)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=None if kind == 'nusc' else aabb, num_layers=1,
                                  color_dims=cd, return_sem=True)
    head = build_head(cfg).head.eval()
    m = GridMeterMapping(**margs)
    planes = synth.random_planes(m, 96, scale=1.0, seed=seed)
    w1, b1, w2, b2 = synth.random_mlp(96, 1 + cd, seed=2)
    _shift_sdf(head, [p[None].to(dev) for p in planes], (w1, b1, w2, b2), dev)
    vol64 = orender.tpv_decode_ref(*[p.double() for p in planes], (m.size_h, m.size_w, m.size_d), w1.double(), b1.double(),
                                   w2.double(), b2.double())
    return head, [p[None].to(dev) for p in planes], GridMeterMappingRef(**margs), aabb, vol64


def _shift_sdf(head, planes, mlp, dev, occupied=0.3):
    """Load the decoder weights and shift the sdf bias (in place, also in ``mlp``) so that the decoded field is <= 0 on
    ``occupied`` of the voxels: the random decoder alone leaves the whole volume on one side of the surface."""
    w1, b1, w2, b2 = mlp
    f = head.model.field
    with torch.no_grad():
        for lin, w, b in ((f.density_net[1], w1, b1), (f.density_net[3], w2, b2)):
            lin.weight.copy_(w); lin.bias.copy_(b)
        head.to(dev)
        head.prepare(planes)
        q = torch.quantile(f.vol_sdf[..., :f.desc.Z].flatten()[::7], occupied).cpu()
        b2[0] -= q
        f.density_net[3].bias.copy_(b2)


def _top2_gap(logits):
    t = logits.topk(2, dim=-1).values
    return t[..., 0] - t[..., 1]


def _check(name, got, ref, band, frac=0.0):
    """Mismatches of got vs ref must lie in ``band`` (bool, same shape) and make up <= frac of the elements."""
    bad = got.cpu() != ref.cpu()
    n_bad, n_out = int(bad.sum()), int((bad & ~band.cpu()).sum())
    print('%s: %d / %d mismatches, %d outside the band' % (name, n_bad, bad.numel(), n_out))
    assert n_out == 0, name
    assert n_bad <= frac * bad.numel(), name


LUT4 = (3, 0, 2, 1)


@pytest.mark.parametrize('kind', ['small', 'nusc'])
def test_lattice_labels_equal_forward_occ(kind):
    dev = _dev()
    head, planes, mref, aabb, _ = _head(kind, dev)
    lut = LUT4 if kind == 'small' else occ_mod.OPENSEED2NUSCENES
    res, thresh = 0.2, (0.05 if kind == 'small' else 0.0)
    out = head.forward_occ(planes, aabb=aabb, resolution=res)
    got = head.occupancy(aabb, res, thresh=thresh, lut=lut)          # the volume forward_occ decoded
    raw = head.occupancy(aabb, res, thresh=thresh, representation=planes)
    ref_occ = (out['sdf'] <= thresh).to(torch.uint8)
    ref_sem = (ref_occ * torch.tensor(lut, device=dev)[out['sem']]).to(torch.uint8)
    assert got['occ'].shape == out['sdf'].shape and got['occ'].dtype == torch.uint8
    band_s = (out['sdf'] - thresh).abs() < 1e-6
    band_l = band_s | (_top2_gap(out['logits']) < 1e-6)
    _check('%s occ' % kind, got['occ'], ref_occ, band_s)
    _check('%s sem' % kind, got['sem'], ref_sem, band_l)
    _check('%s sem (raw argmax)' % kind, raw['sem'], (ref_occ * out['sem']).to(torch.uint8), band_l)
    assert torch.equal(raw['occ'], got['occ'])
    if kind == 'nusc':
        assert got['occ'].shape == (400, 400, 32)
        assert 0.02 < got['occ'].float().mean() < 0.98 and got['sem'].unique().numel() > 8    # a non-degenerate scene


@pytest.mark.parametrize('kind', ['small', 'nusc'])
def test_lattice_labels_match_fp64_oracle(kind):
    """Mismatches only where the fp64 value sits within 1e-5 of the decision (or within the fp32 field's own error of it),
    and at most 1e-4 of the lattice points (a random subset of 200 000 points at the nuscenes_occ size)."""
    dev = _dev()
    from oracle import occupancy as oocc
    head, planes, mref, aabb, vol64 = _head(kind, dev)
    lut = LUT4 if kind == 'small' else occ_mod.OPENSEED2NUSCENES
    res = 0.2
    head.prepare(planes)
    got = head.occupancy(aabb, res, lut=lut)
    out = head.forward_occ(planes, aabb=aabb, resolution=res)      # fp32 field values (bit-equal labels, test above)
    torch.set_num_threads(max(torch.get_num_threads(), 8))
    xyz = out['xyz'].reshape(-1, 3).cpu()
    sel = torch.randperm(xyz.shape[0], generator=torch.Generator().manual_seed(0))[:200000] if kind == 'nusc' else slice(None)
    occ64, sem64, sdf64, lg64 = oocc.point_labels_ref(vol64, mref, xyz[sel].double(), lut=lut)
    sdf32 = out['sdf'].reshape(-1).cpu()[sel].double()
    lg32 = out['logits'].reshape(-1, out['logits'].shape[-1]).cpu()[sel].double()
    band_s = (sdf64.abs() < 1e-5) | (sdf64.abs() <= (sdf32 - sdf64).abs())
    gap = _top2_gap(lg64)
    band_l = band_s | (gap < 1e-5) | (gap <= 2 * (lg32 - lg64).abs().max(-1).values)
    _check('%s occ vs fp64' % kind, got['occ'].reshape(-1).cpu()[sel], occ64, band_s, 1e-4)
    _check('%s sem vs fp64' % kind, got['sem'].reshape(-1).cpu()[sel], sem64, band_l, 1e-4)


def _ego2lidar(yaw_deg, t):
    a = np.deg2rad(yaw_deg)
    e = np.eye(4)
    e[:2, :2] = [[np.cos(a), -np.sin(a)], [np.sin(a), np.cos(a)]]
    e[:3, 3] = t
    return e


@pytest.mark.parametrize('kind', ['small', 'nusc'])
def test_occ3d_resample(kind):
    """The Occ3D branch: the 200 x 200 x 16 ego grid through an ego2lidar with a yaw and a translation (some points leave the
    lattice: zero padding) vs the fp32 torch composition of eval_iou.py:209-250 and, on the small scene, the fp64 oracle."""
    dev = _dev()
    from oracle import occupancy as oocc
    head, planes, mref, aabb, vol64 = _head(kind, dev)
    lut = LUT4 if kind == 'small' else occ_mod.OPENSEED2NUSCENES
    res = 0.2
    e2l = _ego2lidar(12.0, [1.5, -2.0, 0.3])
    if kind == 'small':         # the Occ3D grid scaled into the small scene's 40 m x 40 m x 6 m box (plus a margin outside)
        e2l[:3, :3] *= 0.55
    pts = occ_mod.occ3d_lidar_points(e2l, dev)
    head.prepare(planes)
    expansion = [aabb[3] - aabb[0], aabb[4] - aabb[1], aabb[5] - aabb[2]]
    got = head.occupancy(aabb, res, lut=lut, points=pts, expansion=expansion)
    assert got['occ'].shape == (200, 200, 16)
    # fp32 torch composition (eval_iou.py:209-250)
    out = head.forward_occ(planes, aabb=aabb, resolution=res)
    lp = pts.reshape(-1, 3).clone()
    for i in range(3):
        lp[:, i] = (lp[:, i] - aabb[i]) / expansion[i]
    lp = lp.reshape(1, 200, 200, 16, 3)
    outside = ((lp < 0) | (lp > 1)).any(-1)
    assert 0.01 < outside.float().mean() < 0.9                       # zero padding is exercised
    s = F.grid_sample(out['sdf'][None, None], lp[..., [2, 0, 1]] * 2 - 1, mode='bilinear', align_corners=True).squeeze()
    lg = F.grid_sample(out['logits'].permute(3, 0, 1, 2)[None], lp[..., [2, 0, 1]] * 2 - 1, mode='bilinear',
                       align_corners=True)[0].permute(1, 2, 3, 0)
    ref_occ = (s <= 0).to(torch.uint8)
    ref_sem = (ref_occ * torch.tensor(lut, device=dev)[lg.argmax(-1)]).to(torch.uint8)
    band_s = (s.abs() < 1e-6)
    _check('%s occ3d occ vs torch' % kind, got['occ'], ref_occ, band_s)
    _check('%s occ3d sem vs torch' % kind, got['sem'], ref_sem, band_s | (_top2_gap(lg) < 1e-6))
    assert ((got['occ'] == 1) & (s > 0.5)).sum() == 0
    if kind == 'small':
        u = occ_mod.normalise_points(pts, aabb, expansion).cpu()
        occ64, sem64, s64, lg64 = oocc.sample_labels_ref(vol64, mref, aabb, res, u, lut=lut)
        s32, lg32 = s.cpu().double(), lg.cpu().double()
        band_s = (s64.abs() < 1e-5) | (s64.abs() <= (s32 - s64).abs())
        gap = _top2_gap(lg64)
        band_l = band_s | (gap < 1e-5) | (gap <= 2 * (lg32 - lg64).abs().max(-1).values)
        _check('small occ3d occ vs fp64', got['occ'].cpu(), occ64, band_s, 1e-4)
        _check('small occ3d sem vs fp64', got['sem'].cpu(), sem64, band_l, 1e-4)


@pytest.mark.parametrize('n,n_cls', [(512 * 512 * 40, 17), (10 ** 6 + 3, 150)])
def test_confusion_equals_exact_count(n, n_cls):
    """10.5 M voxels (the OpenOccupancy lattice) with a mask, 255-ignores and labels beyond n_cls; and a class count whose
    histogram does not fit in shared memory, at an odd length (scalar tail)."""
    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(7)
    pred = torch.randint(0, 256, (n,), device=dev, generator=g).to(torch.uint8)
    gt = torch.randint(0, n_cls + 3, (n,), device=dev, generator=g).to(torch.uint8)
    gt[torch.rand(n, device=dev, generator=g) < 0.05] = 255
    pred = torch.where(torch.rand(n, device=dev, generator=g) < 0.5, gt, pred)                # a populated diagonal
    mask = torch.rand(n, device=dev, generator=g) < 0.8
    cm = occ_mod.confusion(pred, gt, n_cls, mask=mask, ignore=255)
    keep = mask & (gt != 255)
    b = gt[keep].long().clamp(max=n_cls) * (n_cls + 1) + pred[keep].long().clamp(max=n_cls)
    assert torch.equal(cm, torch.bincount(b, minlength=(n_cls + 1) ** 2))
    assert torch.equal(cm, occ_mod.confusion(pred, gt, n_cls, mask=mask, ignore=255))          # deterministic
    nomask = occ_mod.confusion(pred[1:], gt[1:], n_cls)                                         # mis-aligned, no mask / ignore
    b = gt[1:].long().clamp(max=n_cls) * (n_cls + 1) + pred[1:].long().clamp(max=n_cls)
    assert torch.equal(nomask, torch.bincount(b, minlength=(n_cls + 1) ** 2))


def _golden():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_golden_occ.npz'))


def _golden_step(G, s, dev):
    names = ('sem_gt', 'sem_pred', 'mask', 'occ_gt', 'occ_pred', 'kitti_gt', 'nonempty')
    return {k: (torch.from_numpy(G['step%d_%s' % (s, k)]).to(dev) if 'step%d_%s' % (s, k) in G else None) for k in names}


def _run_metrics(G, dev):
    from selfocc_b200.metric import IoU, MeanIoU, SSCMetrics
    m1, m16 = MeanIoU([1], 0, ['occupied'], True, 0), MeanIoU(list(range(1, 17)), 0, ['c%d' % i for i in range(16)], True, 0)
    iou, ssc = IoU().to(dev), SSCMetrics(2)
    for m in (m1, m16, iou):
        m.reset()
    xs = [_golden_step(G, s, dev) for s in range(2)]
    pts = []
    for x in xs:
        k = x['kitti_gt'].clone()
        k[k == 255] = 0
        pts.append(torch.nonzero(k))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for x, p in zip(xs, pts):
            m1._after_step(x['occ_pred'], x['occ_gt'], x['mask'])
            m16._after_step(x['sem_pred'], x['sem_gt'], x['mask'])
            iou._after_step(x['occ_pred'], p)
            ssc.add_batch(x['occ_pred'], x['kitti_gt'], x['nonempty'])
    finally:
        torch.cuda.set_sync_debug_mode('default')
    return m1, m16, iou, ssc


def test_device_metrics_reproduce_the_reference():
    dev = _dev()
    G = _golden()
    m1, m16, iou, ssc = _run_metrics(G, dev)
    for tag, m in (('miou1', m1), ('miou16', m16)):
        for k, v in zip(('total_seen', 'total_correct', 'total_positive'), m.counts()):
            assert np.array_equal(v.cpu().numpy(), G['%s_%s' % (tag, k)]), (tag, k)
        miou, occ_iou = m._after_epoch()
        assert miou == pytest.approx(float(G[tag + '_miou']), rel=1e-6)
        assert float(occ_iou) == pytest.approx(float(G[tag + '_occ_iou']), rel=1e-6)
    assert iou._after_epoch() == pytest.approx(float(G['iou_iou']), rel=1e-6)
    assert [int(iou.total_seen), int(iou.total_correct), int(iou.total_positive)] == \
        [int(G['iou_total_' + k][0]) for k in ('seen', 'correct', 'positive')]
    st = ssc.get_stats()
    for k in ('precision', 'recall', 'iou', 'iou_ssc', 'iou_ssc_mean'):
        assert np.allclose(st[k].cpu().numpy(), G['ssc_' + k], rtol=1e-6, atol=0), k
    # nonsurface: the completion counters use it, the semantic ones do not
    x = _golden_step(G, 0, dev)
    ns = torch.rand(x['kitti_gt'].shape, device=dev, generator=torch.Generator(device=dev).manual_seed(3)) < 0.5
    from selfocc_b200.metric import SSCMetrics
    a, b = SSCMetrics(2), SSCMetrics(2)
    a.add_batch(x['occ_pred'], x['kitti_gt'], None, ns)
    b.add_batch(x['occ_pred'], x['kitti_gt'])
    sa, sb = a.get_stats(), b.get_stats()
    assert torch.equal(sa['iou_ssc'], sb['iou_ssc'])
    m = (x['kitti_gt'] != 255) & ns
    p, g = x['occ_pred'][m], x['kitti_gt'][m].long()
    tp, fp = int(((g > 0) & (p > 0)).sum()), int(((g == 0) & (p > 0)).sum())
    assert float(sa['precision']) == pytest.approx(tp / (tp + fp), rel=1e-12)


def test_occupancy_and_metric_steps_do_not_synchronise():
    dev = _dev()
    head, planes, mref, aabb, _ = _head('small', dev)
    pts = occ_mod.occ3d_lidar_points(_ego2lidar(5.0, [0.5, 0.5, 0.0]) * np.array([[.5], [.5], [.5], [1.]]), dev)
    head.prepare(planes)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        a = head.occupancy(aabb, 0.2, lut=(2, 2, 1, 0))
        b = head.occupancy(aabb, 0.2, lut=LUT4, points=pts)
        c = head.occupancy(aabb, 0.4, representation=planes)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    assert a['sem'].max() <= 2 and b['occ'].shape == (200, 200, 16) and c['occ'].shape == (100, 100, 15)
    _run_metrics(_golden(), dev)        # every _after_step / add_batch under the same mode
