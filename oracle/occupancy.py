"""Oracle: occupancy labels and occupancy-metric counters (test infrastructure).

The label compositions are inline code of the reference's evaluation scripts (not importable), restated here in fp64:
* lattice mode, eval_iou.py:196-197,254-270 / eval_iou_kitti.py:160-190: ``occ = sdf <= thresh`` and
  ``sem = occ * lut[argmax(logits)]`` on the lattice of get_uniform_sdf (``render.uniform_sdf_ref``);
* Occ3D resample, eval_iou.py:209-250: ``F.grid_sample(bilinear, zeros, align_corners=True)`` of the sdf and the logit
  lattices at ``u[..., [2, 0, 1]] * 2 - 1``, then the threshold, argmax and LUT.
The counters restate utils/metric_util.py MeanIoU / IoU and utils/scenerf_metric.py SSCMetrics per step as functions of
label volumes (pinned by tests/golden/reference_golden_occ.npz).
"""
import torch
import torch.nn.functional as F

from .render import field_query_ref, uniform_sdf_ref


def _compose(sdf, logits, thresh, lut):
    occ = sdf <= thresh
    if logits is None:
        return occ.to(torch.uint8), None
    arg = logits.argmax(-1)
    lab = arg if lut is None else torch.as_tensor(lut, dtype=torch.int64)[arg]
    return occ.to(torch.uint8), (occ * lab).to(torch.uint8)


def lattice_labels_ref(vol, mapping, aabb, resolution, thresh=0.0, lut=None):
    """vol [Cf, H, W, Z] fp64 -> (occ, sem or None, sdf, logits or None) on the [H, W, D] lattice."""
    sdf, logits, _ = uniform_sdf_ref(vol, mapping, aabb, resolution)
    occ, sem = _compose(sdf, logits, thresh, lut)
    return occ, sem, sdf, logits


def point_labels_ref(vol, mapping, xyz, thresh=0.0, lut=None):
    """The same composition at given lattice points xyz [n, 3] metres (a subset of a large lattice)."""
    h, _ = field_query_ref(vol, mapping, xyz.reshape(-1, 3), with_grad=False)
    sdf, logits = h[:, 0], (h[:, 4:] if h.shape[1] > 4 else None)
    occ, sem = _compose(sdf, logits, thresh, lut)
    return occ, sem, sdf, logits


def sample_labels_ref(vol, mapping, aabb, resolution, u, thresh=0.0, lut=None):
    """Occ3D branch: the lattice resampled at u [..., 3] (points normalised to the lattice's unit cube) ->
    (occ, sem or None, interpolated sdf, interpolated logits or None), shaped like u[..., 0]."""
    sdf, logits, _ = uniform_sdf_ref(vol, mapping, aabb, resolution)
    grid = (u.to(sdf.dtype)[..., [2, 0, 1]] * 2 - 1).reshape(1, -1, 1, 1, 3)
    samp = lambda lat: F.grid_sample(lat[None], grid, mode='bilinear', padding_mode='zeros', align_corners=True)[0, :, :, 0, 0]
    s = samp(sdf[None])[0].reshape(u.shape[:-1])
    lg = None if logits is None else samp(logits.permute(3, 0, 1, 2)).t().reshape(*u.shape[:-1], -1)
    occ, sem = _compose(s, lg, thresh, lut)
    return occ, sem, s, lg


def meaniou_counts_ref(pred, gt, mask, class_indices, empty_label):
    """One MeanIoU._after_step (metric_util.py:86-120, tensor targets) -> (seen, correct, positive) int64 [K + 1]."""
    if mask is not None:
        pred, gt = pred[mask.bool()], gt[mask.bool()]
    seen = [int((gt == c).sum()) for c in class_indices] + [int((gt != empty_label).sum())]
    correct = [int(((gt == c) & (pred == c)).sum()) for c in class_indices] + \
        [int(((gt != empty_label) & (pred != empty_label)).sum())]
    positive = [int((pred == c).sum()) for c in class_indices] + [int((pred != empty_label).sum())]
    return tuple(torch.tensor(v, dtype=torch.int64) for v in (seen, correct, positive))


def iou_counts_ref(outputs, points):
    """One IoU._after_step (metric_util.py:189-199): outputs [H, W, D], points [n, 3] -> (seen, correct, positive)."""
    return int(points.shape[0]), int(outputs[tuple(points.t())].sum()), int(outputs.sum())


def ssc_counts_ref(pred, gt, n_classes, nonempty=None):
    """One SSCMetrics.add_batch (scenerf_metric.py:80-99, 161-238) without `nonsurface` ->
    (completion tp, fp, fn, tps [n], fps [n], fns [n]) int64."""
    m = gt != 255
    if nonempty is not None:
        m = m & nonempty.bool()
    p, g = pred[m].to(torch.int64), gt[m].to(torch.int64)
    tp, fp, fn = int(((g > 0) & (p > 0)).sum()), int(((g == 0) & (p > 0)).sum()), int(((g > 0) & (p == 0)).sum())
    tps = torch.tensor([int(((g == j) & (p == j)).sum()) for j in range(n_classes)])
    fps = torch.tensor([int(((g != j) & (p == j)).sum()) for j in range(n_classes)])
    fns = torch.tensor([int(((g == j) & (p != j)).sum()) for j in range(n_classes)])
    return tp, fp, fn, tps, fps, fns


def confusion_ref(pred, gt, n_cls, mask=None, ignore=-1):
    """so_occ_confusion restated: int64 [(n_cls + 1)^2], bin (n_cls + 1) * g + p, labels >= n_cls in bin n_cls."""
    pred, gt = pred.reshape(-1).to(torch.int64), gt.reshape(-1).to(torch.int64)
    keep = gt != ignore
    if mask is not None:
        keep &= mask.reshape(-1).bool()
    b = gt[keep].clamp(max=n_cls) * (n_cls + 1) + pred[keep].clamp(max=n_cls)
    return torch.bincount(b, minlength=(n_cls + 1) ** 2)
