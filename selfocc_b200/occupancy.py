"""Occupancy labels straight from the decoded volume (eval_iou.py:196-270, eval_iou_kitti.py:160-190).

The reference evaluates occupancy by materialising the whole lattice of field outputs (``forward_occ``: the sdf, 24 fp32
channels per point for a semantic head, the coordinates and an int64 argmax) and then thresholding / arg-maxing /
resampling it with torch ops.  Here one kernel per frame writes only the two byte labels:

* lattice mode (``so_occ_lattice_labels``): ``occ = sdf <= thresh`` and ``sem = occ * lut[argmax(logits)]`` on the lattice
  of ``NeuSHead.get_uniform_sdf``;
* resample mode (``so_occ_sample_labels``, the Occ3D branch): the same lattice resampled with
  ``F.grid_sample(bilinear, zeros, align_corners=True)`` at given points, the lattice corners evaluated on the fly.
"""
import ctypes as C
import torch

from . import _lib
from .ops import _chk, _p, _stream

# utils/metric_util.py openseed2nuscenes: 21 OpenSeeD classes -> the 17 nuScenes occupancy labels (0 = empty)
OPENSEED2NUSCENES = (1, 2, 3, 4, 5, 5, 6, 7, 8, 9, 9, 10, 11, 12, 13, 14, 14, 15, 15, 16, 0)
# utils/metric_util.py cityscapes2semantickitti: 19 Cityscapes classes -> SemanticKITTI labels (0 = unlabeled)
CITYSCAPES2SEMANTICKITTI = (9, 11, 13, 13, 14, 18, 19, 19, 15, 17, 0, 6, 7, 1, 4, 5, 5, 3, 2)


def lattice_axes(aabb, resolution, device=None):
    """The axes of NeuSHead.get_uniform_sdf's lattice (neus_head.py:266-277): inclusive-endpoint ``torch.linspace`` per
    axis with ``int((a1 - a0) / resolution)`` points -> (xs [W], ys [H], zs [D]); the lattice is [H, W, D] = [y, x, z]."""
    xs = torch.linspace(aabb[0], aabb[3], int((aabb[3] - aabb[0]) / resolution), device=device)
    ys = torch.linspace(aabb[1], aabb[4], int((aabb[4] - aabb[1]) / resolution), device=device)
    zs = torch.linspace(aabb[2], aabb[5], int((aabb[5] - aabb[2]) / resolution), device=device)
    return xs, ys, zs


_OCC3D_XYZ = {}


def occ3d_lidar_points(ego2lidar, device):
    """The Occ3D-nuScenes 200 x 200 x 16 ego grid (x, y in [-40, 40] m, z in [-1, 5.4] m) mapped into the lidar frame with
    the torch ops of eval_iou.py:150-163,209-212 -> [200, 200, 16, 3] metres."""
    device = torch.device(device)
    xyz = _OCC3D_XYZ.get(device)
    if xyz is None:
        xx = torch.linspace(-40.0, 40.0, 200)
        yy = torch.linspace(-40.0, 40.0, 200)
        zz = torch.linspace(-1.0, 5.4, 16)
        xyz = torch.stack([xx[:, None, None].expand(-1, 200, 16), yy[None, :, None].expand(200, -1, 16),
                           zz[None, None, :].expand(200, 200, -1), torch.ones(200, 200, 16)], dim=-1).to(device)
        _OCC3D_XYZ[device] = xyz
    e2l = ego2lidar.to(xyz) if torch.is_tensor(ego2lidar) else xyz.new_tensor(ego2lidar)
    pts = torch.matmul(e2l.unsqueeze(0), xyz.reshape(-1, 4, 1)).squeeze(-1)[:, :3]
    return pts.reshape(200, 200, 16, 3)


_LUTS = {}


def as_lut(lut, device):
    """None, a sequence or a tensor -> contiguous uint8 tensor on ``device`` (or None).  A sequence is copied to the device
    once, from pinned memory without blocking, and cached: a per-frame call with a constant table (OPENSEED2NUSCENES, ...)
    never synchronises."""
    if lut is None:
        return None
    device = torch.device(device)
    if torch.is_tensor(lut):
        return lut.to(device=device, dtype=torch.uint8).contiguous()
    key = (tuple(int(v) for v in lut), device)
    if key not in _LUTS:
        _LUTS[key] = torch.tensor(key[0], dtype=torch.uint8).pin_memory().to(device, non_blocking=True)
    return _LUTS[key]


def normalise_points(points, aabb, expansion):
    """Lidar-frame metres [..., 3] -> the lattice's unit cube, (p - aabb_min) / expansion per axis with the scalar ops of
    eval_iou.py:211-215."""
    return torch.stack([(points[..., i] - aabb[i]) / expansion[i] for i in range(3)], -1)


def occupancy_labels(vol_sdf, vol_feat, desc, axes, thresh=0.0, sem_begin=3, n_sem=0, lut=None, points_u=None):
    """Labels of the decoded volume on the lattice ``axes`` = (xs, ys, zs).

    points_u None: lattice mode -> occ, sem uint8 [H, W, D].  Otherwise points_u [..., 3] normalised to the lattice's unit
    cube: resample mode -> occ, sem uint8 [...].  ``sem`` is None when n_sem == 0."""
    lib = _lib.load()
    xs, ys, zs = (a.contiguous() for a in axes)
    _chk(vol_sdf, name='vol_sdf'); _chk(vol_feat, name='vol_feat')
    for a, name in ((xs, 'xs'), (ys, 'ys'), (zs, 'zs')):
        _chk(a, name=name)
    dev = vol_sdf.device
    lut = as_lut(lut, dev)
    if lut is not None and lut.numel() != n_sem:
        raise ValueError('lut has %d entries, the head has %d semantic channels' % (lut.numel(), n_sem))
    lattice = (_p(xs), len(xs), _p(ys), len(ys), _p(zs), len(zs))
    if points_u is None:
        shape = (len(ys), len(xs), len(zs))
    else:
        shape = points_u.shape[:-1]
        points_u = _chk(points_u.reshape(-1, 3).contiguous(), name='points')
    occ = torch.empty(shape, dtype=torch.uint8, device=dev)
    sem = torch.empty(shape, dtype=torch.uint8, device=dev) if n_sem > 0 else None
    if points_u is None:
        rc = lib.so_occ_lattice_labels(_p(vol_sdf), _p(vol_feat), C.byref(desc), *lattice, float(thresh), sem_begin, n_sem, _p(lut),
                                       _p(occ), _p(sem), _stream())
        _lib.check(rc, 'so_occ_lattice_labels')
    elif points_u.shape[0] > 0:
        rc = lib.so_occ_sample_labels(_p(vol_sdf), _p(vol_feat), C.byref(desc), *lattice, _p(points_u), points_u.shape[0], float(thresh),
                                      sem_begin, n_sem, _p(lut), _p(occ), _p(sem), _stream())
        _lib.check(rc, 'so_occ_sample_labels')
    return occ, sem


def confusion(pred, gt, n_cls, mask=None, ignore=-1, out=None):
    """Accumulate the confusion matrix of uint8 label tensors ``pred`` / ``gt`` (same number of elements) into
    ``out`` int64 [(n_cls + 1)^2] (allocated zero-filled when None): bin (n_cls + 1) * g + p, labels >= n_cls in bin n_cls,
    elements with mask == 0 or gt == ignore skipped.  Deterministic."""
    lib = _lib.load()
    pred, gt = pred.reshape(-1).contiguous(), gt.reshape(-1).contiguous()
    _chk(pred, torch.uint8, 'pred'); _chk(gt, torch.uint8, 'gt')
    if pred.numel() != gt.numel():
        raise ValueError('pred has %d labels, gt has %d' % (pred.numel(), gt.numel()))
    if mask is not None:
        mask = mask.reshape(-1).contiguous()
        mask = mask.view(torch.uint8) if mask.dtype == torch.bool else mask
        _chk(mask, torch.uint8, 'mask')
        if mask.numel() != gt.numel():
            raise ValueError('mask has %d entries, gt has %d' % (mask.numel(), gt.numel()))
    if out is None:
        out = torch.zeros((n_cls + 1) ** 2, dtype=torch.int64, device=gt.device)
    if gt.numel() > 0:
        _lib.check(lib.so_occ_confusion(_p(pred), _p(gt), _p(mask), gt.numel(), n_cls, ignore, _p(out), _stream()),
                   'so_occ_confusion')
    return out
