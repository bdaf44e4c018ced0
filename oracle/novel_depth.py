"""Oracle: novel-view depth evaluation (test infrastructure).  Restates in fp64 the per-source loop body of
eval_novel_depth.py:159-208 (eval_novel_depth_kitti.py is its one-camera case): F.grid_sample of the N depth maps at the
source's LiDAR locations -> each camera's points under its mask -> compute_depth_errors_torch (utils/metric_util.py:424-445)
-> summed into the bin ceil(source distance), one frame counted per source."""
import math

import torch
import torch.nn.functional as F

KEYS = ('abs_rel', 'sq_rel', 'rmse', 'rmse_log', 'a1', 'a2', 'a3')


def depth_errors_ref(gt, pred):
    """compute_depth_errors_torch on 1-D gt / pred -> [7] fp64 (an empty input gives NaN, the mean of nothing)."""
    gt, pred = gt.double(), pred.double().clamp(1e-3, 80)
    thresh = torch.maximum(gt / pred, pred / gt)
    sq = (gt - pred) ** 2
    return torch.stack([((gt - pred).abs() / gt).mean(), (sq / gt).mean(), sq.mean().sqrt(),
                        ((gt.log() - pred.log()) ** 2).mean().sqrt(), (thresh < 1.25).double().mean(),
                        (thresh < 1.25 ** 2).double().mean(), (thresh < 1.25 ** 3).double().mean()])


def sample_ref(depth_maps, loc):
    """depth_maps [N, h, w], loc [N, n, 2] in [0, 1] -> [N, n] fp64 (bilinear, padding_mode='border', align_corners=True)."""
    N = depth_maps.shape[0]
    return F.grid_sample(depth_maps.double()[:, None], loc.double()[:, None] * 2 - 1, mode='bilinear', padding_mode='border',
                         align_corners=True).reshape(N, -1)


def source_errors_ref(depth_maps, loc, gt, mask):
    """One source pose: depth_maps [N, h, w], loc [N, n, 2], gt [N, n], mask bool [N, n] -> [N, 7] fp64."""
    pred = sample_ref(depth_maps, loc)
    return torch.stack([depth_errors_ref(gt[c][mask[c]], pred[c][mask[c]]) for c in range(depth_maps.shape[0])])


def frame_errors_ref(depth_maps, meta):
    """One frame: depth_maps [S, N, h, w] (one set per source pose) and the loader's metas -> [(bin, [N, 7] fp64)] per
    source."""
    out = []
    for s, dist in enumerate(meta['frame_dists']):
        t = lambda k, dt=torch.float64: torch.as_tensor(meta[k][s]).to(dt)
        out.append((math.ceil(dist), source_errors_ref(depth_maps[s], t('depth_loc'), t('depth_gt'), t('depth_mask', torch.bool))))
    return out


def aggregate_ref(per_source):
    """[(bin, [N, 7])] over any number of frames -> (agg_depth_errors {bin: [N, 7]}, n_frames {bin: int})."""
    agg, n = {}, {}
    for k, e in per_source:
        agg[k] = e.clone() if k not in agg else agg[k] + e
        n[k] = n.get(k, 0) + 1
    return agg, n
