"""Generate tests/golden/reference_golden_novel_depth.npz from the reference's novel-view depth evaluation arithmetic.

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored vectors):
    python tests/golden/make_golden_novel_depth.py <path to the SelfOcc checkout>
utils/metric_util.py is loaded by file path and executed unmodified, with an ``mmengine`` stand-in whose MMLogger hands out
a standard logger.  Its compute_depth_errors_torch is composed with F.grid_sample, the boolean-mask gather per camera and
the per-distance sums the way eval_novel_depth.py:159-208 composes them (that script imports mmcv / mmseg and the model, so
the loop body is restated here around the reference's function), in fp32 on the CPU.

Inputs (seeded; stored with the outputs): FRAMES frames of N cameras with h x w depth maps and 2-4 source poses each, every
source with its own point count n.  Locations include 0, 1, exact cell edges k / (w - 1), k / (h - 1) and points beyond
[0, 1] (the border padding); one camera of one source has no masked-in point (the reference's NaN row); two sources of a
frame share a distance bin; the distances include an integer (its own bin) and 0.
"""
import importlib.util
import logging
import math
import os
import sys
import types
import numpy as np
import torch
import torch.nn.functional as F

REF = next((a for a in sys.argv[1:] if not a.startswith('--')), None)   # the SelfOcc checkout (required)
HERE = os.path.dirname(os.path.abspath(__file__))
N, H, W = 3, 6, 10
FRAMES = 3
DISTS = ([1.4, 2.0, 1.7], [0.0, 3.2], [2.6, 0.3, 3.9, 1.1])


def inputs(f):
    """Frame f: depth maps [S, N, H, W] and the loader's lists (float64 locations / depths, bool masks, as
    dataset_one_frame_eval.py delivers them)."""
    g = np.random.default_rng(300 + f)
    S = len(DISTS[f])
    maps = (g.random((S, N, H, W)) * 60 + 0.5).astype(np.float32)
    maps[0, 0, 2, 3] = 0.0                                            # below the 1e-3 clamp
    maps[0, 1, 4, 5] = 95.0                                           # above the 80 clamp
    locs, gts, masks = [], [], []
    for s in range(S):
        n = int(g.integers(40, 120))
        loc = g.random((N, n, 2)) * 1.1 - 0.05
        loc[:, :6] = [[0, 0], [1, 1], [0, 1], [1, 0], [3 / (W - 1), 2 / (H - 1)], [7 / (W - 1), 0.5]]
        loc[:, 6:10, 0] = np.arange(4) / (W - 1)
        gt = g.random((N, n)) * 70 + 1.0
        gt[:, ::9] = maps[s, :, None, 0, 0] * (1.0 + 0.2 * g.standard_normal((N, 1)))   # near the prediction: a1-a3 vary
        gt = np.abs(gt) + 1e-2
        mask = g.random((N, n)) < 0.7
        mask[:, :10] = True
        if f == 0 and s == 1:
            mask[2] = False                                           # an empty camera
        locs.append(loc)
        gts.append(gt)
        masks.append(mask)
    return maps, dict(depth_loc=locs, depth_gt=gts, depth_mask=masks, frame_dists=list(DISTS[f]))


def novel_depth_golden():
    mm = types.ModuleType('mmengine')
    mm.MMLogger = type('MMLogger', (), {'get_instance': staticmethod(lambda name: logging.getLogger(name))})
    sys.modules['mmengine'] = mm
    spec = importlib.util.spec_from_file_location('ref_metric_util', os.path.join(REF, 'utils', 'metric_util.py'))
    mu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mu)

    out = {}
    agg, n_frames = {}, {}
    for f in range(FRAMES):
        maps, meta = inputs(f)
        out['f%d_maps' % f] = maps
        out['f%d_dists' % f] = np.asarray(meta['frame_dists'], dtype=np.float64)
        for s, dist in enumerate(meta['frame_dists']):
            for k in ('depth_loc', 'depth_gt', 'depth_mask'):
                out['f%d_s%d_%s' % (f, s, k)] = meta[k][s]
            loc = torch.tensor(meta['depth_loc'][s], dtype=torch.float32)      # input_imgs.new_tensor(...)
            gt = torch.tensor(meta['depth_gt'][s], dtype=torch.float32)
            mask = torch.from_numpy(meta['depth_mask'][s])
            pred = F.grid_sample(torch.from_numpy(maps[s])[:, None], loc[:, None] * 2 - 1, mode='bilinear',
                                 padding_mode='border', align_corners=True).reshape(N, -1)
            cams = torch.stack([torch.stack(mu.compute_depth_errors_torch(gt=gt[c][mask[c]].reshape(-1),
                                                                          pred=pred[c][mask[c]].reshape(-1)))
                                for c in range(N)])
            out['f%d_s%d_sampled' % (f, s)] = pred.numpy()
            out['f%d_s%d_errors' % (f, s)] = cams.numpy()
            k = math.ceil(dist)
            if k not in agg:
                agg[k], n_frames[k] = cams, 1
            else:
                agg[k] = agg[k] + cams
                n_frames[k] += 1
    bins = sorted(agg)
    out['bins'] = np.asarray(bins, dtype=np.int64)
    out['agg_errors'] = np.stack([agg[k].numpy() for k in bins])
    out['n_frames'] = np.asarray([n_frames[k] for k in bins], dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, 'reference_golden_novel_depth.npz'), **out)
    print('wrote novel-depth golden:', len(out), 'arrays')


if __name__ == '__main__':
    if REF is None or not os.path.isfile(os.path.join(REF, 'utils', 'metric_util.py')):
        sys.exit('usage: python tests/golden/make_golden_novel_depth.py <path to a huang-yh/SelfOcc checkout>')
    novel_depth_golden()
