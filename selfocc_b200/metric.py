"""8f-3: DepthMetric on the device (reference utils/metric_util.py:282-397) -- same buffers, same
``_reset / _after_step / _after_epoch`` surface and the same numbers, but the per-camera boolean-mask indexing
(``depth_gt_i[depth_mask_i]``: a device->host sync per camera per frame) is replaced by two small kernels
(``so_depth_metric_sample`` + ``so_depth_metric_sums``) and a sort-based masked median, so a frame's metric step
enqueues without synchronising."""
import ctypes as C
import math
import numpy as np
import torch
import torch.nn as nn

from . import _lib
from .occupancy import confusion as occ_confusion
from .ops import _chk, _p, _stream

KEYS = ('abs_rel', 'sq_rel', 'rmse', 'rmse_log', 'a1', 'a2', 'a3')


def depth_sample(depth_pred, depth_loc):
    """depth_pred [N,h,w], depth_loc [N,n,2] in [0,1] -> [N,n] (grid_sample bilinear / border / align_corners=True)."""
    lib = _lib.load()
    _chk(depth_pred, name='depth_pred'); _chk(depth_loc, name='depth_loc')
    N, h, w = depth_pred.shape
    n = depth_loc.shape[1]
    out = torch.empty(N, n, device=depth_pred.device)
    _lib.check(lib.so_depth_metric_sample(_p(depth_pred), _p(depth_loc), N, n, h, w, _p(out), _stream()), 'so_depth_metric_sample')
    return out


def depth_metric_sums(sampled, depth_gt, mask_u8, scale=None):
    lib = _lib.load()
    _chk(sampled, name='sampled'); _chk(depth_gt, name='depth_gt'); _chk(mask_u8, torch.uint8, 'depth_mask'); _chk(scale, name='scale')
    N, n = sampled.shape
    sums = torch.empty(N, 8, device=sampled.device)
    _lib.check(lib.so_depth_metric_sums(_p(sampled), _p(depth_gt), _p(mask_u8), _p(scale), N, n, _p(sums), _stream()),
               'so_depth_metric_sums')
    return sums


def masked_median(x, mask):
    """torch.median(x_i[mask_i]) per row (the LOWER median, like torch.median) without boolean indexing."""
    filled = torch.where(mask, x, torch.full_like(x, float('inf')))
    srt = filled.sort(dim=1).values
    cnt = mask.sum(1)
    idx = ((cnt - 1).clamp_min(0) // 2).unsqueeze(1)
    return srt.gather(1, idx).squeeze(1)


def metrics_from_sums(sums):
    """[N,8] error sums -> dict of [N] metrics (cal_depth_metric, metric_util.py:247-279)."""
    c = sums[:, 7].clamp_min(1.0)
    return {'abs_rel': sums[:, 0] / c, 'sq_rel': sums[:, 1] / c, 'rmse': (sums[:, 2] / c).sqrt(), 'rmse_log': (sums[:, 3] / c).sqrt(),
            'a1': sums[:, 4] / c, 'a2': sums[:, 5] / c, 'a3': sums[:, 6] / c}


class DepthMetric(nn.Module):
    def __init__(self, camera_names=['front'], eval_types=['raw', 'median']):
        super().__init__()
        self.num_cams, self.camera_names = len(camera_names), camera_names
        self.num_types, self.eval_types = len(eval_types), eval_types
        for k in KEYS + ('scaling',):
            self.register_buffer(k, torch.zeros(self.num_types, self.num_cams))
        self.register_buffer('count', torch.zeros(1))

    def _reset(self):
        for k in KEYS + ('scaling', 'count'):
            getattr(self, k).zero_()

    @torch.no_grad()
    def _after_step(self, depth_loc, depth_gt, depth_mask, depth_pred):
        """depth_loc [N,n,2], depth_gt [N,n], depth_mask bool [N,n], depth_pred [N,h,w] (metric_util.py:311-349)."""
        depth_loc, depth_gt, depth_pred = depth_loc.float().contiguous(), depth_gt.float().contiguous(), depth_pred.float().contiguous()
        mask = depth_mask.bool()
        mask_u8 = mask.to(torch.uint8).contiguous()
        sampled = depth_sample(depth_pred, depth_loc)
        for ti, typ in enumerate(self.eval_types):
            if typ == 'raw':
                scale = torch.ones(self.num_cams, device=sampled.device)
            elif typ == 'median':
                scale = masked_median(depth_gt, mask) / masked_median(sampled, mask)
            else:
                raise NotImplementedError(typ)
            m = metrics_from_sums(depth_metric_sums(sampled, depth_gt, mask_u8, scale.contiguous()))
            self.scaling[ti] += scale
            for k in KEYS:
                getattr(self, k)[ti] += m[k]
        self.count += 1

    def _after_epoch(self, logger=None):
        """metric_util.py:351-397: all-reduce over ranks when torch.distributed is initialised, then average."""
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            dist.barrier()
            for k in ('count',) + KEYS + ('scaling',):
                dist.all_reduce(getattr(self, k))
            dist.barrier()
        res = {k: getattr(self, k) / self.count for k in KEYS + ('scaling',)}
        if logger is not None and (not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0):
            logger.info('Averaging over %s samples.' % self.count.item())
            for ti, typ in enumerate(self.eval_types):
                logger.info('%s evaluation:' % typ)
                for cam, name in enumerate(self.camera_names):
                    logger.info('%12s | ' % name + ' '.join('%s %.3f' % (k, res[k][ti, cam]) for k in KEYS + ('scaling',)))
                logger.info('%12s | ' % 'All' + ' '.join('%s %.3f' % (k, res[k][ti].mean()) for k in KEYS + ('scaling',)))
        return res


# ------------------------------------------------------------------------------------------------------------------------
# Novel-view depth on the device (eval_novel_depth.py:159-208, eval_novel_depth_kitti.py).  The reference renders, samples
# and reduces each of a frame's S source poses separately, with a boolean-mask gather (a host sync) per camera; here the S
# poses are one render_poses launch, the frame's LiDAR points one host-to-device copy and the per-(pose, camera) errors one
# so_novel_depth_errors launch, accumulated into fixed-size per-distance bins on the device.

def novel_depth_errors(depth_maps, offsets, loc, depth_gt, mask_u8, offsets_host=None):
    """depth_maps [S, h, w] (one map per (pose, camera) segment), offsets int64 [S + 1], loc [T, 2] in [0, 1] (x, y),
    depth_gt [T], mask_u8 uint8 [T] -> [S, 7] compute_depth_errors_torch metrics (KEYS order) per segment, NaN where a
    segment has no masked-in point.  ``offsets_host``: the same offsets as a CPU tensor, checked before the launch; when
    omitted they are read back from the device, which synchronises."""
    lib = _lib.load()
    _chk(depth_maps, name='depth_maps'); _chk(offsets, torch.int64, 'offsets'); _chk(loc, name='depth_loc')
    _chk(depth_gt, name='depth_gt'); _chk(mask_u8, torch.uint8, 'depth_mask')
    S, h, w = depth_maps.shape
    T = depth_gt.shape[0]
    if offsets.shape != (S + 1,) or loc.shape != (T, 2) or depth_gt.shape != (T,) or mask_u8.shape != (T,):
        raise ValueError('novel_depth_errors: expected offsets [%d], loc [T, 2], depth_gt [T], mask [T]; got %s, %s, %s, %s'
                         % (S + 1, tuple(offsets.shape), tuple(loc.shape), tuple(depth_gt.shape), tuple(mask_u8.shape)))
    if offsets_host is None:
        offsets_host = offsets.cpu()
    elif offsets_host.is_cuda or offsets_host.dtype != torch.int64 or offsets_host.shape != (S + 1,) or not offsets_host.is_contiguous():
        raise ValueError('offsets_host must be a contiguous int64 CPU tensor of shape [%d]' % (S + 1))
    out = torch.empty(S, 7, device=depth_maps.device)
    _lib.check(lib.so_novel_depth_errors(_p(depth_maps), S, h, w, _p(offsets), _p(offsets_host), T, _p(loc), _p(depth_gt),
                                         _p(mask_u8), _p(out), _stream()), 'so_novel_depth_errors')
    return out


def _align(n, a=16):
    return (n + a - 1) // a * a


def pack_novel_depth(meta, num_cams, max_distance, pin=True):
    """One frame's loader metas (``depth_loc`` [N, n_s, 2], ``depth_gt`` [N, n_s], ``depth_mask`` [N, n_s] per source s,
    numpy, and ``frame_dists`` [S]) -> (buf, layout): every array in one uint8 CPU tensor (pinned unless ``pin`` is False),
    so that a frame is one host-to-device copy.  Sections, each 16-byte aligned, as layout[name] = (byte offset, bytes):
    offsets int64 [S*N + 1] (segment s*N + c = source s, camera c: render_poses' [S, N] order), perm / bins int64 [S] (the
    sources ordered in rounds, each round holding every distance bin at most once, and their bins), loc float32 [T, 2],
    gt float32 [T], mask uint8 [T].  layout['rounds'] holds the [begin, end) of each round in perm / bins."""
    locs, gts, masks, dists = meta['depth_loc'], meta['depth_gt'], meta['depth_mask'], meta['frame_dists']
    S, N = len(dists), num_cams
    if not (len(locs) == len(gts) == len(masks) == S) or S == 0:
        raise ValueError('depth_loc / depth_gt / depth_mask / frame_dists must hold one entry per source pose (got %d, %d, %d, %d)'
                         % (len(locs), len(gts), len(masks), S))
    bins = []
    for d in dists:
        k = math.ceil(float(d))
        if not 0 <= k <= max_distance:
            raise ValueError('source distance %r falls in bin %d, outside the metric\'s bins [0, %d]: construct '
                             'NovelDepthMetric with a larger max_distance' % (d, k, max_distance))
        bins.append(k)
    counts = []
    for s in range(S):
        n = np.shape(gts[s])[-1] if np.ndim(gts[s]) == 2 else -1
        if np.shape(gts[s]) != (N, n) or np.shape(locs[s]) != (N, n, 2) or np.shape(masks[s]) != (N, n):
            raise ValueError('source %d: expected depth_loc [%d, n, 2], depth_gt / depth_mask [%d, n]; got %s, %s, %s'
                             % (s, N, N, np.shape(locs[s]), np.shape(gts[s]), np.shape(masks[s])))
        counts.append(n)
    seg = np.repeat(np.asarray(counts, dtype=np.int64), N)
    T = int(seg.sum())
    seen, rank = {}, []
    for k in bins:
        rank.append(seen.get(k, 0))
        seen[k] = rank[-1] + 1
    perm = sorted(range(S), key=lambda s: (rank[s], s))
    rounds, b = [], 0
    for r in range(max(rank) + 1):
        e = b + rank.count(r)
        rounds.append((b, e))
        b = e
    layout, off = {'S': S, 'N': N, 'T': T, 'rounds': rounds}, 0
    for name, nbytes in (('offsets', 8 * (S * N + 1)), ('perm', 8 * S), ('bins', 8 * S), ('loc', 8 * T), ('gt', 4 * T),
                         ('mask', T)):
        layout[name] = (off, nbytes)
        off += _align(nbytes)
    buf = torch.empty(max(off, 16), dtype=torch.uint8, pin_memory=pin)
    raw = buf.numpy()
    view = lambda name, dt: raw[layout[name][0]:layout[name][0] + layout[name][1]].view(dt)
    offsets = view('offsets', np.int64)
    offsets[0] = 0
    np.cumsum(seg, out=offsets[1:])
    view('perm', np.int64)[:] = perm
    view('bins', np.int64)[:] = [bins[s] for s in perm]
    loc, gt, mask = view('loc', np.float32).reshape(T, 2), view('gt', np.float32), view('mask', np.uint8)
    b = 0
    for s in range(S):
        e = b + N * counts[s]
        loc[b:e] = np.asarray(locs[s]).reshape(-1, 2)
        gt[b:e] = np.asarray(gts[s]).reshape(-1)
        mask[b:e] = np.asarray(masks[s]).reshape(-1)
        b = e
    return buf, layout


class NovelDepthMetric(nn.Module):
    """Per-distance novel-view depth errors of eval_novel_depth.py / eval_novel_depth_kitti.py on the device.

    ``errors`` [B, N, 7] (fp64) and ``n_frames`` [B] (int64) hold one bin per integer distance k = ceil(source distance) in
    [0, max_distance]; a source farther away is refused, not clipped.  ``_after_step(metas, depth_maps)`` takes one frame:
    the loader's metas (``depth_loc`` / ``depth_gt`` / ``depth_mask`` / ``frame_dists``) and the depth maps of its S source
    poses, render_poses' ``ms_depths[0]`` or ``ms_max_depths[0]`` reshaped to [S, N, h, w] (or [S*N, h, w]) with h, w the
    eval ray grid, as the reference reshapes to ``cfg.num_rays``.  Each (source, camera) adds its seven errors to the
    source's bin and each source one frame to the bin's count, as ``agg_depth_errors[k] += cams_depth_errors;
    n_frames[k] += 1`` does; a step enqueues one host-to-device copy and a few launches and reads nothing back.
    ``_after_epoch()`` all-reduces the two buffers when torch.distributed is initialised and returns ``as_dicts()``."""

    def __init__(self, num_cams, max_distance, device='cuda'):
        super().__init__()
        if num_cams < 1 or max_distance < 0:
            raise ValueError('num_cams must be >= 1 and max_distance >= 0')
        self.num_cams, self.max_distance = int(num_cams), int(max_distance)
        self.register_buffer('errors', torch.zeros(self.max_distance + 1, self.num_cams, 7, dtype=torch.float64, device=device))
        self.register_buffer('n_frames', torch.zeros(self.max_distance + 1, dtype=torch.int64, device=device))

    def _reset(self):
        self.errors.zero_()
        self.n_frames.zero_()

    @torch.no_grad()
    def _after_step(self, metas, depth_maps):
        meta = metas[0] if isinstance(metas, (list, tuple)) else metas
        buf, lay = pack_novel_depth(meta, self.num_cams, self.max_distance)
        S, N, T = lay['S'], lay['N'], lay['T']
        h, w = depth_maps.shape[-2:]
        if depth_maps.numel() != S * N * h * w:
            raise ValueError('depth_maps %s: expected the maps of %d source poses x %d cameras, [S, N, h, w] or [S*N, h, w]'
                             % (tuple(depth_maps.shape), S, N))
        dev = self.errors.device
        d = buf.to(dev, non_blocking=True)
        part = lambda name, dt: d[lay[name][0]:lay[name][0] + lay[name][1]].view(dt)
        o0, ob = lay['offsets']
        err = novel_depth_errors(depth_maps.reshape(S * N, h, w).float().contiguous(), part('offsets', torch.int64),
                                 part('loc', torch.float32).view(T, 2), part('gt', torch.float32), part('mask', torch.uint8),
                                 offsets_host=buf[o0:o0 + ob].view(torch.int64))
        err = err.view(S, N, 7).double()
        perm, bins = part('perm', torch.int64), part('bins', torch.int64)
        for b, e in lay['rounds']:                 # every bin once per round: a fixed order of additions
            self.errors.index_add_(0, bins[b:e], err.index_select(0, perm[b:e]))
        self.n_frames.index_add_(0, bins, torch.ones(S, dtype=torch.int64, device=dev))

    def _after_epoch(self):
        d = _dist()
        if d is not None:
            d.all_reduce(self.errors)
            d.all_reduce(self.n_frames)
        return self.as_dicts()

    def as_dicts(self):
        """(agg_depth_errors, n_frames) keyed by distance, bins without a frame left out, as the scripts' print_metrics
        takes them: eval_novel_depth.py's ({k: [N, 7] tensor}, {k: [1] int tensor}); for N = 1 eval_novel_depth_kitti.py's
        ({k: [7] ndarray}, {k: int})."""
        nf = self.n_frames.cpu()
        keep = [k for k in range(self.max_distance + 1) if nf[k] > 0]
        if self.num_cams == 1:
            return {k: self.errors[k, 0].cpu().numpy() for k in keep}, {k: int(nf[k]) for k in keep}
        return {k: self.errors[k] for k in keep}, {k: self.n_frames[k:k + 1] for k in keep}


# ------------------------------------------------------------------------------------------------------------------------
# Occupancy metrics on the device (utils/metric_util.py MeanIoU / IoU, utils/scenerf_metric.py SSCMetrics).  Same
# constructor arguments and reset / _after_step / _after_epoch / add_batch / get_stats surface as the reference; the
# per-step counting is enqueued without reading the host (the reference does three .item() per class per step).  Counts are
# exact int64 (the reference accumulates fp32, which stops counting exactly past 2^24 voxels); the ratios are taken in fp64.

def _dist():
    import torch.distributed as dist
    return dist if dist.is_available() and dist.is_initialized() else None


def _on(t, device):
    """numpy array / tensor -> tensor on ``device`` (a no-op for a tensor already there)."""
    t = torch.as_tensor(t)
    return t if t.device == device else t.to(device)


def _labels(t, n_cls, keep=None):
    """Integer labels -> uint8 for so_occ_confusion: values outside [0, n_cls] (other than ``keep``) become n_cls, the bin
    of every label >= n_cls, so every count the metrics derive stays exact."""
    if t.dtype == torch.uint8:
        return t
    if t.dtype == torch.bool:
        return t.view(torch.uint8)
    over = (t < 0) | (t > n_cls)
    if keep is not None:
        over &= t != keep
    return torch.where(over, torch.full_like(t, n_cls), t).to(torch.uint8)


def counts_from_confusion(cm, class_indices, empty_label):
    """Confusion matrix cm [(n + 1)^2] (bin (n + 1) * gt + pred, any device) -> (seen, correct, positive) int64 [K + 1]:
    for each class c of ``class_indices`` #(gt == c), #(gt == c & pred == c), #(pred == c), and last the same three counts
    of 'not empty_label' -- MeanIoU's total_seen / total_correct / total_positive (metric_util.py:111-120).  SSCMetrics'
    counters are the same numbers: with class_indices = range(n_classes) and empty 0, tps = correct[:-1],
    fps = positive[:-1] - tps, fns = seen[:-1] - tps, and completion tp / fp / fn = correct[-1], positive[-1] - correct[-1],
    seen[-1] - correct[-1]."""
    n1 = int(round(cm.numel() ** 0.5))
    m = cm.reshape(n1, n1).to(torch.int64)
    row, col, diag, total, e = m.sum(1), m.sum(0), m.diagonal(), m.sum(), empty_label
    seen = torch.stack([row[c] for c in class_indices] + [total - row[e]])
    correct = torch.stack([diag[c] for c in class_indices] + [total - row[e] - col[e] + m[e, e]])
    positive = torch.stack([col[c] for c in class_indices] + [total - col[e]])
    return seen, correct, positive


def meaniou_scores(seen, correct, positive):
    """MeanIoU._after_epoch (metric_util.py:122-165) from the counts -> (miou * 100, occupied iou * 100, ious, precs, recas)."""
    s, c, p = (t.double().cpu().tolist() for t in (seen, correct, positive))
    ious, precs, recas = [], [], []
    for i in range(len(s) - 1):
        precs.append(0. if p[i] == 0 else c[i] / p[i])
        if s[i] == 0:
            ious.append(1)
            recas.append(1)
        else:
            ious.append(c[i] / (s[i] + p[i] - c[i]))
            recas.append(c[i] / s[i])
    den = s[-1] + p[-1] - c[-1]
    occ_iou = c[-1] / den if den else float('nan')
    return np.mean(ious) * 100, occ_iou * 100, ious, precs, recas


def iou_score(seen, correct, positive):
    """IoU._after_epoch (metric_util.py:217-237): one class -> iou * 100."""
    s, c, p = (float(t) for t in (seen, correct, positive))
    return np.mean([1 if s == 0 else c / (s + p - c)]) * 100


def ssc_stats(seen, correct, positive):
    """SSCMetrics.get_stats (scenerf_metric.py:101-125) from counts_from_confusion(cm, range(n_classes), 0)."""
    seen, correct, positive = seen.double(), correct.double(), positive.double()
    tp, fp, fn = correct[-1:], positive[-1:] - correct[-1:], seen[-1:] - correct[-1:]
    if float(tp) != 0:
        precision, recall, iou = tp / (tp + fp), tp / (tp + fn), tp / (tp + fp + fn)
    else:
        precision, recall, iou = 0, 0, 0
    tps, fps, fns = correct[:-1], positive[:-1] - correct[:-1], seen[:-1] - correct[:-1]
    iou_ssc = tps / (tps + fps + fns + 1e-5)
    return {'precision': precision, 'recall': recall, 'iou': iou, 'iou_ssc': iou_ssc, 'iou_ssc_mean': torch.mean(iou_ssc[1:])}


class MeanIoU:
    """Drop-in for utils/metric_util.py MeanIoU on the device: each _after_step is one so_occ_confusion launch into an int64
    confusion matrix (exact counts, where the reference accumulates fp32), no host read until _after_epoch, which
    all-reduces when torch.distributed is initialised.  _after_epoch returns (miou * 100, occupied iou * 100 as a 0-dim
    tensor).  The dict-``targets`` branch (Occ3D files with their own crop logic; unused by eval_iou.py) is not provided."""

    def __init__(self, class_indices, empty_label, label_str, use_mask=False, dataset_empty_label=17, name='none'):
        self.class_indices = list(class_indices)
        self.num_classes = len(self.class_indices)
        self.empty_label, self.dataset_empty_label = empty_label, dataset_empty_label
        self.label_str, self.use_mask, self.name = label_str, use_mask, name
        self.n_cls = max(self.class_indices + [empty_label]) + 1
        if self.n_cls > 255:
            raise ValueError('class indices must be < 255 (labels are counted as uint8)')

    def reset(self):
        self.confusion = torch.zeros((self.n_cls + 1) ** 2, dtype=torch.int64, device='cuda')

    def _after_step(self, outputs, targets, mask=None):
        if not isinstance(targets, (torch.Tensor, np.ndarray)):
            raise NotImplementedError('MeanIoU: dict targets (the Occ3D file branch) are not supported; pass label tensors')
        dev = self.confusion.device
        outputs, targets = _on(outputs, dev), _on(targets, dev)
        occ_confusion(_labels(outputs, self.n_cls), _labels(targets, self.n_cls), self.n_cls,
                      mask=None if mask is None else _on(mask, dev).bool(), out=self.confusion)

    def counts(self):
        """(total_seen, total_correct, total_positive) int64 [num_classes + 1] of the reference."""
        return counts_from_confusion(self.confusion, self.class_indices, self.empty_label)

    def _after_epoch(self, logger=None):
        d = _dist()
        if d is not None:
            d.all_reduce(self.confusion)
            d.barrier()
        seen, correct, positive = self.counts()
        miou, occ_iou, ious, precs, recas = meaniou_scores(seen, correct, positive)
        if logger is not None:
            logger.info(f'Validation per class iou {self.name}:')
            for iou, prec, reca, label_str in zip(ious, precs, recas, self.label_str):
                logger.info('%s : %.2f%%, %.2f, %.2f' % (label_str, iou * 100, prec, reca))
            logger.info(seen)
            logger.info(correct)
            logger.info(positive)
        return miou, torch.tensor(occ_iou, dtype=torch.float64, device=seen.device)


class IoU(nn.Module):
    """Drop-in for utils/metric_util.py IoU on the device: the ground-truth points index the prediction as a tensor (the
    reference converts them to Python lists), int64 counters, no host read until _after_epoch, which all-reduces only when
    torch.distributed is initialised.  Occ3D targets may be tensors already on the device (numpy arrays are copied)."""

    def __init__(self, use_mask=False):
        super().__init__()
        self.class_indices, self.num_classes, self.label_str, self.use_mask = [0], 1, ['occupied'], use_mask
        xx = torch.linspace(-40.0, 40.0, 200)
        yy = torch.linspace(-40.0, 40.0, 200)
        zz = torch.linspace(-1.0, 5.4, 16)
        xyz = torch.stack([xx[:, None, None].expand(-1, 200, 16), yy[None, :, None].expand(200, -1, 16),
                           zz[None, None, :].expand(200, 200, -1)], dim=-1)
        self.register_buffer('xyz', xyz, persistent=False)

    def reset(self):
        self.total_seen, self.total_correct, self.total_positive = (torch.zeros(1, dtype=torch.int64, device='cuda')
                                                                     for _ in range(3))

    def _add(self, seen, correct, positive):
        self.total_seen += seen
        self.total_correct += correct.to(torch.int64)
        self.total_positive += positive.to(torch.int64)

    def _after_step(self, outputs, targets, occ3d=False):
        if occ3d:
            self._after_step_occ3d(outputs, targets)
            return
        targets = _on(targets, outputs.device)
        self._add(targets.shape[0], outputs[tuple(targets.t())].sum(), outputs.sum())

    def _after_step_occ3d(self, outputs, targets):
        mask = _on(targets['mask_camera'], outputs.device).bool()
        label = _on(targets['semantics'], outputs.device) != 17
        if self.use_mask:
            label = label & mask
            positive = (outputs * mask).sum()
        else:
            positive = outputs.sum()
        self._add(label.sum(), (outputs * label).sum(), positive)

    def _after_epoch(self, logger=None):
        d = _dist()
        if d is not None:
            for t in (self.total_seen, self.total_correct, self.total_positive):
                d.all_reduce(t)
        miou = iou_score(self.total_seen, self.total_correct, self.total_positive)
        if logger is not None:
            logger.info('Validation per class iou:')
            logger.info('%s : %.2f%%' % (self.label_str[0], miou))
            logger.info(f'Final iou: {miou}')
        return miou


class SSCMetrics:
    """Drop-in for utils/scenerf_metric.py SSCMetrics on the device: add_batch is one so_occ_confusion launch (two when
    ``nonsurface`` is given: the completion counters use it, the semantic ones do not), exact int64 counts, no host read
    until get_stats.  get_stats all-reduces only when torch.distributed is initialised (the reference needs a process
    group); its values are tensors as in the reference, computed in fp64."""

    def __init__(self, n_classes):
        if not 1 <= n_classes <= 255:
            raise ValueError('n_classes must be in [1, 255]')
        self.n_classes = n_classes
        self.reset()

    def reset(self):
        z = lambda: torch.zeros((self.n_classes + 1) ** 2, dtype=torch.int64, device='cuda')
        # steps without `nonsurface` count once into `shared`; the others into `semantic` and `completion` separately
        self.shared, self.semantic, self.completion = z(), z(), z()

    def add_batch(self, y_pred, y_true, nonempty=None, nonsurface=None):
        dev, n = self.shared.device, self.n_classes
        pred, gt = _labels(_on(y_pred, dev), n), _labels(_on(y_true, dev), n, keep=255)
        nonempty = None if nonempty is None else _on(nonempty, dev).bool()
        if nonsurface is None:
            occ_confusion(pred, gt, n, mask=nonempty, ignore=255, out=self.shared)
            return
        nonsurface = _on(nonsurface, dev).bool()
        occ_confusion(pred, gt, n, mask=nonempty, ignore=255, out=self.semantic)
        occ_confusion(pred, gt, n, mask=nonsurface if nonempty is None else nonempty & nonsurface, ignore=255, out=self.completion)

    def get_stats(self):
        d = _dist()
        if d is not None:
            for t in (self.shared, self.semantic, self.completion):
                d.all_reduce(t)
        classes = range(self.n_classes)
        seen, correct, positive = counts_from_confusion(self.shared + self.semantic, classes, 0)
        cs, cc, cp = counts_from_confusion(self.shared + self.completion, classes, 0)
        seen[-1], correct[-1], positive[-1] = cs[-1], cc[-1], cp[-1]
        return ssc_stats(seen, correct, positive)
