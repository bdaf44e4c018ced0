"""Photometric reprojection losses of SelfOcc on the per-ray statistics kernel (SURVEY.md 8f-2):
drop-in ``ReprojLossMonoMultiNewCombine`` (reference loss/reproj_loss_mono_multi_new_combine.py) and
``ReprojLossMonoMultiNew`` (loss/reproj_loss_mono_multi_new.py).

The per-sample work (reprojection of every sample into the previous / next frame, bilinear colour gathers, masks, the
weighted sums over each ray) runs in ``so_reproj_stats_forward`` / ``_backward`` (csrc/reproj.cu) through
``ops.ReprojStatsFunction``, which returns per ray and direction set the weight-normalised photometric error l1 and
colour.  What is left is a function of a few numbers per ray and runs here as torch on [N_cam, R] grids, batched over
cameras, in fp64: SSIM over the ray grid, the 1e3 filter of rays without a valid reprojection, the automask min and the
means.  Nothing in the forward or backward
reads a value on the host, except the optional ``masked/{cam}`` scalars handed to an attached ``writer`` (every 10th
call, as the reference does), whose ``add_scalar`` reads a count.

Input layout: every camera's ``weights`` / ``ts`` (/ ``deltas``) entry holds R * S values ray-major (S samples per ray,
R = len(ms_rays)), which is what ``NeuSHead.forward`` emits (``ray_indices[cam]`` = arange(R).repeat_interleave(S)); the
kernel uses that layout and does not read ``ray_indices``, whose lengths are checked.  Batch size 1, fp32, CUDA.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .registry import LOSSES

_DEFAULT_KEYS = ('curr_imgs', 'prev_imgs', 'next_imgs', 'ray_indices', 'weights', 'ts', 'metas', 'ms_rays')


def ssim(x, y):
    """(1 - SSIM) / 2 clamped to [0, 1] over 3x3 windows with reflection padding (Monodepth2's SSIM), x, y [B, C, h, w]."""
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    x, y = F.pad(x, (1, 1, 1, 1), mode='reflect'), F.pad(y, (1, 1, 1, 1), mode='reflect')
    mu_x, mu_y = F.avg_pool2d(x, 3, 1), F.avg_pool2d(y, 3, 1)
    sigma_x = F.avg_pool2d(x ** 2, 3, 1) - mu_x ** 2
    sigma_y = F.avg_pool2d(y ** 2, 3, 1) - mu_y ** 2
    sigma_xy = F.avg_pool2d(x * y, 3, 1) - mu_x * mu_y
    n = (2 * mu_x * mu_y + c1) * (2 * sigma_xy + c2)
    d = (mu_x ** 2 + mu_y ** 2 + c1) * (sigma_x + sigma_y + c2)
    return torch.clamp((1 - n / d) / 2, 0, 1)


def _mats(metas, key, n, dev):
    m = [meta[key] for meta in metas]
    if isinstance(m[0], torch.Tensor):
        t = torch.stack(m)
    else:
        t = torch.from_numpy(np.asarray(m, dtype=np.float32))
    return t.to(dev, torch.float32, non_blocking=True).reshape(-1, 4, 4)[:n].contiguous()


class _ReprojLoss(nn.Module):
    MODE = None

    def __init__(self, weight=1.0, input_dict=None, no_ssim=False, img_size=(768, 1600), ray_resize=None, no_automask=False,
                 dims=3, **kwargs):
        super().__init__()
        if dims != 3:
            raise NotImplementedError('dims=%r: the reprojection statistics kernel handles RGB images only (dims=3)' % (dims,))
        self.weight = weight
        self.input_dict = dict(input_dict) if input_dict is not None else {k: k for k in _DEFAULT_KEYS}
        self.img_size = list(img_size)
        self.ray_resize = list(ray_resize) if ray_resize is not None else None
        self.no_automask = no_automask
        self.dims = dims
        self.no_ssim = no_ssim or ray_resize is None
        self.writer = None               # a tensorboard-style writer with add_scalar(tag, value, step); None = no logging
        self.iter_counter = 0

    def forward(self, inputs):
        """BaseLoss.forward: weight * loss over the inputs named by input_dict."""
        return self.weight * self.reproj_loss(**{k: inputs[v] for k, v in self.input_dict.items()})

    def _stats(self, curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas):
        bs, num_cams = curr_imgs.shape[:2]
        if bs != 1:
            raise NotImplementedError('batch size %d: the reprojection loss supports batch size 1 (as the reference)' % bs)
        R = ms_rays.shape[0]
        n_cam = len(weights)
        n = weights[0].numel()
        if n % R:
            raise ValueError('each camera must hold R * S samples ray-major, R = %d rays; got %d' % (R, n))
        lists = dict(weights=weights, ts=ts, ray_indices=ray_indices) if deltas is None else \
            dict(weights=weights, ts=ts, ray_indices=ray_indices, deltas=deltas)
        for k, v in lists.items():
            if len(v) != n_cam or any(t.numel() != n for t in v):
                raise ValueError('%s must have %d entries of %d samples (R = %d rays x S = %d), as weights' % (k, n_cam, n, R, n // R))
        if n_cam > num_cams:
            raise ValueError('%d cameras of weights but %d images' % (n_cam, num_cams))
        if not self.no_ssim and R != self.ray_resize[0] * self.ray_resize[1]:
            raise ValueError('SSIM needs the rays to fill ray_resize %s, got %d rays (ray sharding or a partial ray set: '
                             'set no_ssim=True)' % (self.ray_resize, R))
        dev = weights[0].device
        cfg = dict(mode=self.MODE, shape=(n_cam, R, n // R), ts=ops._one_buffer([t.detach() for t in ts], 'ts'),
                   deltas=None if deltas is None else ops._one_buffer([t.detach() for t in deltas], 'deltas'),
                   pix=ms_rays.detach().float().contiguous(), img2prev=_mats(metas, 'img2prevImg', n_cam, dev),
                   img2next=_mats(metas, 'img2nextImg', n_cam, dev),
                   images=tuple(im[0, :n_cam].float().contiguous() for im in (curr_imgs, prev_imgs, next_imgs)),
                   img_size=self.img_size)
        stats, colours = ops.ReprojStatsFunction.apply(cfg, *weights)
        # the tail runs in fp64: SSIM's variances E[x^2] - E[x]^2 cancel badly in fp32, and on [N_cam, R] grids fp64 is free
        return stats.double(), colours.double(), num_cams

    def _grid(self, x):
        """[N, R, 3] -> [N, 3, h, w] over the ray grid."""
        return x.reshape(x.shape[0], *self.ray_resize, 3).permute(0, 3, 1, 2)

    def _photometric(self, pred, target, l1):
        """0.85 SSIM + 0.15 l1 per ray (l1 alone without SSIM); pred, target [N, R, 3], l1 [N, R]."""
        if self.no_ssim:
            return l1
        s = ssim(self._grid(pred), self._grid(target)).mean(1).flatten(1)
        return 0.85 * s + 0.15 * l1

    def _automask(self, colours):
        cur = colours[..., 0:3]
        return [self._photometric(colours[..., k:k + 3], cur, (cur - colours[..., k:k + 3]).abs().mean(-1)) for k in (3, 6)]

    def _log(self, idx, first_masked):
        if self.writer and self.iter_counter % 10 == 0:
            for cam, c in enumerate((idx > first_masked).sum(1)):
                self.writer.add_scalar(f'masked/{cam}', c, self.iter_counter)

    @staticmethod
    def _set(stats, j):
        """(l1, combined colour, any) of direction set j."""
        return stats[..., 6 * j + 1], stats[..., 6 * j + 2:6 * j + 5], stats[..., 6 * j + 5] > 0


@LOSSES.register_module()
class ReprojLossMonoMultiNewCombine(_ReprojLoss):
    """Reprojection loss with the previous and next frame merged per sample (padding 'border'):
    per ray 0.15 l1 + 0.85 SSIM of the weighted colour over the ray grid, min with the two automask terms."""
    MODE = 'combine'

    def reproj_loss(self, curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas=None):
        stats, colours, num_cams = self._stats(curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas)
        cur = colours[..., 0:3]
        l1, rgb, any_valid = self._set(stats, 0)
        loss = self._photometric(rgb, cur, l1)
        if not self.no_automask:
            loss = torch.where(any_valid, loss, torch.full_like(loss, 1e3))
            loss, idx = torch.stack([loss] + self._automask(colours), dim=-1).min(dim=-1)
            self._log(idx, 0)
        self.iter_counter += 1
        return (loss.mean(1).sum() / num_cams).float()


@LOSSES.register_module()
class ReprojLossMonoMultiNew(_ReprojLoss):
    """Reprojection loss with the previous and next frame as separate candidates (padding 'zeros'): per ray the min
    over {prev, next, (automask prev, automask next)} of 0.15 l1 + 0.85 SSIM; a direction without a valid sample scores 1e3."""
    MODE = 'multi_new'

    def __init__(self, weight=1.0, input_dict=None, sdf_loss=False, sdf_loss_weight=0.1, **kwargs):
        if sdf_loss:
            raise NotImplementedError('sdf_loss=True (argmax-weight sdf term) is not implemented by the native reprojection loss')
        super().__init__(weight, input_dict, **kwargs)
        self.sdf_loss = sdf_loss
        self.sdf_loss_weight = sdf_loss_weight

    def reproj_loss(self, curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas=None,
                    sample_sdfs=None):
        stats, colours, num_cams = self._stats(curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas)
        cur = colours[..., 0:3]
        cands = []
        for j in (0, 1):
            l1, rgb, any_valid = self._set(stats, j)
            c = self._photometric(rgb, cur, l1)
            cands.append(torch.where(any_valid, c, torch.full_like(c, 1e3)))
        if not self.no_automask:
            cands += self._automask(colours)
        loss, idx = torch.stack(cands, dim=-1).min(dim=-1)
        self._log(idx, 1)
        self.iter_counter += 1
        return (loss.mean(1).sum() / num_cams).float()
