"""The training objectives of SelfOcc's shipped configs (SURVEY.md 8f-2): drop-in ``MultiLoss`` and every term it builds.

Photometric reprojection losses on the per-ray statistics kernel: ``ReprojLossMonoMultiNewCombine`` (reference
loss/reproj_loss_mono_multi_new_combine.py) and ``ReprojLossMonoMultiNew`` (loss/reproj_loss_mono_multi_new.py).  The other
terms (eikonal, second-grad, sparsity, RGB, semantic, edge) and ``MultiLoss`` follow in the second half of this file.

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

Ray-sharded training (MultiLoss.forward with inputs['ray_shard']): every term splits into ``local_payload`` (the per-ray
quantities of this rank's rays: the reprojection statistics, colours and image values at the ray pixels, depths, the
semantic elements; a per-sample term's sum and count) and ``from_gathered`` (the same tail formulas as the unsharded
term, on the full ray grid).
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
        """BaseLoss.forward: weight * loss over the inputs named by input_dict.  With the fused objective
        (fuse_objective) the head has already computed the per-ray statistics (inputs['reproj_stats'])."""
        if 'reproj_stats' in inputs:
            return self.weight * self.tail(*self._fused(inputs))
        return self.weight * self.reproj_loss(**{k: inputs[v] for k, v in self.input_dict.items()})

    def reproj_loss(self, curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas=None,
                    sample_sdfs=None):
        return self.tail(*self._stats(curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas))

    # ray-sharded evaluation (MultiLoss): the per-ray statistics of this rank's rays, the tail on the gathered grid
    def local_payload(self, inputs, shard):
        if 'reproj_stats' in inputs:
            stats, colours, _ = self._fused(inputs, full_grid=False)
            return [(stats, shard[2]), (colours, shard[2])]
        kw = {k: inputs[v] for k, v in self.input_dict.items() if k != 'sample_sdfs'}
        stats, colours, _ = self._stats(**kw, full_grid=False)
        return [(stats, shard[2]), (colours, shard[2])]

    def _fused(self, inputs, full_grid=True):
        """(stats, colours, num_cams) from the statistics the fused training render emitted, as _stats returns them."""
        stats, colours = inputs['reproj_stats'], inputs['reproj_colours']
        if stats.shape[-1] != 6 * ops.REPROJ_SETS[self.MODE]:
            raise ValueError('reproj_stats hold %d values per ray, %s needs %d: fuse the head with this objective '
                             '(fuse_objective)' % (stats.shape[-1], type(self).__name__, 6 * ops.REPROJ_SETS[self.MODE]))
        R = stats.shape[1]
        if full_grid and not self.no_ssim and R != self.ray_resize[0] * self.ray_resize[1]:
            raise ValueError('SSIM needs the rays to fill ray_resize %s, got %d rays (ray sharding or a partial ray set: '
                             'set no_ssim=True)' % (self.ray_resize, R))
        return stats.double(), colours.double(), inputs[self.input_dict['curr_imgs']].shape[1]

    def from_gathered(self, full, inputs):
        return self.weight * self.tail(full[0], full[1], inputs[self.input_dict['curr_imgs']].shape[1])

    def _stats(self, curr_imgs, prev_imgs, next_imgs, ray_indices, weights, ts, metas, ms_rays, deltas=None, full_grid=True):
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
        if full_grid and not self.no_ssim and R != self.ray_resize[0] * self.ray_resize[1]:
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

    def tail(self, stats, colours, num_cams):
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

    def tail(self, stats, colours, num_cams):
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


# ---------------------------------------------------------------------------------------------------------------------
# The remaining terms of the shipped configs' objectives and MultiLoss.
#
# EikonalLoss, SecondGradLoss and SoftSparsityLoss read the largest per-sample tensors of the objective (eik_grad,
# second_grad: [rays, S, 3]; uniform_sdf: the lattice) and run on so_sample_mean_forward / _backward (csrc/loss_terms.cu):
# one read forward, one read and one write backward, no per-sample temporaries.  SparsityLoss and HardSparsityLoss run on
# the same launches (so_sparsity_*, so_hard_sparsity_*), AdaptiveSparsityLoss per ray (so_adaptive_sparsity_*).  RGBLossMS, SemLossMS, SemCELossMS and
# EdgeLoss3DMS work per ray ([cameras, rays] grids) and stay in torch, batched over cameras.

class _Term(nn.Module):
    """BaseLoss (reference loss/base_loss.py): weight * loss over the inputs named by input_dict."""
    DEFAULT_KEYS = ()

    def __init__(self, weight=1.0, input_dict=None):
        super().__init__()
        self.weight = weight
        self.input_dict = dict(input_dict) if input_dict is not None else {k: k for k in self.DEFAULT_KEYS}
        self.writer = None

    def forward(self, inputs):
        return self.weight * self.loss_func(**self._args(inputs))

    def _args(self, inputs):
        return {k: inputs[v] for k, v in self.input_dict.items()}

    # ray-sharded evaluation (MultiLoss.forward with inputs['ray_shard']): local_payload(inputs, (rank, world, R_full)) ->
    # [(this rank's [L, count, k] slice, its full length)]; from_gathered(full tensors, inputs) -> weight * loss
    def local_payload(self, inputs, shard):
        raise NotImplementedError('%s under ray sharding' % type(self).__name__)


class _SampleMeanTerm(_Term):
    """A per-sample mean over the rays' samples: under ray sharding each rank sends its mean times its element count and
    that count (the full mean is the ratio of the sums; elements per sample cancel)."""

    def local_payload(self, inputs, shard):
        x, = self._args(inputs).values()
        n = x.numel()
        part = self.loss_func(x).double() * n if n else x.new_zeros((), dtype=torch.float64)
        return [(torch.stack([part, part.new_full((), float(n))]).reshape(1, 1, 2), shard[1])]

    def from_gathered(self, full, inputs):
        s = full[0][0].sum(0)                                   # over the ranks: (sum, count)
        return self.weight * (s[0] / s[1]).float()


@LOSSES.register_module()
class EikonalLoss(_SampleMeanTerm):
    """mean over samples of (|eik_grad|_2 - 1)^2 (loss/eikonal_loss.py)."""
    DEFAULT_KEYS = ('eik_grad',)

    def __init__(self, weight=1.0, input_dict=None, **kwargs):
        super().__init__(weight, input_dict)

    def loss_func(self, eik_grad):
        return ops.SampleMeanFunction.apply(eik_grad, 'eikonal')

    # the fused objective (fuse_objective): the head's render has already taken the mean (inputs['eikonal_mean'])
    def forward(self, inputs):
        if 'eikonal_mean' in inputs:
            return self.weight * inputs['eikonal_mean']
        return super().forward(inputs)

    def local_payload(self, inputs, shard):
        if 'eikonal_mean' not in inputs:
            return super().local_payload(inputs, shard)
        n = sum(t.numel() for t in inputs['ray_indices'])        # this rank's samples: the mean's count
        part = inputs['eikonal_mean'].double() * n
        return [(torch.stack([part, part.new_full((), float(n))]).reshape(1, 1, 2), shard[1])]


@LOSSES.register_module()
class SecondGradLoss(_SampleMeanTerm):
    """mean |second_grad| (loss/second_grad_loss.py)."""
    DEFAULT_KEYS = ('second_grad',)

    def __init__(self, weight=1.0, input_dict=None, **kwargs):
        super().__init__(weight, input_dict)

    def loss_func(self, second_grad):
        return ops.SampleMeanFunction.apply(second_grad, 'abs')

    # the fused objective (fuse_objective(..., second_grad=True)): the head's render has already taken the mean
    # (inputs['second_grad_mean'])
    def forward(self, inputs):
        if 'second_grad_mean' in inputs:
            return self.weight * inputs['second_grad_mean']
        return super().forward(inputs)

    def local_payload(self, inputs, shard):
        if 'second_grad_mean' not in inputs:
            return super().local_payload(inputs, shard)
        n = 3 * sum(t.numel() for t in inputs['ray_indices'])    # this rank's elements (3 per sample): the mean's count
        part = inputs['second_grad_mean'].double() * n
        return [(torch.stack([part, part.new_full((), float(n))]).reshape(1, 1, 2), shard[1])]


class _LatticeTerm(_Term):
    """A term on the density lattice; the shipped configs feed it uniform_sdf."""
    DEFAULT_KEYS = ('density',)

    # under ray sharding the uniform_sdf lattice is the same on every rank: each rank computes the whole term, unscaled, and
    # the average over the ranks of its (equal) gradients is the gradient
    def local_payload(self, inputs, shard):
        if self.input_dict['density'] != 'uniform_sdf':
            raise NotImplementedError('%s under ray sharding takes the replicated uniform_sdf, got %r'
                                      % (type(self).__name__, self.input_dict['density']))
        return []

    def from_gathered(self, full, inputs):
        return self(inputs)


@LOSSES.register_module()
class SoftSparsityLoss(_LatticeTerm):
    """mean relu(-density) (loss/sparsity_loss.py SoftSparsityLoss); the shipped configs feed it uniform_sdf."""

    def __init__(self, weight=1.0, input_dict=None, **kwargs):
        super().__init__(weight, input_dict)

    def loss_func(self, density):
        return ops.SampleMeanFunction.apply(density, 'neg_relu')


@LOSSES.register_module()
class SparsityLoss(_LatticeTerm):
    """mean sech^2(density / (2 scale)) (loss/sparsity_loss.py SparsityLoss, StreetSurf style), on so_sparsity_forward /
    _backward: 0 where the reference's 1 / cosh overflows to 1 / inf."""

    def __init__(self, weight=1.0, scale=1.0, input_dict=None, **kwargs):
        super().__init__(weight, input_dict)
        self.scale = scale

    def loss_func(self, density):
        return ops.SparsityFunction.apply(density, self.scale)


@LOSSES.register_module()
class HardSparsityLoss(_LatticeTerm):
    """relu(mean sigmoid(-scale density) - thresh) over the [H, W, D] lattice with the crop borders counted as density 100
    (loss/sparsity_loss.py HardSparsityLoss), on so_hard_sparsity_forward / _backward.  Unlike the reference, which writes
    100 into the caller's tensor, the crop is applied inside the kernel: the input (and every term after this one that
    reads it) is left as it was."""

    def __init__(self, weight=1.0, scale=1.0, thresh=0.2, crop=((0, 0), (0, 0), (0, 0)), input_dict=None, **kwargs):
        super().__init__(weight, input_dict)
        self.scale = scale
        self.thresh = thresh
        self.crop = [[int(v) for v in row] for row in crop]

    def loss_func(self, density):
        return ops.HardSparsityFunction.apply(density, self.scale, self.thresh, self.crop)


@LOSSES.register_module()
class AdaptiveSparsityLoss(_Term):
    """mean relu(-sdf) over the samples more than ``slack`` behind the ray's rendered depth, ts > depth + slack
    (loss/sparsity_loss.py AdaptiveSparsityLoss).  Per ray so_adaptive_sparsity_rays forms (sum, count) in fp64 and
    so_adaptive_sparsity_reduce takes their ratio in a fixed order: no boolean-mask gather, no host read; NaN when no sample
    counts, as the reference's mean of an empty selection.  The gradient reaches the sdf only.

    The reference's default keys name an ``sdfs`` input that NeuSHead does not emit: with ``return_sample_sdf=True`` the
    head's per-sample sdf is ``sample_sdf``, so a config maps input_dict={'sdfs': 'sample_sdf', 'ts': 'ts',
    'ms_depths': 'ms_depths'}.  Under ray sharding each rank sends its rays' (sum, count) pairs; the gathered pairs reduce to
    the unsharded value bit for bit."""
    DEFAULT_KEYS = ('sdfs', 'ts', 'ms_depths')

    def __init__(self, weight=1, input_dict=None, slack=4.0, **kwargs):
        super().__init__(weight, input_dict)
        self.slack = slack

    def _args(self, inputs):
        missing = [(k, v) for k, v in self.input_dict.items() if v not in inputs]
        if missing:
            raise KeyError('AdaptiveSparsityLoss reads %s, which the inputs lack (the head emits its per-sample sdf as '
                           "'sample_sdf' with return_sample_sdf=True: map input_dict {'sdfs': 'sample_sdf', ...})"
                           % ', '.join('%r (input_dict key %r)' % (v, k) for k, v in missing))
        return super()._args(inputs)

    def loss_func(self, sdfs, ts, ms_depths):
        return ops.AdaptiveSparsityReduceFunction.apply(self._rays(sdfs, ts, ms_depths))

    def _rays(self, sdfs, ts, ms_depths):
        """[N, R, 2] fp64 (sum, count) per ray of camera."""
        depths = ms_depths[0]
        bs, num_cams, num_rays = depths.shape
        if bs != 1:
            raise NotImplementedError('batch size %d: AdaptiveSparsityLoss supports batch size 1 (as the reference)' % bs)
        return ops.AdaptiveSparsityRaysFunction.apply(self.slack, [t.detach() for t in ts], depths[0].detach(), *sdfs)

    def local_payload(self, inputs, shard):
        return [(self._rays(**self._args(inputs)), shard[2])]

    def from_gathered(self, full, inputs):
        return self.weight * ops.AdaptiveSparsityReduceFunction.apply(full[0])


def sample_at_rays(imgs, rays, img_size, padding):
    """Bilinear samples of imgs [M, C, H, W] at the ray pixels rays [R, 2] (x, y in img_size pixels) -> [M, C, R]: the
    reference's F.grid_sample(align_corners=True) at (x / img_size[1], y / img_size[0]) * 2 - 1, normalised by the loss's
    img_size, not by the image's shape.  padding: 'zeros' (RGBLossMS) or 'border' (EdgeLoss3DMS)."""
    rays = rays.to(imgs.dtype)
    pix = torch.stack([rays[:, 0] / img_size[1], rays[:, 1] / img_size[0]], -1)     # scalar divisions: no host copy
    grid = (pix * 2 - 1).reshape(1, 1, -1, 2).expand(imgs.shape[0], 1, -1, 2)
    return F.grid_sample(imgs, grid, mode='bilinear', padding_mode=padding, align_corners=True)[:, :, 0]


def _single_rays(ms_rays, what):
    if isinstance(ms_rays, (list, tuple)):
        raise NotImplementedError('%s: list-valued ms_rays is not supported (the reference raises too)' % what)
    return ms_rays


def _check_grid(ray_resize, R, what):
    if R != ray_resize[0] * ray_resize[1]:
        raise ValueError('%s needs the rays to fill ray_resize %s, got %d rays (ray sharding or a partial ray set)'
                         % (what, list(ray_resize), R))


@LOSSES.register_module()
class RGBLossMS(_Term):
    """Per scale mean |colour - gt| at the ray pixels, 0.15 l1 + 0.85 SSIM over the ray grid when SSIM is on
    (loss/rgb_loss_ms.py RGBLossMS)."""
    DEFAULT_KEYS = ('ms_colors', 'ms_rays', 'gt_imgs')

    def __init__(self, weight=1.0, img_size=None, no_ssim=True, ray_resize=None, input_dict=None, **kwargs):
        super().__init__(weight, input_dict)
        assert img_size is not None
        self.img_size = list(img_size)
        self.no_ssim = no_ssim or ray_resize is None
        self.ray_resize = list(ray_resize) if ray_resize is not None else None

    def loss_func(self, ms_colors, ms_rays, gt_imgs):
        rays = _single_rays(ms_rays, 'RGBLossMS')
        if not self.no_ssim:
            _check_grid(self.ray_resize, rays.shape[0], 'RGBLossMS with SSIM')
        return self._tail(ms_colors, self._gt(rays, gt_imgs), gt_imgs)

    def _gt(self, rays, gt_imgs):
        return sample_at_rays(gt_imgs.flatten(0, 1), rays, self.img_size, 'zeros')          # [B*N, 3, R]

    def local_payload(self, inputs, shard):
        a = self._args(inputs)
        gt = self._gt(_single_rays(a['ms_rays'], 'RGBLossMS'), a['gt_imgs'])
        return [(c.flatten(0, 1), shard[2]) for c in a['ms_colors']] + [(gt.transpose(1, 2), shard[2])]

    def from_gathered(self, full, inputs):
        gt_imgs = self._args(inputs)['gt_imgs']
        colors = [c.reshape(*gt_imgs.shape[:2], *c.shape[1:]) for c in full[:-1]]
        return self.weight * self._tail(colors, full[-1].transpose(1, 2).contiguous(), gt_imgs)

    def _tail(self, ms_colors, gt, gt_imgs):
        """The loss from the colours [B, N, R, 3] and the ground truth at the ray pixels [B*N, 3, R] on the ray grid."""
        bs, num_cams = gt_imgs.shape[:2]
        R = gt.shape[-1]
        gt_grid = None if self.no_ssim else gt.reshape(bs * num_cams, 3, *self.ray_resize)
        gt = gt.reshape(bs, num_cams, 3, R).transpose(-1, -2)
        tot = 0.
        for color in ms_colors:
            loss = (color - gt).abs().mean()
            if not self.no_ssim:
                c = color.reshape(bs * num_cams, *self.ray_resize, 3).permute(0, 3, 1, 2)
                loss = 0.15 * loss + 0.85 * ssim(c, gt_grid).mean()
            tot = tot + loss
        return tot / len(ms_colors)


def _sem_labels(metas, rays, dev):
    """metas[b]['sem'] [N, H, W] integer labels -> labels at the ray pixels, int64 [B, N, R] on dev.  numpy labels travel
    once, pinned and non-blocking, in their own dtype; the gather and the widening run on the device."""
    lab = [m['sem'] for m in metas]
    if isinstance(lab[0], np.ndarray):
        t = torch.from_numpy(np.ascontiguousarray(np.stack(lab)))
        if dev.type == 'cuda':
            t = t.pin_memory()
        t = t.to(dev, non_blocking=True)
    elif isinstance(lab[0], torch.Tensor):
        t = torch.stack(lab).to(dev, non_blocking=True)
    else:
        raise NotImplementedError('metas[i]["sem"] must be a numpy array or a tensor')
    r = rays.to(dev).long()
    return t[:, :, r[:, 1], r[:, 0]].long()


class _SemTerm(_Term):
    DEFAULT_KEYS = ('sem', 'metas', 'ms_rays')

    def __init__(self, weight=1.0, img_size=None, ray_resize=None, input_dict=None, **kwargs):
        super().__init__(weight, input_dict)
        assert img_size is not None
        self.img_size = img_size
        self.ray_resize = ray_resize

    def loss_func(self, sem, metas, ms_rays):
        rays = _single_rays(ms_rays, type(self).__name__)
        gt = _sem_labels(metas, rays, sem[0].device)
        return sum(self.term(s, gt) for s in sem) / len(sem)

    # under ray sharding: the elements the term averages, [B, N, count, k] per scale (per_ray), gathered, then their mean
    def local_payload(self, inputs, shard):
        a = self._args(inputs)
        gt = _sem_labels(a['metas'], _single_rays(a['ms_rays'], type(self).__name__), a['sem'][0].device)
        return [(self.per_ray(s, gt).flatten(0, 1), shard[2]) for s in a['sem']]

    def from_gathered(self, full, inputs):
        return self.weight * (sum(e[None].mean() for e in full) / len(full))


@LOSSES.register_module()
class SemLossMS(_SemTerm):
    """Binary cross-entropy of the clamped semantic probabilities against one-hot labels at the ray pixels
    (loss/rgb_loss_ms.py SemLossMS; F.binary_cross_entropy clamps the log at -100)."""

    @staticmethod
    def term(s, gt):
        return F.binary_cross_entropy(torch.clamp(s, 0, 1), F.one_hot(gt, num_classes=s.shape[-1]).to(s.dtype))

    @staticmethod
    def per_ray(s, gt):
        return F.binary_cross_entropy(torch.clamp(s, 0, 1), F.one_hot(gt, num_classes=s.shape[-1]).to(s.dtype), reduction='none')


@LOSSES.register_module()
class SemCELossMS(_SemTerm):
    """Cross-entropy -log(clamp(s, 1e-6, 1)) of the label class, mean over rays (loss/rgb_loss_ms.py SemCELossMS).  The
    reference's sum over one-hot classes has exactly one non-zero term; this gathers it."""

    @staticmethod
    def term(s, gt):
        return SemCELossMS.per_ray(s, gt).mean()

    @staticmethod
    def per_ray(s, gt):
        return -torch.log(torch.clamp(s.gather(-1, gt.unsqueeze(-1)), 1e-6, 1))


def _smooth(disp, img):
    """Edge-aware smoothness of disp [M, 1, h, w] weighted by exp(-|d img|) (edge_loss_3d_ms.py get_smooth_loss)."""
    gx = (disp[:, :, :, :-1] - disp[:, :, :, 1:]).abs() * torch.exp(-(img[:, :, :, :-1] - img[:, :, :, 1:]).abs().mean(1, True))
    gy = (disp[:, :, :-1, :] - disp[:, :, 1:, :]).abs() * torch.exp(-(img[:, :, :-1, :] - img[:, :, 1:, :]).abs().mean(1, True))
    return gx.mean() + gy.mean()


@LOSSES.register_module()
class EdgeLoss3DMS(_Term):
    """Edge-aware smoothness of the mean-normalised depth over the ray grid, weighted by the current image at the ray
    pixels (padding 'border'); with use_inf_mask the depth is blended towards max_depths by 1 - ms_accs
    (loss/edge_loss_3d_ms.py)."""
    DEFAULT_KEYS = ('curr_imgs', 'ms_depths', 'ms_rays')

    def __init__(self, weight=1.0, input_dict=None, **kwargs):
        super().__init__(weight, input_dict)
        self.img_size = list(kwargs.get('img_size', [768, 1600]))
        self.ray_resize = kwargs.get('ray_resize', None)
        self.use_inf_mask = kwargs.get('use_inf_mask', False)
        assert self.ray_resize is not None
        self.ray_resize = list(self.ray_resize)

    def loss_func(self, curr_imgs, ms_depths, ms_rays, ms_accs=None, max_depths=None):
        _check_grid(self.ray_resize, ms_depths[0].shape[2], 'EdgeLoss3DMS')
        return self._tail(self._rays(curr_imgs, ms_depths, ms_rays, ms_accs, max_depths))

    def _rays(self, curr_imgs, ms_depths, ms_rays, ms_accs=None, max_depths=None):
        """Per scale the depth [B, N, R] (blended by the inf mask) and the current image at the ray pixels [B*N, 3, R]."""
        if self.use_inf_mask:
            assert ms_accs is not None and max_depths is not None
        if not isinstance(ms_rays, (list, tuple)):
            ms_rays = [ms_rays] * len(ms_depths)
        imgs = curr_imgs.flatten(0, 1)
        out = []
        for scale, (depth, rays) in enumerate(zip(ms_depths, ms_rays)):
            rgb = sample_at_rays(imgs, rays, self.img_size, 'border')
            if self.use_inf_mask:
                depth = depth * ms_accs[scale] + max_depths[scale] * (1 - ms_accs[scale])
            out.append((depth, rgb))
        return out

    def _tail(self, per_scale):
        tot = 0.
        for depth, rgb in per_scale:
            depth = depth.reshape(-1, 1, *self.ray_resize)
            rgb = rgb.reshape(depth.shape[0], -1, *self.ray_resize)
            norm = depth / (depth.mean(2, True).mean(3, True) + 1e-6)
            tot = tot + _smooth(norm, rgb)
        return tot / len(per_scale)

    def local_payload(self, inputs, shard):
        pay = []
        for depth, rgb in self._rays(**self._args(inputs)):
            pay += [(depth.reshape(-1, depth.shape[-1], 1), shard[2]), (rgb.transpose(1, 2), shard[2])]
        return pay

    def from_gathered(self, full, inputs):
        return self.weight * self._tail([(d, rgb.transpose(1, 2).contiguous()) for d, rgb in zip(full[0::2], full[1::2])])


_PER_SAMPLE_KEYS = ('weights', 'ts', 'deltas', 'eik_grad', 'sample_sdf')


def fuse_objective(head, multi_loss, second_grad=False):
    """Let ``head``'s training render compute ``multi_loss``'s per-sample terms itself (so_render_train_objective_forward):
    the reprojection term's per-ray statistics and the eikonal mean come out of the render, and the per-sample tensors
    weights / ts / deltas / eik_grad are never written.  The losses' values and gradients are those of the unfused step.
    The model is then called with the reprojection images as kwargs: model(..., curr_imgs=, prev_imgs=, next_imgs=).

    Supported: at most one reprojection term (ReprojLossMonoMultiNewCombine or ReprojLossMonoMultiNew on the head's
    outputs, without ``deltas`` / ``sample_sdfs`` inputs or sdf_loss), at most one EikonalLoss on ``eik_grad``, any number of
    terms that read no per-sample output, and a head without two_split or return_sample_sdf; anything else raises
    NotImplementedError and leaves the head unfused.  Returns what it recorded on the head (``head.fused_objective``);
    ``head.fused_objective = None`` undoes it.  Evaluation (head.eval()) is unaffected.

    ``second_grad=True`` fuses SecondGradLoss as well: the render takes the mean of |second_grad| at its own sample points
    and the head emits ``second_grad_mean`` instead of the [rays, S, 3] ``second_grad`` (and no longer asks the render for ts /
    deltas).  It accepts at most one SecondGradLoss, reading ``second_grad``, on a head with return_second_grad and the
    declared-assumption opt-in (second_grad_assumption / SELFOCC_B200_SECOND_GRAD=1); the record then carries
    ``second_grad=True``.  Without the keyword SecondGradLoss stays on the head's second_grad tensor, as before."""
    if head.two_split and head.img2lidar.two_split:
        raise NotImplementedError('fuse_objective: two_split=True renders half the cameras for the reprojection term')
    if head.return_sample_sdf:
        raise NotImplementedError('fuse_objective: return_sample_sdf needs the per-sample sdf tensor')
    reproj, eik, sg = [], [], []
    for term in multi_loss.losses:
        keys = getattr(term, 'input_dict', {})
        if second_grad and isinstance(term, SecondGradLoss):
            if keys != {'second_grad': 'second_grad'}:
                raise NotImplementedError('fuse_objective: SecondGradLoss must read second_grad, got input_dict %r' % (keys,))
            sg.append(term)
            continue
        if isinstance(term, _ReprojLoss):
            if 'deltas' in keys or 'sample_sdfs' in keys or getattr(term, 'sdf_loss', False):
                raise NotImplementedError('fuse_objective: %s with deltas / sample_sdfs / sdf_loss' % type(term).__name__)
            if any(keys.get(k, k) != k for k in _DEFAULT_KEYS):
                raise NotImplementedError('fuse_objective: %s must read the head\'s outputs and the model\'s image kwargs '
                                          'under their own names, got input_dict %r' % (type(term).__name__, keys))
            reproj.append(term)
        elif isinstance(term, EikonalLoss):
            if keys != {'eik_grad': 'eik_grad'}:
                raise NotImplementedError('fuse_objective: EikonalLoss must read eik_grad, got input_dict %r' % (keys,))
            eik.append(term)
        elif any(v in _PER_SAMPLE_KEYS for v in keys.values()):
            raise NotImplementedError('fuse_objective: %s reads per-sample outputs %r' % (type(term).__name__, keys))
    if len(reproj) > 1 or len(eik) > 1:
        raise NotImplementedError('fuse_objective: at most one reprojection term and one EikonalLoss, got %d and %d'
                                  % (len(reproj), len(eik)))
    if len(sg) > 1:
        raise NotImplementedError('fuse_objective: at most one SecondGradLoss, got %d' % len(sg))
    if sg and not getattr(head, 'return_second_grad', False):
        raise NotImplementedError('fuse_objective: SecondGradLoss needs a head with return_second_grad=True')
    if sg and not getattr(head, 'second_grad_assumption', False):
        raise NotImplementedError('fuse_objective: second_grad is a declared assumption: construct the head with '
                                  'second_grad_assumption=True (or set SELFOCC_B200_SECOND_GRAD=1)')
    rec = dict(mode=reproj[0].MODE if reproj else None, img_size=tuple(reproj[0].img_size) if reproj else None, eikonal=bool(eik))
    if second_grad:
        rec['second_grad'] = bool(sg)
    head.fused_objective = rec
    return head.fused_objective


@LOSSES.register_module()
class MultiLoss(nn.Module):
    """Sum of the terms built from loss_cfgs through LOSSES (loss/multi_loss.py) -> (tot_loss, loss_dict).
    loss_dict maps each term's class name to its detached 0-d device tensor, not a Python float: nothing here reads the
    host, and f'{v:.5f}' formats the tensor as it would the float.  An attached ``writer`` (add_scalar(tag, value, step))
    logs every term and the total on every 10th call, as the reference does; that logging reads the host."""

    def __init__(self, loss_cfgs):
        super().__init__()
        assert isinstance(loss_cfgs, list)
        self.num_losses = len(loss_cfgs)
        self.losses = nn.ModuleList([LOSSES.build(c) for c in loss_cfgs])
        self.iter_counter = 0
        self.writer = None
        self.group = None             # process group of a ray-sharded step (None: the default group)
        self.collective = None        # collective(out, buf) of dist.all_gather_ray_payload (None: all_gather_into_tensor)

    def forward(self, inputs):
        """With inputs['ray_shard'] = (rank, world, R_full), world > 1 (NeuSHead under head.ray_shard), the inputs hold this
        rank's slice of every camera's rays and the objective runs in two stages: local_payload (the per-ray quantities of
        this rank's rays), ONE gather of every term's payload, and from_gathered (each term's formulas on the full ray grid).
        Every rank then returns the unsharded loss values; the gradients follow dist.all_gather_ray_payload's contract
        (averaged over the ranks, as DistributedDataParallel does, they are the unsharded gradients)."""
        shard = inputs.get('ray_shard')
        if shard is not None and shard[1] > 1:
            return self.from_gathered(self.gather(self.local_payload(inputs), shard[0], shard[1]), inputs)
        return self._total(loss_func(inputs) for loss_func in self.losses)

    def local_payload(self, inputs):
        """Stage 1 of a ray-sharded step: per term a list of (this rank's [L, count, k] slice, its full length)."""
        shard = inputs['ray_shard']
        return [loss_func.local_payload(inputs, shard) for loss_func in self.losses]

    def gather(self, payload, rank, world):
        """local_payload's slices of every rank -> per term the list of full tensors, in one collective."""
        from .dist import all_gather_ray_payload
        flat = [p for term in payload for p in term]
        if not flat:
            return payload
        full = iter(all_gather_ray_payload([t for t, _ in flat], [n for _, n in flat], rank, world, self.collective, self.group))
        return [[next(full) for _ in term] for term in payload]

    def from_gathered(self, full, inputs):
        """Stage 2 of a ray-sharded step: (tot_loss, loss_dict) from gather's full tensors."""
        return self._total(loss_func.from_gathered(f, inputs) for loss_func, f in zip(self.losses, full))

    def _total(self, losses):
        loss_dict = {}
        tot_loss = 0.
        log = self.writer is not None and self.iter_counter % 10 == 0
        for loss_func, loss in zip(self.losses, losses):
            tot_loss = tot_loss + loss
            name = loss_func.__class__.__name__
            loss_dict[name] = loss.detach()
            if log:
                self.writer.add_scalar(f'loss/{name}', loss.detach().item(), self.iter_counter)
        if log:
            self.writer.add_scalar('loss/total', tot_loss.detach().item(), self.iter_counter)
        self.iter_counter += 1
        return tot_loss, loss_dict
