"""Oracle: the non-reprojection terms of the shipped configs' objectives and MultiLoss (test infrastructure; any dtype,
any device; fp64 for the reference values, fp32 for the reference composition the native path is timed against).

Each function restates one reference term from its source, with autograd through every input:
  * eikonal_ref        loss/eikonal_loss.py:19-21         mean over rows of (|g|_2 - 1)^2
  * second_grad_ref    loss/second_grad_loss.py:19-20     mean |x|
  * soft_sparsity_ref  loss/sparsity_loss.py:80-81        mean relu(-x)
  * rgb_ref            loss/rgb_loss_ms.py:68-99          l1 at the ray pixels (grid_sample, zeros padding), with SSIM
                                                          0.15 l1 + 0.85 SSIM over the ray grid (SSIM class :7-37)
  * sem_bce_ref        loss/rgb_loss_ms.py:126-155        binary cross-entropy of clamp(s, 0, 1) vs one-hot labels, the
                                                          log clamped at -100 as F.binary_cross_entropy does
  * sem_ce_ref         loss/rgb_loss_ms.py:183-213        mean over rays of sum_c -log(clamp(s, 1e-6, 1)) one_hot
  * edge_ref           loss/edge_loss_3d_ms.py:7-79       edge-aware smoothness of the mean-normalised depth over the ray
                                                          grid (grid_sample, border padding), optional inf mask
  * multi_loss_ref     loss/multi_loss.py:24-44           sum of weight * term; loss_dict by class name
The ray pixel (x, y) samples the image at (x / img_size[1], y / img_size[0]) * 2 - 1 with align_corners=True
(rgb_loss_ms.py:73-84, edge_loss_3d_ms.py:56-66): normalised by the loss's img_size, not by the image's shape.
"""
import torch
import torch.nn.functional as F

from .reproj import ssim_ref

# SemCELossMS's clamp bound as the reference's fp32 run sees it: in a fp64 run the value stays the fp32 number, so that
# a probability exactly at the bound passes its gradient as it does in the reference
CE_MIN32 = float(torch.tensor(1e-6, dtype=torch.float32))


def eikonal_ref(g):
    return ((g.norm(2, dim=-1) - 1) ** 2).mean()          # vector_norm's backward is 0 at a zero norm


def second_grad_ref(x):
    return x.abs().mean()


def soft_sparsity_ref(x):
    return torch.relu(-x).mean()


def rays_sample_ref(imgs, rays, img_size, padding):
    """imgs [M, C, H, W], rays [R, 2] -> [M, C, R]."""
    pix = rays.to(imgs.dtype).clone()
    pix[:, 0] = pix[:, 0] / img_size[1]
    pix[:, 1] = pix[:, 1] / img_size[0]
    grid = (pix * 2 - 1).reshape(1, 1, -1, 2).repeat(imgs.shape[0], 1, 1, 1)
    return F.grid_sample(imgs, grid, mode='bilinear', padding_mode=padding, align_corners=True)[:, :, 0]


def rgb_ref(ms_colors, ms_rays, gt_imgs, img_size, ray_resize=None, no_ssim=True):
    bs, n = gt_imgs.shape[:2]
    R = ms_rays.shape[0]
    gt = rays_sample_ref(gt_imgs.flatten(0, 1), ms_rays, img_size, 'zeros').reshape(bs, n, 3, R).transpose(-1, -2)
    tot = 0.
    for c in ms_colors:
        loss = (c - gt).abs().mean()
        if not (no_ssim or ray_resize is None):
            grid = lambda t: t.reshape(bs * n, *ray_resize, 3).permute(0, 3, 1, 2)
            loss = 0.15 * loss + 0.85 * ssim_ref(grid(c), grid(gt)).mean()
        tot = tot + loss
    return tot / len(ms_colors)


def _labels(sem_lab, rays):
    """sem_lab [B, N, H, W] integer labels -> [B, N, R] at the ray pixels (truncated to integers, as .to(torch.long))."""
    r = rays.long()
    return sem_lab.long()[:, :, r[:, 1], r[:, 0]]


class _BCE(torch.autograd.Function):
    """F.binary_cross_entropy(p, y), mean reduction: value -(y max(log p, -100) + (1 - y) max(log(1 - p), -100)), and
    ATen's gradient (p - y) / max(p (1 - p), 1e-12), which does not see the clamp of the log."""

    @staticmethod
    def forward(ctx, p, y):
        ctx.save_for_backward(p, y)
        return (-(y * torch.clamp(torch.log(p), min=-100) + (1 - y) * torch.clamp(torch.log1p(-p), min=-100))).mean()

    @staticmethod
    def backward(ctx, g):
        p, y = ctx.saved_tensors
        return g * (p - y) / torch.clamp(p * (1 - p), min=1e-12) / p.numel(), None


def sem_bce_ref(sem, sem_lab, ms_rays):
    tot = 0.
    for s in sem:
        gt = F.one_hot(_labels(sem_lab, ms_rays), s.shape[-1]).to(s.dtype)
        tot = tot + _BCE.apply(torch.clamp(s, 0, 1), gt)
    return tot / len(sem)


def sem_ce_ref(sem, sem_lab, ms_rays):
    tot = 0.
    for s in sem:
        gt = F.one_hot(_labels(sem_lab, ms_rays), s.shape[-1]).to(s.dtype)
        tot = tot + torch.sum(-torch.log(torch.clamp(s, CE_MIN32, 1)) * gt, dim=-1).mean()
    return tot / len(sem)


def edge_ref(curr_imgs, ms_depths, ms_rays, img_size, ray_resize, ms_accs=None, max_depths=None):
    bs, n, R = ms_depths[0].shape
    tot = 0.
    for k, d in enumerate(ms_depths):
        img = rays_sample_ref(curr_imgs.flatten(0, 1), ms_rays, img_size, 'border').reshape(bs * n, -1, *ray_resize)
        if ms_accs is not None:
            d = d * ms_accs[k] + max_depths[k] * (1 - ms_accs[k])
        d = d.reshape(bs * n, 1, *ray_resize)
        d = d / (d.mean(2, True).mean(3, True) + 1e-6)
        wx = torch.exp(-(img[..., :-1] - img[..., 1:]).abs().mean(1, True))
        wy = torch.exp(-(img[..., :-1, :] - img[..., 1:, :]).abs().mean(1, True))
        tot = tot + ((d[..., :-1] - d[..., 1:]).abs() * wx).mean() + ((d[..., :-1, :] - d[..., 1:, :]).abs() * wy).mean()
    return tot / len(ms_depths)


def term_ref(cfg, inputs, sem_lab=None):
    """weight * term for one loss cfg of a shipped config; inputs by the cfg's input_dict names (the reference's keys)."""
    t = cfg['type']
    keys = cfg.get('input_dict')
    get = lambda k: inputs[keys[k]] if keys and k in keys else inputs[k]
    if t == 'EikonalLoss':
        v = eikonal_ref(get('eik_grad'))
    elif t == 'SecondGradLoss':
        v = second_grad_ref(get('second_grad'))
    elif t == 'SoftSparsityLoss':
        v = soft_sparsity_ref(get('density'))
    elif t == 'RGBLossMS':
        v = rgb_ref(get('ms_colors'), get('ms_rays'), get('gt_imgs'), cfg['img_size'], cfg.get('ray_resize'), cfg.get('no_ssim', True))
    elif t in ('SemLossMS', 'SemCELossMS'):
        v = (sem_bce_ref if t == 'SemLossMS' else sem_ce_ref)(get('sem'), sem_lab, get('ms_rays'))
    elif t == 'EdgeLoss3DMS':
        v = edge_ref(get('curr_imgs'), get('ms_depths'), get('ms_rays'), cfg.get('img_size', [768, 1600]), cfg['ray_resize'],
                     get('ms_accs') if cfg.get('use_inf_mask') else None, get('max_depths') if cfg.get('use_inf_mask') else None)
    else:
        raise KeyError(t)
    return cfg.get('weight', 1.0) * v


def multi_loss_ref(cfgs, inputs, sem_lab=None):
    """(total, {class name: value}) of MultiLoss over the given non-reprojection cfgs."""
    tot, d = 0., {}
    for c in cfgs:
        v = term_ref(c, inputs, sem_lab)
        tot = tot + v
        d[c['type']] = v
    return tot, d
