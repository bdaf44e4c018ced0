"""Oracle: the two photometric reprojection losses (test infrastructure; fp32 or fp64, any device).

Restates ReprojLossMonoMultiNewCombine (reference loss/reproj_loss_mono_multi_new_combine.py:70-248) and
ReprojLossMonoMultiNew (loss/reproj_loss_mono_multi_new.py:72-288) from the algorithm, with autograd through the weights:
  * each sample (u t, v t, t, 1) is mapped through img2prevImg / img2nextImg (:118-133 / :128-144), valid when z > 0 and
    0 < x / max(z, 1e-5) < img_w, 0 < y / max(z, 1e-5) < img_h;
  * colours are F.grid_sample(bilinear, align_corners=True) at x / img_w * 2 - 1 (:140-156 / :151-163), padding 'border'
    for Combine and 'zeros' for MultiNew;
  * optional deltas: w / max(delta, eps), 0 where delta < eps (:111-116 / :120-125);
  * Combine: masked-weight-normalised sums over each ray of the per-sample l1 and colour averaged over the valid
    directions (:158-198); MultiNew: the same per direction (:165-192, 219-239);
  * per-ray tail: SSIM over the ray grid, the 1e3 filters, the automask min, the means (:200-248 / :200-288).
eps of the weight-sum clamp and of the deltas is the fp32 epsilon in every dtype: the reference runs in fp32, and a fp64
run restates that function, not a fp64 variant of it.  Everything else runs in the inputs' dtype.  ``ray_stats_ref``
returns the per-ray sums in the kernel's layout (so_reproj_stats_forward) and ``loss_from_stats_ref`` the tail on them.
"""
import torch
import torch.nn.functional as F

EPS32 = float(torch.finfo(torch.float32).eps)


def ssim_ref(x, y):
    """1 - SSIM over 3x3 reflection-padded windows, halved and clamped (the SSIM class of both loss files, :7-37)."""
    x, y = F.pad(x, (1, 1, 1, 1), mode='reflect'), F.pad(y, (1, 1, 1, 1), mode='reflect')
    pool = lambda t: F.avg_pool2d(t, 3, 1)
    mx, my = pool(x), pool(y)
    sx, sy, sxy = pool(x * x) - mx * mx, pool(y * y) - my * my, pool(x * y) - mx * my
    n = (2 * mx * my + 0.01 ** 2) * (2 * sxy + 0.03 ** 2)
    d = (mx * mx + my * my + 0.01 ** 2) * (sx + sy + 0.03 ** 2)
    return torch.clamp((1 - n / d) / 2, 0, 1)


def _project(M, pix_s, t, img_size):
    """M [4,4], pix_s [n,2] ray pixel of each sample, t [n] -> (pixel [n,2], mask [n])."""
    coords = torch.cat([pix_s * t[:, None], t[:, None], torch.ones_like(t)[:, None]], dim=1)     # (u t, v t, t, 1)
    # the reference's broadcast [1,1,1,4,4] @ [1,1,n,4,1] product: same summation order as its fp32 run
    p = torch.matmul(M.reshape(1, 1, 1, 4, 4), coords.reshape(1, 1, -1, 4, 1)).reshape(-1, 4)
    z = p[:, 2]
    px = p[:, :2] / z.clamp_min(1e-5)[:, None]
    mask = (z > 0) & (px[:, 0] > 0) & (px[:, 0] < img_size[1]) & (px[:, 1] > 0) & (px[:, 1] < img_size[0])
    return px, mask


def _sample(img, px, img_size, padding):
    """img [3,H,W], px [n,2] loss pixels -> [n,3]."""
    g = torch.stack([px[:, 0] / img_size[1], px[:, 1] / img_size[0]], dim=-1) * 2 - 1
    return F.grid_sample(img[None], g[None, None].to(img.dtype), mode='bilinear', padding_mode=padding,
                         align_corners=True)[0, :, 0].transpose(0, 1)


def _per_sample(variant, curr, prev, nxt, weights, ts, img2prev, img2next, ms_rays, img_size, deltas):
    """Per camera: (ray index [R*S], effective weight [R*S], [(mask, diff, rgb) per set], colours [R, 9])."""
    padding = 'border' if variant == 'combine' else 'zeros'
    R = ms_rays.shape[0]
    for cam, (w, t) in enumerate(zip(weights, ts)):
        w, t = w.reshape(-1), t.reshape(-1).detach()
        S = w.numel() // R
        ray = torch.arange(R, device=w.device).repeat_interleave(S)
        if deltas is not None:
            d = deltas[cam].reshape(-1).detach()
            w = torch.where(d < EPS32, torch.zeros_like(w), w / d.clamp_min(EPS32))
        cur_r = _sample(curr[cam], ms_rays, img_size, padding)
        colours = torch.cat([cur_r, _sample(prev[cam], ms_rays, img_size, padding), _sample(nxt[cam], ms_rays, img_size, padding)], -1)
        cur = cur_r[ray]
        terms = []
        for M, img in ((img2prev[cam], prev[cam]), (img2next[cam], nxt[cam])):
            px, m = _project(M, ms_rays[ray], t, img_size)
            rgb = _sample(img, px, img_size, padding)
            rgb = torch.where(m[:, None], rgb, torch.zeros_like(rgb))
            diff = torch.where(m, (cur - rgb).abs().mean(-1), torch.zeros_like(t))
            terms.append((m, diff, rgb))
        if variant == 'combine':
            (pm, dp, rp), (nm, dn, rn) = terms
            cnt = (pm.to(t.dtype) + nm.to(t.dtype)).clamp_min(1.0)
            terms = [(pm | nm, (dp + dn) / cnt, (rp + rn) / cnt[:, None])]
        yield ray, w, terms, colours


def ray_stats_ref(variant, curr, prev, nxt, weights, ts, img2prev, img2next, ms_rays, img_size, deltas=None):
    """-> (stats [N, R, 6 * sets] = per set (W, l1, rgb0, rgb1, rgb2, any) with l1 = L / clamp(W, eps) and
    rgb = C / clamp(W, eps) of the sums L, C over the ray, colours [N, R, 9] = curr / prev / next at the ray pixel).
    curr/prev/nxt [N,3,H,W]; weights/ts/deltas: per-camera lists of R*S ray-major samples; img2prev/img2next [N,4,4]."""
    R = ms_rays.shape[0]
    stats, colours = [], []
    for ray, w, terms, col in _per_sample(variant, curr, prev, nxt, weights, ts, img2prev, img2next, ms_rays, img_size, deltas):
        per = []
        for m, diff, rgb in terms:
            wm = torch.where(m, w, torch.zeros_like(w))
            acc = torch.zeros(R, 5, dtype=w.dtype, device=w.device).index_add(
                0, ray, torch.cat([wm[:, None], (wm * diff)[:, None], wm[:, None] * rgb], dim=1))
            anyv = torch.zeros(R, dtype=w.dtype, device=w.device).index_add(0, ray, m.to(w.dtype)) > 0
            per.append(torch.cat([acc[:, :1], acc[:, 1:] / acc[:, :1].clamp_min(EPS32), anyv.to(w.dtype)[:, None]], dim=1))
        stats.append(torch.cat(per, dim=1))
        colours.append(col)
    return torch.stack(stats), torch.stack(colours)


def _tail(variant, sets, colours, ray_resize, no_ssim, no_automask):
    """sets: per direction set (l1 [N,R], colour [N,R,3], any [N,R]) -> (loss, candidates [N, R, K] before the min)."""
    no_ssim = no_ssim or ray_resize is None
    N, R = colours.shape[:2]
    cur = colours[..., 0:3]

    def grid(x):
        return x.reshape(N, ray_resize[0], ray_resize[1], 3).permute(0, 3, 1, 2)

    def photometric(pred, l1):
        if no_ssim:
            return l1
        return 0.85 * ssim_ref(grid(pred), grid(cur)).mean(1).reshape(N, R) + 0.15 * l1

    auto = [photometric(colours[..., k:k + 3], (cur - colours[..., k:k + 3]).abs().mean(-1)) for k in (3, 6)]
    big = torch.full((N, R), 1e3, dtype=colours.dtype, device=colours.device)
    direction = [(photometric(rgb, l1), a) for l1, rgb, a in sets]
    if variant == 'combine':
        c, anyv = direction[0]
        cands = [c] if no_automask else [torch.where(anyv, c, big)] + auto
    else:
        cands = [torch.where(a, c, big) for c, a in direction] + ([] if no_automask else auto)
    cands = torch.stack(cands, dim=-1)
    return cands.min(dim=-1).values.mean(1).sum() / N, cands


def loss_from_stats_ref(variant, stats, colours, ray_resize=None, no_ssim=False, no_automask=False):
    """The per-ray tail on the statistics of ray_stats_ref -> (loss, candidates [N, R, K] before the min)."""
    sets = [(stats[..., 6 * j + 1], stats[..., 6 * j + 2:6 * j + 5], stats[..., 6 * j + 5] > 0) for j in range(stats.shape[-1] // 6)]
    return _tail(variant, sets, colours, ray_resize, no_ssim, no_automask)


def reproj_loss_ref(variant, curr, prev, nxt, weights, ts, img2prev, img2next, ms_rays, img_size, ray_resize=None,
                    no_ssim=False, no_automask=False, deltas=None, weight=1.0):
    """weight * loss of ReprojLossMonoMultiNewCombine (variant 'combine') / ReprojLossMonoMultiNew ('multi_new').  Each
    sample's weight is divided by its ray's clamped masked weight sum before the sums over the ray, the reference's order
    (:178-198 / :175-189), which keeps a fp32 run within rounding of the reference where W is small."""
    R = ms_rays.shape[0]
    sets, colours = [], []
    for ray, w, terms, col in _per_sample(variant, curr, prev, nxt, weights, ts, img2prev, img2next, ms_rays, img_size, deltas):
        per = []
        for m, diff, rgb in terms:
            wm = torch.where(m, w, torch.zeros_like(w))
            wn = wm / torch.zeros(R, dtype=w.dtype, device=w.device).index_add(0, ray, wm).clamp_min(EPS32)[ray]
            acc = torch.zeros(R, 4, dtype=w.dtype, device=w.device).index_add(0, ray, torch.cat([(wn * diff)[:, None],
                                                                                                 wn[:, None] * rgb], 1))
            anyv = torch.zeros(R, dtype=w.dtype, device=w.device).index_add(0, ray, m.to(w.dtype)) > 0
            per.append((acc[:, 0], acc[:, 1:], anyv))
        sets.append(per)
        colours.append(col)
    sets = [tuple(torch.stack([p[j][k] for p in sets]) for k in range(3)) for j in range(len(sets[0]))]
    return weight * _tail(variant, sets, torch.stack(colours), ray_resize, no_ssim, no_automask)[0]
