"""GPU: the native reprojection losses (so_reproj_stats_forward / _backward + the torch per-ray tail) against the fp64
oracle (oracle/reproj.py, pinned to the reference by tests/test_reproj_cpu.py).

The validity masks are discontinuous in the sample depth, so a strict comparison needs inputs whose masks fp32 and fp64
agree on: every sample whose fp64 reprojection lies within GUARD_PX of an image bound, or whose depth in the other frame
is within GUARD_Z of zero, is moved before the comparison.  Rays whose automask min is a near-tie (relative gap < 1e-6) are
counted and left out of the gradient comparison: the min picks a different branch under rounding there."""
import numpy as np
import pytest
import torch

from selfocc_b200 import synth

pytestmark = pytest.mark.gpu
GUARD_PX, GUARD_Z = 1e-3, 1e-4
SMALL = dict(n_cam=3, ray_resize=(6, 10), S=48, img_size=(96, 160), img_hw=(60, 100))
NUSC = dict(n_cam=6, ray_resize=(48, 100), S=256, img_size=(768, 1600), img_hw=(768, 1600))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _guard_bad(M, pix, t, img_size):
    """fp64: samples within the guard band of a mask bound. M [N,4,4], pix [R*S,2], t [N,R*S]."""
    c = torch.stack([pix[None, :, 0] * t, pix[None, :, 1] * t, t, torch.ones_like(t)], -1)
    p = torch.einsum('nij,nsj->nsi', M, c)
    z = p[..., 2]
    x, y = p[..., 0] / z.clamp_min(1e-5), p[..., 1] / z.clamp_min(1e-5)
    near = lambda a, b: (a - b).abs() < GUARD_PX
    edge = near(x, 0) | near(x, img_size[1]) | near(y, 0) | near(y, img_size[0])
    return (z.abs() < GUARD_Z) | ((z > 0) & edge)


def make_case(dev, n_cam, ray_resize, S, img_size, img_hw, seed=0):
    g = torch.Generator().manual_seed(seed)
    h, w = img_size
    R = ray_resize[0] * ray_resize[1]
    yaws = synth.NUSC_YAWS[:n_cam]
    prev, nxt = synth.temporal_rig(yaws, f=1266.0 * w / 1600, cx=w / 2, cy=h * 450 / 900, forward=0.5, yaw_deg=1.0)
    # the last camera: large pixel shifts, so that rays at the right / bottom have no valid sample in either frame
    prev[-1, 0] += 0.3 * w * prev[-1, 2]
    nxt[-1, 1] += 0.4 * h * nxt[-1, 2]
    ys, xs = torch.meshgrid(torch.arange(ray_resize[0]), torch.arange(ray_resize[1]), indexing='ij')
    rays = torch.stack([(xs.flatten() + torch.rand(R, generator=g)) * w / ray_resize[1],
                        (ys.flatten() + torch.rand(R, generator=g)) * h / ray_resize[0]], -1).float()
    ts = (0.3 + 50.0 * torch.rand(n_cam, R * S, generator=g) ** 2).float()
    ts[:, S:2 * S] = 0.3                                   # a ray close to the camera: behind the next frame's camera
    Mp, Mn = torch.from_numpy(prev), torch.from_numpy(nxt)
    pix = rays.double().repeat_interleave(S, 0)
    for _ in range(20):
        bad = _guard_bad(Mp, pix, ts.double(), img_size) | _guard_bad(Mn, pix, ts.double(), img_size)
        if not bad.any():
            break
        ts = torch.where(bad, ts * 1.0037, ts)
    assert not bad.any()
    wts = torch.rand(n_cam, R * S, generator=g) * (torch.rand(n_cam, R * S, generator=g) < 0.8)
    wts[:, 2 * S:3 * S] = 0.                               # all-zero weights: the eps clamp
    deltas = 0.01 + 0.5 * torch.rand(n_cam, R * S, generator=g)
    deltas[:, ::11] = 0.
    imgs = synth.textured_images(3 * n_cam, *img_hw, seed=seed + 1).reshape(3, 1, n_cam, 3, *img_hw)
    to = lambda t: t.to(dev).contiguous()
    return dict(curr=to(imgs[0]), prev=to(imgs[1]), next=to(imgs[2]), rays=to(rays), ts=to(ts), weights=to(wts), deltas=to(deltas),
                img2prev=to(Mp.float()), img2next=to(Mn.float()), img_size=list(img_size), ray_resize=list(ray_resize), S=S)


def _native(cls, case, ssim, auto, use_deltas):
    keys = {k: k for k in ('curr_imgs', 'prev_imgs', 'next_imgs', 'ray_indices', 'weights', 'ts', 'metas', 'ms_rays')}
    if use_deltas:
        keys['deltas'] = 'deltas'
    m = cls(weight=1.0, input_dict=keys, no_ssim=not ssim, img_size=case['img_size'], ray_resize=case['ray_resize'],
            no_automask=not auto)
    w = case['weights'].clone().requires_grad_(True)
    n_cam = w.shape[0]
    R = case['rays'].shape[0]
    ridx = torch.arange(R, device=w.device).repeat_interleave(case['S'])
    inputs = dict(curr_imgs=case['curr'], prev_imgs=case['prev'], next_imgs=case['next'], ray_indices=[ridx] * n_cam,
                  weights=list(w.unbind(0)), ts=list(case['ts'].unbind(0)), deltas=list(case['deltas'].unbind(0)),
                  metas=[dict(img2prevImg=case['img2prev'], img2nextImg=case['img2next'])], ms_rays=case['rays'])
    return m, w, inputs


def _oracle(variant, case, ssim, auto, use_deltas):
    from oracle.reproj import ray_stats_ref, loss_from_stats_ref
    d = lambda t: t.double()
    w = d(case['weights']).requires_grad_(True)
    stats, colours = ray_stats_ref(variant, d(case['curr'][0]), d(case['prev'][0]), d(case['next'][0]), list(w.unbind(0)),
                                   list(d(case['ts']).unbind(0)), d(case['img2prev']), d(case['img2next']), d(case['rays']),
                                   case['img_size'], list(d(case['deltas']).unbind(0)) if use_deltas else None)
    loss, cands = loss_from_stats_ref(variant, stats, colours, case['ray_resize'], not ssim, not auto)
    g, = torch.autograd.grad(loss, w)
    return stats.detach(), colours, loss.detach(), g, cands.detach()


_CASES = {}


def _case(size):
    if size not in _CASES:
        _CASES[size] = make_case(_dev(), **(SMALL if size == 'small' else NUSC))
    return _CASES[size]


@pytest.mark.parametrize('size', ['small', 'nusc'])
@pytest.mark.parametrize('variant', ['combine', 'multi_new'])
@pytest.mark.parametrize('ssim', [True, False])
@pytest.mark.parametrize('auto', [True, False])
@pytest.mark.parametrize('use_deltas', [False, True])
def test_native_loss_matches_fp64_oracle(size, variant, ssim, auto, use_deltas):
    from selfocc_b200.loss import ReprojLossMonoMultiNew, ReprojLossMonoMultiNewCombine
    case = _case(size)
    cls = ReprojLossMonoMultiNewCombine if variant == 'combine' else ReprojLossMonoMultiNew
    m, w, inputs = _native(cls, case, ssim, auto, use_deltas)
    with torch.no_grad():
        stats, colours, _ = m._stats(inputs['curr_imgs'], inputs['prev_imgs'], inputs['next_imgs'], inputs['ray_indices'],
                                     inputs['weights'], inputs['ts'], inputs['metas'], inputs['ms_rays'],
                                     inputs['deltas'] if use_deltas else None)
    loss = m(inputs)
    loss.backward()
    ostats, ocol, oloss, ograd, cands = _oracle(variant, case, ssim, auto, use_deltas)
    # edge cases present in the inputs
    anys = ostats[..., 5::6]
    assert (anys == 0).any() and (anys == 1).any()
    if variant == 'combine':
        assert ((ostats[..., 0] == 0) & (ostats[..., 5] == 1)).any()       # valid samples, all weights zero
    assert torch.equal(stats[..., 5::6].cpu(), anys.float().cpu())
    for k in range(stats.shape[-1]):
        ref = ostats[..., k]
        err = (stats[..., k].double() - ref).abs().max().item()
        assert err <= 1e-5 * max(ref.abs().max().item(), 1e-30), (k, err)
    assert (colours.double() - ocol).abs().max().item() <= 1e-6
    assert abs(loss.item() - oloss.item()) <= 1e-5 * abs(oloss.item()), (loss.item(), oloss.item())
    # d loss / d weights, without the rays whose min is a near-tie
    # (a tie of two 1e3 filters carries no gradient either way)
    srt = cands.sort(dim=-1).values
    if srt.shape[-1] > 1:
        tie = ((srt[..., 1] - srt[..., 0]).abs() <= 1e-6 * srt[..., 0].abs()) & (srt[..., 0] < 1e3)
    else:
        tie = torch.zeros_like(srt[..., 0], dtype=torch.bool)
    keep = (~tie).repeat_interleave(case['S'], dim=1)
    assert tie.float().mean().item() < 0.05, int(tie.sum())   # includes exact ties, e.g. two zero-weight directions at l1 = 0
    gn, go = w.grad.double()[keep], ograd[keep]
    assert (gn - go).abs().max().item() <= 1e-5 * go.abs().max().item()


def test_native_loss_is_deterministic_and_never_syncs_with_the_host():
    from selfocc_b200.loss import ReprojLossMonoMultiNew, ReprojLossMonoMultiNewCombine
    case = _case('small')
    for cls in (ReprojLossMonoMultiNewCombine, ReprojLossMonoMultiNew):
        res = []
        for _ in range(2):
            m, w, inputs = _native(cls, case, True, True, True)
            torch.cuda.synchronize()
            torch.cuda.set_sync_debug_mode('error')
            try:
                loss = m(inputs)
                loss.backward()
            finally:
                torch.cuda.set_sync_debug_mode(0)
            res.append((loss.detach().clone(), w.grad.clone()))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])


def test_weight_lists_that_are_not_one_buffer_give_the_same_result():
    """Separate per-camera tensors are stacked; the gradients come back in the inputs' shapes."""
    from selfocc_b200.loss import ReprojLossMonoMultiNewCombine
    case = _case('small')
    m, w, inputs = _native(ReprojLossMonoMultiNewCombine, case, True, True, False)
    l0 = m(inputs)
    l0.backward()
    sep = [x.detach().clone().reshape(-1, case['S'], 1).requires_grad_(True) for x in w.unbind(0)]
    inputs['weights'] = sep
    inputs['ts'] = [t.clone() for t in inputs['ts']]
    l1 = m(inputs)
    l1.backward()
    assert torch.equal(l0.detach(), l1.detach())
    for i, s in enumerate(sep):
        assert s.grad.shape == s.shape and torch.equal(s.grad.reshape(-1), w.grad[i])


def test_ray_count_that_does_not_fill_ray_resize_is_refused_with_ssim():
    from selfocc_b200.loss import ReprojLossMonoMultiNewCombine
    case = _case('small')
    m, w, inputs = _native(ReprojLossMonoMultiNewCombine, case, True, True, False)
    m.ray_resize = [6, 11]
    with pytest.raises(ValueError, match='ray_resize'):
        m(inputs)


def test_head_forward_feeds_the_native_loss_and_gradients_match_the_oracle_loss():
    """NeuSHead.forward (training, 6 cams x 48x100 rays of a 768x1600 rig) -> ReprojLossMonoMultiNewCombine -> backward to
    the planes and the decode MLP, against the oracle loss on the same head outputs.  Rays with a sample inside the
    mask guard band are counted (at most 0.1 %) and taken out of both sides, as are automask near-ties: the parameter
    gradients compared are those of d loss / d weights on the other rays, back-propagated through the head."""
    dev = _dev()
    from selfocc_b200 import configs
    from selfocc_b200.registry import build_head
    from selfocc_b200.loss import ReprojLossMonoMultiNewCombine
    import selfocc_b200.segmentor  # noqa: F401
    from oracle.reproj import reproj_loss_ref
    torch.manual_seed(0)
    img_size, ray_resize, S = (768, 1600), [48, 100], 32
    margs, rng = synth.small_mapping(16, 8, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=S, ray_number=tuple(ray_resize), ray_img_size=img_size, color_dims=3)
    head = build_head(cfg['head']).to(dev).train()
    with torch.no_grad():
        head.model.field.deviation_network.variance.fill_(0.25)
    l2i, i2l = synth.camera_rig()
    prev, nxt = synth.temporal_rig()
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=img_size,
                  img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                  img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))]
    H, W, Z = 33, 33, 9
    planes = [(0.5 * torch.randn(1, n, 96, device=dev)).requires_grad_(True) for n in (H * W, Z * H, W * Z)]
    imgs = synth.textured_images(18, 192, 400, seed=3).reshape(3, 1, 6, 3, 192, 400).to(dev)
    R = ray_resize[0] * ray_resize[1]
    jitter = torch.rand(6 * R, S + 1, device=dev)
    f = head.model.field
    params = planes + [f.density_net[1].weight, f.density_net[3].weight]
    out = head(representation=planes, metas=metas, jitter=jitter)
    assert out['ms_rays'].shape[0] == R
    ts = torch.stack(out['ts']).detach().double().cpu()
    pix = out['ms_rays'].detach().double().cpu().repeat_interleave(S, 0)
    bad = _guard_bad(torch.from_numpy(prev), pix, ts, img_size) | _guard_bad(torch.from_numpy(nxt), pix, ts, img_size)
    bad_rays = bad.reshape(6, R, S).any(-1)
    assert bad_rays.float().mean().item() <= 1e-3, int(bad_rays.sum())
    # automask near-ties: the fp32 oracle's SSIM carries ~1e-4 relative rounding, so its min may take the other branch
    from oracle.reproj import ray_stats_ref, loss_from_stats_ref
    d = lambda t: t.detach().double()
    st, col = ray_stats_ref('combine', d(imgs[0][0]), d(imgs[1][0]), d(imgs[2][0]), [d(w) for w in out['weights']],
                            [d(t) for t in out['ts']], d(metas[0]['img2prevImg']), d(metas[0]['img2nextImg']), d(out['ms_rays']),
                            list(img_size))
    srt = loss_from_stats_ref('combine', st, col, ray_resize)[1].sort(dim=-1).values
    tie = ((srt[..., 1] - srt[..., 0]).abs() <= 1e-3 * srt[..., 0].abs()).cpu()
    assert tie.float().mean().item() < 0.01, int(tie.sum())
    keep = (~(bad_rays | tie)).repeat_interleave(S, 1).to(dev).float()

    def grads(loss):
        gw = torch.autograd.grad(loss, out['weights'], retain_graph=True)
        gp = torch.autograd.grad(out['weights'], params, [g * k for g, k in zip(gw, keep)], retain_graph=True)
        return torch.stack(gw) * keep, gp

    inputs = dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], metas=metas)
    ln = ReprojLossMonoMultiNewCombine(img_size=list(img_size), ray_resize=ray_resize)(inputs)
    # the oracle consumes the same head outputs in fp64: in fp32 its autograd through w / W and its SSIM variances cancel
    # to ~1e-2 of the gradient on rays of small total weight
    lo = reproj_loss_ref('combine', d(imgs[0][0]), d(imgs[1][0]), d(imgs[2][0]), [w.double() for w in out['weights']],
                         [d(t) for t in out['ts']], d(metas[0]['img2prevImg']), d(metas[0]['img2nextImg']), d(out['ms_rays']),
                         list(img_size), ray_resize)
    (gwn, gpn), (gwo, gpo) = grads(ln), grads(lo)
    assert abs(ln.item() - lo.item()) <= 1e-5 * abs(lo.item())
    assert (gwn - gwo).abs().max().item() <= 1e-4 * gwo.abs().max().item()
    for a, b in zip(gpn, gpo):
        assert a.abs().sum() > 0 and torch.isfinite(a).all()
        assert (a - b).abs().max().item() <= 1e-4 * b.abs().max().item()
