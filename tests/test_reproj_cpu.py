"""CPU: the reprojection-loss oracle against the reference's own losses (golden vectors), the native loss modules built
from the shipped configs' loss dicts, and argument checking of the statistics entry points."""
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, 'golden', 'reference_golden_reproj.npz')
CFGS = os.path.join(HERE, 'golden', 'reference_loss_cfgs.json')


def _case(dtype):
    z = np.load(GOLD)
    t = lambda k: torch.from_numpy(z[k]).to(dtype)
    return z, dict(curr=t('curr')[0], prev=t('prev')[0], nxt=t('next')[0], ts=list(t('ts').unbind(0)), img2prev=t('img2prev'),
                   img2next=t('img2next'), ms_rays=t('ms_rays'), img_size=[int(v) for v in z['img_size']]), t


@pytest.mark.parametrize('variant', ['combine', 'multi_new'])
@pytest.mark.parametrize('ssim', [True, False])
@pytest.mark.parametrize('auto', [True, False])
@pytest.mark.parametrize('deltas', [False, True])
def test_oracle_matches_reference_golden(variant, ssim, auto, deltas):
    from oracle.reproj import reproj_loss_ref
    z, kw, t = _case(torch.float32)
    w = t('weights').clone().requires_grad_(True)
    loss = reproj_loss_ref(variant, weights=list(w.unbind(0)), ray_resize=[int(v) for v in z['ray_resize']], no_ssim=not ssim,
                           no_automask=not auto, deltas=list(t('deltas').unbind(0)) if deltas else None, **kw)
    loss.backward()
    tag = '%s_ssim%d_auto%d_deltas%d' % (variant, ssim, auto, deltas)
    ref_loss, ref_grad = float(z[tag + '_loss']), z[tag + '_grad']
    assert abs(float(loss) - ref_loss) <= 1e-6 * abs(ref_loss), (float(loss), ref_loss)
    err = np.abs(w.grad.numpy() - ref_grad).max()
    assert err <= 1e-6 * np.abs(ref_grad).max(), (err, np.abs(ref_grad).max())


def test_golden_case_covers_the_edge_cases():
    """The stored case has samples behind the camera, samples that leave the image and rays without a valid sample."""
    from oracle.reproj import ray_stats_ref, _project
    z, kw, t = _case(torch.float64)
    stats, _ = ray_stats_ref('multi_new', kw['curr'], kw['prev'], kw['nxt'], list(t('weights').unbind(0)), kw['ts'],
                             kw['img2prev'], kw['img2next'], kw['ms_rays'], kw['img_size'])
    assert (stats[..., 5] == 0).any() and (stats[..., 11] == 0).any() and (stats[..., 5] == 1).any()
    assert ((stats[..., 5] == 0) & (stats[..., 11] == 0)).any()          # no valid sample in either frame
    R = kw['ms_rays'].shape[0]
    S = kw['ts'][0].numel() // R
    pix = kw['ms_rays'].repeat_interleave(S, 0)
    behind = leave = 0
    for cam in range(2):
        for M in (kw['img2prev'][cam], kw['img2next'][cam]):
            coords = torch.cat([pix * kw['ts'][cam][:, None], kw['ts'][cam][:, None], torch.ones(R * S, 1, dtype=torch.float64)], 1)
            zc = (coords @ M.T)[:, 2]
            _, m = _project(M, pix, kw['ts'][cam], kw['img_size'])
            behind += int((zc <= 0).sum())
            leave += int(((zc > 0) & ~m).sum())
    assert behind > 0 and leave > 0


def _cfgs():
    return json.load(open(CFGS))


def test_loss_modules_build_from_the_shipped_configs():
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss as L
    cfgs = _cfgs()
    assert {c['type'] for c in cfgs.values()} == {'ReprojLossMonoMultiNewCombine', 'ReprojLossMonoMultiNew'}
    for name, c in cfgs.items():
        m = LOSSES.build(c)
        assert type(m).__name__ == c['type'] and isinstance(m, (L.ReprojLossMonoMultiNewCombine, L.ReprojLossMonoMultiNew))
        assert m.img_size == list(c['img_size']) and m.ray_resize == list(c['ray_resize']) and not m.no_ssim
        assert m.input_dict == c['input_dict'] and m.weight == c['weight'] and m.iter_counter == 0, name
        assert m.no_automask == c.get('no_automask', False)


def test_loss_modules_refuse_unsupported_options():
    from selfocc_b200.loss import ReprojLossMonoMultiNew, ReprojLossMonoMultiNewCombine
    with pytest.raises(NotImplementedError, match='sdf_loss'):
        ReprojLossMonoMultiNew(sdf_loss=True, ray_resize=[6, 10])
    for cls in (ReprojLossMonoMultiNew, ReprojLossMonoMultiNewCombine):
        with pytest.raises(NotImplementedError, match='dims'):
            cls(dims=4, ray_resize=[6, 10])
        assert cls(ray_resize=None).no_ssim                # no ray grid: SSIM is off, as in the reference


def test_loss_refuses_batch_above_one_and_a_partial_ray_grid():
    """Both checks run before any device work, so CPU tensors suffice."""
    from selfocc_b200.loss import ReprojLossMonoMultiNewCombine
    m = ReprojLossMonoMultiNewCombine(ray_resize=[6, 10], img_size=[48, 80])
    imgs = torch.zeros(2, 2, 3, 8, 8)
    w = [torch.zeros(60 * 4)] * 2
    args = dict(curr_imgs=imgs, prev_imgs=imgs, next_imgs=imgs, ray_indices=w, weights=w, ts=w, metas=[{}], ms_rays=torch.zeros(60, 2))
    with pytest.raises(NotImplementedError, match='batch size'):
        m.reproj_loss(**args)
    imgs = imgs[:1]
    w = [torch.zeros(30 * 4)] * 2
    with pytest.raises(ValueError, match='ray_resize'):
        m.reproj_loss(**dict(args, curr_imgs=imgs, prev_imgs=imgs, next_imgs=imgs, ray_indices=w, weights=w, ts=w,
                             ms_rays=torch.zeros(30, 2)))
    with pytest.raises(ValueError, match='R \\* S'):
        m.reproj_loss(**dict(args, curr_imgs=imgs, prev_imgs=imgs, next_imgs=imgs, weights=[torch.zeros(61)] * 2))


def test_reproj_entry_points_reject_bad_arguments_without_a_gpu():
    """Null pointers, non-positive sizes, a bad img_size or mode: SO_ERR_INVALID_ARG before any CUDA call."""
    import ctypes as C
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N, one = None, C.c_void_p(16)
    # (weights, ts, deltas, pix, img2prev, img2next, curr, prev, next, n_cam, R, S, img_h, img_w, size_h, size_w, mode)
    good = [one] * 9 + [6, 4800, 256, 90, 160, 768.0, 1600.0, 0]

    def fwd(i=None, bad=None, stats=one):
        a = list(good)
        if i is not None:
            a[i] = bad
        return lib.so_reproj_stats_forward(*a, stats, N, N)

    def bwd(i=None, bad=None, st=one, g=one, gw=one):
        a = list(good[1:])
        if i is not None:
            a[i - 1] = bad
        return lib.so_reproj_stats_backward(*a, st, g, gw, N)

    for i in (0, 1, 3, 4, 5, 6, 7, 8):                     # every required pointer; deltas (2) is optional
        assert fwd(i, N) == -1, i
    assert fwd(stats=N) == -1
    for i, bad in ((9, 0), (10, 0), (11, 0), (12, 0), (13, -1), (14, 0.0), (15, -5.0), (14, float('nan')), (16, 2)):
        assert fwd(i, bad) == -1, (i, bad)
    for i in (1, 3, 4, 5, 6, 7, 8):
        assert bwd(i, N) == -1, i
    assert bwd(st=N) == -1 and bwd(g=N) == -1 and bwd(gw=N) == -1
    for i, bad in ((9, 0), (11, 0), (16, 7), (15, float('inf'))):
        assert bwd(i, bad) == -1, (i, bad)
    a = list(good)
    a[12], a[13] = 65536, 65536                            # image plane beyond 32-bit pixel offsets
    assert lib.so_reproj_stats_forward(*a, one, N, N) == -2
