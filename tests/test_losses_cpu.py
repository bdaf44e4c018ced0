"""CPU: the objective's oracle and torch-side terms against the reference's own losses (golden vectors), MultiLoss built
from every shipped config's loss dict, and argument checking of the per-sample loss-term entry points."""
import json
import os

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, 'golden', 'reference_golden_losses.npz')
CFGS = os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')
IMG_SIZE, RAY_RESIZE = [48, 80], [6, 10]

SHIPPED_TERMS = {
    'nuscenes/nuscenes_occ.py': ['ReprojLossMonoMultiNewCombine', 'RGBLossMS', 'EikonalLoss', 'SecondGradLoss', 'SemCELossMS'],
    'nuscenes/nuscenes_occ_bev.py': ['ReprojLossMonoMultiNewCombine', 'RGBLossMS', 'EikonalLoss', 'SecondGradLoss', 'SemLossMS',
                                     'SoftSparsityLoss'],
    'nuscenes/nuscenes_novel_depth.py': ['ReprojLossMonoMultiNewCombine', 'RGBLossMS', 'EikonalLoss', 'SecondGradLoss'],
    'kitti/kitti_novel_depth.py': ['ReprojLossMonoMultiNew', 'RGBLossMS', 'EikonalLoss', 'SecondGradLoss'],
    'kitti/kitti_occ.py': ['ReprojLossMonoMultiNew', 'RGBLossMS', 'EikonalLoss', 'SecondGradLoss', 'SoftSparsityLoss'],
    'nuscenes/nuscenes_depth.py': ['ReprojLossMonoMultiNewCombine', 'EikonalLoss', 'EdgeLoss3DMS'],
    'kitti_raw/kitti_raw_depth.py': ['ReprojLossMonoMultiNew', 'EikonalLoss', 'EdgeLoss3DMS'],
}


def _gold(dtype=torch.float32):
    z = np.load(GOLD)
    t = lambda k: torch.from_numpy(z[k]).to(dtype) if z[k].dtype.kind == 'f' else torch.from_numpy(z[k])
    return z, t


def _close(loss, grads, z, tag, rtol=1e-6, grad_rtol=None):
    ref = float(z[tag + '_loss'])
    grad_rtol = rtol if grad_rtol is None else grad_rtol
    assert abs(float(loss.detach()) - ref) <= rtol * abs(ref), (tag, float(loss), ref)
    for name, g in grads.items():
        r = z['%s_grad_%s' % (tag, name)]
        err = np.abs(g.detach().double().numpy() - r).max()
        assert err <= grad_rtol * np.abs(r).max(), (tag, name, err, np.abs(r).max())


def _cases():
    out = [('EikonalLoss', None, None), ('SecondGradLoss', None, None), ('SoftSparsityLoss', None, None),
           ('SemLossMS', None, None), ('SemCELossMS', None, None)]
    for rays in ('in', 'out'):
        out += [('RGBLossMS', s, rays) for s in (0, 1)] + [('EdgeLoss3DMS', i, rays) for i in (0, 1)]
    return out


def _run(cls, opt, rays, t, impl, dtype):
    """(tag, loss, {name: leaf}) of one golden case through the oracle (impl='oracle') or the native module."""
    import oracle.losses as O
    import selfocc_b200.loss as L
    leaf = lambda k: t(k).clone().requires_grad_(True)
    metas = [dict(sem=t('sem_lab')[0].numpy())]
    if cls in ('EikonalLoss', 'SecondGradLoss', 'SoftSparsityLoss'):
        name = {'EikonalLoss': 'eik', 'SecondGradLoss': 'sg', 'SoftSparsityLoss': 'dens'}[cls]
        x = leaf(name)
        f = {'EikonalLoss': O.eikonal_ref, 'SecondGradLoss': O.second_grad_ref, 'SoftSparsityLoss': O.soft_sparsity_ref}[cls]
        return cls, f(x), {name: x}
    if cls in ('SemLossMS', 'SemCELossMS'):
        s = leaf('sem')
        if impl == 'oracle':
            loss = (O.sem_bce_ref if cls == 'SemLossMS' else O.sem_ce_ref)([s], t('sem_lab'), t('rays_in'))
        else:
            loss = getattr(L, cls)(img_size=IMG_SIZE)(dict(sem=[s], metas=metas, ms_rays=t('rays_in')))
        return cls, loss, {'sem': s}
    r = t('rays_' + rays)
    if cls == 'RGBLossMS':
        c = leaf('colors')
        if impl == 'oracle':
            loss = O.rgb_ref(list(c.unbind(0)), r, t('gt'), IMG_SIZE, RAY_RESIZE, no_ssim=not opt)
        else:
            loss = L.RGBLossMS(img_size=IMG_SIZE, no_ssim=not opt, ray_resize=RAY_RESIZE)(
                dict(ms_colors=list(c.unbind(0)), ms_rays=r, gt_imgs=t('gt')))
        return 'RGBLossMS_ssim%d_rays%s' % (opt, rays), loss, {'colors': c}
    d, a, mx = leaf('depths'), leaf('accs'), leaf('maxd')
    grads = dict(depths=d, accs=a, maxd=mx) if opt else dict(depths=d)
    if impl == 'oracle':
        loss = O.edge_ref(t('curr'), list(d.unbind(0)), r, IMG_SIZE, RAY_RESIZE, list(a.unbind(0)) if opt else None,
                          list(mx.unbind(0)) if opt else None)
    else:
        keys = dict(curr_imgs='curr_imgs', ms_depths='ms_depths', ms_rays='ms_rays')
        if opt:
            keys.update(ms_accs='ms_accs', max_depths='max_depths')
        loss = L.EdgeLoss3DMS(img_size=IMG_SIZE, ray_resize=RAY_RESIZE, use_inf_mask=bool(opt), input_dict=keys)(
            dict(curr_imgs=t('curr'), ms_depths=list(d.unbind(0)), ms_rays=r, ms_accs=list(a.unbind(0)), max_depths=list(mx.unbind(0))))
    return 'EdgeLoss3DMS_inf%d_rays%s' % (opt, rays), loss, grads


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('cls,opt,rays', _cases())
def test_oracle_matches_reference_golden(cls, opt, rays, dtype):
    """The oracle against the reference's fp32 run: run in fp32 it restates that run within 1e-6; run in fp64 it is within
    1e-6 too, except SSIM's gradient, where the reference's fp32 variances E[x^2] - E[x]^2 cancel to a few 1e-6."""
    z, t = _gold(dtype)
    tag, loss, grads = _run(cls, opt, rays, t, 'oracle', dtype)
    loss.backward()
    ssim64 = dtype == torch.float64 and cls == 'RGBLossMS' and opt
    _close(loss, {k: v.grad for k, v in grads.items()}, z, tag, grad_rtol=1e-5 if ssim64 else 1e-6)


@pytest.mark.parametrize('cls,opt,rays', [c for c in _cases() if c[0] in ('RGBLossMS', 'EdgeLoss3DMS', 'SemLossMS', 'SemCELossMS')])
def test_torch_side_modules_match_reference_golden(cls, opt, rays):
    """The native RGB, semantic and edge terms (torch, batched over cameras) on the CPU, fp32 as the reference ran."""
    z, t = _gold(torch.float32)
    tag, loss, grads = _run(cls, opt, rays, t, 'native', torch.float32)
    loss.backward()
    _close(loss, {k: v.grad for k, v in grads.items()}, z, tag)


def test_golden_case_covers_the_edge_cases():
    z, t = _gold()
    eik = t('eik')
    assert (eik.norm(dim=-1) == 0).sum() >= 3
    assert (t('sg') == 0).any() and (t('dens') == 0).any()
    sem = t('sem')
    assert (sem < 0).any() and (sem > 1).any() and (sem == 0).any() and (sem == 1).any() and (sem == np.float32(1e-6)).any()
    r = t('rays_out')
    assert ((r[:, 0] < 0) | (r[:, 0] > IMG_SIZE[1]) | (r[:, 1] > IMG_SIZE[0])).sum() >= 8
    assert RAY_RESIZE[0] != RAY_RESIZE[1] and t('colors').shape[2] == 2
    # zeros vs border padding differ on the rays that leave the image
    assert float(z['RGBLossMS_ssim0_raysout_loss']) != float(z['RGBLossMS_ssim0_raysin_loss'])
    assert float(z['EdgeLoss3DMS_inf1_raysin_loss']) != float(z['EdgeLoss3DMS_inf0_raysin_loss'])


def _cfgs():
    return json.load(open(CFGS))


def test_every_shipped_loss_dict_builds():
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss as L
    cfgs = _cfgs()
    assert set(cfgs) == set(SHIPPED_TERMS)
    for name, c in cfgs.items():
        m = LOSSES.build(c)
        assert isinstance(m, L.MultiLoss) and m.num_losses == len(c['loss_cfgs'])
        assert [type(t).__name__ for t in m.losses] == SHIPPED_TERMS[name], name
        for term, tc in zip(m.losses, c['loss_cfgs']):
            assert term.weight == tc['weight']
            if 'input_dict' in tc:
                assert term.input_dict == tc['input_dict']


@pytest.mark.parametrize('name', sorted(SHIPPED_TERMS))
def test_multiloss_matches_reference_golden(name, monkeypatch):
    """MultiLoss over each shipped config's non-reprojection terms on the small golden case: the total and every
    loss_dict entry, as 0-d tensors.  The reprojection terms and the kernel behind the eikonal, second-grad and sparsity
    terms need the GPU: here the kernel is stood in for by the oracle (tests/test_gpu_losses.py runs the real one), so
    this checks the composition: building, input_dict routing, weights, keys and the total."""
    import sys
    import oracle.losses as O
    from selfocc_b200 import ops
    ref = {'eikonal': O.eikonal_ref, 'abs': O.second_grad_ref, 'neg_relu': O.soft_sparsity_ref}
    monkeypatch.setattr(ops.SampleMeanFunction, 'apply', lambda x, op: ref[op](x))
    sys.path.insert(0, os.path.join(HERE, 'golden'))
    from make_golden_losses import small_cfg, multi_inputs
    from selfocc_b200.loss import MultiLoss
    z, t = _gold()
    inp = {k: t(k) for k in ('eik', 'sg', 'dens', 'colors', 'gt', 'curr', 'depths', 'rays_in', 'sem', 'sem_lab')}
    terms = [small_cfg(c) for c in _cfgs()[name]['loss_cfgs'] if not c['type'].startswith('ReprojLoss')]
    ml = MultiLoss(terms)
    tot, d = ml(multi_inputs(inp))
    tag = 'multi_' + os.path.splitext(os.path.basename(name))[0]
    assert list(d) == list(z[tag + '_names'])
    for v, ref in zip(d.values(), z[tag + '_values']):
        assert isinstance(v, torch.Tensor) and v.dim() == 0 and not v.requires_grad
        assert abs(float(v) - ref) <= 1e-6 * abs(ref), (name, float(v), ref)
        assert f'{v:.5f}' == f'{float(v):.5f}'
    assert abs(float(tot) - float(z[tag + '_total'])) <= 1e-6 * float(z[tag + '_total'])
    assert ml.iter_counter == 1


def test_multiloss_writer_logs_every_tenth_call():
    from selfocc_b200.loss import MultiLoss

    class W:
        def __init__(self):
            self.log = []

        def add_scalar(self, tag, v, step):
            self.log.append((tag, step))
    ml = MultiLoss([dict(type='SecondGradLoss', weight=0.5), dict(type='SoftSparsityLoss', input_dict={'density': 'second_grad'})])
    ml.writer = W()
    ml.losses[0].loss_func = ml.losses[1].loss_func = lambda **kw: kw[next(iter(kw))].abs().mean()   # CPU stand-in
    for _ in range(12):
        ml({'second_grad': torch.ones(3)})
    assert ml.writer.log == [('loss/SecondGradLoss', 0), ('loss/SoftSparsityLoss', 0), ('loss/total', 0),
                             ('loss/SecondGradLoss', 10), ('loss/SoftSparsityLoss', 10), ('loss/total', 10)]


def test_terms_refuse_what_they_do_not_support():
    import selfocc_b200.loss as L
    rays = torch.zeros(30, 2)
    rgb = L.RGBLossMS(img_size=IMG_SIZE, no_ssim=False, ray_resize=RAY_RESIZE)
    with pytest.raises(NotImplementedError, match='list-valued'):
        rgb.loss_func([torch.zeros(1, 1, 60, 3)], [rays], torch.zeros(1, 1, 3, 8, 8))
    with pytest.raises(ValueError, match='ray_resize'):
        rgb.loss_func([torch.zeros(1, 1, 30, 3)], rays, torch.zeros(1, 1, 3, 8, 8))
    for cls in (L.SemLossMS, L.SemCELossMS):
        with pytest.raises(NotImplementedError, match='list-valued'):
            cls(img_size=IMG_SIZE).loss_func([torch.zeros(1, 1, 30, 5)], [{}], [rays])
    edge = L.EdgeLoss3DMS(img_size=IMG_SIZE, ray_resize=RAY_RESIZE)
    with pytest.raises(ValueError, match='ray_resize'):
        edge.loss_func(torch.zeros(1, 1, 3, 8, 8), [torch.ones(1, 1, 30)], rays)
    assert L.RGBLossMS(img_size=IMG_SIZE, no_ssim=False).no_ssim     # no ray grid: no SSIM, as the reference
    from selfocc_b200 import ops
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        L.EikonalLoss()({'eik_grad': torch.zeros(4, 3)})
    with pytest.raises(ValueError, match='op must be'):
        ops.SampleMeanFunction.apply(torch.zeros(4), 'cosh')


def test_sample_mean_entry_points_reject_bad_arguments_without_a_gpu():
    """Null pointers, non-positive sizes, a bad op, rows not of 3, mis-aligned pointers: SO_ERR_INVALID_ARG (-1) before
    any CUDA call."""
    import ctypes as C
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N, one, ws = None, C.c_void_p(16), C.c_void_p(64)
    fwd, bwd = lib.so_sample_mean_forward, lib.so_sample_mean_backward
    assert fwd(N, 12, 0, ws, one, N) == -1 and fwd(one, 12, 0, N, one, N) == -1 and fwd(one, 12, 0, ws, N, N) == -1
    assert bwd(N, 12, 0, one, one, N) == -1 and bwd(one, 12, 0, N, one, N) == -1 and bwd(one, 12, 0, one, N, N) == -1
    for n in (0, -3):
        assert fwd(one, n, 1, ws, one, N) == -1 and bwd(one, n, 1, one, one, N) == -1
    for op in (-1, 3, 7):
        assert fwd(one, 12, op, ws, one, N) == -1 and bwd(one, 12, op, one, one, N) == -1
    assert fwd(one, 10, 0, ws, one, N) == -1 and bwd(one, 10, 0, one, one, N) == -1     # eikonal: rows of 3
    assert fwd(C.c_void_p(18), 12, 1, ws, one, N) == -1                                   # x not 4-byte aligned
    assert fwd(one, 12, 1, C.c_void_p(20), one, N) == -1                                  # workspace not 8-byte aligned
    assert bwd(one, 12, 1, one, C.c_void_p(18), N) == -1
    assert lib.so_abi_version() == 9
