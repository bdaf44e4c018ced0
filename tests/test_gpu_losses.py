"""GPU: the per-sample loss-term kernels (so_sample_mean_forward / _backward) against the fp64 oracle at nuScenes_occ
sizes, the native loss modules against the reference's golden vectors and against the fp32 reference composition at
shipped sizes, and nuscenes_occ's whole MultiLoss: no host sync, and finite gradients through a real NeuSHead."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from selfocc_b200 import synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
T, S = 6 * 48 * 100, 256                      # nuScenes_occ: 6 cameras x 48x100 rays x 256 samples


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _kernel_input(op, dev, shape=None, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    if op == 'eikonal':
        x = torch.randn(*(shape or (T, S, 3)), device=dev, generator=g) * 0.6
        x.view(-1, 3)[::97] = 0.                                   # zero-norm rows
    elif op == 'abs':
        x = torch.randn(*(shape or (T, S, 3)), device=dev, generator=g)
        x[x.abs() < 0.05] = 0.                                     # exact zeros
    else:
        x = torch.randn(*(shape or (200, 200, 16)), device=dev, generator=g)
        x[x.abs() < 0.05] = 0.
    return x


def _oracle(op, x):
    import oracle.losses as O
    f = {'eikonal': O.eikonal_ref, 'abs': O.second_grad_ref, 'neg_relu': O.soft_sparsity_ref}[op]
    xd = x.double().requires_grad_(True)
    loss = f(xd)
    g, = torch.autograd.grad(loss, xd)
    return loss.detach(), g


def _check_kernel(op, x, g_out=1.0):
    from selfocc_b200 import ops
    xl = x.detach().clone().requires_grad_(True)
    loss = ops.SampleMeanFunction.apply(xl, op)
    gx, = torch.autograd.grad(loss * g_out, xl)
    lo, go = _oracle(op, x)
    go = go * g_out
    assert loss.dtype == torch.float32 and loss.dim() == 0
    assert abs(loss.item() - lo.item()) <= 1e-6 * abs(lo.item()), (op, loss.item(), lo.item())
    assert (gx.double() - go).abs().max().item() <= 1e-6 * go.abs().max().item()
    assert (gx[go == 0] == 0).all()                                # exact zeros where torch's subgradient is zero
    if op != 'eikonal':                                            # (a row whose fp32 norm rounds to 1 has a 0 gradient)
        assert torch.equal(gx == 0, go == 0)
    return loss, gx


@pytest.mark.parametrize('op', ['eikonal', 'abs', 'neg_relu'])
def test_kernel_matches_fp64_oracle_at_shipped_sizes_and_repeats_bitwise(op):
    from selfocc_b200 import ops
    dev = _dev()
    x = _kernel_input(op, dev)
    l1, g1 = _check_kernel(op, x, g_out=0.1)
    l2, g2 = _check_kernel(op, x, g_out=0.1)
    assert torch.equal(l1, l2) and torch.equal(g1, g2)
    assert (g1 == 0).any()


@pytest.mark.parametrize('op', ['eikonal', 'abs', 'neg_relu'])
def test_kernel_handles_unaligned_heads_tails_and_non_contiguous_input(op):
    dev = _dev()
    base = _kernel_input(op, dev, shape=(1000, 7, 3) if op != 'neg_relu' else (21001 * 3,), seed=3).reshape(-1)
    for off in range(4):                                          # every offset inside a 16-byte word, and odd tails
        n = base.numel() - 3 * off - 3 * (off + 1) if op == 'eikonal' else base.numel() - off - 5 * off - 1
        x = base[3 * off:3 * off + n] if op == 'eikonal' else base[off:off + n]
        _check_kernel(op, x.reshape(-1, 3) if op == 'eikonal' else x)
    for n in (3, 6, 9) if op == 'eikonal' else (1, 2, 3, 5):     # smaller than one vector item
        _check_kernel(op, base[:n].reshape(-1, 3) if op == 'eikonal' else base[:n])
    nc = base[:3 * 4000].reshape(4000, 3).t().contiguous().t() if op == 'eikonal' else base[:8000].reshape(80, 100).t()
    assert not nc.is_contiguous()
    _check_kernel(op, nc)


def test_kernel_gradient_scale_stays_on_the_device():
    """The backward reads grad_out on the device: under sync debug 'error' the forward and backward run."""
    from selfocc_b200 import ops
    dev = _dev()
    x = _kernel_input('eikonal', dev, shape=(1000, 3)).requires_grad_(True)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss = ops.SampleMeanFunction.apply(x, 'eikonal') * 0.1 + ops.SampleMeanFunction.apply(x, 'abs')
        g, = torch.autograd.grad(loss, x)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(g).all()


def test_native_modules_match_reference_golden_on_the_device():
    """Every native term on the golden inputs, moved to the GPU: losses within the CPU tests' 1e-6, the kernel terms'
    gradients within 1e-6 of their max-abs.  The torch-side terms' reductions sum in another order on the device than in
    the CPU run that made the golden vectors, so their gradients carry one more fp32 rounding: 2e-6 (the edge term's mean
    normalisation misses 1e-6 by 4 %), and as for the fp64 oracle, 1e-5 for the SSIM gradient, where the reference's fp32
    variances E[x^2] - E[x]^2 cancel to a few 1e-6."""
    sys.path.insert(0, HERE)
    import test_losses_cpu as C
    z = np.load(C.GOLD)
    dev = _dev()
    t = lambda k: torch.from_numpy(z[k]).to(dev).float() if z[k].dtype.kind == 'f' else torch.from_numpy(z[k])
    import selfocc_b200.loss as L
    for cls, key, name in (('EikonalLoss', 'eik_grad', 'eik'), ('SecondGradLoss', 'second_grad', 'sg'),
                           ('SoftSparsityLoss', 'density', 'dens')):
        x = t(name).requires_grad_(True)
        loss = getattr(L, cls)()({key: x})
        loss.backward()
        C._close(loss.cpu(), {name: x.grad.cpu()}, z, cls)
    for cls, opt, rays in C._cases():
        if cls in ('EikonalLoss', 'SecondGradLoss', 'SoftSparsityLoss'):
            continue
        tdev = lambda k: t(k) if k != 'sem_lab' else torch.from_numpy(z[k])        # labels stay numpy-backed
        tag, loss, grads = C._run(cls, opt, rays, tdev, 'native', torch.float32)
        loss.backward()
        assert loss.device.type == 'cuda'
        C._close(loss.cpu(), {k: v.grad.cpu() for k, v in grads.items()}, z, tag,
                 grad_rtol=1e-5 if cls == 'RGBLossMS' and opt else 2e-6)


def _shipped_case(dev, seed=0):
    """nuScenes_occ-sized per-ray head outputs: 6 cams x 48x100 rays of a 768x1600 image, 17 semantic classes."""
    g = torch.Generator().manual_seed(seed)
    R, n, C = 4800, 6, 17
    ys, xs = torch.meshgrid(torch.arange(48), torch.arange(100), indexing='ij')
    rays = torch.stack([(xs.flatten() + torch.rand(R, generator=g)) * 16, (ys.flatten() + torch.rand(R, generator=g)) * 16], -1)
    imgs = synth.textured_images(12, 192, 400, seed=seed + 1).reshape(2, 1, n, 3, 192, 400)
    lab = torch.randint(0, C, (1, n, 768, 1600), generator=g).to(torch.uint8)
    sem = torch.softmax(3 * torch.randn(1, n, R, C, generator=g), -1)
    return dict(rays=rays.to(dev), gt=imgs[0].to(dev), curr=imgs[1].to(dev), colors=torch.rand(1, n, R, 3, generator=g).to(dev),
                depths=(1 + 40 * torch.rand(1, n, R, generator=g)).to(dev), accs=torch.rand(1, n, R, generator=g).to(dev),
                maxd=(40 + 10 * torch.rand(1, n, R, generator=g)).to(dev), sem=sem.to(dev), sem_lab=lab.numpy())


def test_native_modules_match_the_reference_composition_at_shipped_sizes():
    """RGB (SSIM), both semantic terms and the edge term (inf mask) at nuScenes_occ sizes against the oracle run in fp32 on
    the device, as the reference would: loss within 1e-5 relative, gradients within 1e-5 of their max-abs."""
    import oracle.losses as O
    import selfocc_b200.loss as L
    dev = _dev()
    c = _shipped_case(dev)
    img, rr = [768, 1600], [48, 100]
    lab_dev = torch.from_numpy(c['sem_lab']).to(dev)

    def both(native, oracle, names):
        out = []
        for f in (native, oracle):
            leaves = {k: c[k].clone().requires_grad_(True) for k in names}
            loss = f(leaves)
            out.append((loss.detach(), torch.autograd.grad(loss, [leaves[k] for k in names])))
        (ln, gn), (lo, go) = out
        assert abs(ln.item() - lo.item()) <= 1e-5 * abs(lo.item()), (ln.item(), lo.item())
        for a, b in zip(gn, go):
            assert (a - b).abs().max().item() <= 1e-5 * b.abs().max().item()

    both(lambda v: L.RGBLossMS(img_size=img, no_ssim=False, ray_resize=rr)(dict(ms_colors=[v['colors']], ms_rays=c['rays'], gt_imgs=c['gt'])),
         lambda v: O.rgb_ref([v['colors']], c['rays'], c['gt'], img, rr, no_ssim=False), ['colors'])
    for cls, ref in (('SemLossMS', O.sem_bce_ref), ('SemCELossMS', O.sem_ce_ref)):
        both(lambda v: getattr(L, cls)(img_size=img)(dict(sem=[v['sem']], metas=[dict(sem=c['sem_lab'][0])], ms_rays=c['rays'])),
             lambda v: ref([v['sem']], lab_dev, c['rays']), ['sem'])
    keys = dict(curr_imgs='curr_imgs', ms_depths='ms_depths', ms_rays='ms_rays', ms_accs='ms_accs', max_depths='max_depths')
    both(lambda v: L.EdgeLoss3DMS(img_size=img, ray_resize=rr, use_inf_mask=True, input_dict=keys)(
            dict(curr_imgs=c['curr'], ms_depths=[v['depths']], ms_rays=c['rays'], ms_accs=[v['accs']], max_depths=[v['maxd']])),
         lambda v: O.edge_ref(c['curr'], [v['depths']], c['rays'], img, rr, [v['accs']], [v['maxd']]), ['depths', 'accs', 'maxd'])


def _nusc_occ_loss():
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss  # noqa: F401
    cfgs = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))
    return LOSSES.build(cfgs['nuscenes/nuscenes_occ.py'])


def objective_inputs(dev, S=64, seed=0):
    """nuscenes_occ's objective inputs as NeuSHead.forward and the dataset hand them over (seeded, synthetic)."""
    g = torch.Generator().manual_seed(seed)
    c = _shipped_case(dev, seed)
    R, n = 4800, 6
    prev, nxt = synth.temporal_rig()
    imgs = synth.textured_images(3 * n, 192, 400, seed=seed + 5).reshape(3, 1, n, 3, 192, 400).to(dev)
    w = torch.rand(n, R * S, generator=g).to(dev) / S
    ts = (0.5 + 40 * torch.rand(n, R * S, generator=g)).sort(-1).values.to(dev)
    ridx = [torch.arange(R, device=dev).repeat_interleave(S)] * n
    metas = [dict(img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                  img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev), sem=c['sem_lab'][0])]
    leaves = dict(weights=w, ms_colors=c['colors'], sem=c['sem'], eik_grad=_kernel_input('eikonal', dev, (n * R, S, 3)),
                  second_grad=_kernel_input('abs', dev, (n * R, S, 3)))
    leaves = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
    inputs = dict(curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=c['gt'], ray_indices=ridx,
                  weights=list(leaves['weights'].unbind(0)), ts=list(ts.unbind(0)), metas=metas, ms_rays=c['rays'],
                  ms_colors=[leaves['ms_colors']], sem=[leaves['sem']], eik_grad=leaves['eik_grad'],
                  second_grad=leaves['second_grad'])
    return inputs, leaves


def test_nuscenes_occ_multiloss_never_syncs_with_the_host():
    dev = _dev()
    ml = _nusc_occ_loss()
    inputs, leaves = objective_inputs(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        tot, d = ml(inputs)
        grads = torch.autograd.grad(tot, list(leaves.values()))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert list(d) == ['ReprojLossMonoMultiNewCombine', 'RGBLossMS', 'EikonalLoss', 'SecondGradLoss', 'SemCELossMS']
    assert all(v.is_cuda and v.dim() == 0 for v in d.values())
    assert abs(tot.item() - sum(v.item() for v in d.values())) <= 1e-6 * tot.item()
    assert all(torch.isfinite(g).all() and g.abs().sum() > 0 for g in grads)


def test_head_forward_then_nuscenes_occ_objective_gives_finite_gradients():
    """A real NeuSHead.forward (small TPV, color_dims = 24 with semantics, the second-grad opt-in) feeds nuscenes_occ's
    whole MultiLoss; backward() reaches every head parameter with finite values."""
    dev = _dev()
    from selfocc_b200 import configs
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    torch.manual_seed(0)
    img_size, ray_resize, S = (768, 1600), [48, 100], 32
    margs, rng = synth.small_mapping(16, 8, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=S, ray_number=tuple(ray_resize), ray_img_size=img_size,
                                  color_dims=24, return_sem=True)
    cfg['head'].update(return_second_grad=True, second_grad_assumption=True)
    head = build_head(cfg['head']).to(dev).train()
    with torch.no_grad():
        head.model.field.deviation_network.variance.fill_(0.25)
    l2i, i2l = synth.camera_rig()
    prev, nxt = synth.temporal_rig()
    lab = torch.randint(0, 17, (6, 768, 1600), generator=torch.Generator().manual_seed(2)).to(torch.uint8).numpy()
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), img_shape=img_size, sem=lab,
                  img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                  img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))]
    planes = [(0.5 * torch.randn(1, n, 96, device=dev)).requires_grad_(True) for n in (33 * 33, 9 * 33, 33 * 9)]
    imgs = synth.textured_images(24, 192, 400, seed=3).reshape(4, 1, 6, 3, 192, 400).to(dev)
    out = head(representation=planes, metas=metas)
    assert out['sem'][0].shape[-1] == 21 and 'second_grad' in out
    tot, d = _nusc_occ_loss()(dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas))
    tot.backward()
    assert torch.isfinite(tot) and len(d) == 5
    named = [(k, p) for k, p in head.named_parameters() if p.requires_grad]
    for k, p in named + [('plane%d' % i, p) for i, p in enumerate(planes)]:
        assert p.grad is not None and torch.isfinite(p.grad).all(), k
