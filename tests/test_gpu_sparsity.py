"""GPU: the sparsity terms (so_sparsity_*, so_hard_sparsity_*, so_adaptive_sparsity_*) against the fp64 oracle at the
nuscenes_occ lattice and ray sizes and on their edge cases, the reference's golden vectors, bitwise reruns, no host sync in a
MultiLoss step, emulated ray-sharded steps against the unsharded one, and a nuscenes_occ-shaped head step with the configs'
commented terms switched on against the reference's torch terms."""
import os
import sys

import numpy as np
import pytest
import torch

from selfocc_b200 import synth

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
LATTICE = (200, 200, 16)                       # nuscenes_occ's uniform_sdf: 80 x 80 x 6.4 m at 0.4 m
N_CAM, R, S = 6, 48 * 100, 256                 # nuScenes_occ rays: 6 cameras x 48x100 rays x 256 samples
HARD = {'nocrop': (1.0, 0.2, [[0, 0], [0, 0], [0, 0]]), 'crop': (1.0, 0.2, [[5, 7], [3, 0], [2, 1]]),
        'allcrop': (0.02, 0.1, [[0, 0], [100, 100], [0, 0]]), 'inactive': (1.0, 0.99, [[1, 1], [0, 0], [0, 0]]),
        'slope': (0.05, 0.3, [[0, 2], [0, 0], [3, 0]])}


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _lattice(dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(*LATTICE, device=dev, generator=g) * 0.5
    x[x.abs() < 0.01] = 0.
    x.view(-1)[::1013] = 50.                     # |x| / (2 * 0.1) = 250: past fp32 cosh's range
    x.view(-1)[7::1013] = -1e4
    return x


def _rays(dev, seed=0, far=False):
    g = torch.Generator(device=dev).manual_seed(seed)
    ts = (0.5 + 45 * torch.rand(N_CAM, R, S, device=dev, generator=g)).sort(-1).values
    depth = (1 + 40 * torch.rand(1, N_CAM, R, device=dev, generator=g)) if not far else torch.full((1, N_CAM, R), 100., device=dev)
    sdf = torch.randn(N_CAM, R, S, device=dev, generator=g)
    sdf[sdf.abs() < 0.01] = 0.
    return sdf.reshape(N_CAM, R * S), ts.reshape(N_CAM, R * S), depth


def _grad(f, x):
    xl = x.detach().clone().requires_grad_(True)
    loss = f(xl)
    g, = torch.autograd.grad(loss, xl)
    return loss.detach(), g


def _native(kind, cfg=None):
    import selfocc_b200.loss as L
    if kind == 'sparsity':
        return lambda x: L.SparsityLoss(scale=cfg)({'density': x})
    if kind == 'hard':
        s, t, c = cfg
        return lambda x: L.HardSparsityLoss(scale=s, thresh=t, crop=c)({'density': x})
    ts, depth = cfg
    return lambda x: L.AdaptiveSparsityLoss(input_dict=dict(sdfs='sample_sdf', ts='ts', ms_depths='ms_depths'))(
        dict(sample_sdf=list(x.unbind(0)), ts=list(ts.unbind(0)), ms_depths=[depth]))


def _oracle(kind, cfg=None):
    import oracle.sparsity as O
    if kind == 'sparsity':
        return lambda x: O.sparsity_ref(x, cfg)
    if kind == 'hard':
        return lambda x: O.hard_sparsity_ref(x, *cfg)
    ts, depth = cfg
    # the mask stays in fp32, as the reference's (and the kernel's) depth + slack rounds
    return lambda x: O.adaptive_sparsity_ref(list(x.unbind(0)), list(ts.unbind(0)), depth)


def _against_oracle(kind, x, cfg):
    ln, gn = _grad(_native(kind, cfg), x)
    lo, go = _grad(_oracle(kind, cfg), x.double())
    assert ln.dtype == torch.float32 and ln.dim() == 0
    if torch.isnan(lo):
        assert torch.isnan(ln)
    else:
        assert abs(ln.item() - lo.item()) <= 1e-6 * abs(lo.item()), (kind, ln.item(), lo.item())
    assert torch.isfinite(gn).all()
    assert (gn.double() - go).abs().max().item() <= 1e-6 * go.abs().max().item(), kind
    assert (gn[go == 0] == 0).all()                              # exact zeros: crops, inactive relu, unmasked samples
    return ln, gn, go


def test_sparsity_matches_fp64_oracle_at_the_lattice_and_past_the_cosh_range():
    dev = _dev()
    x = _lattice(dev)
    for scale in (0.1, 1.0):
        ln, gn, go = _against_oracle('sparsity', x, scale)
        far = x.abs() / (2 * scale) > 89.
        assert far.sum() > 100 and (gn[far] == 0).all()
    big = torch.tensor([1e3, -3e38, 17.9, -18.0], device=dev)    # cosh overflows in fp32 from |x| / 0.2 > 89.4
    loss, g = _grad(_native('sparsity', 0.1), big)
    assert loss.item() == 0 and torch.equal(g, torch.zeros_like(g))


@pytest.mark.parametrize('case', sorted(HARD))
def test_hard_sparsity_matches_fp64_oracle_and_leaves_the_input(case):
    dev = _dev()
    x = _lattice(dev, seed=1)
    before = x.clone()
    ln, gn, go = _against_oracle('hard', x, HARD[case])
    assert torch.equal(x, before)
    if case == 'inactive':
        assert ln.item() == 0 and torch.equal(gn, torch.zeros_like(gn))
    elif case == 'allcrop':
        assert ln.item() > 0 and torch.equal(gn, torch.zeros_like(gn))
    else:
        assert ln.item() > 0 and (gn != 0).any()
    if case == 'crop':
        assert not gn[:5].any() and not gn[-7:].any() and not gn[:, :3].any() and not gn[..., :2].any() and not gn[..., -1].any()
    # the module leaves its input to the next term: SoftSparsityLoss after it sees the uncropped lattice
    from selfocc_b200.loss import MultiLoss
    from selfocc_b200 import ops
    s, t, c = HARD[case]
    _, d = MultiLoss([dict(type='HardSparsityLoss', scale=s, thresh=t, crop=c, input_dict={'density': 'uniform_sdf'}),
                      dict(type='SoftSparsityLoss', input_dict={'density': 'uniform_sdf'})])({'uniform_sdf': x})
    assert torch.equal(x, before) and torch.equal(d['SoftSparsityLoss'], ops.SampleMeanFunction.apply(before, 'neg_relu'))


@pytest.mark.parametrize('far', [False, True])
def test_adaptive_sparsity_matches_fp64_oracle_at_shipped_rays(far):
    dev = _dev()
    sdf, ts, depth = _rays(dev, far=far)
    ln, gn, go = _against_oracle('adaptive', sdf, (ts, depth))
    if far:                                                      # empty mask: NaN, as torch's mean of nothing; no gradient
        assert torch.isnan(ln) and torch.equal(gn, torch.zeros_like(gn))
    else:
        assert (gn != 0).any() and (gn == 0).any()


def test_native_terms_match_reference_golden_on_the_device():
    sys.path.insert(0, HERE)
    import test_sparsity_cpu as C
    z = np.load(C.GOLD)
    dev = _dev()
    t = lambda k: torch.from_numpy(z[k]).to(dev).float()
    for tag, scale in (('s01', 0.1), ('s1', 1.0)):
        loss, g = _grad(_native('sparsity', scale), t('dens'))
        fin = C._check(loss.cpu(), g.cpu(), z, 'SparsityLoss_' + tag, 'dens')
        assert (g.cpu().numpy()[~fin] == 0).all()                # 0 where the reference's gradient is 0 * inf
    for tag in ('nocrop', 'crop', 'allcrop', 'inactive', 'slope'):
        loss, g = _grad(_native('hard', C._hard_cfg(z, tag)), t('dens'))
        C._check(loss.cpu(), g.cpu(), z, 'HardSparsityLoss_' + tag, 'dens')
    for tag, dk in (('masked', 'depths'), ('empty', 'depths_far')):
        loss, g = _grad(_native('adaptive', (t('ts'), t(dk))), t('sdfs'))
        C._check(loss.cpu(), g.cpu(), z, 'AdaptiveSparsityLoss_' + tag, 'sdfs')


def test_reruns_are_bit_identical():
    dev = _dev()
    x = _lattice(dev, seed=2)
    sdf, ts, depth = _rays(dev, seed=2)
    for kind, inp, cfg in (('sparsity', x, 0.1), ('hard', x, HARD['crop']), ('adaptive', sdf, (ts, depth))):
        a, b = _grad(_native(kind, cfg), inp), _grad(_native(kind, cfg), inp)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]), kind


CFG_TERMS = [dict(type='SparsityLoss', weight=0.001, scale=0.1, input_dict={'density': 'uniform_sdf'}),
             dict(type='HardSparsityLoss', weight=0.01, crop=[[5, 7], [3, 0], [2, 1]], input_dict={'density': 'uniform_sdf'}),
             dict(type='AdaptiveSparsityLoss', weight=0.001, slack=4.0,
                  input_dict={'sdfs': 'sample_sdf', 'ts': 'ts', 'ms_depths': 'ms_depths'})]


def _multi_inputs(x, sdf, ts, depth):
    return dict(uniform_sdf=x, sample_sdf=list(sdf.unbind(0)), ts=list(ts.unbind(0)), ms_depths=[depth])


@pytest.mark.parametrize('term', [c['type'] for c in CFG_TERMS])
def test_multiloss_step_with_each_term_never_syncs_with_the_host(term):
    from selfocc_b200.loss import MultiLoss
    dev = _dev()
    x = _lattice(dev, seed=3).requires_grad_(True)
    sdf, ts, depth = _rays(dev, seed=3)
    sdf.requires_grad_(True)
    ml = MultiLoss([c for c in CFG_TERMS if c['type'] == term])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        tot, d = ml(_multi_inputs(x, sdf, ts, depth))
        g = torch.autograd.grad(tot, [x if term != 'AdaptiveSparsityLoss' else sdf])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert list(d) == [term] and torch.isfinite(tot) and g[0].abs().sum() > 0


@pytest.mark.parametrize('world', [2, 3])
def test_emulated_ray_sharded_steps_equal_the_unsharded_step(world):
    """Each rank holds its slice of every camera's rays (sample_sdf, ts, depths) and the replicated lattice; the adaptive
    term's per-ray pairs gathered from the ranks reduce to the unsharded value bit for bit, and the ranks' own-slice
    gradients / world are the unsharded ones."""
    sys.path.insert(0, HERE)
    from test_ray_shard_cpu import emulated_ranks
    from selfocc_b200.dist import ray_slice
    from selfocc_b200.loss import MultiLoss
    dev = _dev()
    x = _lattice(dev, seed=4)
    sdf, ts, depth = _rays(dev, seed=4)
    sdf3, ts3 = sdf.reshape(N_CAM, R, S), ts.reshape(N_CAM, R, S)
    ml = MultiLoss(CFG_TERMS)
    full = sdf.clone().requires_grad_(True)
    tot, ref = ml(_multi_inputs(x, full, ts, depth))
    g_ref, = torch.autograd.grad(tot, full)
    ranks = []
    for r in range(world):
        b, c = ray_slice(R, world, r)
        own = sdf3[:, b:b + c].reshape(N_CAM, -1).clone().requires_grad_(True)
        inp = dict(_multi_inputs(x, own, ts3[:, b:b + c].reshape(N_CAM, -1), depth[:, :, b:b + c]), ray_shard=(r, world, R))
        ranks.append((own, inp, b, c))
    res = emulated_ranks(ml, [inp for _, inp, _, _ in ranks], world)
    g_ref3 = g_ref.reshape(N_CAM, R, S)
    for (tot_r, d), (own, _, b, c) in zip(res, ranks):
        assert list(d) == list(ref)
        for k in ref:
            assert torch.equal(d[k], ref[k]), (k, d[k].item(), ref[k].item())
        g, = torch.autograd.grad(tot_r, own)
        want = g_ref3[:, b:b + c].reshape(N_CAM, -1)
        assert (g / world - want).abs().max().item() <= 1e-7 * g_ref.abs().max().item()


def test_nuscenes_occ_shaped_step_with_the_commented_terms_matches_the_reference_terms():
    """A NeuSHead training step (small TPV, nuScenes_occ's 6 x 48x100 rays, return_uniform_sdf and return_sample_sdf) under
    nuscenes_occ's MultiLoss plus its commented AdaptiveSparsityLoss and SparsityLoss blocks; the same step with those two
    terms computed by the reference's torch expressions on the same outputs gives the same head gradients."""
    import json
    dev = _dev()
    from selfocc_b200 import configs
    from selfocc_b200.registry import LOSSES, build_head
    import selfocc_b200.segmentor  # noqa: F401
    torch.manual_seed(0)
    img_size, ray_resize, Sh = (768, 1600), [48, 100], 32
    margs, rng = synth.small_mapping(16, 8, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=Sh, ray_number=tuple(ray_resize), ray_img_size=img_size,
                                  color_dims=24, return_sem=True)
    cfg['head'].update(return_second_grad=True, second_grad_assumption=True, return_uniform_sdf=True, return_sample_sdf=True)
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
    inputs = dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas)
    assert out['uniform_sdf'].dim() == 3 and len(out['sample_sdf']) == 6
    base = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))['nuscenes/nuscenes_occ.py']
    extra = [CFG_TERMS[2], CFG_TERMS[0]]
    ml = LOSSES.build(dict(base, loss_cfgs=base['loss_cfgs'] + extra))
    params = [p for p in head.parameters() if p.requires_grad] + planes

    def step():
        tot, d = ml(inputs)
        return d, torch.autograd.grad(tot, params, retain_graph=True, allow_unused=True)
    d_nat, g_nat = step()
    _, g_nat2 = step()                                           # the render backward's atomics: the step's own spread
    # the reference's torch terms (loss/sparsity_loss.py) on the same outputs, in fp32
    sp, ad = ml.losses[-1], ml.losses[-2]
    sp.loss_func = lambda density: torch.pow(1.0 / torch.cosh(density / (2.0 * 0.1)), 2).mean()

    def adaptive_ref(sdfs, ts, ms_depths):
        depths = ms_depths[0]
        bs, nc, nr = depths.shape
        t = torch.stack(ts, dim=0).reshape(bs, nc, nr, -1)
        s = torch.stack(sdfs, dim=0).reshape(bs, nc, nr, -1)
        return torch.relu(-1 * s[t > (depths + 4.0).unsqueeze(-1)]).mean()
    ad.loss_func = adaptive_ref
    d_ref, g_ref = step()
    for k in ('SparsityLoss', 'AdaptiveSparsityLoss'):
        assert abs(d_nat[k].item() - d_ref[k].item()) <= 1e-5 * abs(d_ref[k].item()), (k, d_nat[k].item(), d_ref[k].item())
    assert d_nat['SparsityLoss'].item() > 0 and torch.isfinite(d_nat['AdaptiveSparsityLoss'])
    n = 0
    for a, a2, b in zip(g_nat, g_nat2, g_ref):
        if b is None:
            continue
        assert torch.isfinite(a).all()
        spread = (a - a2).abs().max().item()
        assert (a - b).abs().max().item() <= max(1e-5 * b.abs().max().item(), 4 * spread)
        n += 1
    assert n >= len(planes) + 4
