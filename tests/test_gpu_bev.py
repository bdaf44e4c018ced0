"""GPU: the BEV-only model (config/nuscenes/nuscenes_occ_bev.py) against the fp64 oracle (oracle/bev.py):

* the BEV decode (so_bev_decode) at the shipped volume and at geometries picked from its tile arithmetic, into NaN-filled
  buffers: every voxel, the sdf pads, the untouched feature pad channels;
* its backward (BEVDecodeFunction) against fp64 autograd, dense and sparse cotangents, at the bars of
  tests/test_gpu_decode_parity.py;
* the encoder at the shipped attention geometry (C = 96, 6 heads x 16; self-attention 1 level x 12 points; cross-attention
  4 levels x 8 points; 6 cameras; the 257 x 257 BEV plane), with and without focal ratios, both attention-kernel
  generations, through the shared layer routine;
* one layer's training routine against fp64 autograd, and a training step of a small nuscenes_occ_bev-shaped model
  through its whole objective;
* inference through the module API: prepare -> render against oracle/parity.render_parity, occupancy against forward_occ.
"""
import copy
import ctypes as C
import json
import os

import pytest
import torch

from selfocc_b200 import synth
from selfocc_b200.mapping import GridMeterMapping
from selfocc_b200.registry import build_head
import selfocc_b200.segmentor  # noqa: F401  registers the modules

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
CFG = json.load(open(os.path.join(HERE, 'golden', 'reference_model_cfgs_bev.json')))['nuscenes/nuscenes_occ_bev.py']
LAYER_BAR, ENCODER_BAR = 5e-5, 2e-4          # as tests/test_gpu_encoder_parity.py


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _margs(h, w, d, rng=(40.0, 40.0), z=(-1.0, 5.4)):
    return dict(nonlinear_mode='linear', h_size=[h, 0], h_range=[rng[0], 0], h_half=False, w_size=[w, 0], w_range=[rng[1], 0],
                w_half=False, d_size=[d, 0], d_range=[z[0], z[1], z[1]])


def _mlp(n_out, g, C_=96):
    return [t.cuda() for t in (torch.randn(C_, C_, generator=g) / C_ ** 0.5, 0.1 * torch.randn(C_, generator=g),
                               torch.randn(n_out, C_, generator=g) / C_ ** 0.5, 0.1 * torch.randn(n_out, generator=g))]


# --------------------------------------------------------------------------------------------- decode forward
# (h, w, d) half sizes -> H = 2h + 1, W = 2w + 1, Z = d + 1; n_feat.  The kernel works on 128-row tiles of BEV cells and
# 32-column n-tiles of the Z * Cf outputs.
DECODE_CASES = {
    'shipped 257x257, Z 25, Cf 25': ((128, 128, 24), 24),
    'one partial tile (5x7), Cf 1': ((2, 3, 24), 0),
    'ragged last tile (13x11), Z*Cf 12 < one n-tile, Cf 4': ((6, 5, 2), 3),
    'ragged tile and n-tile (21x9), Z*Cf 175': ((10, 4, 6), 24),
}


@pytest.mark.parametrize('case', list(DECODE_CASES))
def test_bev_decode_matches_fp64_oracle_into_nan_buffers(case):
    dev = _dev()
    from oracle.bev import bev_decode_ref
    from selfocc_b200 import _lib, ops
    (h, w, d), n_feat = DECODE_CASES[case]
    desc = GridMeterMapping(**_margs(h, w, d)).volume_desc(n_feat)
    H, W, Z, Cf = desc.H, desc.W, desc.Z, 1 + n_feat
    g = torch.Generator().manual_seed(H * 31 + Cf)
    bev = (0.7 * torch.randn(H * W, 96, generator=g)).to(dev)
    w1, b1, w2, b2 = _mlp(Z * Cf, g)
    vs = torch.full((H, W, desc.zpitch), float('nan'), device=dev)
    vf = torch.full((H, W, Z, desc.feat_pitch), float('nan'), device=dev) if n_feat else None
    p = lambda t: C.c_void_p(0 if t is None else t.data_ptr())
    lib = _lib.load()
    assert lib.so_bev_decode(p(bev), 96, p(w1), p(b1), p(w2), p(b2), C.byref(desc), p(vs), p(vf),
                             C.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    ref = bev_decode_ref(bev.double(), (H, W, Z), w1.double(), b1.double(), w2.double(), b2.double())
    smax = ref[0].abs().max().item()
    es = (vs[..., :Z].double() - ref[0]).abs().max().item()
    print('%s: sdf max abs err %.2e (|sdf| max %.2f)' % (case, es, smax))
    assert es <= 2e-5 * max(1.0, smax)
    assert torch.all(vs[..., Z:] == 0)                                     # sdf pads written as 0
    if n_feat:
        rf = ref[1:].permute(1, 2, 3, 0)
        ef = ((vf[..., :n_feat].double() - rf).abs() - 1e-5 * rf.abs()).max().item()
        print('%s: feature max (abs err - 1e-5 |ref|) %.2e' % (case, ef))
        assert ef <= 5e-5
        assert torch.isnan(vf[..., n_feat:]).all()                         # feature pad channels never written
    s2, f2 = ops.bev_decode(bev, w1, b1, w2, b2, desc)                     # the ops front end: same launch, same bits
    assert torch.equal(s2[..., :Z], vs[..., :Z]) and (f2 is None or torch.equal(f2[..., :n_feat], vf[..., :n_feat]))


# --------------------------------------------------------------------------------------------- decode backward
def _rel(got, ref):
    return (got.double() - ref).abs().max().item() / ref.abs().max().item()


@pytest.mark.parametrize('n_feat', [24, 3])
@pytest.mark.parametrize('kind', ['dense', 'sparse'])
def test_bev_decode_backward_matches_fp64_autograd(n_feat, kind, monkeypatch):
    dev = _dev()
    from oracle.bev import bev_decode_ref
    from selfocc_b200 import ops
    monkeypatch.setattr(ops.BEVDecodeFunction, 'SLAB_ROWS', 37)            # several slabs, a ragged last one
    desc = GridMeterMapping(**_margs(4, 5, 24)).volume_desc(n_feat)
    H, W, Z = desc.H, desc.W, desc.Z
    g = torch.Generator().manual_seed(5 + n_feat)
    bev = (0.7 * torch.randn(H * W, 96, generator=g)).to(dev).requires_grad_(True)
    ws = [t.requires_grad_(True) for t in _mlp(Z * (1 + n_feat), g)]
    g_vs = torch.randn(H, W, desc.zpitch, generator=g).to(dev)             # pads carry values: they must be ignored
    g_vf = torch.randn(H, W, Z, desc.feat_pitch, generator=g).to(dev)
    if kind == 'sparse':                                                    # a render's gradient: few voxels, spiky
        keep = torch.rand(H, W, Z, generator=g).to(dev) < 0.02
        g_vs[..., :Z] = g_vs[..., :Z] * keep * 30
        g_vf = g_vf * keep[..., None] * 30
    vs, vf = ops.BEVDecodeFunction.apply(bev, *ws, desc)
    torch.autograd.backward([vs, vf], [g_vs, g_vf])
    b64, w64 = bev.detach().double().requires_grad_(True), [t.detach().double().requires_grad_(True) for t in ws]
    vol = bev_decode_ref(b64, (H, W, Z), *w64)
    loss = (vol[0] * g_vs[..., :Z].double()).sum() + (vol[1:].permute(1, 2, 3, 0) * g_vf[..., :n_feat].double()).sum()
    loss.backward()
    for name, a, b in [('bev', bev, b64)] + [(n, x, y) for n, x, y in zip(('w1', 'b1', 'w2', 'b2'), ws, w64)]:
        e = _rel(a.grad, b.grad)
        print('%s %s n_feat=%d: grad %s %.2e of max-abs' % (kind, 'backward', n_feat, name, e))
        assert e < 1e-5, name
    for name, a, b, dim in (('bev channel', bev, b64, 0), ('w1 row', ws[0], w64[0], 1), ('w1 column', ws[0], w64[0], 0)):
        err = (a.grad.double() - b.grad).abs().amax(dim) / b.grad.abs().amax(dim).clamp_min(1e-30)
        print('%s: worst %s %.2e of its max-abs' % (kind, name, err.max().item()))
        assert err.max().item() < 2e-5, name


# --------------------------------------------------------------------------------------------- encoder at the shipped geometry
RIG = dict(f=126.6, cx=80., cy=45., height=1.0, radius=0.2)
IMG, FPN = (90, 160), [(12, 20), (6, 10), (3, 5), (2, 3)]
FOCAL = ([1.0, 0.9, 1.1, 0.95, 1.05, 0.8], [1.0, 0.85, 1.1, 1.0, 0.9, 1.2])


def _bev_model(cfg, seed=0):
    """Lifter + encoder of the config with every parameter away from its trivial value (as tests/test_gpu_encoder_parity)."""
    torch.manual_seed(seed)
    lifter, enc = build_head(cfg['lifter']), build_head(cfg['encoder'])
    enc.init_weights()
    g = torch.Generator().manual_seed(seed + 1)
    rn = lambda t: torch.randn(t.shape, generator=g)
    with torch.no_grad():
        for n, p in enc.named_parameters():
            if 'sampling_offsets.weight' in n or 'attention_weights.weight' in n:
                p.copy_(0.05 * rn(p))
            elif '.norms.' in n:
                p.copy_(1.0 + 0.3 * rn(p) if n.endswith('.weight') else 0.1 * rn(p))
            elif n.endswith('.bias'):
                p.add_(0.1 * rn(p))
        for p in lifter.parameters():
            p.mul_(0.5)
    return lifter, enc


def _ocfg(cfg):
    e = cfg['encoder']
    pe, layer = e['positional_encoding'], e['transformerlayers'][0]
    return dict(num_freqs=pe['num_freqs'], tot_range=pe['tot_range'], num_points_cross=e['num_points_cross'],
                num_points_self=e['num_points_self'], num_heads=layer['attn_cfgs'][0]['num_heads'], num_cams=e['num_cams'],
                num_layers=e['num_layers'])


def _frame(seed=0, focal=False, img=IMG, fpn=FPN, rig=RIG):
    g = torch.Generator().manual_seed(seed + 2)
    l2i, i2l = synth.camera_rig(synth.NUSC_YAWS, **rig)
    metas = [dict(lidar2img=list(l2i), img2lidar=list(i2l), temImg2lidar=list(i2l), img_shape=img)]
    if focal:
        metas[0].update(focal_ratios_x=FOCAL[0], focal_ratios_y=FOCAL[1])
    feats = [torch.randn(1, 6, 96, h, w, generator=g) for h, w in fpn]
    return metas, feats, torch.tensor(l2i, dtype=torch.float32), torch.tensor(i2l, dtype=torch.float32)


@pytest.mark.parametrize('focal', [False, True])
def test_bev_encoder_and_each_layer_match_oracle_at_shipped_geometry(focal, monkeypatch):
    dev = _dev()
    from oracle import bev as ob
    from oracle.mapping import GridMeterMappingRef
    from selfocc_b200 import _lib
    from selfocc_b200.encoder import TPVFormerLayer
    lifter, enc = _bev_model(CFG)
    ocfg = _ocfg(CFG)
    H, W = enc.bev_size
    assert (H, W) == (257, 257) and ocfg['num_heads'] == 6 and (ocfg['num_points_self'], ocfg['num_points_cross']) == (12, 8)
    metas, feats, l2i, _ = _frame(focal=focal)
    mref = GridMeterMappingRef(**CFG['encoder']['mapping_args'])
    p = {k: v.detach().cpu().double() for k, v in enc.state_dict().items()}
    torch.set_num_threads(max(torch.get_num_threads(), 8))
    feats64 = [f.double() for f in feats]
    fr = FOCAL if focal else None
    ref = ob.bev_encoder_ref(p, mref, lifter.bev.detach().double(), feats64, l2i[None], IMG, ocfg, focal_ratios=fr)
    # the per-layer oracle's operands, as bev_encoder_ref builds them
    pos = torch.nn.functional.linear(ob.bev_pos_features(mref, ocfg['num_freqs'], ocfg['tot_range']).double(),
                                     p['positional_encoding.position_layer.weight'], p['positional_encoding.position_layer.bias'])
    from oracle.lifting import flatten_img_feats, point_sampling_ref
    from oracle.focal import focal_scale_ref
    feat, shapes = flatten_img_feats(p, feats64)
    ref_3d, ref_2d = ob.bev_ref_tables(mref, ocfg['num_points_cross'])
    ref_cam, mask = point_sampling_ref(ref_3d[None], l2i[None], IMG)
    if focal:
        ref_cam = focal_scale_ref(ref_cam, *FOCAL)
    ref_2d = ref_2d.double().reshape(1, -1, 1, 2)
    lifter.to(dev)
    enc.to(dev).eval()
    rows = TPVFormerLayer.forward_rows
    calls = []
    monkeypatch.setattr(TPVFormerLayer, 'forward_rows', lambda self, *a: calls.append(a[4]) or rows(self, *a))
    for force_v1 in (0, 1):
        seen = []
        hooks = [l.register_forward_hook(lambda m, a, o: seen.append((a[0].detach().cpu(), o.detach().cpu()))) for l in enc.layers]
        _lib.load().so_attn_force_v1(force_v1)
        calls.clear()
        try:
            with torch.no_grad():
                fd = [f.to(dev) for f in feats]
                out = enc(representation=lifter(ms_img_feats=fd)['representation'], ms_img_feats=fd, metas=metas)['representation']
        finally:
            _lib.load().so_attn_force_v1(0)
            for hk in hooks:
                hk.remove()
        tag = '%s focal=%s' % ('v1' if force_v1 else 'v2', focal)
        assert calls == [[(0, H * W)]] * ocfg['num_layers']                # the shared routine, one plane, every layer
        for i, (inp, got) in enumerate(seen):
            lref = ob.bev_layer_ref(p, 'layers.%d.' % i, inp.double(), pos[None], feat, shapes, ref_2d, ref_cam.double(), mask,
                                    (H, W), ocfg)
            e = (got.double() - lref).abs().max().item()
            print('%s layer %d: max abs err %.2e (|x| max %.2f)' % (tag, i, e, lref.abs().max().item()))
            assert e < LAYER_BAR, (tag, i)
        e = (out.cpu().double() - ref).abs().max().item()
        print('%s encoder: max abs err %.2e' % (tag, e))
        assert e < ENCODER_BAR, tag


# --------------------------------------------------------------------------------------------- training
def _small_cfg(h=4, w=5, d=4, layers=1):
    cfg = copy.deepcopy(CFG)
    margs = _margs(h, w, d, rng=(8.0, 10.0), z=(-1.0, 3.0))
    cfg['lifter'].update(bev_h=2 * h + 1, bev_w=2 * w + 1)
    cfg['encoder'].update(mapping_args=margs, num_layers=layers, transformerlayers=cfg['encoder']['transformerlayers'][:layers])
    cfg['encoder']['positional_encoding']['tot_range'] = [-10.0, -8.0, -1.0, 10.0, 8.0, 3.0]
    cfg['head'].update(mapping_args=margs, roi_aabb=[-10.0, -8.0, -1.0, 10.0, 8.0, 3.0])
    return cfg


def test_bev_layer_training_matches_fp64_oracle():
    """One BEVFormerLayer in train() at dropout 0 through the training routine (forward_rows_train) against fp64 autograd of
    oracle.bev.bev_layer_ref: outputs, every parameter's gradient, the gradients of the query, positional embedding and
    image features, at the bars of tests/test_gpu_attn_train.py."""
    dev = _dev()
    from oracle import bev as ob
    from oracle.mapping import GridMeterMappingRef
    from test_gpu_attn_train import _assert_grads_match, _leaf64, _tol
    cfg = _small_cfg()
    lifter, enc = _bev_model(cfg, seed=3)
    enc.to(dev).train()
    for m in enc.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
    metas, feats, l2i, _ = _frame(seed=4)
    g = torch.Generator().manual_seed(5)
    H, W = enc.bev_size
    layer = enc.layers[0]
    feat, shapes, lsi = enc.flatten_features([f.to(dev) for f in feats])
    feat = feat.detach().requires_grad_(True)
    uvs, masks, vises = enc.project_tables((enc.ref_3d,), metas, dev)
    q = (0.5 * torch.randn(1, H * W, 96, generator=g)).to(dev).requires_grad_(True)
    pos = (0.5 * torch.randn(1, H * W, 96, generator=g)).to(dev).requires_grad_(True)
    ref_2d = enc.ref_2d.reshape(1, -1, 1, 2)
    out = layer(q, feat, feat, bev_pos=pos, ref_2d=ref_2d, spatial_shapes=shapes, level_start_index=lsi,
                reference_points_cams=uvs[0], bev_masks=masks[0], bev_size=(H, W), bev_vis=vises[0])
    go = torch.randn(out.shape, generator=g)
    (out * go.to(dev)).sum().backward()
    p64 = _leaf64(layer, 'l.')
    q64, pos64, f64 = (t.detach().cpu().double().requires_grad_(True) for t in (q, pos, feat))
    ocfg = _ocfg(cfg)
    ref = ob.bev_layer_ref(p64, 'l.', q64, pos64, f64, [tuple(s) for s in shapes.tolist()], ref_2d.cpu().double(),
                           uvs[0].cpu().double(), masks[0].cpu().bool(), (H, W), ocfg)
    e = (out.detach().cpu().double() - ref.detach()).abs().max().item()
    print('layer output max abs err %.2e' % e)
    assert e < 1e-4
    (ref * go.double()).sum().backward()
    _assert_grads_match(layer, p64, 'l.', _tol)
    for name, got, want, tol in (('query', q, q64, 1e-3), ('pos', pos, pos64, 1e-3), ('image features', feat, f64, 2e-4)):
        e = (got.grad.cpu().double() - want.grad).abs().max().item() / want.grad.abs().max().item()
        print('%s grad %.2e of max-abs' % (name, e))
        assert e < tol, name


def test_bev_model_training_step_through_the_whole_objective():
    """A small nuscenes_occ_bev-shaped model (head as the config sets it, second_grad opt-in) and the config's MultiLoss:
    loss finite, every parameter with a finite gradient."""
    dev = _dev()
    from selfocc_b200.registry import LOSSES
    import selfocc_b200.loss  # noqa: F401
    cfg = _small_cfg(8, 8, 8)
    cfg['head'].update(second_grad_assumption=True)
    torch.manual_seed(0)
    model = build_head(dict(type='TPVHotPath', **cfg)).to(dev).train()
    with torch.no_grad():
        model.head.model.field.deviation_network.variance.fill_(0.25)
    img_size = tuple(cfg['head']['ray_img_size'])
    metas, feats, _, _ = _frame(seed=6, img=img_size, fpn=synth.fpn_level_shapes(*img_size), rig={})
    prev, nxt = synth.temporal_rig()
    lab = torch.randint(0, 17, (6,) + img_size, generator=torch.Generator().manual_seed(2)).to(torch.uint8).numpy()
    metas[0].update(sem=lab, img2prevImg=torch.tensor(prev, dtype=torch.float32, device=dev),
                    img2nextImg=torch.tensor(nxt, dtype=torch.float32, device=dev))
    imgs = synth.textured_images(24, 192, 400, seed=3).reshape(4, 1, 6, 3, 192, 400).to(dev)
    out = model(ms_img_feats=[f.to(dev) for f in feats], metas=metas)
    cfgs = json.load(open(os.path.join(HERE, 'golden', 'reference_multiloss_cfgs.json')))
    loss = LOSSES.build(cfgs['nuscenes/nuscenes_occ_bev.py'])
    tot, parts = loss(dict(out, curr_imgs=imgs[0], prev_imgs=imgs[1], next_imgs=imgs[2], color_imgs=imgs[3], metas=metas))
    tot.backward()
    print('loss %.4f %r' % (tot.item(), {k: round(v.item(), 4) for k, v in parts.items()}))
    assert torch.isfinite(tot) and len(parts) == 6
    for k, p in model.named_parameters():
        if p.requires_grad:
            assert p.grad is not None and torch.isfinite(p.grad).all(), k


# --------------------------------------------------------------------------------------------- inference through the module API
def test_prepare_render_matches_oracle_and_occupancy_equals_forward_occ():
    dev = _dev()
    from oracle import rays as orays
    from oracle.bev import bev_decode_ref
    from oracle.mapping import GridMeterMappingRef
    from oracle.parity import render_parity
    from selfocc_b200 import ops
    cfg = _small_cfg(12, 12, 8)
    S = 64
    hcfg = dict(cfg['head'], color_dims=0, return_sem=False, return_uniform_sdf=False, return_second_grad=False,
                ray_sample_mode='fixed', ray_number=[12, 20], ray_img_size=[90, 160], num_samples=S, render_bkgd='white',
                trans_kw='img2lidar')
    torch.manual_seed(1)
    head = build_head(hcfg).to(dev).eval()
    f = head.model.field
    with torch.no_grad():
        f.density_net[3].bias.add_(torch.linspace(-1.5, 1.5, f.density_net[3].bias.numel(), device=dev))
        f.deviation_network.variance.fill_(0.3)
    H, W = f.mapping.size_h, f.mapping.size_w
    bev = (0.8 * torch.randn(1, H * W, 96)).to(dev)
    metas, _, _, i2l = _frame(seed=8)
    head.prepare(bev, metas)
    out = head.render(metas)
    l1, l2 = f.density_net[1], f.density_net[3]
    vol64 = bev_decode_ref(bev[0].double(), (H, W, f.mapping.size_d), l1.weight.double(), l1.bias.double(),
                           l2.weight.double(), l2.bias.double())
    pix = head.ray_sampler_eval.rays
    rays = ops.make_ray_desc(6, grid=head.ray_sampler_eval._grid)
    got = ops.render_infer(f.vol_sdf, None, f.desc, i2l.to(dev), rays, head._params(False), want=['depth', 'max_idx', 'acc'],
                           pack=f.render_pack(), probe_grid=True)
    assert torch.equal(got['depth'], out['ms_depths'][0].reshape(-1)) and torch.equal(got['acc'], out['ms_accs'][0].reshape(-1))
    origin, direction = orays.img2lidar_rays(i2l[None], pix.cpu())
    rep = render_parity(got, vol64, GridMeterMappingRef(**hcfg['mapping_args']), origin, direction, hcfg['roi_aabb'],
                        head._inv_s(), S, bkgd='white')
    print('render parity: %r' % {k: rep[k] for k in rep if k != 'independent'})
    assert rep['ok']
    # occupancy labels of a semantic BEV head equal forward_occ's composition
    head = build_head(dict(cfg['head'], return_second_grad=False)).to(dev).eval()
    aabb, res = hcfg['roi_aabb'], 0.4
    occ_out = head.forward_occ(bev, aabb=aabb, resolution=res)
    labels = head.occupancy(aabb, res, thresh=0.0)
    ref_occ = (occ_out['sdf'] <= 0).to(torch.uint8)
    band = occ_out['sdf'].abs() < 1e-6
    top2 = occ_out['logits'].topk(2, -1).values
    band_l = band | ((top2[..., 0] - top2[..., 1]) < 1e-6)
    assert torch.equal(labels['occ'][~band], ref_occ[~band])
    assert torch.equal(labels['sem'][~band_l], (ref_occ * occ_out['sem'])[~band_l].to(torch.uint8))
