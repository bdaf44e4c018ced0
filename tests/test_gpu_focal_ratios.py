"""GPU: frames with the focal-ratio rescale of point_sampling (bevformer/utils.py:198-204), the metas['focal_ratios_x' / '_y']
RandomScaleImageMultiViewImage writes for every nuScenes config and for kitti_raw_depth / kitti_novel_depth, through each
lifting path: the kernel (so_point_sampling_scaled), encoder inference, the unsharded and the query-sharded training step,
ShardedLifter and GraphedFrame, and a whole kitti_raw_depth model fed a frame shaped like the reference loader's.

The geometry, models and bars are those of tests/test_gpu_encoder_parity.py (NUSC: 6 cameras, KITTI: 1 camera with a half
h axis; whole encoder 2e-4, one layer 5e-5 against the fp64 oracle), tests/test_gpu_attn_train.py (training gradients) and
tests/test_gpu_encoder_shard.py / tests/test_gpu_dist.py (sharded paths, bit for bit).  The ratio sets:

  nuscenes          scale_rate 0.5, pad rate 0.5: 1.0 on each of 6 cameras (exactly: the rescale is the identity)
  kitti_raw_depth   scale_rate 0.84, pad_scale_rate [0.8649, 0.8421]: x 0.99750626, y 0.97121054 (1 camera)
  kitti_novel_depth pad_scale_rate [1.038, 1.0]: x 1.0, y 0.96339114 (1 camera)
  above_one         x 1.08, y 1.05 on the KITTI camera: visible samples land outside [0, 1]
  straddle          six per-camera ratios between 0.91 and 1.08 (the random_scale option), visible samples outside [0, 1]
  broadcast         one ratio pair for the six cameras (a length-1 list, as view(-1, 1, 1, 1, 1) broadcasts it)
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import focal as of
import test_gpu_encoder_parity as ep
from test_gpu_encoder_parity import NUSC, KITTI, ENCODER_BAR, _dev

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))

STRADDLE = ([0.91, 1.08, 0.97, 1.05, 1.0, 0.94], [1.06, 0.92, 1.08, 0.99, 1.03, 0.95])
RATIOS = {
    'nuscenes': (NUSC, [0.5 / 0.5] * 6, [0.5 / 0.5] * 6),
    'kitti_raw_depth': (KITTI, [0.84 / 0.8421], [0.84 / 0.8649]),
    'kitti_novel_depth': (KITTI, [1.0 / 1.0], [1.0 / 1.038]),
    'above_one': (KITTI, [1.08], [1.05]),
    'straddle': (NUSC, STRADDLE[0], STRADDLE[1]),
    'broadcast': (NUSC, [1.07], [0.96]),
}


def _with_ratios(metas, rx, ry, **extra):
    return [dict(metas[0], focal_ratios_x=list(rx), focal_ratios_y=list(ry), **extra)]


def _outside_visible(uv, mask):
    """number of in-frustum samples whose rescaled uv lies outside [0, 1]"""
    return int(((uv < 0) | (uv > 1)).any(-1)[mask.bool()].sum())


# --------------------------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize('name', sorted(RATIOS))
def test_point_sampling_with_ratios_is_bit_exact(name):
    """project_reference_points on metas shaped like the wrapper's (ratios as lists) against point_sampling_ref +
    focal_scale_ref: uv, mask, vis and the visible-index lists, bit for bit, on all three planes."""
    dev = _dev()
    from oracle import lifting as ol
    from selfocc_b200 import ops
    case, rx, ry = RATIOS[name]
    _, enc, _ = ep._model(case, num_layers=1)
    enc.to(dev)
    metas, _, l2i = ep._frame(case)
    metas = _with_ratios(metas, rx, ry, scale_rate=0.5, flip=False)
    uvs, masks, vises = enc.project_reference_points(metas, dev)
    outside = 0
    for i, r3 in enumerate((enc.ref_3d_hw, enc.ref_3d_zh, enc.ref_3d_wz)):
        uv0, m_ref = ol.point_sampling_ref(r3.cpu()[None], l2i[None], case['img'])
        uv_ref = of.focal_scale_ref(uv0, rx, ry)
        assert torch.equal(uvs[i].cpu(), uv_ref) and torch.equal(masks[i].cpu().bool(), m_ref), i
        assert torch.equal(vises[i].cpu().bool(), m_ref[:, 0].any(-1)), i
        lists, lens = ops.visible_index_lists(masks[i][:, 0].contiguous())
        for c, idx in enumerate(ol.visible_index_lists(m_ref)):
            assert torch.equal(lists[c, :int(lens[c])].cpu(), idx), (i, c)
        outside += _outside_visible(uv_ref, m_ref)
        if name == 'nuscenes':
            assert torch.equal(uv_ref, uv0)
    print('%s: %d visible samples outside [0, 1]' % (name, outside))
    if name in ('above_one', 'straddle'):
        assert outside > 0


def test_no_ratios_and_unit_ratios_equal_the_plain_entry_point():
    dev = _dev()
    from oracle import lifting as ol
    from oracle.mapping import GridMeterMappingRef
    from selfocc_b200 import ops, _lib
    lib = _lib.load()
    l2i = ep._frame(NUSC)[2].to(dev)
    for r3 in ol.ref_3d_tables(GridMeterMappingRef(**NUSC['margs']), [48, 48, 8]):
        r3 = r3.contiguous().to(dev)
        D, Q, _ = r3.shape
        uv = torch.empty(6, Q, D, 2, device=dev)
        mask = torch.empty(6, Q, D, device=dev, dtype=torch.uint8)
        vis = torch.empty(6, Q, device=dev, dtype=torch.uint8)
        _lib.check(lib.so_point_sampling(ops._p(r3), ops._p(l2i), D, Q, 6, 90.0, 160.0, ops._p(uv), ops._p(mask), ops._p(vis),
                                         ops._stream()), 'so_point_sampling')
        for scale in (None, torch.ones(6, 2, device=dev)):
            got = ops.point_sampling(r3, l2i, (90, 160), scale)
            assert all(torch.equal(a, b) for a, b in zip(got, (uv, mask, vis)))
    with pytest.raises(ValueError, match='scale_xy'):
        ops.point_sampling(r3, l2i, (90, 160), torch.ones(1, 2, device=dev))
    with pytest.raises(TypeError):
        ops.point_sampling(r3, l2i, (90, 160), torch.ones(6, 2, device=dev, dtype=torch.float64))


# --------------------------------------------------------------------------------------------- encoder inference
def _oracle(monkeypatch, case, lifter, enc, ocfg, feats, l2i, ratios):
    """ep._oracle_case with the ratios: oracle.focal.tpv_encoder_ref and the per-layer operands rescaled alike."""
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    ep._promote_oracle_tables(monkeypatch)
    p = {k: v.detach().cpu().double() for k, v in enc.state_dict().items()}
    mref = GridMeterMappingRef(**case['margs'])
    planes = [t.detach().cpu().double() for t in (lifter.tpv_hw, lifter.tpv_zh, lifter.tpv_wz)]
    feats64 = [f.double() for f in feats]
    ref = of.tpv_encoder_ref(p, mref, planes, feats64, l2i[None], case['img'], ocfg, ratios)
    tpv_pos, feat, shapes, ref_2d, ref_cams, masks = ep._oracle_layer_inputs(p, mref, feats64, l2i, case['img'], ocfg)
    ref_cams = [of.focal_scale_ref(rc, *ratios) for rc in ref_cams]
    return p, mref, ref, (tpv_pos, feat, shapes, ref_2d, ref_cams, masks)


@pytest.mark.parametrize('ratios', ['kitti_raw_depth', 'above_one'])
@pytest.mark.parametrize('name', ['nuscenes', 'kitti'])
def test_encoder_and_each_layer_with_ratios_match_oracle(name, ratios, monkeypatch):
    """The 4-layer encoder and every layer at the NUSC / KITTI geometry, on the second-generation fused kernels.  On the six
    nuScenes cameras the kitti_raw_depth pair is given once (broadcast) and 'above_one' is the straddling per-camera set."""
    dev = _dev()
    case = dict(nuscenes=NUSC, kitti=KITTI)[name]
    rx, ry = RATIOS[ratios][1:]
    if name == 'nuscenes' and ratios == 'above_one':
        rx, ry = STRADDLE
    lifter, enc, ocfg = ep._model(case)
    metas, feats, l2i = ep._frame(case)
    p, mref, ref, layer_ops = _oracle(monkeypatch, case, lifter, enc, ocfg, feats, l2i, (rx, ry))
    outside = sum(_outside_visible(rc, m) for rc, m in zip(layer_ops[4], layer_ops[5]))
    if ratios == 'above_one':
        assert outside > 0
    lifter.to(dev)
    enc.to(dev)
    spies = ep._Spies(monkeypatch)
    out, seen = ep._run_gpu(lifter, enc, feats, _with_ratios(metas, rx, ry), dev)
    ep._check_against_oracle('%s %s' % (name, ratios), out, seen, ref, p, mref, layer_ops, ocfg)
    L = ocfg['num_layers']
    assert spies.rows == L and len(spies.self_calls) == L and len(spies.cross_calls) == 3 * L
    assert all(ep._self_v2(c['Dh'], c['n']) for c in spies.self_calls)
    assert all(ep._cross_v2(c['Dh'], c['n']) for c in spies.cross_calls)


def test_unit_ratios_change_nothing():
    """nuScenes metas with focal_ratios_x = focal_ratios_y = [1.0] * 6 give the planes of metas without the keys, bit for
    bit, in inference and in a training forward."""
    dev = _dev()
    import test_gpu_attn_train as at
    lifter, enc, _ = ep._model(NUSC)
    metas, feats, _ = ep._frame(NUSC)
    lifter.to(dev)
    enc.to(dev)
    ones = _with_ratios(metas, [1.0] * 6, [1.0] * 6)
    a, _ = ep._run_gpu(lifter, enc, feats, metas, dev)
    b, _ = ep._run_gpu(lifter, enc, feats, ones, dev)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    enc, feats, metas = at._small_encoder(dev, 2, seed=31)
    g = torch.Generator().manual_seed(32)
    H, W, Z = enc.tpv_size
    rep = [torch.randn(1, n, 96, generator=g).to(dev).requires_grad_(True) for n in (H * W, Z * H, W * Z)]
    a = enc(representation=rep, ms_img_feats=feats, metas=metas)['representation']
    b = enc(representation=rep, ms_img_feats=feats, metas=_with_ratios(metas, [1.0] * 6, [1.0] * 6))['representation']
    assert a[0].requires_grad and all(torch.equal(x, y) for x, y in zip(a, b))


# --------------------------------------------------------------------------------------------- training
def test_layer_training_routine_with_ratios_above_one_matches_fp64():
    """One layer's training routine (forward_rows_train) on projections rescaled by the straddling ratios against fp64
    autograd of tpv_layer_ref, at the bars of test_gpu_attn_train.test_tpv_layer_training_matches_fp64_oracle."""
    dev = _dev()
    import test_gpu_attn_train as at
    from oracle import lifting as ol
    enc, feats, metas = at._small_encoder(dev, 1, seed=23)
    metas = _with_ratios(metas, *STRADDLE)
    layer = enc.layers[0]
    g = torch.Generator().manual_seed(24)
    planes, pos, feat, kw = at._layer_inputs(enc, feats, metas, g)
    l2i = torch.tensor(np.asarray(metas[0]['lidar2img']), dtype=torch.float32)
    outside = 0
    for r3, uv, m in zip((enc.ref_3d_hw, enc.ref_3d_zh, enc.ref_3d_wz), kw['reference_points_cams'], kw['tpv_masks']):
        uv_ref = of.focal_scale_ref(ol.point_sampling_ref(r3.cpu()[None], l2i[None], (90, 160))[0], *STRADDLE)
        assert torch.equal(uv.cpu(), uv_ref)
        outside += _outside_visible(uv_ref, m.cpu())
    assert outside > 0
    outs = layer(planes, feat, feat, **kw)
    gouts = [torch.randn(o.shape, generator=g) for o in outs]
    sum((o * go.to(dev)).sum() for o, go in zip(outs, gouts)).backward()
    p64 = at._leaf64(layer, 'l.')
    planes64, pos64 = ([t.detach().cpu().double().requires_grad_(True) for t in ts] for ts in (planes, pos))
    f64 = feat.detach().cpu().double().requires_grad_(True)
    shapes = [tuple(s) for s in kw['spatial_shapes'].tolist()]
    ocfg = dict(num_heads=layer.attentions[0].num_heads, num_points_self=layer.attentions[0].num_points, num_cams=6)
    ref = ol.tpv_layer_ref(p64, 'l.', planes64, pos64, f64, shapes, kw['ref_2d'].cpu().double(),
                           [uv.cpu().double() for uv in kw['reference_points_cams']], [m.cpu().bool() for m in kw['tpv_masks']],
                           enc.tpv_size, ocfg)
    for i, (o, r) in enumerate(zip(outs, ref)):
        assert (o.detach().cpu().double() - r.detach()).abs().max().item() < 1e-4, i
    sum((r * go.double()).sum() for r, go in zip(ref, gouts)).backward()
    at._assert_grads_match(layer, p64, 'l.', at._tol)
    for name, got, want, tol in [('plane %d' % i, a, b, 1e-3) for i, (a, b) in enumerate(zip(planes, planes64))] + \
            [('pos %d' % i, a, b, 1e-3) for i, (a, b) in enumerate(zip(pos, pos64))] + [('image features', feat, f64, 2e-4)]:
        e = (got.grad.cpu().double() - want.grad).abs().max().item() / want.grad.abs().max().item()
        assert e < tol, name


def test_cross_attn_core_gradients_on_rescaled_uv_match_fp64():
    """The image cross-attention core's backward on uv rescaled by ratios above 1 against fp64 autograd at the kernel's fp32
    sampling locations: 5e-5 abs for value and logits, 5e-4 of max-abs for offsets (test_gpu_attn_train's bars)."""
    dev = _dev()
    import test_gpu_attn_train as at
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    from selfocc_b200 import ops, synth
    g = torch.Generator().manual_seed(41)
    n_cam, D, Hd, Dh = 6, 20, 6, 16
    shapes = [(12, 20), (6, 10), (3, 5), (2, 3)]
    Nv = sum(h * w for h, w in shapes)
    margs, _ = synth.small_mapping(10, 4, rng=30.0)
    r3 = ol.ref_3d_tables(GridMeterMappingRef(**margs), [48, D, 8])[1]
    Q = r3.shape[1]
    scale = torch.tensor(STRADDLE, dtype=torch.float32).t().contiguous()
    uv, mask, vis = ops.point_sampling(r3.contiguous().to(dev), at._rig(n_cam).to(dev), (90, 160), scale.to(dev))
    assert _outside_visible(uv[:, None].cpu(), mask[:, None].cpu()) > 0
    vis[:, [0, 7, 11]] = 0
    uv, vis = uv.cpu(), vis.cpu()
    t = dict(value=torch.randn(n_cam, Nv, Hd, Dh, generator=g), offsets=3.0 * torch.randn(Q, Hd, 4, D, 2, generator=g),
             logits=torch.randn(Q, Hd, 4, D, generator=g), grad=torch.randn(Q, Hd * Dh, generator=g))
    slots_ref, grads_ref = at._cross_ref64(t, uv, vis, shapes)
    ss, lsi = at._levels(shapes, dev)
    v, o, lg = (t[k].to(dev).requires_grad_(True) for k in ('value', 'offsets', 'logits'))
    slots = ops.TPVCrossAttnFunction.apply(v, ss, lsi, o, lg, uv.to(dev), vis.to(dev))
    assert (slots.detach().cpu() - slots_ref).abs().max().item() < 2e-5
    slots.backward(t['grad'].to(dev))
    at._assert_core_grads((v.grad, o.grad, lg.grad), grads_ref, 'cross on rescaled uv')


@pytest.mark.parametrize('world', [2, 3])
def test_query_sharded_step_with_ratios_equals_unsharded(world):
    """test_gpu_encoder_shard's emulated ranks on a frame with the straddling ratios: planes bit for bit, DDP-mean
    gradients within 1e-5 of each tensor's max-abs."""
    dev = _dev()
    import test_gpu_encoder_shard as es
    from test_gpu_ray_shard import _check_values
    model, ml, feats, metas, imgs = es.small_training_model(dev, dropout=0.0)
    plain, _ = es.unsharded_step(model, feats, metas, imgs)
    metas = _with_ratios(metas, *STRADDLE)
    rep1, inp1 = es.unsharded_step(model, feats, metas, imgs)
    assert not torch.equal(plain[0], rep1[0])                 # the ratios reach the training step
    del plain
    tot1, ref = ml(inp1)
    ref_g = es._grads(tot1, model, feats)
    del inp1
    planes, inputs, _, _ = es.lockstep_step(model, feats, metas, imgs, world)
    for rep in planes:
        assert all(torch.equal(a, b) for a, b in zip(rep, rep1))
    res, got = es._sharded_grads(ml, model, feats, inputs, world, True)
    for _, d in res:
        _check_values(ref, d)
    es._check_grads(got, ref_g)


# --------------------------------------------------------------------------------------------- sharded lifter and graph
@pytest.mark.parametrize('world', [2, 3, 8])
def test_sharded_lifter_with_ratios_is_bit_identical(world):
    from test_gpu_pipeline import _setup
    from selfocc_b200.dist import ShardedLifter
    model, cfg, margs, rng, metas, feats, l2i, i2l = _setup()
    dev = torch.device('cuda:0')
    model.to(dev)
    feats = [f.to(dev) for f in feats]
    metas_r = _with_ratios(metas, *STRADDLE)
    with torch.no_grad():
        rep = model.lifter(ms_img_feats=feats)['representation']
        plain = model.encoder(representation=rep, ms_img_feats=feats, metas=metas)['representation']
        ref = model.encoder(representation=rep, ms_img_feats=feats, metas=metas_r)['representation']
        sl = ShardedLifter(model.encoder)
        st = sl.prepare(feats, metas_r)
        qfull = torch.cat([p[0] for p in rep], 0).contiguous()
        for li in range(len(model.encoder.layers)):
            bufs = [sl.pad_local(sl.layer_local(li, qfull, st, r, world), r, world) for r in range(world)]
            qfull = sl.assemble(torch.stack(bufs, 0), world)
        got = torch.split(qfull, sl.sizes, 0)
    assert not torch.equal(plain[0], ref[0])
    for a, b in zip(got, ref):
        assert torch.equal(a, b[0])


def test_graphed_frame_reads_device_ratios_at_replay():
    """GraphedFrame at world size 1 with the ratios as device tensors in the metas: rewritten in place between replays, the
    replay equals an eager frame on the new ratios, bit for bit."""
    from test_gpu_pipeline import _setup
    from selfocc_b200.dist import GraphedFrame, frame_sharded
    model, cfg, margs, rng, metas, feats, l2i, i2l = _setup(color_dims=3)
    dev = torch.device('cuda:0')
    model.to(dev)
    model.head.num_samples = 64
    model.head.render_bkgd = 'white'
    feats = [f.to(dev) for f in feats]
    fx = torch.tensor(STRADDLE[0], dtype=torch.float32, device=dev)
    fy = torch.tensor(STRADDLE[1], dtype=torch.float32, device=dev)
    metas_d = [dict(lidar2img=torch.tensor(np.asarray(metas[0]['lidar2img']), dtype=torch.float32, device=dev),
                    img2lidar=torch.tensor(np.asarray(metas[0]['img2lidar']), dtype=torch.float32, device=dev),
                    img_shape=metas[0]['img_shape'], focal_ratios_x=fx, focal_ratios_y=fy)]
    with torch.no_grad():
        eager = frame_sharded(model, feats, metas_d)
        gf = GraphedFrame(model, feats, metas_d)
        rep = gf.replay()
        torch.cuda.synchronize()
        for k in eager:
            assert torch.equal(rep[k], eager[k]), k
        fx.copy_(fx.flip(0))                             # the next frame's ratios, through the same device tensors
        fy.fill_(1.07)
        eager2 = frame_sharded(model, feats, metas_d)
        rep2 = gf.replay()
        torch.cuda.synchronize()
        for k in eager2:
            assert torch.equal(rep2[k], eager2[k]), k
        assert not torch.equal(eager2['depth'], eager['depth'])


# --------------------------------------------------------------------------------------------- a loader-shaped frame
def test_kitti_raw_depth_model_on_a_loader_shaped_frame():
    """Lifter + encoder + head of the shipped kitti_raw_depth config (tests/golden/reference_model_cfgs.json) at a reduced FPN
    size, fed metas with exactly the keys dataset_wrapper_temporal.py emits for it (lidar2img a list of numpy arrays,
    img_shape a tuple, scale_rate, focal_ratios_x / _y lists, flip) plus the head's temImg2lidar: prepare() and render()
    run, and the encoder output matches the fp64 oracle within the 2e-4 bar."""
    dev = _dev()
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    from selfocc_b200 import synth
    from selfocc_b200.segmentor import TPVHotPath
    cfg = json.load(open(os.path.join(HERE, 'golden', 'reference_model_cfgs.json')))['kitti_raw/kitti_raw_depth.py']
    torch.manual_seed(0)
    model = TPVHotPath(lifter=cfg['lifter'], encoder=cfg['encoder'], head=cfg['head'])
    enc = model.encoder
    enc.init_weights()
    g = torch.Generator().manual_seed(1)
    rn = lambda t: torch.randn(t.shape, generator=g)
    with torch.no_grad():                                 # away from the trivial initialisation, as ep._model
        for n, p in enc.named_parameters():
            if 'sampling_offsets.weight' in n or 'attention_weights.weight' in n:
                p.copy_(0.05 * rn(p))
            elif '.norms.' in n:
                p.copy_(1.0 + 0.3 * rn(p) if n.endswith('.weight') else 0.1 * rn(p))
            elif n.endswith('.bias'):
                p.add_(0.1 * rn(p))
        for p in model.lifter.parameters():
            p.mul_(0.5)
    model.eval().to(dev)
    img_h, img_w = cfg['head']['ray_img_size']
    l2i, i2l = synth.camera_rig((0.,), f=721.5, cx=img_w / 2, cy=img_h / 2, height=1.65, radius=0.0)
    scale_rate, pad = 0.84, [0.8649, 0.8421]
    metas = [dict(lidar2img=list(l2i), img_shape=(img_h, img_w), scale_rate=scale_rate,
                  focal_ratios_x=[scale_rate / pad[1]], focal_ratios_y=[scale_rate / pad[0]], flip=False,
                  temImg2lidar=list(i2l))]
    fpn = [(12, 38), (6, 19), (3, 10), (2, 5)]
    feats = [torch.randn(1, 1, 96, h, w, generator=g) for h, w in fpn]
    with torch.no_grad():
        res = model(ms_img_feats=[f.to(dev) for f in feats], metas=metas, prepare=True)
        out = model.head.render(metas=metas)
    depth = out['ms_depths'][0]
    assert depth.numel() == cfg['head']['ray_number'][0] * cfg['head']['ray_number'][1] and torch.isfinite(depth).all()
    # fp64 oracle of the encoder (the geometry tables promoted as ep._promote_oracle_tables does)
    mp = pytest.MonkeyPatch()
    try:
        ep._promote_oracle_tables(mp)
        p = {k: v.detach().cpu().double() for k, v in enc.state_dict().items()}
        e = cfg['encoder']
        ocfg = dict(num_freqs=e['positional_encoding']['num_freqs'], tot_range=e['positional_encoding']['tot_range'],
                    num_points_cross=e['num_points_cross'], num_points_self=e['num_points_self'][0], num_layers=e['num_layers'],
                    num_heads=6, num_cams=1)
        planes = [t.detach().cpu().double() for t in (model.lifter.tpv_hw, model.lifter.tpv_zh, model.lifter.tpv_wz)]
        ref = of.tpv_encoder_ref(p, GridMeterMappingRef(**e['mapping_args']), planes, [f.double() for f in feats],
                                 torch.tensor(l2i, dtype=torch.float32)[None], (img_h, img_w), ocfg,
                                 (metas[0]['focal_ratios_x'], metas[0]['focal_ratios_y']))
    finally:
        mp.undo()
    errs = ep._max_err([t.cpu() for t in res['representation']], ref)
    print('kitti_raw_depth encoder: max abs err per plane %s' % ' / '.join('%.2e' % x for x in errs))
    assert max(errs) < ENCODER_BAR
