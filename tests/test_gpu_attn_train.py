"""Training through the fused attention cores: the backward kernels (so_tpv_cross_attn_backward / so_tpv_self_attn_backward)
against fp64 autograd of the oracle, their determinism, the encoder layer's training routine (forward_rows_train) and the
attention modules' reference formulation (the MSDA op's backward) against the fp64 oracle, which path a training forward
takes, the full-size cores against the reference-contract composition, and the training step's freedom from host syncs.
The C-ABI argument checks run without a GPU."""
import importlib.util
import os

import pytest
import torch

from selfocc_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
gpu = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _levels(shapes, dev):
    ss = torch.tensor(shapes, dtype=torch.int64)
    lsi = torch.cat([ss.new_zeros(1), ss.prod(1).cumsum(0)[:-1]])
    return ss.to(dev), lsi.to(dev)


def _rig(n_cam):
    l2i, _ = synth.camera_rig(synth.NUSC_YAWS[:n_cam], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    return torch.tensor(l2i, dtype=torch.float32)


def _fp32_locations(offsets, ref, shapes):
    """The kernels' sampling locations fmaf(o, 1/W_l, r) in fp32 (1/W_l rounded to fp32 as the kernel does).  o * (1/W_l) is
    exact in fp64 (24 x 24 mantissa bits); adding r rounds at most once more, far below fp32 resolution, so rounding the
    fp64 result to fp32 gives the fused multiply-add's single rounding (barring an exact fp32 tie, ~2^-29 per value).
    offsets [..., L, P, 2] and ref broadcastable to it."""
    rcp = torch.tensor([[1.0 / w, 1.0 / h] for h, w in shapes], dtype=torch.float32).double()
    return (offsets.double() * rcp[:, None, :] + ref.double()).float()


def _at_kernel_locations(loc64, loc32):
    """fp64 locations whose VALUE is the kernel's fp32 location and whose gradient is that of the fp64 location arithmetic.
    The bilinear gradient jumps at pixel faces: a sample within fp32 rounding of a face lies in one cell in fp32 and possibly
    in the neighbour in fp64, so the fp64 reference must sample the same cells as the kernel (DESIGN section 2(b))."""
    return loc64 + (loc32.double() - loc64).detach()


def _assert_core_grads(got, ref, what):
    gv, go, gl = got
    rv, ro, rl = ref
    ev, el = (gv.cpu() - rv).abs().max().item(), (gl.cpu() - rl).abs().max().item()
    eo = (go.cpu() - ro).abs().max().item() / ro.abs().max().item()
    print('%s: grad_value %.2e, grad_logits %.2e abs; grad_offsets %.2e of max-abs' % (what, ev, el, eo))
    assert ev < 5e-5 and el < 5e-5        # the MSDA backward tolerances of DESIGN section 2
    assert eo < 5e-4


# --------------------------------------------------------------------------------------------- CPU: the C ABI
def test_backward_entry_points_reject_bad_arguments_without_a_gpu():
    """Null pointers return SO_ERR_INVALID_ARG (-1), an unsupported head width SO_ERR_UNSUPPORTED (-2), before any CUDA call."""
    import ctypes as C
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N = None
    one = C.c_void_p(16)   # non-null, 16-byte aligned dummy (never dereferenced on these paths)
    assert lib.so_tpv_cross_attn_backward(*[N] * 12, 6, 100, 6, 16, 10, 4, 8, N) == -1
    assert lib.so_tpv_cross_attn_backward(*[one] * 7, N, *[one] * 4, 6, 100, 6, 16, 10, 4, 8, N) == -1      # no count
    assert lib.so_tpv_cross_attn_backward(*[one] * 12, 6, 100, 6, 24, 10, 4, 8, N) == -2                   # Dh = 24
    assert lib.so_tpv_cross_attn_backward(*[one] * 12, 6, 100, 6, 16, 0, 4, 8, N) == -1                    # Q = 0
    assert lib.so_tpv_cross_attn_backward(*[one] * 9, C.c_void_p(24), one, one, 6, 100, 6, 16, 10, 4, 8, N) == -1  # grad_value not float4-aligned
    assert lib.so_tpv_self_attn_backward(*[N] * 10, 100, 6, 16, 10, 3, 12, N) == -1
    assert lib.so_tpv_self_attn_backward(*[one] * 6, N, one, one, one, 100, 6, 16, 10, 3, 12, N) == -1      # no grad_out
    assert lib.so_tpv_self_attn_backward(*[one] * 10, 100, 6, 8, 10, 3, 12, N) == -2                       # Dh = 8
    assert lib.so_tpv_self_attn_backward(*[one] * 8, C.c_void_p(20), one, 100, 6, 16, 10, 3, 12, N) == -1   # odd grad_offsets
    assert lib.so_tpv_self_attn_backward(*[one] * 10, 100, 6, 16, 10, 9, 12, N) == -2                      # L > 8 levels


# --------------------------------------------------------------------------------------------- core gradients vs fp64
def _cross_case(n_cam, D, Hd, Dh, seed):
    """Pillar tables of a small grid projected into a `_rig` camera set; queries 0, 7, 11 are made visible in no camera."""
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    g = torch.Generator().manual_seed(seed)
    shapes = [(12, 20), (6, 10), (3, 5), (2, 3)]
    Nv = sum(h * w for h, w in shapes)
    margs, _ = synth.small_mapping(10, 4, rng=30.0)
    r3 = {8: 0, 20: 1, 48: 2}
    r3 = ol.ref_3d_tables(GridMeterMappingRef(**margs), [48, 20, 8])[r3[D]]
    Q = r3.shape[1]
    from selfocc_b200 import ops
    uv, _, vis = ops.point_sampling(r3.contiguous().cuda(), _rig(n_cam).cuda(), (90, 160))
    vis[:, [0, 7, 11]] = 0
    t = dict(value=torch.randn(n_cam, Nv, Hd, Dh, generator=g), offsets=3.0 * torch.randn(Q, Hd, 4, D, 2, generator=g),
             logits=torch.randn(Q, Hd, 4, D, generator=g), grad=torch.randn(Q, Hd * Dh, generator=g))
    return t, uv.cpu(), vis.cpu(), shapes


def _cross_ref64(t, uv, vis, shapes):
    from oracle import lifting as ol
    v, o, lg = (t[k].double().requires_grad_(True) for k in ('value', 'offsets', 'logits'))
    N = v.shape[0]
    Q, Hd, L, D, _ = o.shape
    loc = ol.deform_locations(uv.double(), o[None], shapes, per_level_ref=False)                  # [N, Q, Hd, L, D, 2]
    loc32 = _fp32_locations(t['offsets'][None], uv[:, :, None, None], shapes)
    assert ((loc32 < 0) | (loc32 > 1)).any()                                                      # zero padding is exercised
    aw = lg.view(Q, Hd, L * D).softmax(-1).view(1, Q, Hd, L, D).expand(N, -1, -1, -1, -1)
    per_cam = ol.msda_ref(v, shapes, _at_kernel_locations(loc, loc32), aw)                          # [N, Q, Hd*Dh]
    visd = vis.double()[..., None]
    slots = (per_cam * visd).sum(0) / visd.sum(0).clamp(min=1)
    slots.backward(t['grad'].double())
    return slots.detach(), (v.grad, o.grad, lg.grad)


@gpu
@pytest.mark.parametrize('n_cam,D,Hd,Dh', [(6, 8, 6, 16), (6, 20, 6, 16), (6, 48, 6, 16), (6, 20, 3, 32), (2, 48, 6, 16)])
def test_cross_attn_core_gradients_match_fp64(n_cam, D, Hd, Dh):
    dev = _dev()
    from selfocc_b200 import ops
    t, uv, vis, shapes = _cross_case(n_cam, D, Hd, Dh, seed=D + Dh + n_cam)
    slots_ref, grads_ref = _cross_ref64(t, uv, vis, shapes)
    ss, lsi = _levels(shapes, dev)
    v, o, lg = (t[k].to(dev).requires_grad_(True) for k in ('value', 'offsets', 'logits'))
    slots = ops.TPVCrossAttnFunction.apply(v, ss, lsi, o, lg, uv.to(dev), vis.to(dev))
    assert (slots.detach().cpu() - slots_ref).abs().max().item() < 2e-5
    slots.backward(t['grad'].to(dev))
    _assert_core_grads((v.grad, o.grad, lg.grad), grads_ref, 'cross N=%d D=%d Dh=%d' % (n_cam, D, Dh))
    # a query visible in no camera has output 0: exactly zero gradients, and nothing reaches grad_value from it
    blind = (vis.sum(0) == 0).nonzero().squeeze(-1)
    assert blind.numel() >= 3
    assert not o.grad[blind.to(dev)].any() and not lg.grad[blind.to(dev)].any()
    g_blind = torch.zeros_like(t['grad'])
    g_blind[blind] = t['grad'][blind]
    gv, go, gl = ops.tpv_cross_attn_backward(v.detach(), ss, lsi, o.detach(), lg.detach(), uv.to(dev), vis.to(dev),
                                             vis.to(dev).sum(0, dtype=torch.int32), g_blind.to(dev))
    assert not gv.any() and not go.any() and not gl.any()


@gpu
@pytest.mark.parametrize('P,Hd,Dh', [(5, 6, 16), (12, 6, 16), (12, 3, 32)])
def test_self_attn_core_gradients_match_fp64(P, Hd, Dh):
    dev = _dev()
    from oracle import lifting as ol
    from selfocc_b200 import ops
    g = torch.Generator().manual_seed(P + Dh)
    H, W, Z = 9, 7, 4
    shapes = [(H, W), (Z, H), (W, Z)]
    Q = H * W + Z * H + W * Z
    ref2d = ol.cross_view_ref_points(H, W, Z, [P, P, P])                                            # [Q, 3, P, 2]
    t = dict(value=torch.randn(Q, Hd, Dh, generator=g), offsets=2.0 * torch.randn(Q, Hd, 3, P, 2, generator=g),
             logits=torch.randn(Q, Hd, 3, P, generator=g), grad=torch.randn(Q, Hd * Dh, generator=g))
    v64, o64, l64 = (t[k].double().requires_grad_(True) for k in ('value', 'offsets', 'logits'))
    loc = ol.deform_locations(ref2d[None].double(), o64[None], shapes, per_level_ref=True)
    loc32 = _fp32_locations(t['offsets'][None], ref2d[None, :, None], shapes)
    assert ((loc32 < 0) | (loc32 > 1)).any()
    aw = l64.view(1, Q, Hd, 3 * P).softmax(-1).view(1, Q, Hd, 3, P)
    out_ref = ol.msda_ref(v64[None], shapes, _at_kernel_locations(loc, loc32), aw)[0]
    out_ref.backward(t['grad'].double())
    ss, lsi = _levels(shapes, dev)
    v, o, lg = (t[k].to(dev).requires_grad_(True) for k in ('value', 'offsets', 'logits'))
    out = ops.TPVSelfAttnFunction.apply(v, ss, lsi, o, lg, ref2d.contiguous().to(dev))
    assert (out.detach().cpu() - out_ref.detach()).abs().max().item() < 2e-5
    out.backward(t['grad'].to(dev))
    _assert_core_grads((v.grad, o.grad, lg.grad), (v64.grad, o64.grad, l64.grad), 'self P=%d Dh=%d' % (P, Dh))


@gpu
def test_backward_offsets_and_logits_are_deterministic():
    dev = _dev()
    from selfocc_b200 import ops
    t, uv, vis, shapes = _cross_case(6, 48, 6, 16, seed=3)
    ss, lsi = _levels(shapes, dev)
    a = [t[k].to(dev) for k in ('value', 'offsets', 'logits')]
    count = vis.to(dev).sum(0, dtype=torch.int32)
    r1 = ops.tpv_cross_attn_backward(*a[:1], ss, lsi, *a[1:], uv.to(dev), vis.to(dev), count, t['grad'].to(dev))
    r2 = ops.tpv_cross_attn_backward(*a[:1], ss, lsi, *a[1:], uv.to(dev), vis.to(dev), count, t['grad'].to(dev))
    assert torch.equal(r1[1], r2[1]) and torch.equal(r1[2], r2[2])
    from oracle import lifting as ol
    H, W, Z, P = 9, 7, 4, 12
    Q = H * W + Z * H + W * Z
    g = torch.Generator().manual_seed(4)
    ss, lsi = _levels([(H, W), (Z, H), (W, Z)], dev)
    args = (torch.randn(Q, 6, 16, generator=g).to(dev), ss, lsi, (2.0 * torch.randn(Q, 6, 3, P, 2, generator=g)).to(dev),
            torch.randn(Q, 6, 3, P, generator=g).to(dev), ol.cross_view_ref_points(H, W, Z, [P] * 3).contiguous().to(dev),
            torch.randn(Q, 96, generator=g).to(dev))
    r1, r2 = ops.tpv_self_attn_backward(*args), ops.tpv_self_attn_backward(*args)
    assert torch.equal(r1[1], r2[1]) and torch.equal(r1[2], r2[2])


# --------------------------------------------------------------------------------------------- modules vs the fp64 oracle
def _perturb(mod, g):
    with torch.no_grad():
        for n, p in mod.named_parameters():
            if 'sampling_offsets.weight' in n or 'attention_weights.weight' in n:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            elif 'bias' in n and 'sampling_offsets' not in n:
                p.copy_(0.1 * torch.randn(p.shape, generator=g))


def _leaf64(mod, pre):
    return {pre + k: v.detach().cpu().double().requires_grad_(True) for k, v in mod.state_dict().items()}


def _assert_grads_match(mod, p64, pre, tol):
    """every parameter's gradient within tol(name) of the largest fp64 gradient entry"""
    for n, prm in mod.named_parameters():
        ref = p64[pre + n].grad
        err = (prm.grad.cpu().double() - ref).abs().max().item() / ref.abs().max().item()
        print('grad %s: %.2e of max-abs' % (n, err))
        assert err < tol(n), n


# Tolerances of the module tests (relative to the largest |entry| of the fp64 gradient): 2e-4 for the projections that see
# only continuous functions of the sampling locations (value_proj, attention_weights, output_proj, the image features), 1e-3
# where the location gradient enters (sampling_offsets, the query).  The module computes its offsets in fp32 and the oracle
# in fp64, so a sample within rounding of a pixel face could take the other cell's bilinear slope; the inputs are seeded and
# small enough that none does, and 1e-3 would not hide a wrong cell.
def _tol(name):
    return 1e-3 if 'sampling_offsets' in name else 2e-4


@gpu
def test_image_cross_attention_training_matches_fp64_oracle():
    dev = _dev()
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    from selfocc_b200 import ops
    from selfocc_b200.encoder import TPVCrossAttention
    g = torch.Generator().manual_seed(21)
    C, Hd, N = 96, 6, 6
    shapes = [(12, 20), (6, 10), (3, 5), (2, 3)]
    Nv = sum(h * w for h, w in shapes)
    att = TPVCrossAttention(embed_dims=C, num_cams=N, dropout=0.0, batch_first=True, num_heads=Hd, num_levels=4,
                            num_points=[12, 8, 4])
    _perturb(att, g)
    att.to(dev).train()
    margs, _ = synth.small_mapping(6, 3, rng=30.0)
    tables = ol.ref_3d_tables(GridMeterMappingRef(**margs), [12, 8, 4])
    l2i = _rig(N).to(dev)
    uvs, masks, vises = [], [], []
    for r3 in tables:
        uv, mask, vis = ops.point_sampling(r3.contiguous().to(dev), l2i, (90, 160))
        uvs.append(uv[:, None]); masks.append(mask[:, None]); vises.append(vis)
    queries = [torch.randn(1, r3.shape[1], C, generator=g) for r3 in tables]
    feat = torch.randn(N, Nv, 1, C, generator=g)
    gouts = [torch.randn(q.shape, generator=g) for q in queries]
    qd = [q.to(dev).requires_grad_(True) for q in queries]
    fd = feat.to(dev).requires_grad_(True)
    ss, lsi = _levels(shapes, dev)
    outs = att(qd, fd, fd, None, spatial_shapes=ss, level_start_index=lsi, reference_points_cams=uvs, tpv_masks=masks)
    sum((o * go.to(dev)).sum() for o, go in zip(outs, gouts)).backward()
    f64 = feat.double().requires_grad_(True)
    names = ('attn_hw', 'attn_zh', 'attn_wz')
    for i, name in enumerate(names):
        plane = getattr(att, name)
        p64 = _leaf64(plane, 'x.')
        q64 = queries[i].double().requires_grad_(True)
        ref, _ = ol.image_cross_attn_ref(p64, 'x.', q64, f64, shapes, uvs[i].cpu().double(), masks[i].cpu().bool(), Hd, N)
        err = (outs[i].detach().cpu().double() - ref.detach()).abs().max().item()
        print('%s output max abs err %.2e' % (name, err))
        assert err < 1e-4
        ref.backward(gouts[i].double())
        _assert_grads_match(plane, p64, 'x.', _tol)
        eq = (qd[i].grad.cpu().double() - q64.grad).abs().max().item() / q64.grad.abs().max().item()
        assert eq < 1e-3, (name, eq)
    ef = (fd.grad.cpu().double() - f64.grad).abs().max().item() / f64.grad.abs().max().item()
    print('image feature grad %.2e of max-abs' % ef)
    assert ef < 2e-4


@gpu
def test_cross_view_hybrid_attention_training_matches_fp64_oracle():
    dev = _dev()
    from oracle import lifting as ol
    from selfocc_b200.encoder import CrossViewHybridAttention
    g = torch.Generator().manual_seed(22)
    C, Hd, P = 96, 6, 4
    H, W, Z = 9, 7, 4
    shapes = [(H, W), (Z, H), (W, Z)]
    Q = H * W + Z * H + W * Z
    att = CrossViewHybridAttention(embed_dims=C, num_heads=Hd, num_levels=3, num_points=P, dropout=0.0, batch_first=True)
    _perturb(att, g)
    att.to(dev).train()
    ref2d = ol.cross_view_ref_points(H, W, Z, [P] * 3)[None]
    query, pos, gout = (torch.randn(1, Q, C, generator=g) for _ in range(3))
    qd, posd = query.to(dev).requires_grad_(True), pos.to(dev).requires_grad_(True)
    ss, lsi = _levels(shapes, dev)
    out = att(qd, qd, qd, None, query_pos=posd, reference_points=ref2d.to(dev), spatial_shapes=ss, level_start_index=lsi)
    (out * gout.to(dev)).sum().backward()
    p64 = _leaf64(att, 'a.')
    q64, pos64 = query.double().requires_grad_(True), pos.double().requires_grad_(True)
    ref = ol.cross_view_self_attn_ref(p64, 'a.', q64, pos64, ref2d.double(), shapes, Hd, P)
    err = (out.detach().cpu().double() - ref.detach()).abs().max().item()
    print('self-attn module output max abs err %.2e' % err)
    assert err < 1e-4
    ref.backward(gout.double())
    _assert_grads_match(att, p64, 'a.', _tol)
    for name, a, b in (('query', qd, q64), ('query_pos', posd, pos64)):
        e = (a.grad.cpu().double() - b.grad).abs().max().item() / b.grad.abs().max().item()
        print('%s grad %.2e of max-abs' % (name, e))
        assert e < 1e-3, name


# --------------------------------------------------------------------------------------------- the layer's training routine
def _small_encoder(dev, num_layers, seed):
    """The encoder of test_tpv_layer_training_step_runs_without_host_sync's geometry at dropout 0, weights `_perturb`ed, in
    train(); returns it with a frame's FPN features and metas."""
    from selfocc_b200 import configs
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    torch.manual_seed(seed)
    margs, rng = synth.small_mapping(8, 4, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=num_layers,
                                  num_points_cross=(6, 6, 4), num_points_self=4, dropout=0.0)
    enc = build_head(cfg['encoder'])
    enc.init_weights()
    g = torch.Generator().manual_seed(seed + 1)
    _perturb(enc, g)
    enc.to(dev).train()
    l2i, _ = synth.camera_rig(synth.NUSC_YAWS, f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    metas = [dict(lidar2img=list(l2i), img_shape=(90, 160))]
    feats = [torch.randn(1, 6, 96, h, w, generator=g).to(dev) for h, w in [(12, 20), (6, 10), (3, 5), (2, 3)]]
    return enc, feats, metas


def _layer_inputs(enc, feats, metas, g):
    """One layer's operands as leaves: planes and positional embeddings [1, Q_i, C] x 3, image features [N, sum(hw), 1, C];
    the layer's keyword arguments; the camera projections and masks."""
    dev = feats[0].device
    feat, ss, lsi = enc.flatten_features(feats)
    H, W, Z = enc.tpv_size
    C = feat.shape[-1]
    planes = [torch.randn(1, n, C, generator=g).to(dev).requires_grad_(True) for n in (H * W, Z * H, W * Z)]
    pos = [torch.randn(1, n, C, generator=g).to(dev).requires_grad_(True) for n in (H * W, Z * H, W * Z)]
    feat = feat.detach().requires_grad_(True)
    uvs, masks, vises = enc.project_reference_points(metas, dev)
    kw = dict(tpv_pos=pos, ref_2d=enc.cross_view_ref_points[None], spatial_shapes=ss, level_start_index=lsi,
              reference_points_cams=uvs, tpv_masks=masks, tpv_size=enc.tpv_size, tpv_vis=vises,
              tpv_levels=(enc.tpv_spatial_shapes, enc.tpv_level_start))
    return planes, pos, feat, kw


@gpu
def test_tpv_layer_training_matches_fp64_oracle():
    """One TPVFormerLayer in train() at dropout 0 through its training routine (forward_rows_train: the fused cores with their
    backward kernels, train_linear, nn.LayerNorm) against fp64 autograd of oracle.lifting.tpv_layer_ref: the layer's
    outputs, every parameter's gradient and the gradients of the input planes, positional embeddings and image features,
    at the module tests' bars."""
    dev = _dev()
    from oracle import lifting as ol
    enc, feats, metas = _small_encoder(dev, 1, seed=23)
    layer = enc.layers[0]
    g = torch.Generator().manual_seed(24)
    planes, pos, feat, kw = _layer_inputs(enc, feats, metas, g)
    outs = layer(planes, feat, feat, **kw)
    gouts = [torch.randn(o.shape, generator=g) for o in outs]
    sum((o * go.to(dev)).sum() for o, go in zip(outs, gouts)).backward()
    p64 = _leaf64(layer, 'l.')
    planes64, pos64 = ([t.detach().cpu().double().requires_grad_(True) for t in ts] for ts in (planes, pos))
    f64 = feat.detach().cpu().double().requires_grad_(True)
    shapes = [tuple(s) for s in kw['spatial_shapes'].tolist()]
    ocfg = dict(num_heads=layer.attentions[0].num_heads, num_points_self=layer.attentions[0].num_points, num_cams=6)
    ref = ol.tpv_layer_ref(p64, 'l.', planes64, pos64, f64, shapes, kw['ref_2d'].cpu().double(),
                           [uv.cpu().double() for uv in kw['reference_points_cams']], [m.cpu().bool() for m in kw['tpv_masks']],
                           enc.tpv_size, ocfg)
    for i, (o, r) in enumerate(zip(outs, ref)):
        err = (o.detach().cpu().double() - r.detach()).abs().max().item()
        print('plane %d output max abs err %.2e' % (i, err))
        assert err < 1e-4, i
    sum((r * go.double()).sum() for r, go in zip(ref, gouts)).backward()
    _assert_grads_match(layer, p64, 'l.', _tol)
    for name, got, want, tol in [('plane %d' % i, a, b, 1e-3) for i, (a, b) in enumerate(zip(planes, planes64))] + \
            [('pos %d' % i, a, b, 1e-3) for i, (a, b) in enumerate(zip(pos, pos64))] + [('image features', feat, f64, 2e-4)]:
        e = (got.grad.cpu().double() - want.grad).abs().max().item() / want.grad.abs().max().item()
        print('%s grad %.2e of max-abs' % (name, e))
        assert e < tol, name


@gpu
def test_training_forward_takes_the_row_routine(monkeypatch):
    """A training forward through TPVFormerEncoder.forward runs forward_rows_train once per layer and never the MSDA op; a
    layer called with a key_padding_mask (all False) runs its op-order loop, the attention modules' reference formulation,
    and computes what the routine computes."""
    dev = _dev()
    from selfocc_b200 import ops
    from selfocc_b200.encoder import TPVFormerLayer
    enc, feats, metas = _small_encoder(dev, 2, seed=25)
    rows, msda = TPVFormerLayer.forward_rows_train, ops.MultiScaleDeformableAttnFunction
    calls = dict(rows=[], msda=0)

    def rows_spy(layer, *a, **k):
        calls['rows'].append(layer)
        return rows(layer, *a, **k)

    class MsdaSpy:
        @staticmethod
        def apply(*a):
            calls['msda'] += 1
            return msda.apply(*a)

    monkeypatch.setattr(TPVFormerLayer, 'forward_rows_train', rows_spy)
    monkeypatch.setattr(ops, 'MultiScaleDeformableAttnFunction', MsdaSpy)
    H, W, Z = enc.tpv_size
    g = torch.Generator().manual_seed(26)
    rep = [torch.randn(1, n, 96, generator=g).to(dev).requires_grad_(True) for n in (H * W, Z * H, W * Z)]
    assert torch.is_grad_enabled() and enc.training
    out = enc(representation=rep, ms_img_feats=feats, metas=metas)['representation']
    sum(o.sum() for o in out).backward()
    assert calls['rows'] == list(enc.layers) and calls['msda'] == 0
    layer = enc.layers[0]
    planes, _, feat, kw = _layer_inputs(enc, feats, metas, g)
    calls['rows'].clear()
    routine = layer(planes, feat, feat, **kw)
    assert calls['rows'] == [layer]
    calls['rows'].clear()
    mask = torch.zeros(1, sum(p.shape[1] for p in planes), dtype=torch.bool, device=dev)
    loop = layer(planes, feat, feat, key_padding_mask=mask, **kw)
    assert calls['rows'] == [] and calls['msda'] == 4        # the self-attention and the three planes' cross-attention
    for a, b in zip(loop, routine):
        assert (a - b).abs().max().item() < 1e-4


# --------------------------------------------------------------------------------------------- full size
def _bench_module():
    spec = importlib.util.spec_from_file_location('bench_train_attn', os.path.join(ROOT, 'scripts', 'bench_train_attn.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@gpu
def test_full_size_cores_match_the_reference_contract_composition():
    """One layer's attention at configs[4] sizes (TPV 257 x 257 x 25; 6 cameras x 4 FPN levels of 768 x 1600), fused Functions
    vs the reference-contract composition (rebatch + mmcv-contract op), both fp32.  Outputs, grad_value and grad_logits are
    continuous in the sampling locations and agree within 1e-4 of their largest entry.  The two compositions round the
    locations differently (fmaf with 1/W against a division), so at these sizes a few hundred of the millions of samples
    sit on the other side of a pixel face, where the location gradient jumps: grad_offsets must agree within 1e-3 of its
    largest entry on all but 0.1 % of its entries."""
    dev = _dev()
    b = _bench_module()
    inp = b.make_inputs(dev)
    cores = [('self', inp['self'], b.self_fused, b.self_reference)] + \
            [('cross_%d' % i, t, b.cross_fused, b.cross_reference) for i, t in enumerate(inp['cross'])]
    for name, t, fa, fb in cores:
        ra, rb = fa(t), fb(t)
        d = b.diffs(ra, rb)
        print(name, d)
        for k in ('out', 'grad_value', 'grad_logits'):
            assert d[k]['max_rel'] < 1e-4, (name, k)
        off = (ra[2] - rb[2]).abs() > 1e-3 * rb[2].abs().max()
        print('%s: grad_offsets entries beyond 1e-3 of max-abs: %d of %d' % (name, int(off.sum()), off.numel()))
        assert off.float().mean().item() < 1e-3, name
        del ra, rb
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- no host sync
@gpu
def test_tpv_layer_training_step_runs_without_host_sync():
    """A whole TPVFormerLayer in train() -- self-attention, the three planes' image cross-attention, norms, FFN -- forward and
    backward with every input already on the device: torch's sync debug mode raises on any synchronising call."""
    dev = _dev()
    from selfocc_b200 import configs
    from selfocc_b200.registry import build_head
    import selfocc_b200.segmentor  # noqa: F401
    torch.manual_seed(0)
    margs, rng = synth.small_mapping(8, 4, rng=20.0, z0=-2.0, z1=4.0)
    cfg = configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=6, num_layers=1, num_points_cross=(6, 6, 4),
                                  num_points_self=4, num_samples=48, ray_number=(9, 16), ray_img_size=(90, 160))
    model = build_head(cfg)
    model.encoder.init_weights()
    model.to(dev).train()
    enc = model.encoder
    l2i, _ = synth.camera_rig(synth.NUSC_YAWS, f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    metas = [dict(lidar2img=list(l2i), img_shape=(90, 160))]
    feats = [torch.randn(1, 6, 96, h, w, device=dev) for h, w in [(12, 20), (6, 10), (3, 5), (2, 3)]]
    feat, ss, lsi = enc.flatten_features(feats)
    feat = feat.detach().requires_grad_(True)                  # the layer's inputs are leaves: two passes share them
    uvs, masks, vises = enc.project_reference_points(metas, dev)
    pos = [p[None].detach() for p in enc._tpv_pos()]
    planes = [p.detach().clone().requires_grad_(True) for p in model.lifter(ms_img_feats=feats)['representation']]
    layer = enc.layers[0]
    kw = dict(tpv_pos=pos, ref_2d=enc.cross_view_ref_points[None], spatial_shapes=ss, level_start_index=lsi,
              reference_points_cams=uvs, tpv_masks=masks, tpv_size=enc.tpv_size, tpv_vis=vises,
              tpv_levels=(enc.tpv_spatial_shapes, enc.tpv_level_start))
    out = layer(planes, feat, feat, **kw)                       # warm-up: library load, weight splits, cuBLAS handles
    sum(o.sum() for o in out).backward()
    torch.cuda.synchronize()
    model.zero_grad(set_to_none=True)
    torch.cuda.set_sync_debug_mode('error')
    try:
        out = layer(planes, feat, feat, **kw)
        sum(o.sum() for o in out).backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    for n, p in layer.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
