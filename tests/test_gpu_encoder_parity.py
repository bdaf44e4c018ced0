"""The encoder's inference routine (``TPVFormerLayer.forward_rows``) against the fp64 oracle at the attention geometry of every
shipped config: C = 96, 6 heads x 16 channels, num_points_cross = [48, 48, 8], num_points_self = 12, 4 FPN levels, FFN 192,
4 layers, on 6 cameras (nuScenes-like) and on 1 camera with a half h axis (KITTI-like), both on a non-square H x W x Z grid.

* whole encoder vs ``oracle.lifting.tpv_encoder_ref`` and every layer on its own vs ``tpv_layer_ref`` run on the layer's own
  fp32 input, in both attention-kernel generations, with spies proving which path ran (fused offsets / logits GEMM, the
  fused 3-plane value projection, LayerNorm in the GEMM epilogue, second-generation dispatch conditions);
* the strided attention entry points (``so_tpv_*_attn_forward_strided``) called directly on column slices of wider buffers
  whose other columns are NaN, against fp64 and bit for bit against the contiguous entry points;
* ``forward_rows``' fallback branches (32-channel heads with unfusable offsets / logits; cuBLAS projections with a separate
  LayerNorm) against the oracle;
* (CPU) the strided entry points' argument checks.

Measured on one H100 80GB HBM3 (700 W power limit), max abs error of the fp32 kernels vs the fp64 oracle; the planes are
LayerNorm outputs with |x| max 5.6 (KITTI-like) to 7.8 (nuScenes-like):

  whole encoder, 4 layers       nuScenes-like 2.4e-5 (v1) / 2.3e-5 (v2), KITTI-like 1.9e-5 / 2.0e-5      bar 2e-4
  one layer on its own input    at most 9.9e-6 over both cases, both kernel generations, all 4 layers    bar 5e-5
  fallback layers               C = 96, 3 heads, P = 5: 9.0e-6; C = 128, 8 heads (cuBLAS): 1.3e-6        bar 5e-5
  strided attention cores       at most 1.1e-6 (cross), 5.5e-7 (self)                                    bar 2e-5

The per-layer bar is the attention-core bar of DESIGN section 2 (5e-5): each layer ends in a LayerNorm, so its output has
the scale of the core outputs, and a layer may not be less accurate than one attention core.  The 4-layer bar stays at the
2e-4 of tests/test_gpu_pipeline.py::test_encoder_matches_oracle."""
import ctypes as C

import pytest
import torch

from selfocc_b200 import synth, configs
from selfocc_b200.registry import build_head
import selfocc_b200.segmentor  # noqa: F401  registers the modules

gpu = pytest.mark.gpu

ENCODER_BAR = 2e-4      # whole encoder (4 layers), as tests/test_gpu_pipeline.py::test_encoder_matches_oracle
LAYER_BAR = 5e-5        # one layer on its own fp32 input: the attention-core bar (module docstring)
CORE_BAR = 2e-5         # one attention core (the MSDA forward bar of DESIGN section 2)

NUSC = dict(margs=dict(nonlinear_mode='linear', h_size=[6, 0], h_range=[20.0, 0], h_half=False, w_size=[4, 0], w_range=[16.0, 0],
                       w_half=False, d_size=[5, 0], d_range=[-2.0, 4.0, 4.0]),
            rng=[-20.0, -16.0, -2.0, 20.0, 16.0, 4.0], yaws=synth.NUSC_YAWS, rig=dict(f=126.6, cx=80., cy=45., height=0.5, radius=0.2),
            img=(90, 160), fpn=[(12, 20), (6, 10), (3, 5), (2, 3)])
KITTI = dict(margs=dict(nonlinear_mode='linear', h_size=[6, 0], h_range=[25.6, 0], h_half=True, w_size=[4, 0], w_range=[12.8, 0],
                        w_half=False, d_size=[5, 0], d_range=[-2.0, 4.4, 4.4]),
             rng=[-12.8, 0.0, -2.0, 12.8, 25.6, 4.4], yaws=(0.,), rig=dict(f=180., cx=152., cy=44., height=0.3, radius=0.1),
             img=(88, 304), fpn=[(11, 38), (6, 19), (3, 10), (2, 5)])


def _dev():
    if not torch.cuda.is_available():
        pytest.skip('needs CUDA')
    return torch.device('cuda:0')


def _levels(shapes, dev):
    ss = torch.tensor(shapes, dtype=torch.int64)
    lsi = torch.cat([ss.new_zeros(1), ss.prod(1).cumsum(0)[:-1]])
    return ss.to(dev), lsi.to(dev)


def _split_groups(D):
    """The cross-attention kernels' sample groups per (query, head) (msda.cu: so_tpv_cross_attn_forward_strided)."""
    return 4 if D >= 32 else (2 if D >= 16 else 1)


def _cross_v2(Dh, D):
    return Dh == 16 and D % (4 * _split_groups(D)) == 0


def _self_v2(Dh, P):
    return Dh == 16 and P % 4 == 0


# --------------------------------------------------------------------------------------------- model and oracle set-up
def _model(case, dim=96, num_heads=6, num_layers=4, num_points_cross=(48, 48, 8), num_points_self=12, seed=0):
    """Lifter + encoder of hot_path_config with every parameter away from its trivial value: offsets / logits projections
    N(0, 0.05), every bias shifted by 0.1 N, LayerNorm gamma = 1 + 0.3 N, beta = 0.1 N."""
    torch.manual_seed(seed)
    cfg = configs.hot_path_config(mapping_args=case['margs'], pc_range=case['rng'], dim=dim, num_heads=num_heads,
                                  num_cams=len(case['yaws']), num_layers=num_layers, num_points_cross=num_points_cross,
                                  num_points_self=num_points_self)
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
    ocfg = dict(num_freqs=[12] * 3, tot_range=case['rng'], num_points_cross=list(num_points_cross), num_points_self=num_points_self,
                num_layers=num_layers, num_heads=num_heads, num_cams=len(case['yaws']))
    return lifter.eval(), enc.eval(), ocfg


def _frame(case, dim=96, seed=0):
    g = torch.Generator().manual_seed(seed + 2)
    l2i, _ = synth.camera_rig(case['yaws'], **case['rig'])
    metas = [dict(lidar2img=list(l2i), img_shape=case['img'])]
    feats = [torch.randn(1, len(case['yaws']), dim, h, w, generator=g) for h, w in case['fpn']]
    return metas, feats, torch.tensor(l2i, dtype=torch.float32)


def _promote_oracle_tables(monkeypatch):
    """Run the oracle in fp64 on the fp32 geometry tables (positional features, camera projections, cross-view reference
    points), promoted as tests/test_gpu_pipeline.py does; the camera masks stay the fp32 ones, which are bit-exact with
    so_point_sampling."""
    from oracle import lifting as ol
    pos, ps, cv = ol.tpv_pos_features, ol.point_sampling_ref, ol.cross_view_ref_points
    monkeypatch.setattr(ol, 'tpv_pos_features', lambda *a, **k: [f.double() for f in pos(*a, **k)])
    monkeypatch.setattr(ol, 'point_sampling_ref', lambda r, m, s: tuple(t.double() if t.dtype.is_floating_point else t
                                                                         for t in ps(r, m, s)))
    monkeypatch.setattr(ol, 'cross_view_ref_points', lambda *a: cv(*a).double())


def _record_oracle_samples(monkeypatch, stats):
    """Wrap the oracle's two attention modules to count, from their own masks and recomputed sampling locations, the
    queries visible in 0 / >= 2 cameras and the sampled locations outside [0, 1]."""
    from oracle import lifting as ol
    self_ref, cross_ref = ol.cross_view_self_attn_ref, ol.image_cross_attn_ref

    def outside(loc):
        return int(((loc < 0) | (loc > 1)).any(-1).sum())

    def self_spy(p, pre, query, query_pos, ref_2d, spatial_shapes, num_heads, num_points):
        B, Q, _ = query.shape
        off = ol._lin(p, pre + 'sampling_offsets', query + query_pos).view(B, Q, num_heads, len(spatial_shapes), num_points, 2)
        loc = ol.deform_locations(ref_2d, off, spatial_shapes, per_level_ref=True)
        stats['self_outside'] += outside(loc)
        stats['self_samples'] += loc[..., 0].numel()
        return self_ref(p, pre, query, query_pos, ref_2d, spatial_shapes, num_heads, num_points)

    def cross_spy(p, pre, query, feat, spatial_shapes, ref_cam, mask, num_heads, num_cams):
        B, Q, _ = query.shape
        D = ref_cam.shape[3]
        off = ol._lin(p, pre + 'deformable_attention.sampling_offsets', query).view(B, Q, num_heads, len(spatial_shapes), D, 2)
        vis = mask[:, 0].any(-1)                                                  # [N, Q]: the query is attended in that camera
        for i in range(num_cams):
            loc = ol.deform_locations(ref_cam[i], off, spatial_shapes, per_level_ref=False)[0][vis[i]]
            stats['cross_outside'] += outside(loc)
            stats['cross_samples'] += loc[..., 0].numel()
        n_vis = vis.sum(0)
        stats['blind'] += int((n_vis == 0).sum())
        stats['multi'] += int((n_vis >= 2).sum())
        stats['queries'] += Q
        return cross_ref(p, pre, query, feat, spatial_shapes, ref_cam, mask, num_heads, num_cams)

    monkeypatch.setattr(ol, 'cross_view_self_attn_ref', self_spy)
    monkeypatch.setattr(ol, 'image_cross_attn_ref', cross_spy)


def _oracle_layer_inputs(p, mref, feats64, l2i, img, ocfg):
    """The per-frame operands tpv_encoder_ref hands every layer (tpvformer_encoder.py:192-290), for tpv_layer_ref."""
    from oracle import lifting as ol
    H, W, Z = mref.size_h, mref.size_w, mref.size_d
    tpv_pos = [ol._lin(p, 'positional_encoding.position_layer_' + n, f)[None]
               for n, f in zip(('hw', 'zh', 'wz'), ol.tpv_pos_features(mref, ocfg['num_freqs'], ocfg['tot_range']))]
    feat, shapes = ol.flatten_img_feats(p, feats64)
    ref_cams, masks = [], []
    for r3 in ol.ref_3d_tables(mref, ocfg['num_points_cross']):
        rc, m = ol.point_sampling_ref(r3[None], l2i[None], img)
        ref_cams.append(rc)
        masks.append(m)
    ref_2d = ol.cross_view_ref_points(H, W, Z, [ocfg['num_points_self']] * 3)[None]
    return tpv_pos, feat, shapes, ref_2d, ref_cams, masks


def _max_err(got, ref):
    return [(g.double() - r).abs().max().item() for g, r in zip(got, ref)]


class _Spies:
    """Pass-through spies on the ops forward_rows calls, recording what each call was handed."""

    def __init__(self, monkeypatch):
        from selfocc_b200 import ops
        from selfocc_b200.encoder import TPVFormerLayer
        self.rows, self.self_calls, self.cross_calls, self.gemm = 0, [], [], 0
        self.ln_epilogue, self.ln_separate = [], []        # the gamma of every LayerNorm, by where it ran
        rows, self_rows, cross_rows = TPVFormerLayer.forward_rows, ops.tpv_self_attn_forward_rows, ops.tpv_cross_attn_forward_rows
        lin, ln = ops.linear_3xtf32, ops.layer_norm

        def rows_spy(layer, *a, **k):
            self.rows += 1
            return rows(layer, *a, **k)

        def operands(value, offs, logits, Hd, Dh, L, n):
            return dict(Hd=Hd, Dh=Dh, L=L, n=n, value_ld=value.stride(0), off_ld=offs.stride(0), lg_ld=logits.stride(0),
                        off_w=offs.shape[1], lg_w=logits.shape[1],
                        one_buffer=offs.untyped_storage().data_ptr() == logits.untyped_storage().data_ptr(),
                        lg_at=(logits.data_ptr() - offs.data_ptr()) // 4)

        def self_spy(value, Hd, Dh, ss, lsi, offs, logits, ref, L, P):
            self.self_calls.append(operands(value, offs, logits, Hd, Dh, L, P))
            return self_rows(value, Hd, Dh, ss, lsi, offs, logits, ref, L, P)

        def cross_spy(value, n_cam, Hd, Dh, ss, lsi, offs, logits, uv, vis, L, D):
            self.cross_calls.append(dict(operands(value, offs, logits, Hd, Dh, L, D), cells=value.shape[0]))
            return cross_rows(value, n_cam, Hd, Dh, ss, lsi, offs, logits, uv, vis, L, D)

        def lin_spy(*a, **k):
            self.gemm += 1
            if k.get('ln') is not None:
                self.ln_epilogue.append(k['ln'][0].data_ptr())
            return lin(*a, **k)

        def ln_spy(x, gamma, *a, **k):
            self.ln_separate.append(gamma.data_ptr())
            return ln(x, gamma, *a, **k)

        monkeypatch.setattr(TPVFormerLayer, 'forward_rows', rows_spy)
        monkeypatch.setattr(ops, 'tpv_self_attn_forward_rows', self_spy)
        monkeypatch.setattr(ops, 'tpv_cross_attn_forward_rows', cross_spy)
        monkeypatch.setattr(ops, 'linear_3xtf32', lin_spy)
        monkeypatch.setattr(ops, 'layer_norm', ln_spy)


def _layer_norm_order(enc):
    """The LayerNorm gammas forward_rows applies, in order: norms[0] after the self-attention, norms[1] after each plane's
    cross-attention output projection, norms[2] after the FFN."""
    out = []
    for layer in enc.layers:
        n0, n1, n2 = (n.weight.data_ptr() for n in layer.norms)
        out += [n0, n1, n1, n1, n2]
    return out


def _run_gpu(lifter, enc, feats, metas, dev):
    """Encoder output planes and every layer's (input, output) planes, fp32 on the CPU."""
    seen = []
    hooks = [layer.register_forward_hook(lambda m, a, o: seen.append(([t.detach().cpu().clone() for t in a[0]],
                                                                       [t.detach().cpu().clone() for t in o])))
             for layer in enc.layers]
    try:
        with torch.no_grad():
            fd = [f.to(dev) for f in feats]
            rep = lifter(ms_img_feats=fd)['representation']
            out = enc(representation=rep, ms_img_feats=fd, metas=metas)['representation']
    finally:
        for h in hooks:
            h.remove()
    assert len(seen) == len(enc.layers)
    return [o.cpu() for o in out], seen


def _oracle_case(monkeypatch, case, lifter, enc, ocfg, feats, l2i):
    """fp64 oracle of the whole encoder plus the per-layer operands; also returns the edge-case counts of the oracle's own
    masks and locations."""
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    _promote_oracle_tables(monkeypatch)
    stats = dict.fromkeys(('self_outside', 'self_samples', 'cross_outside', 'cross_samples', 'blind', 'multi', 'queries'), 0)
    _record_oracle_samples(monkeypatch, stats)
    p = {k: v.detach().cpu().double() for k, v in enc.state_dict().items()}
    mref = GridMeterMappingRef(**case['margs'])
    planes = [t.detach().cpu().double() for t in (lifter.tpv_hw, lifter.tpv_zh, lifter.tpv_wz)]
    feats64 = [f.double() for f in feats]
    ref = ol.tpv_encoder_ref(p, mref, planes, feats64, l2i[None], case['img'], ocfg)
    layer_ops = _oracle_layer_inputs(p, mref, feats64, l2i, case['img'], ocfg)
    return p, mref, ref, layer_ops, stats


def _check_against_oracle(tag, out, seen, ref, p, mref, layer_ops, ocfg):
    from oracle import lifting as ol
    tpv_pos, feat, shapes, ref_2d, ref_cams, masks = layer_ops
    errs = _max_err(out, ref)
    print('%s encoder (%d layers): max abs err per plane hw / zh / wz %s  (|x| max %.2f)'
          % (tag, ocfg['num_layers'], ' / '.join('%.2e' % e for e in errs), max(r.abs().max().item() for r in ref)))
    layer_errs = []
    for i, (inp, got) in enumerate(seen):
        lref = ol.tpv_layer_ref(p, 'layers.%d.' % i, [t.double() for t in inp], tpv_pos, feat, shapes, ref_2d, ref_cams, masks,
                                (mref.size_h, mref.size_w, mref.size_d), ocfg)
        layer_errs.append(_max_err(got, lref))
        print('%s layer %d: max abs err per plane %s' % (tag, i, ' / '.join('%.2e' % e for e in layer_errs[-1])))
    for i, e in enumerate(layer_errs):
        assert max(e) < LAYER_BAR, '%s layer %d: %r' % (tag, i, e)
    assert max(errs) < ENCODER_BAR, '%s encoder: %r' % (tag, errs)


# --------------------------------------------------------------------------------------------- 1 + 2: shipped geometry
@gpu
@pytest.mark.parametrize('name', ['nuscenes', 'kitti'])
def test_encoder_and_each_layer_match_oracle_at_shipped_geometry(name, monkeypatch):
    dev = _dev()
    from selfocc_b200 import _lib
    case = dict(nuscenes=NUSC, kitti=KITTI)[name]
    lifter, enc, ocfg = _model(case)
    metas, feats, l2i = _frame(case)
    p, mref, ref, layer_ops, stats = _oracle_case(monkeypatch, case, lifter, enc, ocfg, feats, l2i)
    print('%s: oracle edge cases %r' % (name, stats))
    assert stats['blind'] > 0                                    # queries visible in no camera (output: the residual alone)
    if len(case['yaws']) > 1:
        assert stats['multi'] > 0                                # queries averaged over two or more cameras
    assert stats['cross_outside'] > 0 and stats['self_outside'] > 0   # zero padding on both attentions
    assert (mref.size_h, mref.size_w) != (mref.size_w, mref.size_h) and len({mref.size_h, mref.size_w, mref.size_d}) == 3
    lifter.to(dev)
    enc.to(dev)
    L = ocfg['num_layers']
    for force_v1 in (0, 1):
        spies = _Spies(monkeypatch)
        _lib.load().so_attn_force_v1(force_v1)
        try:
            out, seen = _run_gpu(lifter, enc, feats, metas, dev)
        finally:
            _lib.load().so_attn_force_v1(0)
        _check_against_oracle('%s %s' % (name, 'v1' if force_v1 else 'v2'), out, seen, ref, p, mref, layer_ops, ocfg)
        # the routed path: one forward_rows per layer, one self- and three cross-attention calls per layer
        assert spies.rows == L and len(spies.self_calls) == L and len(spies.cross_calls) == 3 * L
        # every LayerNorm in the epilogue of the GEMM before it, none as a separate launch
        assert spies.ln_epilogue == _layer_norm_order(enc) and spies.ln_separate == []
        for c in spies.self_calls + spies.cross_calls:
            width = c['Hd'] * c['L'] * c['n']
            # offsets and logits: adjacent column slices of one GEMM output of row pitch 3 Hd L n
            assert c['one_buffer'] and c['lg_at'] == 2 * width and c['off_w'] == 2 * width and c['lg_w'] == width
            assert c['off_ld'] == c['lg_ld'] == 3 * width
            assert (c['Hd'], c['Dh']) == (6, 16)
        for c in spies.self_calls:
            assert c['n'] == 12 and c['L'] == 3 and c['value_ld'] == 96 and _self_v2(c['Dh'], c['n'])
        for c in spies.cross_calls:
            # the three planes' value projections are one GEMM: each plane's value is a column slice of pitch 3 C
            assert c['value_ld'] == 3 * 96 and c['L'] == 4
            assert _cross_v2(c['Dh'], c['n']) and c['cells'] < 2 ** 31
        assert {c['n'] for c in spies.cross_calls} == {8, 48}


# --------------------------------------------------------------------------------------------- 4: fallback branches
@gpu
@pytest.mark.parametrize('dim,heads,p_self', [(96, 3, 5), (128, 8, 12)])
def test_forward_rows_fallback_branches_match_oracle(dim, heads, p_self, monkeypatch):
    """(96, 3 heads, P_self = 5): 32-channel heads, first-generation kernels only; the self-attention's attention-weights
    width 3 x 3 x 5 = 45 is odd, so its offsets and logits take two projections.  (128, 8 heads): K = 128 is not a GEMM shape,
    so every projection runs on cuBLAS, each plane projects its own value, and every LayerNorm is a separate so_layer_norm."""
    dev = _dev()
    lifter, enc, ocfg = _model(NUSC, dim=dim, num_heads=heads, num_layers=1, num_points_self=p_self)
    metas, feats, l2i = _frame(NUSC, dim=dim)
    p, mref, ref, layer_ops, stats = _oracle_case(monkeypatch, NUSC, lifter, enc, ocfg, feats, l2i)
    assert stats['blind'] > 0 and stats['multi'] > 0 and stats['cross_outside'] > 0 and stats['self_outside'] > 0
    lifter.to(dev)
    enc.to(dev)
    spies = _Spies(monkeypatch)
    out, seen = _run_gpu(lifter, enc, feats, metas, dev)
    _check_against_oracle('fallback C=%d Hd=%d P=%d' % (dim, heads, p_self), out, seen, ref, p, mref, layer_ops, ocfg)
    assert spies.rows == 1 and len(spies.self_calls) == 1 and len(spies.cross_calls) == 3
    s = spies.self_calls[0]
    assert not s['one_buffer'] and s['lg_ld'] == s['lg_w'] == heads * 3 * p_self
    for c in spies.cross_calls:
        assert c['Dh'] == dim // heads
    if dim == 96:
        assert s['Dh'] == 32 and not _self_v2(s['Dh'], s['n'])
        assert all(not _cross_v2(c['Dh'], c['n']) for c in spies.cross_calls)
        assert spies.ln_epilogue == _layer_norm_order(enc) and spies.ln_separate == []
    else:
        assert spies.gemm == 0 and spies.ln_epilogue == [] and spies.ln_separate == _layer_norm_order(enc)
        for c in spies.self_calls + spies.cross_calls:
            assert not c['one_buffer'] and c['value_ld'] == dim


# --------------------------------------------------------------------------------------------- 3: strided entry points
def _nan_buffer_slices(rows, widths, dev, front=2):
    """One [rows, ld] NaN buffer holding adjacent column slices of the given widths, starting at an even column `front`
    (float2 offsets need 8-byte alignment) with NaN columns before and after them; ld is even."""
    total = sum(widths)
    ld = front + total + 2 + (total & 1)
    buf = torch.full((rows, ld), float('nan'), device=dev)
    views, c0 = [], front
    for w in widths:
        views.append(buf[:, c0:c0 + w])
        c0 += w
    return buf, views


def _value_slice(rows, Hd, Dh, g, dev):
    """The middle column slice of a [rows, 3 Hd Dh] NaN buffer, filled with N(0, 1)."""
    buf = torch.full((rows, 3 * Hd * Dh), float('nan'), device=dev)
    v = buf[:, Hd * Dh:2 * Hd * Dh]
    v.copy_(torch.randn(rows, Hd * Dh, generator=g))
    return buf, v


@gpu
@pytest.mark.parametrize('n_cam', [1, 6])
@pytest.mark.parametrize('Dh', [16, 32])
@pytest.mark.parametrize('D', [6, 8, 16, 20, 32, 48])
def test_strided_cross_attention_matches_fp64_and_contiguous_form(D, Dh, n_cam):
    dev = _dev()
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    from selfocc_b200 import ops
    g = torch.Generator().manual_seed(100 * D + Dh + n_cam)
    Hd, shapes = 96 // Dh, [(12, 20), (6, 10), (3, 5), (2, 3)]
    L, Nv = len(shapes), sum(h * w for h, w in shapes)
    margs, _ = synth.small_mapping(10, 4, rng=30.0)
    r3 = ol.ref_3d_tables(GridMeterMappingRef(**margs), [D, D, D])[0]            # hw plane: Q = 441 pillars of D points
    l2i, _ = synth.camera_rig(synth.NUSC_YAWS[:n_cam], f=126.6, cx=80., cy=45., height=0.5, radius=0.2)
    uv_full, mask = ol.point_sampling_ref(r3[None], torch.tensor(l2i, dtype=torch.float32)[None], (90, 160))
    uv_full, vis_full = uv_full[:, 0].contiguous(), mask[:, 0].any(-1).to(torch.uint8)
    b, c = 41, 300                                                                # the rows of one shard of the plane
    vis_full[:, b + 3] = 0                                                        # a query visible in no camera
    uv, vis = uv_full[:, b:b + c].contiguous(), vis_full[:, b:b + c].contiguous()
    n_vis = vis.long().sum(0)
    assert (n_vis == 0).any() and (n_vis > 0).any() and (n_cam == 1 or (n_vis >= 2).any())
    vbuf, value = _value_slice(n_cam * Nv, Hd, Dh, g, dev)
    obuf, (offs, logits) = _nan_buffer_slices(c, [Hd * L * D * 2, Hd * L * D], dev)
    offs.copy_(3.0 * torch.randn(c, Hd * L * D * 2, generator=g))
    logits.copy_(torch.randn(c, Hd * L * D, generator=g))
    ss, lsi = _levels(shapes, dev)
    got = ops.tpv_cross_attn_forward_rows(value, n_cam, Hd, Dh, ss, lsi, offs, logits, uv.to(dev), vis.to(dev), L, D)
    contiguous = ops.tpv_cross_attn_forward(value.contiguous().view(n_cam, Nv, Hd, Dh), ss, lsi,
                                            offs.contiguous().view(c, Hd, L, D, 2), logits.contiguous().view(c, Hd, L, D),
                                            uv.to(dev), vis.to(dev))
    assert torch.equal(got, contiguous)
    # fp64: per camera MSDA at ref + offset / (w_l, h_l), averaged over the cameras that see the query
    v64 = value.cpu().double().view(n_cam, Nv, Hd, Dh)
    o64 = offs.cpu().double().view(1, c, Hd, L, D, 2)
    loc = ol.deform_locations(uv.double(), o64, shapes, per_level_ref=False)                    # [N, c, Hd, L, D, 2]
    sampled = loc[vis.bool()]
    assert ((sampled < 0) | (sampled > 1)).any() and ((sampled > 0) & (sampled < 1)).all(-1).any()
    aw = logits.cpu().double().view(c, Hd, L * D).softmax(-1).view(1, c, Hd, L, D).expand(n_cam, -1, -1, -1, -1)
    per_cam = ol.msda_ref(v64, shapes, loc, aw)
    w = vis.double()[..., None]
    ref = (per_cam * w).sum(0) / w.sum(0).clamp(min=1)
    err = (got.cpu().double() - ref).abs().max().item()
    print('strided cross D=%d Dh=%d N=%d (%s): max abs err %.2e' % (D, Dh, n_cam, 'v2' if _cross_v2(Dh, D) else 'v1', err))
    assert torch.isfinite(got).all() and err < CORE_BAR
    assert torch.equal(got[n_vis.to(dev) == 0], torch.zeros_like(got[n_vis.to(dev) == 0]))


@gpu
@pytest.mark.parametrize('Dh', [16, 32])
@pytest.mark.parametrize('P', [5, 12])
def test_strided_self_attention_matches_fp64_and_contiguous_form(P, Dh):
    dev = _dev()
    from oracle import lifting as ol
    from selfocc_b200 import ops
    g = torch.Generator().manual_seed(10 * P + Dh)
    Hd = 96 // Dh
    H, W, Z = 9, 7, 4
    shapes = [(H, W), (Z, H), (W, Z)]
    L, Nv = 3, H * W + Z * H + W * Z
    ref_full = ol.cross_view_ref_points(H, W, Z, [P, P, P])                        # [Nv, 3, P, 2]
    b, c = 20, 80
    ref = ref_full[b:b + c].contiguous()
    vbuf, value = _value_slice(Nv, Hd, Dh, g, dev)
    obuf, (offs, logits) = _nan_buffer_slices(c, [Hd * L * P * 2, Hd * L * P], dev)
    offs.copy_(3.0 * torch.randn(c, Hd * L * P * 2, generator=g))
    logits.copy_(torch.randn(c, Hd * L * P, generator=g))
    ss, lsi = _levels(shapes, dev)
    got = ops.tpv_self_attn_forward_rows(value, Hd, Dh, ss, lsi, offs, logits, ref.to(dev), L, P)
    contiguous = ops.tpv_self_attn_forward(value.contiguous().view(Nv, Hd, Dh), ss, lsi, offs.contiguous().view(c, Hd, L, P, 2),
                                           logits.contiguous().view(c, Hd, L, P), ref.to(dev))
    assert torch.equal(got, contiguous)
    loc = ol.deform_locations(ref.double()[None], offs.cpu().double().view(1, c, Hd, L, P, 2), shapes, per_level_ref=True)
    assert ((loc < 0) | (loc > 1)).any()
    aw = logits.cpu().double().view(1, c, Hd, L * P).softmax(-1).view(1, c, Hd, L, P)
    out_ref = ol.msda_ref(value.cpu().double().view(1, Nv, Hd, Dh), shapes, loc, aw)[0]
    err = (got.cpu().double() - out_ref).abs().max().item()
    print('strided self P=%d Dh=%d (%s): max abs err %.2e' % (P, Dh, 'v2' if _self_v2(Dh, P) else 'v1', err))
    assert torch.isfinite(got).all() and err < CORE_BAR


# --------------------------------------------------------------------------------------------- 5: CPU argument checks
_BAD_STRIDED = ['value_ld_below_row', 'value_ld_not_float4', 'offsets_ld_below_row', 'logits_ld_below_row',
                'value_misaligned', 'offsets_ld_odd']


@pytest.mark.parametrize('bad', [None] + _BAD_STRIDED)
@pytest.mark.parametrize('entry', ['cross', 'self'])
def test_strided_entry_points_reject_bad_pitches_without_a_gpu(entry, bad):
    """Each bad pitch or pointer returns SO_ERR_INVALID_ARG (-1) before any CUDA call.  The control (bad = None) is the same
    call with valid pitches and L = 9 > 8 levels: it passes every argument check and returns SO_ERR_UNSUPPORTED (-2), still
    without a launch, so each -1 comes from the one operand that was made bad."""
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    Hd, Dh, L, n = 6, 16, 9, 8
    a = dict(value=C.c_void_p(16), value_ld=Hd * Dh, offsets_ld=Hd * L * n * 2, logits_ld=Hd * L * n)
    if bad == 'value_ld_below_row':
        a['value_ld'] = Hd * Dh - 4
    elif bad == 'value_ld_not_float4':
        a['value_ld'] = Hd * Dh + 2
    elif bad == 'offsets_ld_below_row':
        a['offsets_ld'] = Hd * L * n * 2 - 2
    elif bad == 'logits_ld_below_row':
        a['logits_ld'] = Hd * L * n - 1
    elif bad == 'value_misaligned':
        a['value'] = C.c_void_p(24)
    elif bad == 'offsets_ld_odd':
        a['offsets_ld'] = Hd * L * n * 2 + 1
    one = C.c_void_p(16)   # non-null, 16-byte aligned dummy (never dereferenced on these paths)
    if entry == 'cross':
        code = lib.so_tpv_cross_attn_forward_strided(a['value'], one, one, one, one, one, one, one, None, 6, 100, Hd, Dh, 10, L, n,
                                                     a['value_ld'], a['offsets_ld'], a['logits_ld'], None)
    else:
        code = lib.so_tpv_self_attn_forward_strided(a['value'], one, one, one, one, one, one, 100, Hd, Dh, 10, L, n,
                                                    a['value_ld'], a['offsets_ld'], a['logits_ld'], None)
    assert code == (-2 if bad is None else -1)
