"""CPU: registry / constructor / state_dict contract of the drop-in modules (no kernel calls)."""
import os
import sys
import torch
import pytest
from selfocc_b200 import synth, configs

ROOT_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from selfocc_b200.registry import MODELS, build_head
import selfocc_b200.segmentor  # noqa: F401  (registers everything)


def _small_cfg(**kw):
    margs, rng = synth.small_mapping(6, 3)
    return configs.hot_path_config(mapping_args=margs, pc_range=rng, num_cams=3, num_layers=2, num_points_cross=(5, 5, 3),
                                   num_points_self=4, num_samples=32, ray_number=(6, 10), ray_img_size=(90, 160), **kw)


def test_registry_builds_reference_style_config():
    model = build_head(_small_cfg())
    for name in ('TPVQueryLifter', 'TPVFormerEncoder', 'TPVFormerLayer', 'TPVPositionalEncoding', 'CrossViewHybridAttention',
                 'TPVCrossAttention', 'BEVCrossAttention', 'BEVDeformableAttention', 'NeuSHead'):
        assert name in MODELS
    keys = set(model.state_dict().keys())
    # checkpoint key names of the reference modules (SURVEY.md section 5: state-dict keys are part of the boundary)
    for k in ('lifter.tpv_hw', 'lifter.tpv_zh', 'lifter.tpv_wz', 'encoder.level_embeds', 'encoder.cams_embeds',
              'encoder.positional_encoding.position_layer_hw.weight',
              'encoder.layers.0.attentions.0.sampling_offsets.weight', 'encoder.layers.0.attentions.0.output_proj.bias',
              'encoder.layers.1.attentions.1.attn_zh.deformable_attention.value_proj.weight',
              'encoder.layers.1.attentions.1.attn_wz.output_proj.weight', 'encoder.layers.0.ffns.0.layers.0.0.weight',
              'encoder.layers.0.ffns.0.layers.1.bias', 'encoder.layers.1.norms.2.weight',
              'head.model.field.density_net.1.weight', 'head.model.field.density_net.3.bias',
              'head.model.field.deviation_network.variance'):
        assert k in keys, k
    # non-persistent buffers (reference registers them with persistent=False)
    assert not any('ref_3d' in k or 'freq_feat' in k or 'cross_view_ref_points' in k for k in keys)
    enc = model.encoder
    assert enc.ref_3d_hw.shape == (3, 13 * 13, 3) and enc.ref_3d_zh.shape == (5, 4 * 13, 3)
    assert enc.cross_view_ref_points.shape == (13 * 13 + 2 * 4 * 13, 3, 4, 2)


def test_tables_match_oracle():
    from oracle.mapping import GridMeterMappingRef
    from oracle import lifting as ol
    margs, rng = synth.small_mapping(6, 3)
    model = build_head(_small_cfg())
    mref = GridMeterMappingRef(**margs)
    for a, b in zip((model.encoder.ref_3d_hw, model.encoder.ref_3d_zh, model.encoder.ref_3d_wz), ol.ref_3d_tables(mref, [5, 5, 3])):
        assert torch.equal(a, b)
    assert torch.equal(model.encoder.cross_view_ref_points, ol.cross_view_ref_points(13, 13, 4, [4, 4, 4]))
    feats = ol.tpv_pos_features(mref, [12] * 3, rng)
    pe = model.encoder.positional_encoding
    for a, b in zip((pe.hw_freq_feat, pe.zh_freq_feat, pe.wz_freq_feat), feats):
        assert torch.equal(a, b)
    pts = (torch.rand(50, 3) - 0.5) * 30
    assert torch.equal(model.encoder.mapping.meter2grid(pts, True), mref.meter2grid(pts, True))


def test_deformable_init_matches_reference_recipe():
    model = build_head(_small_cfg())
    sa = model.encoder.layers[0].attentions[0]
    assert torch.count_nonzero(sa.sampling_offsets.weight) == 0 and torch.count_nonzero(sa.attention_weights.weight) == 0
    b = sa.sampling_offsets.bias.view(6, 3, 4, 2)
    assert torch.allclose(b[0, 0, :, 0], torch.tensor([1., 2., 3., 4.]))      # mmcv MSDA: point i scaled by i+1
    ca = model.encoder.layers[0].attentions[1].attn_hw.deformable_attention
    assert torch.allclose(ca.sampling_offsets.bias.view(6, 4, 3, 2)[0, :, :, 0], torch.ones(4, 3))  # no scaling (:238-239)


def test_fork_only_options_are_rejected():
    cfg = _small_cfg()['head']
    cfg.pop('type')
    from selfocc_b200.head import NeuSHead
    for k, v in (('anneal_aabb', True), ('disp_sampler', True), ('num_samples_importance', 64), ('use_numerical_gradients', True),
                 ('estimate_flow', True), ('beta_hand_tune', True)):
        with pytest.raises(NotImplementedError):
            NeuSHead(**{**cfg, k: v})
    with pytest.raises(NotImplementedError):
        NeuSHead(**{**cfg, 'mapping_args': {**cfg['mapping_args'], 'nonlinear_mode': 'linear_upscale'}})


def test_ray_sampler_grid_equals_table(golden):
    import numpy as np
    from selfocc_b200.head import RaySampler
    rs = RaySampler('fixed', [6, 10], [90, 160])
    assert torch.equal(rs(), torch.from_numpy(golden['rays_fixed_6x10_90x160']))
    np.random.seed(123)
    rc = RaySampler('cellular', [6, 10], [90, 160], ray_upper_crop=8)
    assert torch.allclose(rc(), torch.from_numpy(golden['rays_cell_6x10_90x160']), atol=1e-5)


def test_product_mapping_matches_reference_golden(golden):
    """The product-side GridMeterMapping (construction-time tables, C-ABI axis table) against the reference's own outputs,
    including half axes and outer rings."""
    from selfocc_b200.mapping import GridMeterMapping
    T = lambda a: torch.from_numpy(golden[a])
    ring = GridMeterMapping(nonlinear_mode='linear', h_size=[8, 4], h_range=[10., 20.], h_half=True, w_size=[6, 2],
                            w_range=[12., 8.], w_half=False, d_size=[4, 2], d_range=[-2.0, 2.0, 6.0])
    assert (ring.size_h, ring.size_w, ring.size_d) == (13, 17, 7)
    assert torch.equal(ring.meter2grid(T('map_ring_meter'), True), T('map_ring_m2g'))
    assert torch.equal(ring.grid2meter(T('map_ring_grid')), T('map_ring_g2m'))
    nus = GridMeterMapping(**synth.NUSC_MAPPING)
    assert torch.equal(nus.meter2grid(T('map_nus_meter')), T('map_nus_m2g'))
    assert torch.equal(nus.grid2meter(T('map_nus_grid')), T('map_nus_g2m'))
    d = ring.volume_desc(3)
    assert (d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch) == (13, 17, 7, 8, 3, 4)
    assert d.axis[0].offset == 0.0 and d.axis[1].offset == 8.0 and d.axis[2].start == -2.0 and d.axis[2].size1 == 2.0


def test_modules_build_from_the_reference_config_dicts():
    """Drop-in check at the config boundary: the lifter / encoder / head dicts of EVERY shipped TPV experiment config
    (tests/golden/reference_model_cfgs.json, dumped from the reference's own config files) construct the H100 modules."""
    import json, os
    cfgs = json.load(open(os.path.join(os.path.dirname(__file__), 'golden', 'reference_model_cfgs.json')))
    assert sorted(cfgs) == ['kitti/kitti_novel_depth.py', 'kitti/kitti_occ.py', 'kitti_raw/kitti_raw_depth.py',
                            'nuscenes/nuscenes_depth.py', 'nuscenes/nuscenes_novel_depth.py', 'nuscenes/nuscenes_occ.py']
    for name, c in cfgs.items():
        lifter, enc, head = build_head(c['lifter']), build_head(c['encoder']), build_head(c['head'])
        H, W, Z = enc.tpv_size
        assert lifter.tpv_hw.shape == (1, H * W, 96) and lifter.tpv_zh.shape == (1, Z * H, 96)
        assert (head.bev_size, head.z_size) == ([H, W], Z)
        assert enc.ref_3d_hw.shape == (8, H * W, 3) and enc.ref_3d_zh.shape[0] == 48
        assert head.num_samples == 256 and head.ray_sampler.ray_sample_mode == 'cellular'
        assert head.model.field.desc.n_feat == c['head']['color_dims']
        if c['head'].get('return_second_grad'):
            with pytest.raises(NotImplementedError, match='second_grad'):
                head.forward(representation=None, metas=None)


def test_layer_token_buffer_detection():
    """TPVFormerLayer keeps the three planes as torch.split views of one [1, Q, C] buffer; `_whole` must recognise exactly
    that situation (and nothing else), otherwise the layer falls back to torch.cat like the reference."""
    from selfocc_b200.encoder import _whole
    split = [6, 2, 3]
    buf = torch.randn(1, 11, 4)
    views = torch.split(buf, split, 1)
    assert _whole(views, split) is buf
    assert _whole([v.clone() for v in views], split) is None                     # independent tensors
    assert _whole(torch.split(torch.randn(2, 11, 4), split, 1), split) is None   # batch > 1 is not one contiguous token range
    assert _whole(torch.split(buf, [3, 5, 3], 1), split) is None                 # other split
    assert _whole((views[1], views[0], views[2]), split) is None                 # other order
    wide = torch.randn(1, 11, 8)
    assert _whole(torch.split(wide[..., :4], split, 1), split) is None           # column slice of a wider buffer


def test_modules_register_into_a_real_mmengine_style_registry(tmp_path):
    """Boundary (SURVEY 8b): with mmengine importable the classes must land in mmengine's MODELS registry (the one
    mmseg.models.builder.build_head reads, base_segmentor.py:27-32) and build from the reference's config dicts through it.
    mmengine is not installed here, so a minimal stand-in with the same public surface (Registry.register_module as plain /
    called decorator, .get, .build(cfg) -> cls(**cfg without 'type')) is put on the path in a subprocess."""
    import subprocess
    import textwrap
    pkg = tmp_path / 'mmengine'
    pkg.mkdir()
    (pkg / '__init__.py').write_text('')
    (pkg / 'registry.py').write_text(textwrap.dedent('''
        class Registry:
            def __init__(self, name):
                self.name, self.module_dict = name, {}
            def register_module(self, name=None, force=False, module=None):
                def _reg(cls):
                    key = name or cls.__name__
                    if key in self.module_dict and not force:
                        raise KeyError(key + ' is already registered in ' + self.name)
                    self.module_dict[key] = cls
                    return cls
                return _reg(module) if module is not None else _reg
            def get(self, key):
                return self.module_dict.get(key)
            def build(self, cfg, *args, **kwargs):
                cfg = dict(cfg)
                cls = self.get(cfg.pop('type'))
                if cls is None:
                    raise KeyError('not in the ' + self.name + ' registry')
                return cls(**cfg)
        MODELS = Registry('model')
    '''))
    code = textwrap.dedent('''
        import json, os, sys
        sys.path.insert(0, %r); sys.path.insert(0, %r)
        import mmengine.registry as mr
        import selfocc_b200.segmentor
        from selfocc_b200 import registry
        assert registry.HAVE_MMENGINE and registry.MODELS is mr.MODELS
        names = ['TPVQueryLifter', 'TPVFormerEncoder', 'TPVFormerLayer', 'TPVPositionalEncoding', 'CrossViewHybridAttention',
                 'TPVCrossAttention', 'BEVCrossAttention', 'BEVDeformableAttention', 'NeuSHead']
        missing = [n for n in names if mr.MODELS.get(n) is None]
        assert not missing, missing
        cfgs = json.load(open(os.path.join(%r, 'tests', 'golden', 'reference_model_cfgs.json')))
        m = cfgs['nuscenes/nuscenes_depth.py']
        lifter, encoder, head = (mr.MODELS.build(m[k]) for k in ('lifter', 'encoder', 'head'))     # what build_head does
        assert type(head).__name__ == 'NeuSHead' and len(encoder.layers) == 4
        print('OK', len(mr.MODELS.module_dict))
    ''') % (str(tmp_path), ROOT_DIR, ROOT_DIR)
    r = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and 'OK' in r.stdout, r.stdout + r.stderr


def test_head_checkpoint_key_map():
    """INTEGRATION.md section 1: field parameters stored under another module path (a fork checkpoint) load into
    head.model.field.* -- by unambiguous suffix, or through an explicit {regex: replacement} map."""
    model = build_head(_small_cfg())
    sd = model.state_dict()
    moved = {}
    for k, v in sd.items():
        if k.startswith('head.model.field.density_net.') or k.startswith('head.model.field.deviation_network.'):
            moved[k.replace('head.model.field.', 'head.model.some_fork_field.')] = v + 1.0
        else:
            moved[k] = v
    m2 = build_head(_small_cfg())
    missing, unexpected = m2.load_state_dict(dict(moved), strict=False)
    assert not missing and not unexpected
    for k, v in m2.head.state_dict().items():
        if 'density_net' in k or 'deviation_network' in k:
            assert torch.equal(v, sd['head.' + k] + 1.0)
    # explicit map
    m3 = build_head(_small_cfg())
    m3.head.checkpoint_key_map = {r'^net\.mlp\.': 'model.field.density_net.', r'^net\.var$': 'model.field.deviation_network.variance'}
    alt = {}
    for k, v in sd.items():
        k2 = k.replace('head.model.field.density_net.', 'head.net.mlp.').replace('head.model.field.deviation_network.variance', 'head.net.var')
        alt[k2] = v
    missing, unexpected = m3.load_state_dict(alt, strict=False)
    assert not missing and not unexpected


def test_masked_median_and_metric_assembly_cpu():
    """Host side of the device DepthMetric (selfocc_b200/metric.py): the sort-based masked LOWER median equals
    torch.median(x[mask]) (utils/metric_util.py:331-333), and sums -> metrics is cal_depth_metric's arithmetic."""
    from selfocc_b200.metric import masked_median, metrics_from_sums
    g = torch.Generator().manual_seed(0)
    x = torch.rand(5, 101, generator=g) * 50
    mask = torch.rand(5, 101, generator=g) < 0.6
    mask[3] = False
    mask[3, 7] = True                                              # a single valid element
    mask[4, :] = True
    ref = torch.stack([torch.median(x[i][mask[i]]) for i in range(5)])
    assert torch.equal(masked_median(x, mask), ref)
    gt, pred = torch.rand(3, 40, generator=g) * 60 + 1, torch.rand(3, 40, generator=g) * 60 + 1
    d = gt - pred
    th = torch.maximum(gt / pred, pred / gt)
    sums = torch.stack([(d.abs() / gt).sum(1), (d * d / gt).sum(1), (d * d).sum(1), ((gt.log() - pred.log()) ** 2).sum(1),
                        (th < 1.25).float().sum(1), (th < 1.25 ** 2).float().sum(1), (th < 1.25 ** 3).float().sum(1),
                        torch.full((3,), 40.0)], 1)
    m = metrics_from_sums(sums)
    from oracle.metric import cal_depth_metric_ref
    for i in range(3):
        r = cal_depth_metric_ref(pred[i], gt[i])
        for k in ('abs_rel', 'sq_rel', 'rmse', 'rmse_log', 'a1', 'a2', 'a3'):
            assert torch.allclose(m[k][i], r[k].float(), rtol=1e-5, atol=1e-7), k


def test_ffn_training_path_equals_the_sequential_stack():
    """FFN.forward's autograd path spells the nn.Sequential out (so that its two Linear layers can go through
    encoder.train_linear); on CPU train_linear is nn.Linear, so output and gradients must equal `self.layers(x)` exactly,
    including the dropout draws (same generator state, same order)."""
    import torch
    from selfocc_b200.encoder import FFN, train_linear
    torch.manual_seed(0)
    ffn = FFN(embed_dims=96, feedforward_channels=192, ffn_drop=0.1).train()
    x = torch.randn(2, 37, 96, requires_grad=True)
    torch.manual_seed(5)
    y = ffn(x)
    gx, = torch.autograd.grad(y.sum(), x)
    x2 = x.detach().clone().requires_grad_(True)
    torch.manual_seed(5)
    y_ref = x2 + ffn.layers(x2)
    gx_ref, = torch.autograd.grad(y_ref.sum(), x2)
    assert torch.equal(y, y_ref) and torch.equal(gx, gx_ref)
    lin = torch.nn.Linear(96, 96)
    assert torch.equal(train_linear(lin, x), lin(x))          # CPU tensors: the stock layer
