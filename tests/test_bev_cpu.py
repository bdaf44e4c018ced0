"""CPU: the BEV-only model (config/nuscenes/nuscenes_occ_bev.py) -- oracle against the reference's own outputs
(tests/golden/reference_golden_bev.npz, make_golden_bev.py), module construction from the shipped config, the C entry
points' argument checks, and the sharding entry points' refusal."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bev as ob
from oracle.mapping import GridMeterMappingRef
from oracle.render import C0, field_query_ref
from selfocc_b200.registry import MODELS, build_head
import selfocc_b200.segmentor  # noqa: F401  (registers everything)

HERE = os.path.dirname(os.path.abspath(__file__))
CFG_NAME = 'nuscenes/nuscenes_occ_bev.py'


@pytest.fixture(scope='module')
def gb():
    return np.load(os.path.join(HERE, 'golden', 'reference_golden_bev.npz'))


@pytest.fixture(scope='module')
def cfg():
    return json.load(open(os.path.join(HERE, 'golden', 'reference_model_cfgs_bev.json')))[CFG_NAME]


def _t(a):
    return torch.from_numpy(np.asarray(a))


def test_oracle_tables_and_features_equal_the_reference(gb, cfg):
    pe = cfg['encoder']['positional_encoding']
    for name in ('ship', 'small'):
        m = GridMeterMappingRef(**json.loads(str(gb[name + '_margs'])))
        s = int(gb[name + '_stride'])
        assert torch.equal(ob.bev_pos_features(m, pe['num_freqs'], pe['tot_range'])[::s], _t(gb[name + '_freq_feat']))
        ref_3d, ref_2d = ob.bev_ref_tables(m, cfg['encoder']['num_points_cross'])
        assert torch.equal(ref_3d[:, ::s], _t(gb[name + '_ref_3d']))
        assert torch.equal(ref_2d.flatten(0, 1)[::s], _t(gb[name + '_ref_2d']))


def test_encoder_tables_equal_the_reference(gb, cfg):
    """BEVFormerEncoder built from the shipped config holds the reference's freq_feat / ref_3d / ref_2d bit for bit."""
    e = dict(cfg['encoder'])
    for name in ('ship', 'small'):
        e['mapping_args'] = json.loads(str(gb[name + '_margs']))
        enc = build_head(e)
        s = int(gb[name + '_stride'])
        assert enc.bev_size == list(gb[name + '_bev_size'])
        assert torch.equal(enc.positional_encoding.freq_feat[::s], _t(gb[name + '_freq_feat']))
        assert torch.equal(enc.ref_3d[:, ::s], _t(gb[name + '_ref_3d']))
        assert torch.equal(enc.ref_2d.flatten(0, 1)[::s], _t(gb[name + '_ref_2d']))


@pytest.mark.parametrize('case', ['a', 'b'])
def test_oracle_decode_and_field_query_equal_the_reference(gb, case):
    C_, cd, H, W, Z = [int(v) for v in gb[case + '_dims']]
    m = GridMeterMappingRef(**json.loads(str(gb[case + '_margs'])))
    T = lambda k: _t(gb[case + '_' + k])
    vol = ob.bev_decode_ref(T('bev')[0], (H, W, Z), T('w1'), T('b1'), T('w2'), T('b2'))
    ref_vol = T('vol')[0]
    assert vol.shape == ref_vol.shape == (1 + cd, H, W, Z)
    assert torch.allclose(vol, ref_vol, atol=1e-6, rtol=0)
    h, _ = field_query_ref(vol, m, T('x'), with_grad=False)
    assert torch.allclose(F.softplus(h[:, :1]), T('sigma'), atol=1e-6, rtol=0)
    assert torch.allclose(F.softplus(h[:, :1]), T('sigma_geo'), atol=1e-6, rtol=0)
    if cd:
        assert torch.allclose(torch.relu(C0 * h[:, 1:4] + 0.5), T('rgb'), atol=1e-6, rtol=0)


def test_hot_path_builds_from_the_shipped_config(gb, cfg):
    for name in ('BEVQueryLifter', 'BEVFormerEncoder', 'BEVFormerLayer', 'BEVPositionalEncoding', 'MultiScaleDeformableAttention'):
        assert name in MODELS
    model = build_head(dict(type='TPVHotPath', **cfg))
    keys = set(model.state_dict().keys())
    assert sorted(k[len('lifter.'):] for k in keys if k.startswith('lifter.')) == list(gb['lifter_keys'])
    for k in ('lifter.bev', 'encoder.level_embeds', 'encoder.cams_embeds', 'encoder.positional_encoding.position_layer.weight',
              'encoder.layers.0.attentions.0.sampling_offsets.weight', 'encoder.layers.0.attentions.0.attention_weights.bias',
              'encoder.layers.0.attentions.0.value_proj.weight', 'encoder.layers.0.attentions.0.output_proj.bias',
              'encoder.layers.3.attentions.1.deformable_attention.sampling_offsets.weight',
              'encoder.layers.3.attentions.1.deformable_attention.value_proj.bias', 'encoder.layers.3.attentions.1.output_proj.weight',
              'encoder.layers.0.ffns.0.layers.0.0.weight', 'encoder.layers.0.ffns.0.layers.1.bias', 'encoder.layers.2.norms.2.weight',
              'head.model.field.density_net.1.weight', 'head.model.field.density_net.3.bias', 'head.model.field.deviation_network.variance'):
        assert k in keys, k
    assert not any('ref_3d' in k or 'ref_2d' in k or 'freq_feat' in k for k in keys)   # persistent=False, as the reference
    H, W = model.encoder.bev_size
    Z = model.head.z_size
    assert (H, W, Z) == (257, 257, 25)
    assert model.lifter.bev.shape == (1, H * W, 96) and tuple(gb['lifter_rep_shape']) == (1, 12, 8)
    assert model.encoder.ref_3d.shape == (8, H * W, 3)
    f = model.head.model.field
    assert not f.tpv and f.density_net[3].weight.shape == (Z * 25, 96) and f.desc.n_feat == 24
    sa = model.encoder.layers[0].attentions[0]
    assert (sa.num_heads, sa.num_levels, sa.num_points) == (6, 1, 12)
    assert torch.count_nonzero(sa.sampling_offsets.weight) == 0 and torch.count_nonzero(sa.attention_weights.weight) == 0
    b = sa.sampling_offsets.bias.view(6, 1, 12, 2)
    assert torch.equal(b[0, 0, :, 0], torch.arange(1., 13.))                 # mmcv init: point i scaled by i + 1
    th = torch.arange(6, dtype=torch.float32) * (2.0 * torch.pi / 6)
    ring = torch.stack([th.cos(), th.sin()], -1)
    assert torch.equal(b[:, 0, 0], ring / ring.abs().max(-1, keepdim=True)[0])     # unit ring over the heads
    ca = model.encoder.layers[0].attentions[1].deformable_attention
    assert (ca.num_levels, ca.num_points) == (4, 8)
    # checkpoints of the field keep loading under the existing suffix lookup
    sd = {'head.some.other.path.density_net.3.weight': torch.zeros(Z * 25, 96)}
    missing = model.load_state_dict(sd, strict=False).missing_keys
    assert 'head.model.field.density_net.3.weight' not in missing


def test_bev_entry_points_reject_bad_arguments_without_a_gpu():
    from selfocc_b200 import _lib, build
    build.build()
    lib = _lib.load()
    N, one = None, C.c_void_p(16)
    d = _lib.VolumeDesc()
    d.H, d.W, d.Z, d.zpitch, d.n_feat, d.feat_pitch = 5, 7, 25, 32, 24, 24
    for i in range(3):
        d.axis[i].range0, d.axis[i].size0 = 10.0, 4.0
    assert lib.so_bev_decode(N, 96, one, one, one, one, C.byref(d), one, one, N) == -1
    assert lib.so_bev_decode(one, 96, one, one, one, one, C.byref(d), one, N, N) == -1       # features without vol_feat
    assert lib.so_bev_decode(one, 128, one, one, one, one, C.byref(d), one, one, N) == -2     # C other than 96
    wide = _lib.VolumeDesc()
    C.pointer(wide)[0] = d
    wide.Z, wide.zpitch, wide.n_feat, wide.feat_pitch = 90, 96, 24, 24                        # Z * Cf = 2250 > 2048
    assert lib.so_bev_decode(one, 96, one, one, one, one, C.byref(wide), one, one, N) == -2
    assert lib.so_bev_decode(C.c_void_p(20), 96, one, one, one, one, C.byref(d), one, one, N) == -1   # misaligned bev
    bad = _lib.VolumeDesc()
    C.pointer(bad)[0] = d
    bad.zpitch = 8                                                                            # zpitch < Z
    assert lib.so_bev_decode(one, 96, one, one, one, one, C.byref(bad), one, one, N) == -1
    assert lib.so_bev_decode_bwd_gather(N, N, C.byref(d), 0, 1, N, N) == -1
    assert lib.so_bev_decode_bwd_gather(N, N, C.byref(d), 30, 6, one, N) == -1               # rows past H * W
    assert lib.so_bev_decode_bwd_gather(N, N, C.byref(d), 35, 0, one, N) == 0                # nothing to gather
    assert lib.so_bev_decode_bwd_features(N, 4, one, N) == -1 and lib.so_bev_decode_bwd_features(one, 0, one, N) == 0
    assert lib.so_bev_decode_bwd_hidden(one, N, 4, N) == -1 and lib.so_bev_decode_bwd_hidden(one, one, -1, N) == -1


def test_sharding_entry_points_refuse_a_bev_model(cfg):
    from selfocc_b200 import dist
    c = dict(cfg)
    margs = dict(nonlinear_mode='linear', h_size=[3, 0], h_range=[6.0, 0], h_half=False, w_size=[3, 0], w_range=[6.0, 0],
                 w_half=False, d_size=[2, 0], d_range=[-1.0, 2.0, 2.0])
    c['lifter'] = dict(c['lifter'], bev_h=7, bev_w=7)
    c['encoder'] = dict(c['encoder'], mapping_args=margs, num_layers=1, transformerlayers=c['encoder']['transformerlayers'][:1])
    c['head'] = dict(c['head'], mapping_args=margs)
    model = build_head(dict(type='TPVHotPath', **c))
    with pytest.raises(NotImplementedError, match='ShardedLifter'):
        dist.ShardedLifter(model.encoder)
    with pytest.raises(NotImplementedError, match='ShardedLifter'):
        dist.GraphedFrame(model, None, None)
    with pytest.raises(NotImplementedError, match='decode_sharded'):
        dist.decode_sharded(model.head, model.lifter.bev)
    model.encoder.query_shard = (0, 2)
    with pytest.raises(NotImplementedError, match='query_shard'):
        model.encoder(model.lifter.bev, ms_img_feats=None, metas=None)
