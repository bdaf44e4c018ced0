"""Golden fixtures of the BEV-only model (config/nuscenes/nuscenes_occ_bev.py), from the reference's own modules.

    python tests/golden/make_golden_bev.py <path to a huang-yh/SelfOcc checkout>

Runs these reference files UNMODIFIED, with the stand-in technique of make_golden.py --bevnerf (minimal stand-ins for the
mmengine / mmseg / mmcv names they import, a synthetic package tree so their relative imports resolve to the reference's
own files loaded by path):
  * model/lifter/bev_query_lifter.py          BEVQueryLifter
  * model/encoder/bevformer/bevformer_pos_embed.py   BEVPositionalEncoding
  * model/encoder/bevformer/bevformer_encoder.py     BEVFormerEncoder, construction only (build_transformer_layer is stubbed,
                                                     build_positional_encoding builds the real BEVPositionalEncoding)
  * model/head/nerfacc_head/bev_nerf.py      BEVNeRF, tpv=False
Writes tests/golden/reference_golden_bev.npz and tests/golden/reference_model_cfgs_bev.json (the lifter / encoder / head
config dicts of nuscenes_occ_bev.py).
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
REF = sys.argv[1] if len(sys.argv) > 1 else None
CFG = 'nuscenes/nuscenes_occ_bev.py'


class _Registry:
    def register_module(self, *a, **k):
        return lambda cls: cls


class _BaseModule(nn.Module):
    def __init__(self, init_cfg=None, **kwargs):
        super().__init__()


class _StubLayer(nn.Module):
    pre_norm = False


def _install_stand_ins(built):
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__path__ = []
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m
    mod('mmengine', model=None)
    mod('mmengine.model', BaseModule=_BaseModule, ModuleList=nn.ModuleList)
    mod('mmengine.registry', MODELS=_Registry())
    mod('mmengine.logging', MMLogger=types.SimpleNamespace(get_instance=lambda name: types.SimpleNamespace(info=print)))
    mod('mmseg')
    mod('mmseg.registry', MODELS=_Registry())
    mod('mmcv')
    mod('mmcv.ops')
    mod('mmcv.ops.multi_scale_deform_attn', MultiScaleDeformableAttention=type('MultiScaleDeformableAttention', (nn.Module,), {}))
    mod('mmcv.cnn')
    mod('mmcv.cnn.bricks')
    mod('mmcv.cnn.bricks.transformer',
        build_positional_encoding=lambda cfg: built['pe'](**{k: v for k, v in cfg.items() if k != 'type'}),
        build_transformer_layer=lambda cfg: _StubLayer())
    for pkg in ('refpkg', 'refpkg.lifter', 'refpkg.encoder', 'refpkg.encoder.bevformer', 'refpkg.head', 'refpkg.head.utils',
                'refpkg.head.nerfacc_head'):
        mod(pkg)
    sys.modules['refpkg.lifter.base_lifter'] = types.SimpleNamespace(BaseLifter=_BaseModule)
    sys.modules['refpkg.encoder.base_encoder'] = types.SimpleNamespace(BaseEncoder=_BaseModule)
    sys.modules['refpkg.encoder.bevformer.utils'] = types.SimpleNamespace(point_sampling=None)
    sys.modules['refpkg.encoder.bevformer.attention'] = types.SimpleNamespace(
        BEVCrossAttention=type('BEVCrossAttention', (nn.Module,), {}),
        BEVDeformableAttention=type('BEVDeformableAttention', (nn.Module,), {}))


def _load_as(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def model_cfgs():
    ns = {}
    f = os.path.join(REF, 'config', CFG)
    exec(compile(open(f).read(), f, 'exec'), ns)
    return {CFG: {k: ns['model'][k] for k in ('lifter', 'encoder', 'head')}}


def main():
    built = {}
    _install_stand_ins(built)
    _load_as('model/encoder/bevformer/mappings.py', 'refpkg.encoder.bevformer.mappings')
    _load_as('model/head/utils/sh_render.py', 'refpkg.head.utils.sh_render')
    pe_mod = _load_as('model/encoder/bevformer/bevformer_pos_embed.py', 'refpkg.encoder.bevformer.bevformer_pos_embed')
    built['pe'] = pe_mod.BEVPositionalEncoding
    enc_mod = _load_as('model/encoder/bevformer/bevformer_encoder.py', 'refpkg.encoder.bevformer.bevformer_encoder')
    lift_mod = _load_as('model/lifter/bev_query_lifter.py', 'refpkg.lifter.bev_query_lifter')
    bn = _load_as('model/head/nerfacc_head/bev_nerf.py', 'refpkg.head.nerfacc_head.bev_nerf')

    cfgs = model_cfgs()
    json.dump(cfgs, open(os.path.join(HERE, 'reference_model_cfgs_bev.json'), 'w'), indent=1, sort_keys=True)
    cfg = cfgs[CFG]
    out = {}
    # encoder tables: the shipped geometry (strided rows) and a small one (whole)
    small = dict(nonlinear_mode='linear', h_size=[3, 0], h_range=[6.0, 0], h_half=False, w_size=[2, 0], w_range=[4.0, 0],
                 w_half=False, d_size=[3, 0], d_range=[-1.0, 2.0, 2.0])
    for name, margs, stride in (('ship', cfg['encoder']['mapping_args'], 97), ('small', small, 1)):
        e = cfg['encoder']
        enc = enc_mod.BEVFormerEncoder(mapping_args=margs, embed_dims=e['embed_dims'], num_cams=e['num_cams'],
                                       num_feature_levels=e['num_feature_levels'],
                                       positional_encoding=dict(e['positional_encoding']), num_points_cross=e['num_points_cross'],
                                       num_points_self=e['num_points_self'], transformerlayers=e['transformerlayers'],
                                       num_layers=e['num_layers'])
        out[name + '_margs'] = np.array(json.dumps(margs, sort_keys=True))
        out[name + '_stride'] = np.array(stride)
        out[name + '_freq_feat'] = enc.positional_encoding.freq_feat[::stride].numpy()
        out[name + '_ref_3d'] = enc.ref_3d[:, ::stride].numpy()
        out[name + '_ref_2d'] = enc.ref_2d.flatten(0, 1)[::stride].numpy()
        out[name + '_bev_size'] = np.array(enc.bev_size)
    torch.manual_seed(3)
    lifter = lift_mod.BEVQueryLifter(bev_h=3, bev_w=4, dim=8)
    out['lifter_keys'] = np.array(sorted(lifter.state_dict()))
    out['lifter_rep_shape'] = np.array(lifter([torch.zeros(1, 6, 8, 2, 2)])['representation'].shape)

    # decode + field queries at a small geometry, C = 96 (the kernel's width), Cf = 1 + color_dims as NeuSHead builds it
    for name, margs, cd in (('a', dict(nonlinear_mode='linear', h_size=[3, 0], h_range=[4.8, 0], h_half=False, w_size=[2, 0],
                                        w_range=[3.2, 0], w_half=False, d_size=[3, 0], d_range=[-1.0, 2.0, 2.0]), 3),
                            ('b', dict(nonlinear_mode='linear', h_size=[2, 0], h_range=[3.2, 0], h_half=True, w_size=[3, 0],
                                       w_range=[4.8, 0], w_half=False, d_size=[4, 0], d_range=[-1.0, 3.0, 3.0]), 0)):
        torch.manual_seed(17 if name == 'a' else 19)
        net = bn.BEVNeRF(mapping_args=margs, embed_dims=96, color_dims=cd, density_layers=2, sh_deg=0, sh_act='relu', tpv=False)
        H, W, Z = net.h_size, net.w_size, net.z_size
        bev = 0.7 * torch.randn(1, H * W, 96)
        with torch.no_grad():
            net.pre_compute_density_color(bev)
            vol = net.density_color.clone()                         # [1, Cf, H, W, Z]
            lo = torch.tensor([-margs['w_range'][0] * 1.2, (0.0 if margs['h_half'] else -margs['h_range'][0]) * 1.2 - 0.5,
                               margs['d_range'][0] - 0.7])
            hi = torch.tensor([margs['w_range'][0] * 1.2, margs['h_range'][0] * 1.2, margs['d_range'][1] + 0.7])
            x = lo + (hi - lo) * torch.rand(193, 3)
            dirs = torch.nn.functional.normalize(torch.randn(x.shape[0], 3), dim=-1)
            rgb, sigma, _ = net(x, condition=dirs)
            sigma_geo, _ = net.forward_geo(x)
        out[name + '_margs'] = np.array(json.dumps(margs, sort_keys=True))
        out[name + '_dims'] = np.array([96, cd, H, W, Z])
        out[name + '_bev'] = bev.numpy()
        for k, t in (('w1', net.density_net[1].weight), ('b1', net.density_net[1].bias), ('w2', net.density_net[3].weight),
                     ('b2', net.density_net[3].bias)):
            out[name + '_' + k] = t.detach().numpy()
        out[name + '_vol'] = vol.numpy()
        out[name + '_x'], out[name + '_rgb'], out[name + '_sigma'] = x.numpy(), rgb.numpy(), sigma.numpy()
        out[name + '_sigma_geo'] = sigma_geo.numpy()
    np.savez_compressed(os.path.join(HERE, 'reference_golden_bev.npz'), **out)
    print('wrote bev golden:', len(out), 'arrays')


if __name__ == '__main__':
    if REF is None or not os.path.isfile(os.path.join(REF, 'model', 'lifter', 'bev_query_lifter.py')):
        sys.exit('usage: python tests/golden/make_golden_bev.py <path to a huang-yh/SelfOcc checkout>')
    main()
