"""Generate golden vectors from the importable pure-torch pieces of the reference.

Run once, on a machine with a checkout of huang-yh/SelfOcc (the tests only read the stored vectors):
    python tests/golden/make_golden.py <path to the SelfOcc checkout>
Writes ``tests/golden/reference_golden.npz``.  Only reference modules that import without
mmcv/mmengine/nerfstudio are used (SURVEY.md section 8c); they are loaded by file path and
executed unmodified.  Inputs are seeded and stored beside the outputs.
"""
import importlib.util
import os
import sys
import numpy as np
import torch

REF = next((a for a in sys.argv[1:] if not a.startswith('--')), None)   # the SelfOcc checkout (required)
HERE = os.path.dirname(os.path.abspath(__file__))


def load(rel, name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    torch.manual_seed(0)
    np.random.seed(0)
    out = {}
    mp = load('model/encoder/bevformer/mappings.py', 'ref_mappings')
    # (i) the reference's own __main__ smoke inputs (mappings.py:300-329)
    m = mp.GridMeterMapping(nonlinear_mode='linear', h_size=[2, 2], h_range=[2, 4], h_half=False, w_size=[2, 2],
                            w_range=[2, 4], w_half=False, d_size=[2, 2], d_range=[-1., 1., 5.])
    grid = torch.tensor([[4, 0, 0], [0, 4, 1], [4, 4, 2], [5, 6, 4], [1, 0, 1.5], [7.5, 8, 2.5]])
    meter = torch.tensor([[-6., 0., -1.], [0., -6., 0.], [0., 0., 1.], [2., 1., 5.], [-6., -3.6667, 0.5],
                          [6., 4.8333, 1.8333]])
    out['map_small_grid'] = grid.numpy()
    out['map_small_g2m'] = m.grid2meter(grid).numpy()
    out['map_small_meter'] = meter.numpy()
    out['map_small_m2g'] = m.meter2grid(meter).numpy()
    # (ii) the nuScenes depth mapping (config/nuscenes/nuscenes_depth.py:188-198) on random points
    args = dict(nonlinear_mode='linear', h_size=[128, 0], h_range=[51.2, 0], h_half=False, w_size=[128, 0],
                w_range=[51.2, 0], w_half=False, d_size=[30, 0], d_range=[-4.0, 5.0, 5.0])
    m2 = mp.GridMeterMapping(**args)
    pts = (torch.rand(64, 3) - 0.5) * torch.tensor([120., 120., 12.])
    out['map_nus_meter'] = pts.numpy()
    out['map_nus_m2g'] = m2.meter2grid(pts).numpy()
    out['map_nus_m2g_norm'] = m2.meter2grid(pts, True).numpy()
    g = torch.rand(64, 3) * torch.tensor([256., 256., 30.])
    out['map_nus_grid'] = g.numpy()
    out['map_nus_g2m'] = m2.grid2meter(g).numpy()
    # (iii) a mapping with outer rings + half axes
    args3 = dict(nonlinear_mode='linear', h_size=[8, 4], h_range=[10., 20.], h_half=True, w_size=[6, 2],
                 w_range=[12., 8.], w_half=False, d_size=[4, 2], d_range=[-2.0, 2.0, 6.0])
    m3 = mp.GridMeterMapping(**args3)
    pts3 = (torch.rand(64, 3) - 0.3) * torch.tensor([40., 30., 10.])
    out['map_ring_meter'] = pts3.numpy()
    out['map_ring_m2g'] = m3.meter2grid(pts3, True).numpy()
    g3 = torch.rand(64, 3) * torch.tensor([12., 16., 6.])
    out['map_ring_grid'] = g3.numpy()
    out['map_ring_g2m'] = m3.grid2meter(g3).numpy()

    # cross-view reference points (tpvformer/utils.py:5-71)
    tu = load('model/encoder/tpvformer/utils.py', 'ref_tpv_utils')
    out['cvref_5_7_3_p4'] = tu.get_cross_view_ref_points(5, 7, 3, [4, 4, 4]).numpy()
    out['cvref_4_3_6_p3'] = tu.get_cross_view_ref_points(4, 3, 6, [3, 3, 3]).numpy()

    # point_sampling (bevformer/utils.py:116-206)
    bu = load('model/encoder/bevformer/utils.py', 'ref_bev_utils')
    ref3d = (torch.rand(1, 5, 40, 3) - 0.5) * torch.tensor([80., 80., 8.])
    K = np.array([[1266., 0, 800, 0], [0, 1266., 450, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    l2i = []
    for yaw in (0., -55., 110.):
        a = np.deg2rad(yaw)
        c2l = np.eye(4)
        # camera axes (x right, y down, z forward) expressed in the lidar frame (x right, y fwd, z up)
        fwd = np.array([np.sin(-a), np.cos(-a), 0.])
        right = np.array([np.cos(-a), -np.sin(-a), 0.])
        down = np.array([0., 0., -1.])
        c2l[:3, 0], c2l[:3, 1], c2l[:3, 2], c2l[:3, 3] = right, down, fwd, [0.3, 0.5, 1.5]
        l2i.append(K @ np.linalg.inv(c2l))
    l2i = np.stack(l2i)[None]
    metas = [dict(lidar2img=list(l2i[0]), img_shape=(900, 1600))]
    rc, mk = bu.point_sampling(ref3d, metas)
    out['ps_ref3d'] = ref3d.numpy()
    out['ps_lidar2img'] = l2i
    out['ps_uv'] = rc.numpy()
    out['ps_mask'] = mk.numpy()

    # ray sampler (ray_sampler.py) fixed + cellular
    rs = load('model/head/nerfacc_head/ray_sampler.py', 'ref_ray_sampler')
    out['rays_fixed_6x10_90x160'] = rs.RaySampler('fixed', [6, 10], [90, 160])().numpy()
    out['rays_fixed_450x800'] = rs.RaySampler('fixed', [450, 800], [900, 1600])()[::997].numpy()
    np.random.seed(123)
    u4 = np.random.uniform(size=4)
    np.random.seed(123)
    out['rays_cell_u4'] = u4
    out['rays_cell_6x10_90x160'] = rs.RaySampler('cellular', [6, 10], [90, 160], ray_upper_crop=8)().numpy()

    # SH bases (sh_render.py)
    sh = load('model/head/utils/sh_render.py', 'ref_sh')
    dirs = torch.nn.functional.normalize(torch.randn(16, 3), dim=-1)
    feats = torch.randn(16, 3)
    out['sh_dirs'] = dirs.numpy()
    out['sh_feats'] = feats.numpy()
    out['sh_deg0_relu'] = sh.SHRender(None, dirs, feats, 0, 'relu').numpy()
    out['sh_deg0_sigmoid'] = sh.SHRender(None, dirs, feats, 0, 'sigmoid').numpy()

    # depth metric arithmetic (utils/metric_util.py:247-279; module import needs mmengine, so the
    # function source is exec'd on its own)
    src = open(os.path.join(REF, 'utils/metric_util.py')).read().split('\n')
    s = next(i for i, l in enumerate(src) if l.startswith('def cal_depth_metric'))
    e = next(i for i in range(s + 1, len(src)) if src[i].startswith('class '))
    ns = {'torch': torch}
    exec('\n'.join(src[s:e]), ns)
    gt = torch.rand(200) * 60 + 1
    pred = gt * (1 + 0.2 * torch.randn(200))
    md = ns['cal_depth_metric'](pred, gt)
    out['dm_gt'], out['dm_pred'] = gt.numpy(), pred.numpy()
    out['dm_vals'] = np.array([float(md[k]) for k in ('abs_rel', 'sq_rel', 'rmse', 'rmse_log', 'a1', 'a2', 'a3')])

    np.savez_compressed(os.path.join(HERE, 'reference_golden.npz'), **out)
    print('wrote', len(out), 'arrays')




def dump_reference_model_configs():
    """The lifter / encoder / head config dicts of every shipped TPV experiment config, as the reference's own config
    files define them (plain `exec` of config/<set>/<name>.py: they are self-contained python apart from `_base_`).
    Written to tests/golden/reference_model_cfgs.json; tests/test_modules_cpu.py builds the H100 modules from them."""
    import glob
    import json
    out = {}
    for f in sorted(glob.glob(os.path.join(REF, 'config', '*', '*.py'))):
        if '_base_' in f:
            continue
        ns = {}
        exec(compile(open(f).read(), f, 'exec'), ns)
        m = ns['model']
        if m['encoder']['type'] != 'TPVFormerEncoder':
            continue                      # nuscenes_occ_bev.py: the BEV-only variant is out of scope (SURVEY.md 2.1)
        out[os.path.relpath(f, os.path.join(REF, 'config'))] = {k: m[k] for k in ('lifter', 'encoder', 'head')}
    json.dump(out, open(os.path.join(HERE, 'reference_model_cfgs.json'), 'w'), indent=1, sort_keys=True)
    print('wrote model configs of', sorted(out))




def bevnerf_golden():
    """Pins oracle rows B5/B7 (TPV -> decoded volume, trilinear field query) to the reference's only in-tree statement of
    them: model/head/nerfacc_head/bev_nerf.py:62-175 (``BEVNeRF``, tpv=True).  The module is executed UNMODIFIED; its two
    non-torch imports are satisfied by (a) a 3-line stand-in for ``mmengine.model.BaseModule`` (an nn.Module that accepts
    ``init_cfg``) and (b) a synthetic package tree so that its relative imports resolve to the reference's own
    ``mappings.py`` / ``sh_render.py`` loaded by file path.  Writes tests/golden/reference_golden_bevnerf.npz."""
    import types
    import torch.nn as nn

    class BaseModule(nn.Module):
        def __init__(self, init_cfg=None):
            super().__init__()
    mm, mmm = types.ModuleType('mmengine'), types.ModuleType('mmengine.model')
    mmm.BaseModule = BaseModule
    mm.model = mmm
    sys.modules.setdefault('mmengine', mm)
    sys.modules.setdefault('mmengine.model', mmm)
    for pkg in ('refpkg', 'refpkg.encoder', 'refpkg.encoder.bevformer', 'refpkg.head', 'refpkg.head.utils',
                'refpkg.head.nerfacc_head'):
        p = types.ModuleType(pkg)
        p.__path__ = []
        sys.modules[pkg] = p

    def load_as(rel, name):
        spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod
    load_as('model/encoder/bevformer/mappings.py', 'refpkg.encoder.bevformer.mappings')
    load_as('model/head/utils/sh_render.py', 'refpkg.head.utils.sh_render')
    bn = load_as('model/head/nerfacc_head/bev_nerf.py', 'refpkg.head.nerfacc_head.bev_nerf')

    out = {}
    cases = {
        # name: (mapping args, embed dims, color dims, sem dims)
        'a': (dict(nonlinear_mode='linear', h_size=[4, 0], h_range=[6.4, 0], h_half=False, w_size=[5, 0], w_range=[8.0, 0],
                   w_half=False, d_size=[6, 0], d_range=[-2.0, 4.0, 4.0]), 32, 3, 5),
        'b': (dict(nonlinear_mode='linear', h_size=[6, 0], h_range=[9.6, 0], h_half=True, w_size=[3, 0], w_range=[4.8, 0],
                   w_half=False, d_size=[4, 0], d_range=[-1.0, 3.0, 3.0]), 16, 0, 0),
    }
    for name, (margs, C, cd, sd) in cases.items():
        torch.manual_seed(7 if name == 'a' else 11)
        net = bn.BEVNeRF(mapping_args=margs, embed_dims=C, color_dims=cd, sem_dims=sd, density_layers=2, sh_deg=0,
                         sh_act='relu', tpv=True)
        H, W, Z = net.h_size, net.w_size, net.z_size
        planes = [0.5 * torch.randn(1, n, C) for n in (H * W, Z * H, W * Z)]
        with torch.no_grad():
            net.pre_compute_density_color(planes)
            vol = net.density_color.clone()                       # [1, Cf, H, W, Z]
            lo = torch.tensor([-margs['w_range'][0] * 1.2, (0.0 if margs['h_half'] else -margs['h_range'][0]) * 1.2 - 0.5,
                               margs['d_range'][0] - 0.7])
            hi = torch.tensor([margs['w_range'][0] * 1.2, margs['h_range'][0] * 1.2, margs['d_range'][1] + 0.7])
            x = lo + (hi - lo) * torch.rand(257, 3)               # includes points outside the volume (zeros padding)
            dirs = torch.nn.functional.normalize(torch.randn(x.shape[0], 3), dim=-1)   # SH degree 0 ignores them (sh_render.py:48)
            rgb, sigma, sems = net(x, condition=dirs)
            sigma_geo, sems_geo = net.forward_geo(x)
            dens = net.query_density(x)
        out[name + '_margs'] = np.array(json_dumps(margs))
        out[name + '_dims'] = np.array([C, cd, sd, H, W, Z])
        for i, p in enumerate(planes):
            out['%s_plane%d' % (name, i)] = p.numpy()
        out[name + '_w1'], out[name + '_b1'] = net.density_net[1].weight.detach().numpy(), net.density_net[1].bias.detach().numpy()
        out[name + '_w2'], out[name + '_b2'] = net.density_net[3].weight.detach().numpy(), net.density_net[3].bias.detach().numpy()
        out[name + '_vol'] = vol.numpy()
        out[name + '_x'] = x.numpy()
        out[name + '_rgb'], out[name + '_sigma'], out[name + '_sems'] = rgb.numpy(), sigma.numpy(), sems.numpy()
        out[name + '_sigma_geo'], out[name + '_sems_geo'], out[name + '_dens'] = sigma_geo.numpy(), sems_geo.numpy(), dens.numpy()
    np.savez_compressed(os.path.join(HERE, 'reference_golden_bevnerf.npz'), **out)
    print('wrote bevnerf golden:', len(out), 'arrays')


def json_dumps(o):
    import json
    return json.dumps(o, sort_keys=True)


if __name__ == '__main__' and (REF is None or not os.path.isfile(os.path.join(REF, 'model', 'head', 'nerfacc_head', 'bev_nerf.py'))):
    sys.exit('usage: python tests/golden/make_golden.py <path to a huang-yh/SelfOcc checkout> [--bevnerf]')

if __name__ == '__main__' and '--bevnerf' in sys.argv:
    bevnerf_golden()

if __name__ == '__main__' and '--bevnerf' not in sys.argv:
    main()
    dump_reference_model_configs()
    bevnerf_golden()
